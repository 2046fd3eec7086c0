"""TEST HARNESS ONLY: the mass-matrix device functions compiled for the host (tests/host_emul/emul_mm.cpp, which builds on emul.cpp)."""
import ctypes
import os
import subprocess

import numpy as np

from tests.host_emul.binding import EmulWorld, _p

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.join(_HERE, "..", "..")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libemul_mm.so")
        srcs = [os.path.join(_HERE, f) for f in ("emul_mm.cpp", "emul.cpp")] + [
            os.path.join(_ROOT, "nimblephysics_b200", "csrc", f)
            for f in ("nb2_mm.cuh", "nb2_dyn.cuh", "nb2_math.cuh", "nb2_model.h", "nb2_host_model.h", "nb2_cw.cuh", "nb2_geom.cuh")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so,
                                   os.path.join(_HERE, "emul_mm.cpp")])
        _LIB = ctypes.CDLL(so)
    return _LIB


class EmulMmWorld(EmulWorld):
    """EmulWorld + M, M^-1 and their backward (rows in float64 if fp64, else float32)."""

    def mass_matrix(self, pos, inverse=False, fp64=False, world_inertia=None):
        dt = np.float64 if fp64 else np.float32
        pos = np.ascontiguousarray(pos, dt)
        B = pos.shape[0]
        out = np.empty((B, self.n, self.n), dt)
        assert lib().emul_mass_matrix(ctypes.byref(self.desc), int(inverse), B, _p(pos), _p(self._wi(world_inertia, B)), _p(out), int(fp64)) == 0
        return out

    def mass_matrix_backward(self, pos, grad, minv=None, fp64=False, world_inertia=None):
        """-> (grad_pos [B, n], grad_inertia fp64 [10*nb, B]); minv: the forward's M^-1 for the inverse's backward, else None"""
        dt = np.float64 if fp64 else np.float32
        pos = np.ascontiguousarray(pos, dt)
        grad = np.ascontiguousarray(grad, dt)
        mi = np.ascontiguousarray(minv, dt) if minv is not None else None
        B = pos.shape[0]
        gp = np.empty((B, self.n), dt)
        gi = np.zeros((10 * self.cm.nb, B), np.float64)
        assert lib().emul_mass_matrix_backward(ctypes.byref(self.desc), B, _p(pos), _p(self._wi(world_inertia, B)), _p(grad), _p(mi), _p(gp),
                                               _p(gi), int(fp64)) == 0
        return gp, gi
