"""TEST HARNESS ONLY: the dense dynamics-Jacobian device functions compiled for the host (tests/host_emul/emul_djac.cpp, which builds on
emul.cpp)."""
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
        so = os.path.join(_HERE, "libemul_djac.so")
        srcs = [os.path.join(_HERE, f) for f in ("emul_djac.cpp", "emul.cpp")] + [
            os.path.join(_ROOT, "nimblephysics_b200", "csrc", f)
            for f in ("nb2_djac.cuh", "nb2_dyn.cuh", "nb2_math.cuh", "nb2_model.h", "nb2_host_model.h", "nb2_cw.cuh", "nb2_geom.cuh")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so,
                                   os.path.join(_HERE, "emul_djac.cpp")])
        _LIB = ctypes.CDLL(so)
    return _LIB


class EmulDjacWorld(EmulWorld):
    """EmulWorld + the dense Jacobians of inverse and forward dynamics (rows in float64 if fp64, else float32)."""

    def dynamics_jacobians(self, state, x, fd, fp64=False, world_inertia=None, slots=32):
        """fd: forward dynamics (x = tau), else inverse dynamics (x = next_vel).  -> (out [B, n], J_q, J_qdot, J_x [B, n, n])"""
        dt = np.float64 if fp64 else np.float32
        state = np.ascontiguousarray(state, dt)
        x = np.ascontiguousarray(x, dt)
        B, n = state.shape[0], self.n
        out = np.empty((B, n), dt)
        J = [np.empty((B, n, n), dt) for _ in range(3)]
        rc = lib().emul_dynamics_jacobians(ctypes.byref(self.desc), int(fd), int(slots), B, _p(state), _p(x), _p(out), _p(J[0]), _p(J[1]), _p(J[2]),
                                           int(fp64), _p(self._wi(world_inertia, B)))
        assert rc == 0
        return (out, *J)
