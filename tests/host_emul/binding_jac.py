"""TEST HARNESS ONLY: the world-Jacobian device functions compiled for the host (tests/host_emul/emul_jac.cpp, which builds on emul.cpp)."""
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
        so = os.path.join(_HERE, "libemul_jac.so")
        srcs = [os.path.join(_HERE, f) for f in ("emul_jac.cpp", "emul.cpp")] + [
            os.path.join(_ROOT, "nimblephysics_b200", "csrc", f)
            for f in ("nb2_jac.cuh", "nb2_mm.cuh", "nb2_dyn.cuh", "nb2_math.cuh", "nb2_model.h", "nb2_host_model.h", "nb2_cw.cuh", "nb2_geom.cuh")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so,
                                   os.path.join(_HERE, "emul_jac.cpp")])
        _LIB = ctypes.CDLL(so)
    return _LIB


class EmulJacWorld(EmulWorld):
    """EmulWorld + the body-point and COM Jacobians and their backward (rows in float64 if fp64, else float32).
    Nodes are given as canonical bodies [k] and body <- node transforms [k, 4, 4]."""

    @staticmethod
    def _nodes(bodies, T):
        b = np.ascontiguousarray(bodies, np.int32)
        T = np.asarray(T, np.float64).reshape(len(b), 4, 4)
        T12 = np.ascontiguousarray(np.concatenate([T[:, :3, :3].reshape(-1, 9), T[:, :3, 3]], 1))
        return b, T12

    def world_jacobian(self, pos, bodies, T, offsets=None, fp64=False):
        dt = np.float64 if fp64 else np.float32
        pos = np.ascontiguousarray(pos, dt)
        B = pos.shape[0]
        b, T12 = self._nodes(bodies, T)
        off = None if offsets is None else np.ascontiguousarray(offsets, dt)
        J = np.empty((B, len(b), 6, self.n), dt)
        assert lib().emul_world_jacobian(ctypes.byref(self.desc), B, _p(pos), len(b), _p(b), _p(T12), _p(off),
                                         int(off is not None and off.ndim == 3), _p(J), None, None, None, int(fp64)) == 0
        return J

    def world_jacobian_backward(self, pos, bodies, T, grad, offsets=None, fp64=False):
        """-> (grad_pos [B, n], grad_offsets [B, k, 3] per world)"""
        dt = np.float64 if fp64 else np.float32
        pos = np.ascontiguousarray(pos, dt)
        B = pos.shape[0]
        b, T12 = self._nodes(bodies, T)
        off = None if offsets is None else np.ascontiguousarray(offsets, dt)
        g = np.ascontiguousarray(grad, dt)
        gp, go = np.empty((B, self.n), dt), np.empty((B, len(b), 3), dt)
        assert lib().emul_world_jacobian(ctypes.byref(self.desc), B, _p(pos), len(b), _p(b), _p(T12), _p(off),
                                         int(off is not None and off.ndim == 3), None, _p(g), _p(gp), _p(go), int(fp64)) == 0
        return gp, go

    def com_jacobian(self, pos, root, fp64=False, world_inertia=None):
        dt = np.float64 if fp64 else np.float32
        pos = np.ascontiguousarray(pos, dt)
        B = pos.shape[0]
        J = np.empty((B, 3, self.n), dt)
        assert lib().emul_com_jacobian(ctypes.byref(self.desc), B, _p(pos), int(root), _p(self._wi(world_inertia, B)), _p(J), None, None, None,
                                       int(fp64)) == 0
        return J

    def com_jacobian_backward(self, pos, root, grad, fp64=False, world_inertia=None):
        """-> (grad_pos [B, n], grad_inertia fp64 [10*nb, B])"""
        dt = np.float64 if fp64 else np.float32
        pos = np.ascontiguousarray(pos, dt)
        B = pos.shape[0]
        g = np.ascontiguousarray(grad, dt)
        gp = np.empty((B, self.n), dt)
        gi = np.full((10 * self.cm.nb, B), np.nan, np.float64)
        assert lib().emul_com_jacobian(ctypes.byref(self.desc), B, _p(pos), int(root), _p(self._wi(world_inertia, B)), None, _p(g), _p(gp), _p(gi),
                                       int(fp64)) == 0
        return gp, gi
