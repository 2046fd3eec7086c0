"""TEST HARNESS ONLY: the Jacobian-derivative device functions compiled for the host (tests/host_emul/emul_jacd.cpp, which builds on
emul.cpp)."""
import ctypes
import os
import subprocess

import numpy as np

from tests.host_emul.binding import _p
from tests.host_emul.binding_jac import EmulJacWorld

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.join(_HERE, "..", "..")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libemul_jacd.so")
        srcs = [os.path.join(_HERE, f) for f in ("emul_jacd.cpp", "emul.cpp")] + [
            os.path.join(_ROOT, "nimblephysics_b200", "csrc", f)
            for f in ("nb2_jac.cuh", "nb2_mm.cuh", "nb2_dyn.cuh", "nb2_math.cuh", "nb2_model.h", "nb2_host_model.h", "nb2_cw.cuh", "nb2_geom.cuh")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so,
                                   os.path.join(_HERE, "emul_jacd.cpp")])
        _LIB = ctypes.CDLL(so)
    return _LIB


class EmulJacdWorld(EmulJacWorld):
    """EmulJacWorld + the time derivatives of the body-point and COM Jacobians and their backward, at states [B, 2n] (rows in float64 if
    fp64, else float32)."""

    def world_jacobian_deriv(self, state, bodies, T, offsets=None, fp64=False):
        dt = np.float64 if fp64 else np.float32
        st = np.ascontiguousarray(state, dt)
        B = st.shape[0]
        b, T12 = self._nodes(bodies, T)
        off = None if offsets is None else np.ascontiguousarray(offsets, dt)
        dJ = np.empty((B, len(b), 6, self.n), dt)
        assert lib().emul_world_jacobian_deriv(ctypes.byref(self.desc), B, _p(st), len(b), _p(b), _p(T12), _p(off),
                                               int(off is not None and off.ndim == 3), _p(dJ), None, None, None, int(fp64)) == 0
        return dJ

    def world_jacobian_deriv_backward(self, state, bodies, T, grad, offsets=None, fp64=False):
        """-> (grad_state [B, 2n], grad_offsets [B, k, 3] per world)"""
        dt = np.float64 if fp64 else np.float32
        st = np.ascontiguousarray(state, dt)
        B = st.shape[0]
        b, T12 = self._nodes(bodies, T)
        off = None if offsets is None else np.ascontiguousarray(offsets, dt)
        g = np.ascontiguousarray(grad, dt)
        gs, go = np.empty((B, 2 * self.n), dt), np.empty((B, len(b), 3), dt)
        assert lib().emul_world_jacobian_deriv(ctypes.byref(self.desc), B, _p(st), len(b), _p(b), _p(T12), _p(off),
                                               int(off is not None and off.ndim == 3), None, _p(g), _p(gs), _p(go), int(fp64)) == 0
        return gs, go

    def com_jacobian_deriv(self, state, root, fp64=False, world_inertia=None):
        dt = np.float64 if fp64 else np.float32
        st = np.ascontiguousarray(state, dt)
        B = st.shape[0]
        dJ = np.empty((B, 3, self.n), dt)
        assert lib().emul_com_jacobian_deriv(ctypes.byref(self.desc), B, _p(st), int(root), _p(self._wi(world_inertia, B)), _p(dJ), None, None,
                                             None, int(fp64)) == 0
        return dJ

    def com_jacobian_deriv_backward(self, state, root, grad, fp64=False, world_inertia=None):
        """-> (grad_state [B, 2n], grad_inertia fp64 [10*nb, B])"""
        dt = np.float64 if fp64 else np.float32
        st = np.ascontiguousarray(state, dt)
        B = st.shape[0]
        g = np.ascontiguousarray(grad, dt)
        gs = np.empty((B, 2 * self.n), dt)
        gi = np.full((10 * self.cm.nb, B), np.nan, np.float64)
        assert lib().emul_com_jacobian_deriv(ctypes.byref(self.desc), B, _p(st), int(root), _p(self._wi(world_inertia, B)), None, _p(g), _p(gs),
                                             _p(gi), int(fp64)) == 0
        return gs, gi
