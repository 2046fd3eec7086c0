"""TEST HARNESS ONLY: the constrained forward-dynamics program compiled for the host (tests/host_emul/emul_cfd.cpp, which builds on
emul.cpp)."""
import ctypes
import os
import subprocess

import numpy as np

from tests.host_emul.binding import EmulWorld, _p
from tests.host_emul.binding_jac import EmulJacWorld

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.join(_HERE, "..", "..")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libemul_cfd.so")
        srcs = [os.path.join(_HERE, f) for f in ("emul_cfd.cpp", "emul.cpp")] + [
            os.path.join(_ROOT, "nimblephysics_b200", "csrc", f)
            for f in ("nb2_cfd.cuh", "nb2_djac.cuh", "nb2_jac.cuh", "nb2_mm.cuh", "nb2_dyn.cuh", "nb2_math.cuh", "nb2_model.h", "nb2_host_model.h",
                      "nb2_cw.cuh", "nb2_geom.cuh")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so,
                                   os.path.join(_HERE, "emul_cfd.cpp")])
        _LIB = ctypes.CDLL(so)
        _LIB.emul_constrained_forward_dynamics.argtypes = ([ctypes.c_void_p] + [ctypes.c_int] * 4 + [ctypes.c_void_p] * 2 + [ctypes.c_int]
                                                           + [ctypes.c_void_p] * 3 + [ctypes.c_int, ctypes.c_void_p, ctypes.c_double]
                                                           + [ctypes.c_void_p] * 8 + [ctypes.c_int])
    return _LIB


class EmulCfdWorld(EmulWorld):
    """EmulWorld + constrained forward dynamics and its backward (rows in float64 if fp64, else float32).  bodies: canonical bodies [k],
    T: body <- node transforms [k, 4, 4]; offsets None, [k, 3] or [B, k, 3]."""

    def _call(self, bwd, state, tau, bodies, T, offsets, point, rho, fp64, world_inertia, slots, gqdd=None, gw=None):
        dt = np.float64 if fp64 else np.float32
        st, ta = np.ascontiguousarray(state, dt), np.ascontiguousarray(tau, dt)
        B, n = st.shape[0], self.n
        b, T12 = EmulJacWorld._nodes(bodies, T)
        k, r = len(b), 3 if point else 6
        off = None if offsets is None else np.ascontiguousarray(offsets, dt)
        qdd = wr = gs = gt = go = gi = None
        if bwd:
            gqdd, gw = np.ascontiguousarray(gqdd, dt), np.ascontiguousarray(gw, dt)
            gs, gt, go = np.empty((B, 2 * n), dt), np.empty((B, n), dt), np.empty((B, k, 3), dt)
            gi = np.full((10 * self.cm.nb, B), np.nan, np.float64)
        else:
            qdd, wr = np.empty((B, n), dt), np.empty((B, k, r), dt)
        rc = lib().emul_constrained_forward_dynamics(ctypes.byref(self.desc), int(bwd), int(slots), k, int(point), _p(b), _p(T12), B, _p(st),
                                                     _p(ta), _p(off), int(off is not None and off.ndim == 3), _p(self._wi(world_inertia, B)),
                                                     float(rho), _p(qdd), _p(wr), _p(gqdd), _p(gw), _p(gs), _p(gt), _p(go), _p(gi), int(fp64))
        assert rc == 0
        return (gs, gt, go, gi) if bwd else (qdd, wr)

    def constrained_forward_dynamics(self, state, tau, bodies, T, offsets=None, point=False, rho=0.0, fp64=False, world_inertia=None, slots=8):
        """-> (qdd [B, n], wrenches [B, k, 6 or 3])"""
        return self._call(False, state, tau, bodies, T, offsets, point, rho, fp64, world_inertia, slots)

    def constrained_forward_dynamics_backward(self, state, tau, bodies, T, gqdd, gw, offsets=None, point=False, rho=0.0, fp64=False,
                                              world_inertia=None, slots=8):
        """-> (grad_state [B, 2n], grad_tau [B, n], grad_offsets [B, k, 3], grad_inertia fp64 [10 nb, B])"""
        return self._call(True, state, tau, bodies, T, offsets, point, rho, fp64, world_inertia, slots, gqdd, gw)
