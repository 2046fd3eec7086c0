"""TEST HARNESS ONLY: the impulse-dynamics program compiled for the host (tests/host_emul/emul_imp.cpp, which builds on emul.cpp)."""
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
        so = os.path.join(_HERE, "libemul_imp.so")
        srcs = [os.path.join(_HERE, f) for f in ("emul_imp.cpp", "emul.cpp")] + [
            os.path.join(_ROOT, "nimblephysics_b200", "csrc", f)
            for f in ("nb2_imp.cuh", "nb2_cfd.cuh", "nb2_djac.cuh", "nb2_jac.cuh", "nb2_mm.cuh", "nb2_dyn.cuh", "nb2_math.cuh", "nb2_model.h",
                      "nb2_host_model.h", "nb2_cw.cuh", "nb2_geom.cuh")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so,
                                   os.path.join(_HERE, "emul_imp.cpp")])
        _LIB = ctypes.CDLL(so)
        _LIB.emul_impulse_dynamics.argtypes = ([ctypes.c_void_p] + [ctypes.c_int] * 4 + [ctypes.c_void_p] * 2 + [ctypes.c_int]
                                               + [ctypes.c_void_p] * 2 + [ctypes.c_int, ctypes.c_void_p, ctypes.c_double, ctypes.c_double]
                                               + [ctypes.c_void_p] * 7 + [ctypes.c_int])
    return _LIB


class EmulImpWorld(EmulWorld):
    """EmulWorld + impulse dynamics and its backward (rows in float64 if fp64, else float32).  bodies: canonical bodies [k], T: body <- node
    transforms [k, 4, 4]; offsets None, [k, 3] or [B, k, 3]."""

    def _call(self, bwd, state, bodies, T, offsets, point, e, rho, fp64, world_inertia, slots, gvel=None, gimp=None):
        dt = np.float64 if fp64 else np.float32
        st = np.ascontiguousarray(state, dt)
        B, n = st.shape[0], self.n
        b, T12 = EmulJacWorld._nodes(bodies, T)
        k, r = len(b), 3 if point else 6
        off = None if offsets is None else np.ascontiguousarray(offsets, dt)
        vel = imp = gs = go = gi = None
        if bwd:
            gvel, gimp = np.ascontiguousarray(gvel, dt), np.ascontiguousarray(gimp, dt)
            gs, go = np.empty((B, 2 * n), dt), np.empty((B, k, 3), dt)
            gi = np.full((10 * self.cm.nb, B), np.nan, np.float64)
        else:
            vel, imp = np.empty((B, n), dt), np.empty((B, k, r), dt)
        rc = lib().emul_impulse_dynamics(ctypes.byref(self.desc), int(bwd), int(slots), k, int(point), _p(b), _p(T12), B, _p(st), _p(off),
                                         int(off is not None and off.ndim == 3), _p(self._wi(world_inertia, B)), float(e), float(rho), _p(vel),
                                         _p(imp), _p(gvel), _p(gimp), _p(gs), _p(go), _p(gi), int(fp64))
        assert rc == 0
        return (gs, go, gi) if bwd else (vel, imp)

    def impulse_dynamics(self, state, bodies, T, offsets=None, point=False, e=0.0, rho=0.0, fp64=False, world_inertia=None, slots=8):
        """-> (qdot_after [B, n], impulses [B, k, 6 or 3])"""
        return self._call(False, state, bodies, T, offsets, point, e, rho, fp64, world_inertia, slots)

    def impulse_dynamics_backward(self, state, bodies, T, gvel, gimp, offsets=None, point=False, e=0.0, rho=0.0, fp64=False, world_inertia=None,
                                  slots=8):
        """-> (grad_state [B, 2n], grad_offsets [B, k, 3], grad_inertia fp64 [10 nb, B])"""
        return self._call(True, state, bodies, T, offsets, point, e, rho, fp64, world_inertia, slots, gvel, gimp)
