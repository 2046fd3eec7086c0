"""TEST HARNESS ONLY: the dense-Jacobian program of impulse dynamics compiled for the host (tests/host_emul/emul_impj.cpp, which builds on
emul.cpp), next to the forward and VJP of binding_imp."""
import ctypes
import os
import subprocess

import numpy as np

from tests.host_emul.binding import _p
from tests.host_emul.binding_imp import EmulImpWorld
from tests.host_emul.binding_jac import EmulJacWorld

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.join(_HERE, "..", "..")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libemul_impj.so")
        srcs = [os.path.join(_HERE, f) for f in ("emul_impj.cpp", "emul.cpp")] + [
            os.path.join(_ROOT, "nimblephysics_b200", "csrc", f)
            for f in ("nb2_imp.cuh", "nb2_cfd.cuh", "nb2_djac.cuh", "nb2_jac.cuh", "nb2_mm.cuh", "nb2_dyn.cuh", "nb2_math.cuh", "nb2_model.h",
                      "nb2_host_model.h", "nb2_cw.cuh", "nb2_geom.cuh")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so,
                                   os.path.join(_HERE, "emul_impj.cpp")])
        _LIB = ctypes.CDLL(so)
        _LIB.emul_impulse_dynamics_jacobians.argtypes = ([ctypes.c_void_p] + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 2 + [ctypes.c_int]
                                                         + [ctypes.c_void_p] * 2 + [ctypes.c_int, ctypes.c_void_p, ctypes.c_double, ctypes.c_double]
                                                         + [ctypes.c_void_p] * 3 + [ctypes.c_int])
    return _LIB


class EmulImpjWorld(EmulImpWorld):
    """EmulImpWorld + the dense Jacobians of impulse dynamics (rows in float64 if fp64, else float32)."""

    def impulse_dynamics_jacobians(self, state, bodies, T, offsets=None, point=False, e=0.0, rho=0.0, fp64=False, world_inertia=None, slots=8):
        """-> (qdot_after [B, n], impulses [B, k, r], dv_dq, dv_dqdot [B, n, n], dimp_dq, dimp_dqdot [B, k, r, n])"""
        dt = np.float64 if fp64 else np.float32
        st = np.ascontiguousarray(state, dt)
        B, n = st.shape[0], self.n
        b, T12 = EmulJacWorld._nodes(bodies, T)
        k, r = len(b), 3 if point else 6
        off = None if offsets is None else np.ascontiguousarray(offsets, dt)
        vel, imp = np.full((B, n), np.nan, dt), np.full((B, k, r), np.nan, dt)
        J = [np.full((B, n, n), np.nan, dt) for _ in range(2)] + [np.full((B, k, r, n), np.nan, dt) for _ in range(2)]
        ptrs = (ctypes.c_void_p * 4)(*[x.ctypes.data for x in J])
        rc = lib().emul_impulse_dynamics_jacobians(ctypes.byref(self.desc), int(slots), k, int(point), _p(b), _p(T12), B, _p(st), _p(off),
                                                   int(off is not None and off.ndim == 3), _p(self._wi(world_inertia, B)), float(e), float(rho),
                                                   _p(vel), _p(imp), ptrs, int(fp64))
        assert rc == 0
        return (vel, imp, *J)
