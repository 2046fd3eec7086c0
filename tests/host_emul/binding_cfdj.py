"""TEST HARNESS ONLY: the dense-Jacobian program of constrained forward dynamics compiled for the host (tests/host_emul/emul_cfdj.cpp,
which builds on emul.cpp), next to the forward and VJP of binding_cfd."""
import ctypes
import os
import subprocess

import numpy as np

from tests.host_emul.binding import _p
from tests.host_emul.binding_cfd import EmulCfdWorld
from tests.host_emul.binding_jac import EmulJacWorld

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.join(_HERE, "..", "..")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libemul_cfdj.so")
        srcs = [os.path.join(_HERE, f) for f in ("emul_cfdj.cpp", "emul.cpp")] + [
            os.path.join(_ROOT, "nimblephysics_b200", "csrc", f)
            for f in ("nb2_cfd.cuh", "nb2_djac.cuh", "nb2_jac.cuh", "nb2_mm.cuh", "nb2_dyn.cuh", "nb2_math.cuh", "nb2_model.h", "nb2_host_model.h",
                      "nb2_cw.cuh", "nb2_geom.cuh")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so,
                                   os.path.join(_HERE, "emul_cfdj.cpp")])
        _LIB = ctypes.CDLL(so)
        _LIB.emul_constrained_forward_dynamics_jacobians.argtypes = ([ctypes.c_void_p] + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 2
                                                                     + [ctypes.c_int] + [ctypes.c_void_p] * 3
                                                                     + [ctypes.c_int, ctypes.c_void_p, ctypes.c_double]
                                                                     + [ctypes.c_void_p] * 3 + [ctypes.c_int])
    return _LIB


class EmulCfdjWorld(EmulCfdWorld):
    """EmulCfdWorld + the dense Jacobians of constrained forward dynamics (rows in float64 if fp64, else float32)."""

    def constrained_forward_dynamics_jacobians(self, state, tau, bodies, T, offsets=None, point=False, rho=0.0, fp64=False, world_inertia=None,
                                               slots=8):
        """-> (qdd [B, n], wrenches [B, k, r], dqdd_dq, dqdd_dqdot, dqdd_dtau [B, n, n], dwrench_dq, dwrench_dqdot, dwrench_dtau [B, k, r, n])"""
        dt = np.float64 if fp64 else np.float32
        st, ta = np.ascontiguousarray(state, dt), np.ascontiguousarray(tau, dt)
        B, n = st.shape[0], self.n
        b, T12 = EmulJacWorld._nodes(bodies, T)
        k, r = len(b), 3 if point else 6
        off = None if offsets is None else np.ascontiguousarray(offsets, dt)
        qdd, wr = np.full((B, n), np.nan, dt), np.full((B, k, r), np.nan, dt)
        J = [np.full((B, n, n), np.nan, dt) for _ in range(3)] + [np.full((B, k, r, n), np.nan, dt) for _ in range(3)]
        ptrs = (ctypes.c_void_p * 6)(*[x.ctypes.data for x in J])
        rc = lib().emul_constrained_forward_dynamics_jacobians(ctypes.byref(self.desc), int(slots), k, int(point), _p(b), _p(T12), B, _p(st), _p(ta),
                                                               _p(off), int(off is not None and off.ndim == 3), _p(self._wi(world_inertia, B)),
                                                               float(rho), _p(qdd), _p(wr), ptrs, int(fp64))
        assert rc == 0
        return (qdd, wr, *J)
