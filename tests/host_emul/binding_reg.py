"""TEST HARNESS ONLY: the regressor device functions compiled for the host (tests/host_emul/emul_reg.cpp, which builds on emul.cpp)."""
import ctypes
import os
import subprocess

import numpy as np

from tests.host_emul.binding import _p
from tests.host_emul.binding_id import EmulIdWorld

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.join(_HERE, "..", "..")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libemul_reg.so")
        srcs = [os.path.join(_HERE, f) for f in ("emul_reg.cpp", "emul.cpp")] + [
            os.path.join(_ROOT, "nimblephysics_b200", "csrc", f)
            for f in ("nb2_reg.cuh", "nb2_djac.cuh", "nb2_jac.cuh", "nb2_mm.cuh", "nb2_dyn.cuh", "nb2_math.cuh", "nb2_model.h", "nb2_host_model.h",
                      "nb2_cw.cuh", "nb2_geom.cuh")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so,
                                   os.path.join(_HERE, "emul_reg.cpp")])
        _LIB = ctypes.CDLL(so)
    return _LIB


class EmulRegWorld(EmulIdWorld):
    """EmulIdWorld + the inverse-dynamics and energy regressors (rows in float64 if fp64, else float32)."""

    def id_regressor(self, state, next_vel, fp64=False):
        """-> (Y [B, n, nb, 10], tau_passive [B, n])"""
        dt = np.float64 if fp64 else np.float32
        st, nv = np.ascontiguousarray(state, dt), np.ascontiguousarray(next_vel, dt)
        B = st.shape[0]
        Y = np.full((B, self.n, self.cm.nb, 10), np.nan, dt)
        tp = np.full((B, self.n), np.nan, dt)
        assert lib().emul_regressor(ctypes.byref(self.desc), B, _p(st), _p(nv), _p(Y), _p(tp), None, None, None, int(fp64)) == 0
        return Y, tp

    def energy_regressor(self, state, fp64=False):
        """-> (Y_T [B, nb, 10], Y_U [B, nb, 10], U_spring [B])"""
        dt = np.float64 if fp64 else np.float32
        st = np.ascontiguousarray(state, dt)
        B = st.shape[0]
        YT, YU, Us = np.full((B, self.cm.nb, 10), np.nan, dt), np.full((B, self.cm.nb, 10), np.nan, dt), np.full(B, np.nan, dt)
        assert lib().emul_regressor(ctypes.byref(self.desc), B, _p(st), None, None, None, _p(YT), _p(YU), _p(Us), int(fp64)) == 0
        return YT, YU, Us
