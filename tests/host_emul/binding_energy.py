"""TEST HARNESS ONLY: the energy-and-momentum device functions compiled for the host (tests/host_emul/emul_energy.cpp, which builds on
emul.cpp)."""
import ctypes
import os
import subprocess

import numpy as np

from tests.host_emul.binding import _p
from tests.host_emul.binding_jacd import EmulJacdWorld

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.join(_HERE, "..", "..")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libemul_energy.so")
        srcs = [os.path.join(_HERE, f) for f in ("emul_energy.cpp", "emul.cpp")] + [
            os.path.join(_ROOT, "nimblephysics_b200", "csrc", f)
            for f in ("nb2_energy.cuh", "nb2_jac.cuh", "nb2_mm.cuh", "nb2_dyn.cuh", "nb2_math.cuh", "nb2_model.h", "nb2_host_model.h", "nb2_cw.cuh",
                      "nb2_geom.cuh")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so,
                                   os.path.join(_HERE, "emul_energy.cpp")])
        _LIB = ctypes.CDLL(so)
    return _LIB


class EmulEnergyWorld(EmulJacdWorld):
    """EmulJacdWorld + the kinetic and potential energy and momentum of a tree and their backward, at states [B, 2n] (rows in float64 if
    fp64, else float32)."""

    def energy_momentum(self, state, root, fp64=False, world_inertia=None):
        """-> (kinetic [B], potential [B], momentum [B, 6])"""
        dt = np.float64 if fp64 else np.float32
        st = np.ascontiguousarray(state, dt)
        B = st.shape[0]
        T, U, h = np.empty(B, dt), np.empty(B, dt), np.empty((B, 6), dt)
        assert lib().emul_energy_momentum(ctypes.byref(self.desc), B, _p(st), int(root), _p(self._wi(world_inertia, B)), _p(T), _p(U), _p(h),
                                          None, None, None, None, None, int(fp64)) == 0
        return T, U, h

    def energy_momentum_backward(self, state, root, gT, gU, gh, fp64=False, world_inertia=None):
        """-> (grad_state [B, 2n], grad_inertia fp64 [10*nb, B])"""
        dt = np.float64 if fp64 else np.float32
        st = np.ascontiguousarray(state, dt)
        B = st.shape[0]
        gT, gU, gh = (np.ascontiguousarray(x, dt) for x in (gT, gU, gh))
        gs = np.empty((B, 2 * self.n), dt)
        gi = np.full((10 * self.cm.nb, B), np.nan, np.float64)
        assert lib().emul_energy_momentum(ctypes.byref(self.desc), B, _p(st), int(root), _p(self._wi(world_inertia, B)), None, None, None, _p(gT),
                                          _p(gU), _p(gh), _p(gs), _p(gi), int(fp64)) == 0
        return gs, gi
