"""TEST HARNESS ONLY: the multiple-contact inverse-dynamics device functions compiled for the host (tests/host_emul/emul_mcid.cpp, which
builds on emul_cid.cpp and emul_id.cpp)."""
import ctypes
import os
import subprocess

import numpy as np

from tests.host_emul.binding import _p
from tests.host_emul.binding_cid import EmulCidWorld

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.join(_HERE, "..", "..")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libemul_mcid.so")
        srcs = [os.path.join(_HERE, f) for f in ("emul_mcid.cpp", "emul_cid.cpp", "emul_id.cpp", "emul.cpp")] + [
            os.path.join(_ROOT, "nimblephysics_b200", "csrc", f)
            for f in ("nb2_dyn.cuh", "nb2_math.cuh", "nb2_model.h", "nb2_host_model.h", "nb2_cw.cuh", "nb2_geom.cuh")] + [
            os.path.join(_ROOT, "include", "nb2.h")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so,
                                   os.path.join(_HERE, "emul_mcid.cpp")])
        _LIB = ctypes.CDLL(so)
    return _LIB


class EmulMcidWorld(EmulCidWorld):
    """EmulCidWorld + the multiple-contact inverse-dynamics forward and backward (bodies: canonical indices [k], points [k, 3]: each body's
    origin in its canonical frame; rows in float64 if fp64, else float32)."""

    @staticmethod
    def _set(bodies, points):
        b = np.ascontiguousarray(bodies, np.int32)
        return len(b), b, np.ascontiguousarray(points, np.float64).reshape(len(b), 3)

    def multiple_contact_inverse_dynamics(self, bodies, points, state, next_vel, guess=None, fp64=False, world_inertia=None):
        """-> (tau [B, n], wrenches [B, k, 6], the saved stream [words, B])"""
        k, b, p = self._set(bodies, points)
        dt = np.float64 if fp64 else np.float32
        state = np.ascontiguousarray(state, dt)
        next_vel = np.ascontiguousarray(next_vel, dt)
        guess = np.ascontiguousarray(guess, dt) if guess is not None else None
        B = state.shape[0]
        tau = np.empty((B, self.n), dt)
        wrench = np.empty((B, k, 6), dt)
        saved = np.zeros((self.sw, B), dt)
        rc = lib().emul_multiple_contact_inverse_dynamics(ctypes.byref(self.desc), B, k, _p(b), _p(p), _p(state), _p(next_vel), _p(guess),
                                                          _p(tau), _p(wrench), _p(saved), int(fp64), _p(self._wi(world_inertia, B)))
        assert rc == 0, rc
        return tau, wrench, saved

    def multiple_contact_inverse_dynamics_backward(self, bodies, points, state, saved, wrench, grad_tau, grad_wrench, guess=None, fp64=False,
                                                   world_inertia=None):
        """-> (grad_state [B, 2n], grad_next_vel [B, n], grad_inertia fp64 [10*nb, B], grad_guess [B, k, 6])"""
        k, b, p = self._set(bodies, points)
        dt = np.float64 if fp64 else np.float32
        state = np.ascontiguousarray(state, dt)
        wrench = np.ascontiguousarray(wrench, dt)
        guess = np.ascontiguousarray(guess, dt) if guess is not None else None
        grad_tau = np.ascontiguousarray(grad_tau, dt)
        grad_wrench = np.ascontiguousarray(grad_wrench, dt)
        B = state.shape[0]
        gs = np.empty((B, 2 * self.n), dt)
        gn = np.empty((B, self.n), dt)
        gi = np.zeros((10 * self.cm.nb, B), np.float64)
        gg = np.empty((B, k, 6), dt)
        rc = lib().emul_multiple_contact_inverse_dynamics_backward(ctypes.byref(self.desc), B, k, _p(b), _p(p), _p(state), _p(saved), _p(wrench),
                                                                   _p(guess), _p(grad_tau), _p(grad_wrench), _p(gs), _p(gn), _p(gi), _p(gg),
                                                                   int(fp64), _p(self._wi(world_inertia, B)))
        assert rc == 0, rc
        return gs, gn, gi, gg
