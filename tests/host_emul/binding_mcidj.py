"""TEST HARNESS ONLY: the dense contact-inverse-dynamics Jacobian device functions compiled for the host (tests/host_emul/emul_mcidj.cpp,
which builds on emul.cpp)."""
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
        so = os.path.join(_HERE, "libemul_mcidj.so")
        srcs = [os.path.join(_HERE, f) for f in ("emul_mcidj.cpp", "emul.cpp")] + [
            os.path.join(_ROOT, "nimblephysics_b200", "csrc", f)
            for f in ("nb2_mcidj.cuh", "nb2_djac.cuh", "nb2_dyn.cuh", "nb2_math.cuh", "nb2_model.h", "nb2_host_model.h", "nb2_cw.cuh",
                      "nb2_geom.cuh")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so,
                                   os.path.join(_HERE, "emul_mcidj.cpp")])
        _LIB = ctypes.CDLL(so)
    return _LIB


class EmulMcidjWorld(EmulWorld):
    """EmulWorld + the dense Jacobians of multiple-contact (k = 1: one-body) contact inverse dynamics (bodies: canonical indices [k],
    points [k, 3]: each body's origin in its canonical frame; rows in float64 if fp64, else float32)."""

    def contact_jacobians(self, bodies, points, state, next_vel, guess=None, fp64=False, world_inertia=None, slots=32):
        """-> (tau [B, n], wrenches [B, k, 6], T_q, T_qdot, T_next_vel [B, n, n], T_guess [B, n, 6k], W_q, W_qdot, W_next_vel [B, 6k, n],
        W_guess [B, 6k, 6k])"""
        b = np.ascontiguousarray(bodies, np.int32)
        k = len(b)
        p = np.ascontiguousarray(points, np.float64).reshape(k, 3)
        dt = np.float64 if fp64 else np.float32
        state = np.ascontiguousarray(state, dt)
        next_vel = np.ascontiguousarray(next_vel, dt)
        guess = np.ascontiguousarray(guess, dt) if guess is not None else None
        B, n, m = state.shape[0], self.n, 6 * k
        tau, w = np.empty((B, n), dt), np.empty((B, k, 6), dt)
        J = [np.empty((B, n, n), dt) for _ in range(3)] + [np.empty((B, n, m), dt)] + [np.empty((B, m, n), dt) for _ in range(3)] + [
            np.empty((B, m, m), dt)]
        ptrs = (ctypes.c_void_p * 8)(*[a.ctypes.data for a in J])
        rc = lib().emul_contact_inverse_dynamics_jacobians(ctypes.byref(self.desc), int(slots), B, k, _p(b), _p(p), _p(state), _p(next_vel),
                                                           _p(guess), _p(tau), _p(w), ptrs, int(fp64), _p(self._wi(world_inertia, B)))
        assert rc == 0, rc
        return (tau, w, *J)
