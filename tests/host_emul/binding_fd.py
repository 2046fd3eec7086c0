"""TEST HARNESS ONLY: the forward-dynamics device functions compiled for the host (tests/host_emul/emul_fd.cpp, which builds on emul.cpp)."""
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
        so = os.path.join(_HERE, "libemul_fd.so")
        srcs = [os.path.join(_HERE, f) for f in ("emul_fd.cpp", "emul.cpp")] + [
            os.path.join(_ROOT, "nimblephysics_b200", "csrc", f)
            for f in ("nb2_dyn.cuh", "nb2_math.cuh", "nb2_model.h", "nb2_host_model.h", "nb2_cw.cuh", "nb2_geom.cuh")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so,
                                   os.path.join(_HERE, "emul_fd.cpp")])
        _LIB = ctypes.CDLL(so)
    return _LIB


class EmulFdWorld(EmulWorld):
    """EmulWorld + the forward-dynamics forward and backward (rows in float64 if fp64, else float32)."""

    def forward_dynamics(self, state, tau, fp64=False, world_inertia=None, split=False):
        """-> (qdd [B, n], the saved stream [words, B]).  split: read q and qdot from two separate [B, n] arrays (the legacy entry's layout)
        instead of the state rows."""
        dt = np.float64 if fp64 else np.float32
        state = np.ascontiguousarray(state, dt)
        tau = np.ascontiguousarray(tau, dt)
        B, n = state.shape[0], self.n
        if split:
            q, v = np.ascontiguousarray(state[:, :n]), np.ascontiguousarray(state[:, n:])
            qa, qs, va, vs = _p(q), n, _p(v), n
        else:
            qa, qs, va, vs = _p(state), 2 * n, ctypes.c_void_p(state.ctypes.data + n * state.itemsize), 2 * n
        qdd = np.empty((B, n), dt)
        saved = np.zeros((self.sw, B), dt)
        rc = lib().emul_forward_dynamics(ctypes.byref(self.desc), B, qa, qs, va, vs, _p(tau), _p(qdd), _p(saved), int(fp64),
                                         _p(self._wi(world_inertia, B)))
        assert rc == 0
        return qdd, saved

    def forward_dynamics_backward(self, state, saved, grad_qdd, fp64=False, world_inertia=None):
        """-> (grad_state [B, 2n], grad_tau [B, n], grad_inertia fp64 [10*nb, B])"""
        dt = np.float64 if fp64 else np.float32
        state = np.ascontiguousarray(state, dt)
        grad_qdd = np.ascontiguousarray(grad_qdd, dt)
        B = state.shape[0]
        gs = np.empty((B, 2 * self.n), dt)
        gt = np.empty((B, self.n), dt)
        gi = np.zeros((10 * self.cm.nb, B), np.float64)
        rc = lib().emul_forward_dynamics_backward(ctypes.byref(self.desc), B, _p(state), _p(saved), _p(grad_qdd), _p(gs), _p(gt), _p(gi),
                                                  int(fp64), _p(self._wi(world_inertia, B)))
        assert rc == 0
        return gs, gt, gi
