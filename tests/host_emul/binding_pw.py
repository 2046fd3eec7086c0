"""TEST HARNESS ONLY: the per-world-inertia harness (tests/host_emul/emul_pw.cpp) — csrc/nb2_dyn.cuh compiled for the host with
every world of the batch stepping with its own canonical inertia table."""
import ctypes
import os
import subprocess

import numpy as np

from tests.host_emul.binding import EmulWorld, _p
from tests.host_emul.binding import lib as emul_lib

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.join(_HERE, "..", "..")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libemul_pw.so")
        srcs = [os.path.join(_HERE, "emul_pw.cpp")] + [os.path.join(_ROOT, "nimblephysics_b200", "csrc", f)
                                                         for f in ("nb2_dyn.cuh", "nb2_math.cuh", "nb2_model.h", "nb2_host_model.h", "nb2_cw.cuh", "nb2_geom.cuh")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so,
                                   os.path.join(_HERE, "emul_pw.cpp")])
        _LIB = ctypes.CDLL(so)
    return _LIB


class EmulWorldPW(EmulWorld):
    """EmulWorld whose four step calls take an optional per-world canonical inertia `world_inertia` [B, nb, 10]
    (None: the model's table, i.e. exactly EmulWorld's computation)."""

    def _wi(self, world_inertia, B):
        if world_inertia is None:
            return None
        wi = np.asarray(world_inertia, np.float64).reshape(B, 10 * self.cm.nb)
        return np.ascontiguousarray(wi.T)  # word-major [10*nb, B], the layout of the *_pw entry points

    @staticmethod
    def _pp(a):
        return _p(a) if a is not None else None

    def forward(self, state, action, fp64=False, world_inertia=None):
        state = np.ascontiguousarray(state, np.float32)
        action = np.ascontiguousarray(action, np.float32)
        B = state.shape[0]
        nxt = np.empty_like(state)
        saved = np.zeros((self.sw, B), np.float64 if fp64 else np.float32)
        wi = self._wi(world_inertia, B)
        rc = lib().emulpw_forward(ctypes.byref(self.desc), B, _p(state), _p(action), _p(nxt), _p(saved), int(fp64), self._pp(wi))
        assert rc == 0
        return nxt, saved

    def backward(self, state, action, saved, gnext, fp64=False, want_inertia_grad=False, world_inertia=None):
        state = np.ascontiguousarray(state, np.float32)
        action = np.ascontiguousarray(action, np.float32)
        gnext = np.ascontiguousarray(gnext, np.float32)
        B = state.shape[0]
        gs, ga = np.empty_like(state), np.empty_like(action)
        gi = np.zeros((10 * self.cm.nb, B), np.float32) if want_inertia_grad else None
        wi = self._wi(world_inertia, B)
        rc = lib().emulpw_backward(ctypes.byref(self.desc), B, _p(state), _p(action), _p(saved), _p(gnext), _p(gs), _p(ga), int(fp64),
                                   self._pp(gi), self._pp(wi))
        assert rc == 0
        return (gs, ga, gi) if want_inertia_grad else (gs, ga)

    def forward_contact(self, state, action, x_lcp=None, m_lcp=None, small_mc=8, reverse=False, world_inertia=None):
        from nimblephysics_b200._cabi import MAX_CONTACTS, MAX_ROWS

        state = np.ascontiguousarray(state, np.float32)
        action = np.ascontiguousarray(action, np.float32)
        B = state.shape[0]
        nxt = np.empty_like(state)
        saved = np.zeros((B, self.sw), np.float64)  # world-major
        x = np.zeros((B, MAX_ROWS)) if x_lcp is None else np.ascontiguousarray(x_lcp, np.float64).copy()
        m = np.full(B, -1, np.int32) if m_lcp is None else np.ascontiguousarray(m_lcp, np.int32).copy()
        labels = np.zeros((B, MAX_ROWS), np.int32)
        status = np.zeros(B, np.int32)
        nc = np.zeros(B, np.int32)
        cinfo = np.zeros((B, MAX_CONTACTS, 10), np.float32)
        crec = np.zeros((B, emul_lib().emul_contact_rec_doubles(ctypes.byref(self.desc))), np.float64)
        wi = self._wi(world_inertia, B)
        rc = lib().emulpw_forward_contact(ctypes.byref(self.desc), B, _p(state), _p(action), _p(nxt), _p(saved), _p(x), _p(m), _p(labels),
                                          _p(status), _p(nc), _p(cinfo), _p(crec), int(small_mc), int(reverse), self._pp(wi))
        assert rc == 0
        return dict(next=nxt, saved=saved, x=x, m=m, labels=labels, status=status, nc=nc, cinfo=cinfo, crec=crec)

    def backward_contact(self, state, action, saved, crec, gnext, want_inertia_grad=False, small_mc=8, reverse=False, world_inertia=None):
        state = np.ascontiguousarray(state, np.float32)
        action = np.ascontiguousarray(action, np.float32)
        gnext = np.ascontiguousarray(gnext, np.float32)
        B = state.shape[0]
        gs, ga = np.empty_like(state), np.empty_like(action)
        gi = np.zeros((10 * self.cm.nb, B), np.float32) if want_inertia_grad else None
        self.bwd_status = np.zeros(B, np.int32)
        wi = self._wi(world_inertia, B)
        rc = lib().emulpw_backward_contact(ctypes.byref(self.desc), B, _p(state), _p(action), _p(saved), _p(crec), _p(gnext), _p(gs), _p(ga),
                                           self._pp(gi), _p(self.bwd_status), int(small_mc), int(reverse), self._pp(wi))
        assert rc == 0
        return (gs, ga, gi) if want_inertia_grad else (gs, ga)
