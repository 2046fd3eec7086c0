"""TEST HARNESS ONLY: runs csrc/nb2_dyn.cuh compiled for the host (tests/host_emul/emul.cpp)."""
import ctypes
import os
import subprocess

import numpy as np

from nimblephysics_b200._cabi import Nb2ModelDesc, make_desc

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.join(_HERE, "..", "..")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libemul.so")
        srcs = [os.path.join(_HERE, "emul.cpp")] + [os.path.join(_ROOT, "nimblephysics_b200", "csrc", f)
                                                      for f in ("nb2_dyn.cuh", "nb2_math.cuh", "nb2_model.h", "nb2_host_model.h", "nb2_cw.cuh", "nb2_geom.cuh")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so,
                                   os.path.join(_HERE, "emul.cpp")])
        _LIB = ctypes.CDLL(so)
    return _LIB


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


class EmulWorld:
    """The four step calls take an optional per-world canonical inertia `world_inertia` [B, nb, 10] as their last keyword argument
    (None: the model's table)."""

    def __init__(self, cm):
        self.cm = cm
        self.desc, self._keep = make_desc(cm)
        self.n, self.na = cm.ndof, len(cm.action_map)
        self.sw = lib().emul_saved_words(ctypes.byref(self.desc))

    def _wi(self, world_inertia, B):
        if world_inertia is None:
            return None
        wi = np.asarray(world_inertia, np.float64).reshape(B, 10 * self.cm.nb)
        return np.ascontiguousarray(wi.T)  # word-major [10*nb, B], the layout of the *_pw entry points

    def forward(self, state, action, fp64=False, world_inertia=None):
        state = np.ascontiguousarray(state, np.float32)
        action = np.ascontiguousarray(action, np.float32)
        B = state.shape[0]
        nxt = np.empty_like(state)
        saved = np.zeros((self.sw, B), np.float64 if fp64 else np.float32)
        rc = lib().emul_forward(ctypes.byref(self.desc), B, _p(state), _p(action), _p(nxt), _p(saved), int(fp64),
                                _p(self._wi(world_inertia, B)))
        assert rc == 0
        return nxt, saved

    def backward(self, state, action, saved, gnext, fp64=False, want_inertia_grad=False, world_inertia=None):
        state = np.ascontiguousarray(state, np.float32)
        action = np.ascontiguousarray(action, np.float32)
        gnext = np.ascontiguousarray(gnext, np.float32)
        B = state.shape[0]
        gs = np.empty_like(state)
        ga = np.empty_like(action)
        gi = np.zeros((10 * self.cm.nb, B), np.float32) if want_inertia_grad else None
        rc = lib().emul_backward(ctypes.byref(self.desc), B, _p(state), _p(action), _p(saved), _p(gnext), _p(gs),
                                 _p(ga), int(fp64), _p(gi), _p(self._wi(world_inertia, B)))
        assert rc == 0
        return (gs, ga, gi) if want_inertia_grad else (gs, ga)

    def forward_contact(self, state, action, x_lcp=None, m_lcp=None, small_mc=8, reverse=False, world_inertia=None):
        """fp64 ABA + warp-cooperative contact stage (host build).  -> dict(next, saved, x, m, labels, status, nc, cinfo, crec).
        small_mc: contact capacity of the emulated shared-memory workspace (worlds beyond it retry in the large one);
        reverse: run every CW_FOR of the odd worlds backwards."""
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
        crec = np.zeros((B, lib().emul_contact_rec_doubles(ctypes.byref(self.desc))), np.float64)
        rc = lib().emul_forward_contact(ctypes.byref(self.desc), B, _p(state), _p(action), _p(nxt), _p(saved), _p(x), _p(m),
                                        _p(labels), _p(status), _p(nc), _p(cinfo), _p(crec), int(small_mc), int(reverse),
                                        _p(self._wi(world_inertia, B)))
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
        rc = lib().emul_backward_contact(ctypes.byref(self.desc), B, _p(state), _p(action), _p(saved), _p(crec),
                                         _p(gnext), _p(gs), _p(ga), _p(gi), _p(self.bwd_status),
                                         int(small_mc), int(reverse), _p(self._wi(world_inertia, B)))
        assert rc == 0
        return (gs, ga, gi) if want_inertia_grad else (gs, ga)


def cw_solve_chain(A, b, lo, hi, findex, x0=None, fallback_cfm=1e-4, reverse=False):
    """The warp-cooperative solve chain (csrc/nb2_cw.cuh lcp_chain, host build: one lane) -> (x, mapping, status)."""
    A = np.ascontiguousarray(A, np.float64); b = np.ascontiguousarray(b, np.float64)
    lo = np.ascontiguousarray(lo, np.float64); hi = np.ascontiguousarray(hi, np.float64)
    fi = np.ascontiguousarray(findex, np.int32)
    m = len(b)
    x = np.zeros(m); mp = np.zeros(m, np.int32)
    x0a = np.ascontiguousarray(x0, np.float64) if x0 is not None else np.zeros(m)
    L = lib()
    L.emul_cw_solve_chain.argtypes = [ctypes.c_int] + [ctypes.c_void_p] * 6 + [ctypes.c_int, ctypes.c_double, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    st = L.emul_cw_solve_chain(m, _p(A), _p(b), _p(lo), _p(hi), _p(fi), _p(x0a), int(x0 is not None), float(fallback_cfm), _p(x), _p(mp), int(reverse))
    return x, mp, st
