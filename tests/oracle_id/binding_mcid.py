"""TEST INFRASTRUCTURE ONLY — ctypes binding of the multiple-contact inverse-dynamics oracle (tests/oracle_id/mcid_oracle.cpp, built on
cid_oracle.cpp and id_oracle.cpp)."""
import ctypes
import os
import subprocess

import numpy as np

from tests.oracle_id.binding import IdOracle, _ORACLE, _p
from tests.oracle_id.binding_cid import CidOracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libmcidoracle.so")
        srcs = [os.path.join(_HERE, f) for f in ("mcid_oracle.cpp", "cid_oracle.cpp", "id_oracle.cpp")] + [
            os.path.join(_ORACLE, f) for f in os.listdir(_ORACLE) if f.endswith((".cpp", ".hpp"))]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["g++", "-O3", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(_HERE, "mcid_oracle.cpp")])
        _LIB = ctypes.CDLL(so)
        _LIB.orc_model_create.restype = ctypes.c_void_p
    return _LIB


class McidOracle(CidOracle):
    """CidOracle + multiple-contact inverse dynamics; its model lives in this oracle's library (same model code)."""

    def __init__(self, raw):
        import tests.oracle_id.binding as b

        prev, b._LIB = b._LIB, lib()
        try:
            IdOracle.__init__(self, raw)
        finally:
            b._LIB = prev
        self._lib = lib()

    def multiple_contact_inverse_dynamics(self, bodies, state, next_vel, guess=None, want_jac=False):
        """bodies: raw body indices [k]; guess [k, 6] or None.  -> tau [n], wrenches [k, 6], and with want_jac
        d[tau; wrenches] / d[q; qdot; v'; guess] [n + 6k, 3n + 6k]."""
        k = len(bodies)
        bi = np.ascontiguousarray(bodies, np.int32)
        s = np.ascontiguousarray(state, np.float64)
        vn = np.ascontiguousarray(next_vel, np.float64)
        g = np.ascontiguousarray(guess, np.float64).reshape(k, 6) if guess is not None else None
        tau, w = np.empty(self.n), np.empty((k, 6))
        J = np.empty((self.n + 6 * k, 3 * self.n + 6 * k)) if want_jac else None
        self._lib.orc_multiple_contact_inverse_dynamics(self.h, ctypes.c_int(k), _p(bi, ctypes.c_int), _p(s), _p(vn),
                                                        _p(g) if g is not None else None, _p(tau), _p(w), _p(J) if want_jac else None)
        return (tau, w, J) if want_jac else (tau, w)
