"""TEST INFRASTRUCTURE ONLY — ctypes binding of the contact inverse-dynamics oracle (tests/oracle_id/cid_oracle.cpp, built on id_oracle.cpp)."""
import ctypes
import os
import subprocess

import numpy as np

from tests.oracle_id.binding import IdOracle, _ORACLE, _p

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libcidoracle.so")
        srcs = [os.path.join(_HERE, f) for f in ("cid_oracle.cpp", "id_oracle.cpp")] + [
            os.path.join(_ORACLE, f) for f in os.listdir(_ORACLE) if f.endswith((".cpp", ".hpp"))]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["g++", "-O3", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(_HERE, "cid_oracle.cpp")])
        _LIB = ctypes.CDLL(so)
        _LIB.orc_model_create.restype = ctypes.c_void_p
    return _LIB


class CidOracle(IdOracle):
    """IdOracle + contact inverse dynamics; its model lives in the contact oracle's library (same model code)."""

    def __init__(self, raw):
        import tests.oracle_id.binding as b

        prev, b._LIB = b._LIB, lib()
        try:
            super().__init__(raw)
        finally:
            b._LIB = prev
        self._lib = lib()

    def __del__(self):
        try:
            self._lib.orc_model_destroy(self.h)
        except Exception:
            pass

    def inverse_dynamics(self, state, next_vel, want_jac=False):
        s = np.ascontiguousarray(state, np.float64)
        vn = np.ascontiguousarray(next_vel, np.float64)
        tau = np.empty(self.n)
        J = np.empty((self.n, 3 * self.n)) if want_jac else None
        self._lib.orc_inverse_dynamics(self.h, _p(s), _p(vn), _p(tau), _p(J) if want_jac else None)
        return (tau, J) if want_jac else tau

    def contact_inverse_dynamics(self, body, state, next_vel, want_jac=False):
        """body: raw body index.  -> tau [n], wrench [6], and with want_jac d[tau; wrench] / d[q; qdot; v'] [n + 6, 3n]."""
        s = np.ascontiguousarray(state, np.float64)
        vn = np.ascontiguousarray(next_vel, np.float64)
        tau, w = np.empty(self.n), np.empty(6)
        J = np.empty((self.n + 6, 3 * self.n)) if want_jac else None
        self._lib.orc_contact_inverse_dynamics(self.h, ctypes.c_int(int(body)), _p(s), _p(vn), _p(tau), _p(w), _p(J) if want_jac else None)
        return (tau, w, J) if want_jac else (tau, w)
