"""TEST INFRASTRUCTURE ONLY — ctypes binding of the inverse-dynamics oracle (tests/oracle_id/id_oracle.cpp, built on oracle/nb_oracle.cpp)."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(_HERE, "..", "..", "oracle")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libidoracle.so")
        srcs = [os.path.join(_HERE, "id_oracle.cpp")] + [os.path.join(_ORACLE, f) for f in os.listdir(_ORACLE) if f.endswith((".cpp", ".hpp"))]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["g++", "-O3", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(_HERE, "id_oracle.cpp")])
        _LIB = ctypes.CDLL(so)
        _LIB.orc_model_create.restype = ctypes.c_void_p
    return _LIB


def _p(a, t=ctypes.c_double):
    return a.ctypes.data_as(ctypes.POINTER(t))


class IdOracle:
    """Contact-free inverse dynamics of one fp64 world built from a RawModel (the step oracle's model)."""

    def __init__(self, raw):
        L = lib()
        self.n = raw.ndof
        f = lambda a: np.ascontiguousarray(a, dtype=np.float64)
        i = lambda a: np.ascontiguousarray(a, dtype=np.int32)
        self._keep = k = [i(raw.parent), i(raw.jtype), i(raw.dof_off), i(raw.mobile), f(raw.axis), f(raw.Tpj), f(raw.Tcj),
                          f(raw.mass), f(raw.com), f(raw.moment), f(raw.damping), f(raw.spring), f(raw.rest),
                          f(raw.pos_lo), f(raw.pos_hi), f(raw.vel_lo), f(raw.vel_hi), f(raw.force_lo), f(raw.force_hi),
                          f(raw.gravity), i(raw.action_map)]
        I = ctypes.c_int
        self.h = ctypes.c_void_p(L.orc_model_create(
            I(raw.nb), I(raw.ndof), _p(k[0], I), _p(k[1], I), _p(k[2], I), _p(k[3], I), _p(k[4]), _p(k[5]), _p(k[6]),
            _p(k[7]), _p(k[8]), _p(k[9]), _p(k[10]), _p(k[11]), _p(k[12]), _p(k[13]), _p(k[14]), _p(k[15]), _p(k[16]),
            _p(k[17]), _p(k[18]), _p(k[19]), ctypes.c_double(raw.dt), I(len(raw.action_map)), _p(k[20], I)))

    def __del__(self):
        try:
            lib().orc_model_destroy(self.h)
        except Exception:
            pass

    def inverse_dynamics(self, state, next_vel, want_jac=False):
        """tau [n], and with want_jac d tau / d[q; qdot; v'] [n, 3n] (dual numbers)."""
        s = np.ascontiguousarray(state, np.float64)
        vn = np.ascontiguousarray(next_vel, np.float64)
        tau = np.empty(self.n)
        J = np.empty((self.n, 3 * self.n)) if want_jac else None
        lib().orc_inverse_dynamics(self.h, _p(s), _p(vn), _p(tau), _p(J) if want_jac else None)
        return (tau, J) if want_jac else tau
