"""TEST INFRASTRUCTURE ONLY — ctypes binding of oracle/liboracle.so (fp64 restatement) and, when present,
oracle/_ref/libodelcp.so (the reference's own ODE LCP solver, `make -C oracle REF=<nimblephysics tree>`).
May be imported only by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build(force=False):
    so = os.path.join(_HERE, "liboracle.so")
    src_m = max(os.path.getmtime(os.path.join(_HERE, f)) for f in os.listdir(_HERE) if f.endswith((".cpp", ".hpp")))
    if force or not os.path.exists(so) or os.path.getmtime(so) < src_m:
        subprocess.check_call(["make", "-C", _HERE, "all"], stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(build())
        _LIB.orc_model_create.restype = ctypes.c_void_p
    return _LIB


def _p(a, t=ctypes.c_double):
    return a.ctypes.data_as(ctypes.POINTER(t))


class OracleWorld:
    """One fp64 world built from a RawModel (nimblephysics_b200.modelspec.RawModel)."""

    def __init__(self, raw):
        L = lib()
        self.raw = raw
        self.n = raw.ndof
        self.na = len(raw.action_map)
        f = lambda a: np.ascontiguousarray(a, dtype=np.float64)
        i = lambda a: np.ascontiguousarray(a, dtype=np.int32)
        self._keep = [i(raw.parent), i(raw.jtype), i(raw.dof_off), i(raw.mobile), f(raw.axis), f(raw.Tpj), f(raw.Tcj),
                      f(raw.mass), f(raw.com), f(raw.moment), f(raw.damping), f(raw.spring), f(raw.rest),
                      f(raw.pos_lo), f(raw.pos_hi), f(raw.vel_lo), f(raw.vel_hi), f(raw.force_lo), f(raw.force_hi),
                      f(raw.gravity), i(raw.action_map)]
        k = self._keep
        I = ctypes.c_int
        self.h = ctypes.c_void_p(L.orc_model_create(
            I(raw.nb), I(raw.ndof), _p(k[0], I), _p(k[1], I), _p(k[2], I), _p(k[3], I), _p(k[4]), _p(k[5]), _p(k[6]),
            _p(k[7]), _p(k[8]), _p(k[9]), _p(k[10]), _p(k[11]), _p(k[12]), _p(k[13]), _p(k[14]), _p(k[15]), _p(k[16]),
            _p(k[17]), _p(k[18]), _p(k[19]), ctypes.c_double(raw.dt), I(self.na), _p(k[20], I)))

    def __del__(self):
        try:
            lib().orc_model_destroy(self.h)
        except Exception:
            pass

    def step(self, state, action, want_qdd=False):
        s = np.ascontiguousarray(state, np.float64)
        a = np.ascontiguousarray(action, np.float64)
        out = np.empty(2 * self.n)
        qdd = np.empty(self.n)
        lib().orc_step(self.h, _p(s), _p(a), _p(out), _p(qdd))
        return (out, qdd) if want_qdd else out

    def step_f32(self, state, action):
        s = np.ascontiguousarray(state, np.float64)
        a = np.ascontiguousarray(action, np.float64)
        out = np.empty(2 * self.n)
        lib().orc_step_f32(self.h, _p(s), _p(a), _p(out))
        return out

    def jacobian(self, state, action):
        """d[q+;v+]/d[q;v;tau]  [2n,3n]"""
        s = np.ascontiguousarray(state, np.float64)
        a = np.ascontiguousarray(action, np.float64)
        J = np.empty((2 * self.n, 3 * self.n))
        lib().orc_jacobian(self.h, _p(s), _p(a), _p(J))
        return J

    def backprop(self, state, action, grad_next):
        s = np.ascontiguousarray(state, np.float64)
        a = np.ascontiguousarray(action, np.float64)
        g = np.ascontiguousarray(grad_next, np.float64)
        gs = np.empty(2 * self.n)
        ga = np.empty(self.na)
        lib().orc_backprop(self.h, _p(s), _p(a), _p(g), _p(gs), _p(ga))
        return gs, ga

    def ik(self, state, types, bodies, want_jac=True):
        """IKMapping outputs for raw body indices `bodies` (types: 0 spatial, 1 linear, 2 angular, 3 COM of that body's skeleton):
        (pos, vel, d pos/d q, d vel/d qdot)."""
        s = np.ascontiguousarray(state, np.float64)
        t = np.ascontiguousarray(types, np.int32); b = np.ascontiguousarray(bodies, np.int32)
        sk = np.ascontiguousarray(self.raw.skel_id, np.int32)
        dim = int(sum(6 if k == 0 else 3 for k in t))
        pos, vel = np.empty(dim), np.empty(dim)
        Jp, Jv = np.zeros((dim, self.n)), np.zeros((dim, self.n))
        I = ctypes.c_int
        lib().orc_ik(self.h, _p(s), I(len(t)), _p(t, I), _p(b, I), _p(sk, I), I(dim), _p(pos), _p(vel),
                     _p(Jp) if want_jac else None, _p(Jv) if want_jac else None)
        return pos, vel, Jp, Jv


# ---------------------------------------------------------------------------------------------- contact stage
def _pi(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))


class OracleContactWorld(OracleWorld):
    """OracleWorld + the contact / LCP stage (ConstraintSolver::solve)."""

    MAXC, MAXR = 64, 192

    def __init__(self, raw):
        super().__init__(raw)
        f = lambda a: np.ascontiguousarray(a, dtype=np.float64)
        i = lambda a: np.ascontiguousarray(a, dtype=np.int32)
        k = [i(raw.skel_id), i(raw.shape_body), i(raw.shape_type), f(raw.shape_dims), f(raw.shape_T), f(raw.friction),
             f(raw.restitution)]
        self._keep2 = k
        lib().orc_model_set_contact(self.h, _pi(k[0]), ctypes.c_int(raw.ns), _pi(k[1]), _pi(k[2]), _p(k[3]), _p(k[4]), _p(k[5]),
                                    _p(k[6]), ctypes.c_int(int(raw.penetration_correction)),
                                    ctypes.c_double(raw.contact_clipping_depth), ctypes.c_double(raw.fallback_cfm))
        le = getattr(raw, "limit_enforced", None)
        if le is not None and np.any(le):
            self._keep4 = i(le)
            lib().orc_model_set_limits(self.h, _pi(self._keep4))
        sc = getattr(raw, "self_collision", None)
        if sc is not None and np.any(sc):
            k2 = [i(raw.self_collision), i(raw.adjacent_check)]
            self._keep3 = k2
            lib().orc_model_set_self_collision(self.h, _pi(k2[0]), _pi(k2[1]))

    def step_contact(self, state, action, x_warm=None):
        """-> dict(next_state, nc, point, normal, depth, bodies, type, A, b, lo, hi, findex, x, mapping, status, vstar)"""
        s = np.ascontiguousarray(state, np.float64)
        a = np.ascontiguousarray(action, np.float64)
        C, R = self.MAXC, self.MAXR
        out = np.empty(2 * self.n)
        nc = ctypes.c_int(0)
        status = ctypes.c_int(0)
        pt, nr, dp = np.zeros((C, 3)), np.zeros((C, 3)), np.zeros(C)
        bod, typ = np.zeros((C, 2), np.int32), np.zeros(C, np.int32)
        A, b, lo, hi, x = np.zeros(R * R), np.zeros(R), np.zeros(R), np.zeros(R), np.zeros(R)
        fi, mp = np.zeros(R, np.int32), np.zeros(R, np.int32)
        vstar = np.zeros(self.n)
        if x_warm is None:
            xw, mw = np.zeros(1), -1
        else:
            xw = np.ascontiguousarray(x_warm, np.float64)
            mw = xw.size
        m = lib().orc_step_contact(self.h, _p(s), _p(a), _p(xw), ctypes.c_int(mw), _p(out), ctypes.c_int(C), ctypes.c_int(R),
                                   ctypes.byref(nc), _p(pt), _p(nr), _p(dp), _pi(bod), _pi(typ), _p(A), _p(b), _p(lo), _p(hi),
                                   _pi(fi), _p(x), _pi(mp), ctypes.byref(status), _p(vstar))
        if m < 0:
            raise RuntimeError("oracle contact buffers too small")
        k = nc.value
        return dict(next_state=out, nc=k, point=pt[:k], normal=nr[:k], depth=dp[:k], bodies=bod[:k], type=typ[:k],
                    A=A[:m * m].reshape(m, m), b=b[:m], lo=lo[:m], hi=hi[:m], findex=fi[:m], x=x[:m], mapping=mp[:m],
                    status=status.value, vstar=vstar, m=m)


def solve_chain(A, b, lo, hi, findex, x0=None, fallback_cfm=1e-4):
    n = len(b)
    A = np.ascontiguousarray(A, np.float64)
    b, lo, hi = (np.ascontiguousarray(v, np.float64) for v in (b, lo, hi))
    fi = np.ascontiguousarray(findex, np.int32)
    x = np.zeros(n)
    mp = np.zeros(n, np.int32)
    x0a = np.zeros(n) if x0 is None else np.ascontiguousarray(x0, np.float64)
    st = lib().orc_solve_chain(ctypes.c_int(n), _p(A), _p(b), _p(lo), _p(hi), _pi(fi), _p(x0a), ctypes.c_int(0 if x0 is None else 1),
                               ctypes.c_double(fallback_cfm), _p(x), _pi(mp))
    return x, mp, st


def lcp_valid(A, x, b, hi, lo, findex):
    n = len(b)
    A, x, b, hi, lo = (np.ascontiguousarray(v, np.float64) for v in (A, x, b, hi, lo))
    fi = np.ascontiguousarray(findex, np.int32)
    return bool(lib().orc_lcp_valid(ctypes.c_int(n), _p(A), _p(x), _p(b), _p(hi), _p(lo), _pi(fi)))


def dantzig(A, b, lo, hi, findex, early=False):
    n = len(b)
    A, b, lo, hi = (np.ascontiguousarray(v, np.float64) for v in (A, b, lo, hi))
    fi = np.ascontiguousarray(findex, np.int32)
    x = np.zeros(n)
    ok = lib().orc_dantzig(ctypes.c_int(n), _p(A), _p(b), _p(lo), _p(hi), _pi(fi), ctypes.c_int(int(early)), _p(x))
    return x, bool(ok)


def pinv_solve(Q, b):
    Q = np.ascontiguousarray(Q, np.float64)
    b = np.ascontiguousarray(b, np.float64)
    m, n = Q.shape
    x = np.zeros(n)
    lib().orc_pinv_solve(ctypes.c_int(m), ctypes.c_int(n), _p(Q), _p(b), _p(x))
    return x


_REF = None


def ref_ode():
    """The reference's own dSolveLCP (compiled from a nimblephysics tree by oracle/Makefile) or None."""
    global _REF
    if _REF is None:
        path = os.path.join(_HERE, "_ref", "libodelcp.so")
        _REF = ctypes.CDLL(path) if os.path.exists(path) else False
    return _REF or None


def ref_dsolve_lcp(A, b, lo, hi, findex, early=False):
    L = ref_ode()
    n = len(b)
    pad = L.ref_dPAD(ctypes.c_int(n))
    Ap = np.zeros((n, pad))
    Ap[:, :n] = A
    x, w = np.zeros(n), np.zeros(n)
    bb, ll, hh = (np.array(v, np.float64).copy() for v in (b, lo, hi))
    fi = np.array(findex, np.int32).copy()
    ok = L.ref_dSolveLCP(ctypes.c_int(n), _p(Ap), _p(x), _p(bb), _p(w), ctypes.c_int(0), _p(ll), _p(hh), _pi(fi), ctypes.c_int(int(early)))
    return x, bool(ok)


def _jc(self, state, action, x_warm=None):
    s = np.ascontiguousarray(state, np.float64)
    a = np.ascontiguousarray(action, np.float64)
    J = np.empty((2 * self.n, 3 * self.n))
    xw = np.zeros(1) if x_warm is None else np.ascontiguousarray(x_warm, np.float64)
    rc = lib().orc_jacobian_contact(self.h, _p(s), _p(a), _p(xw), ctypes.c_int(-1 if x_warm is None else xw.size), _p(J))
    return J, rc


def _bc(self, state, action, grad_next, x_warm=None):
    s = np.ascontiguousarray(state, np.float64)
    a = np.ascontiguousarray(action, np.float64)
    g = np.ascontiguousarray(grad_next, np.float64)
    gs, ga = np.empty(2 * self.n), np.empty(self.na)
    xw = np.zeros(1) if x_warm is None else np.ascontiguousarray(x_warm, np.float64)
    rc = lib().orc_backprop_contact(self.h, _p(s), _p(a), _p(xw), ctypes.c_int(-1 if x_warm is None else xw.size), _p(g), _p(gs), _p(ga))
    return gs, ga, rc


OracleContactWorld.jacobian_contact = _jc
OracleContactWorld.backprop_contact = _bc
