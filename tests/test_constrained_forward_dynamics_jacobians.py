"""Dense Jacobians of constrained forward dynamics on the CPU: the host-emulated program (csrc/nb2_cfd.cuh cfdj_world,
tests/host_emul/emul_cfdj.cpp) against the emulated VJP seeded with each unit vector, on every lane schedule and row-slot count; all six
blocks against central differences of the fp64 oracle; the closed forms of the tau and qdot blocks in the oracle's M, J, Jdot and
A = J M^-1 J^T + rho I; the singular set; and the argument checks of nimblephysics_b200.constrained_forward_dynamics_jacobians."""
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import nimblephysics_b200 as nb
from oracle.binding import OracleWorld
from tests.host_emul.binding_cfdj import EmulCfdjWorld
from tests.test_constrained_forward_dynamics import FEET, LIMBS, _setup, oracle_cfd
from tests.test_forward_dynamics import fd_inputs
from tests.test_inverse_dynamics import _compile
from tests.test_world_jacobian_deriv import oracle_point_deriv
from tests.util import load_raw, rel_err

ROW_CASES = [("atlas", FEET, False), ("atlas", LIMBS, False), ("atlas", LIMBS, True), ("atlas_sdf", FEET, False), ("free_child", None, True)]


def vjp_rows(ew, s, tau, bodies, T, off, point, rho=0.0, slots=8):
    """the six blocks assembled from the emulated VJP seeded with e_i on qdd and e_r on the wrenches, [B, n or m, n] each"""
    B, n, k, r = s.shape[0], ew.n, len(bodies), 3 if point else 6
    m = k * r
    blocks = [np.empty((B, n, n)) for _ in range(3)] + [np.empty((B, m, n)) for _ in range(3)]
    for i in range(n + m):
        gq, gw = np.zeros((B, n)), np.zeros((B, m))
        (gq[:, i] if i < n else gw[:, i - n])[...] = 1.0
        gs, gt, _, _ = ew.constrained_forward_dynamics_backward(s, tau, bodies, T, gq, gw.reshape(B, k, r), off, point=point, rho=rho, fp64=True,
                                                                slots=slots)
        o, row = (0, i) if i < n else (3, i - n)
        blocks[o][:, row], blocks[o + 1][:, row], blocks[o + 2][:, row] = gs[:, :n], gs[:, n:], gt
    return blocks


@pytest.mark.parametrize("name,names,point", ROW_CASES)
def test_emulated_rows_are_the_vjp_bit_for_bit(name, names, point):
    raw, cm, ris, (bodies, T) = _setup(name, names)
    ew = EmulCfdjWorld(cm)
    B, k, n = 2, len(ris), raw.ndof
    s, tau = fd_inputs(raw, B, seed=41)
    s, tau = s.astype(np.float64), tau.astype(np.float64)
    off = np.random.default_rng(42).uniform(-0.1, 0.1, (B, k, 3))
    out = ew.constrained_forward_dynamics_jacobians(s, tau, bodies, T, off, point=point, fp64=True)
    q, w = ew.constrained_forward_dynamics(s, tau, bodies, T, off, point=point, fp64=True)
    assert np.array_equal(out[0], q) and np.array_equal(out[1], w)
    m = k * (3 if point else 6)
    ref = vjp_rows(ew, s, tau, bodies, T, off, point)
    for got, want in zip(out[2:5] + tuple(x.reshape(B, m, n) for x in out[5:]), ref):
        # the per-seed code is the VJP's own (cfd_point_form, the mu / g / FD-backward arithmetic, cfd_point_vjps): equal bit for bit
        assert np.array_equal(got, want), rel_err(got, want)


@pytest.mark.parametrize("lanes", [2, 4, 8])
def test_emulated_lane_schedules_and_slot_counts_agree(lanes):
    raw, cm1, ris, (bodies, T) = _setup("atlas", LIMBS)
    e1, ek = EmulCfdjWorld(cm1), EmulCfdjWorld(_compile(raw, lanes))
    s, tau = fd_inputs(raw, 3, seed=lanes)
    off = np.random.default_rng(lanes).uniform(-0.1, 0.1, (3, 4, 3))
    ref = e1.constrained_forward_dynamics_jacobians(s, tau, bodies, T, off, fp64=True)
    for ew, slots in ((ek, 8), (ek, 1), (e1, 1)):
        got = ew.constrained_forward_dynamics_jacobians(s, tau, bodies, T, off, fp64=True, slots=slots)
        for a, b in zip(got, ref):
            assert rel_err(a, b) < 1e-12


def _central(f, x, h=1e-5):
    cols = []
    for c in range(x.size):
        xp, xm = x.copy(), x.copy()
        xp[c] += h
        xm[c] -= h
        cols.append((f(xp) - f(xm)) / (2 * h))
    return np.stack(cols, -1)


@pytest.mark.parametrize("name,names,point", [("free_child", None, True), ("atlas", FEET, False), ("atlas", ["l_foot", "r_hand"], True)])
def test_emulated_blocks_match_oracle_differences(name, names, point):
    raw, cm, ris, (bodies, T) = _setup(name, names)
    ew = EmulCfdjWorld(cm)
    k, n = len(ris), raw.ndof
    s, tau = fd_inputs(raw, 1, seed=31)
    s, tau = s.astype(np.float64), tau.astype(np.float64)
    off = np.random.default_rng(32).uniform(-0.1, 0.1, (1, k, 3))
    out = ew.constrained_forward_dynamics_jacobians(s, tau, bodies, T, off, point=point, fp64=True)
    flat = lambda q, w: np.concatenate([q, w.reshape(-1)])
    Ds = _central(lambda x: flat(*oracle_cfd(raw, x, tau[0], ris, off[0], point)), s[0])
    Dt = _central(lambda x: flat(*oracle_cfd(raw, s[0], x, ris, off[0], point)), tau[0])
    m = k * (3 if point else 6)
    want = [Ds[:n, :n], Ds[:n, n:], Dt[:n], Ds[n:, :n], Ds[n:, n:], Dt[n:]]
    for got, ref in zip([x[0] for x in out[2:5]] + [x[0].reshape(m, n) for x in out[5:]], want):
        assert rel_err(got, ref) < 1e-6, rel_err(got, ref)


def _point_form(raw, q, ris, offs, dW, point):
    """d lam from d wrench [m, ...]: lam_a = w_a - p x w_l for a 6-D contact (p does not depend on qdot or tau)"""
    if point:
        return dW
    ow, out = OracleWorld(raw), dW.copy()
    for i, (ri, o) in enumerate(zip(ris, offs)):
        pos = ow.ik(np.concatenate([q, 0 * q]), [0], [ri], want_jac=False)[0]
        p = pos[3:6] + Rotation.from_rotvec(pos[:3]).as_matrix() @ o
        out[6 * i:6 * i + 3] -= np.cross(p, dW[6 * i + 3:6 * i + 6], axis=0)
    return out


@pytest.mark.parametrize("rho", [0.0, 1e-3])
@pytest.mark.parametrize("names,point", [(FEET, False), (LIMBS, True)])
def test_emulated_closed_forms(rho, names, point):
    raw, cm, ris, (bodies, T) = _setup("atlas", names)
    ew = EmulCfdjWorld(cm)
    B, k, n = 2, len(ris), raw.ndof
    s, tau = fd_inputs(raw, B, seed=51)
    s, tau = s.astype(np.float64), tau.astype(np.float64)
    off = np.random.default_rng(52).uniform(-0.1, 0.1, (k, 3))
    rows = slice(3, 6) if point else slice(0, 6)
    out = ew.constrained_forward_dynamics_jacobians(s, tau, bodies, T, off, point=point, rho=rho, fp64=True)
    m = k * (3 if point else 6)
    for w in range(B):
        q, qd = s[w, :n], s[w, n:]
        _, _, J, _, M, _ = oracle_cfd(raw, s[w], tau[w], ris, off, point, rho, full=True)
        Jdv = lambda v: np.concatenate([oracle_point_deriv(raw, q, v, ri, o)[rows] for ri, o in zip(ris, off)]) @ v
        dJdv = _central(Jdv, qd)  # d(Jdot qdot)/dqdot
        Mi = np.linalg.inv(M)
        A = J @ Mi @ J.T + rho * np.eye(m)
        dqdd_dtau, dqdd_dqdot = out[4][w], out[3][w]
        dlam_dtau = _point_form(raw, q, ris, off, out[7][w].reshape(m, n), point)
        dlam_dqdot = _point_form(raw, q, ris, off, out[6][w].reshape(m, n), point)
        assert rel_err(dqdd_dtau, Mi - Mi @ J.T @ np.linalg.solve(A, J @ Mi)) < 1e-9
        assert rel_err(dqdd_dtau, dqdd_dtau.T) < 1e-10
        assert rel_err(dlam_dtau, -np.linalg.solve(A, J @ Mi)) < 1e-9
        scale = np.abs(J @ dqdd_dtau).max() + np.abs(dlam_dtau).max()
        assert np.abs(J @ dqdd_dtau + rho * dlam_dtau).max() < 1e-10 * scale
        # J qdd + Jdot qdot = -rho lam, differentiated in qdot: J dqdd/dqdot + d(Jdot qdot)/dqdot = -rho dlam/dqdot.  Jdot is linear in qdot,
        # but Jdot(qdot) qdot = sum_jc D_rcj qdot_j qdot_c with D not symmetric in (c, j) (the brackets of a chain's screws; a free root's
        # ad_v v = 0), so its derivative is not 2 Jdot; it is taken from central differences of the oracle's Jdot qdot.
        scale = np.abs(dJdv).max() + np.abs(J @ dqdd_dqdot).max()
        assert np.abs(J @ dqdd_dqdot + dJdv + rho * dlam_dqdot).max() < 1e-7 * scale


def singular_middle_world():
    """free_child's three-joint arm held at a point of its last link: at the link's origin, which lies on the last joint's axis, the point
    moves in two directions only and J M^-1 J^T is singular.  Three worlds, the middle one held there: (raw, cm, bodies, T, s, tau, off)."""
    raw, cm, _, (bodies, T) = _setup("free_child", None)
    s, tau = fd_inputs(raw, 3, seed=61)
    off = np.zeros((3, 1, 3))
    off[0, 0], off[2, 0] = [0.05, -0.03, 0.2], [0.1, 0.1, -0.1]
    return raw, cm, bodies[1:], T[1:], s.astype(np.float64), tau.astype(np.float64), off


def test_emulated_singular_world_is_nan_and_isolated():
    """the singular world's outputs and blocks are all NaN; the other worlds' are their own single-world results; damping makes it finite"""
    raw, cm, bodies, T, s, tau, off = singular_middle_world()
    ew = EmulCfdjWorld(cm)
    for fp64 in (False, True):
        out = ew.constrained_forward_dynamics_jacobians(s, tau, bodies, T, off, point=True, fp64=fp64)
        for w in (0, 2):
            one = ew.constrained_forward_dynamics_jacobians(s[w:w + 1], tau[w:w + 1], bodies, T, off[w:w + 1], point=True, fp64=fp64)
            for a, b in zip(out, one):
                assert np.isnan(a[1]).all() and np.isfinite(b).all() and np.array_equal(a[w:w + 1], b)
    out = ew.constrained_forward_dynamics_jacobians(s, tau, bodies, T, off, point=True, rho=1e-3, fp64=True)
    assert all(np.isfinite(x).all() for x in out)


def test_emulated_empty_batch():
    raw, cm, ris, (bodies, T) = _setup("atlas", FEET)
    n = raw.ndof
    out = EmulCfdjWorld(cm).constrained_forward_dynamics_jacobians(np.zeros((0, 2 * n)), np.zeros((0, n)), bodies, T, fp64=True)
    assert [x.shape for x in out] == [(0, n), (0, 2, 6)] + [(0, n, n)] * 3 + [(0, 2, 6, n)] * 3


def test_value_errors():
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    n = raw.ndof
    s, t = torch.zeros(2, 2 * n), torch.zeros(2, n)
    nodes = world.skeletons[0]._ordered_bodies()
    feet = [b for b in nodes if b.name in FEET]
    f = nb.constrained_forward_dynamics_jacobians
    for bad in ([], feet + feet[:1], nodes[:5]):
        with pytest.raises(ValueError, match="constrained_forward_dynamics_jacobians"):
            f(world, s, t, bad)
    other = nb.World.from_raw(raw).skeletons[0]._ordered_bodies()[0]
    with pytest.raises(ValueError):
        f(world, s, t, [other])
    for rho in (-1.0, float("nan"), float("inf"), torch.tensor(1.0)):
        with pytest.raises(ValueError):
            f(world, s, t, feet, damping=rho)
    for off in (torch.zeros(3, 3), torch.zeros(2, 3, 3), torch.zeros(2, 3, dtype=torch.int64), torch.zeros(2, 2, 3)[None]):
        with pytest.raises(ValueError):
            f(world, s, t, feet, offsets=off)
    for bad_s, bad_t in ((torch.zeros(2, 2 * n + 1), t), (s, torch.zeros(3, n)), (s.long(), t), (s, t.long()), (s[0], t)):
        with pytest.raises(ValueError):
            f(world, bad_s, bad_t, feet)
    with pytest.raises(ValueError):
        f(world, s, t, feet, mass=torch.zeros(3, world.getMassDims(), dtype=torch.float64))
    gw = nb.World.from_raw(load_raw("atlas_ground"))
    ground = [b for sk in gw.skeletons if not sk.mobile or sk.getNumDofs() == 0 for b in sk._ordered_bodies()]
    gn = gw.getNumDofs()
    with pytest.raises(ValueError):
        f(gw, torch.zeros(2, 2 * gn), torch.zeros(2, gn), ground[:1])
