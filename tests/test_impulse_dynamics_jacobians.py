"""Dense Jacobians of impulse dynamics on the CPU: the host-emulated program (csrc/nb2_imp.cuh impj_world, tests/host_emul/emul_impj.cpp)
against the emulated VJP seeded with each unit vector, on every lane schedule and row-slot count; all four blocks against central
differences of the fp64 oracle; the closed forms of the qdot- blocks, linearity in qdot-, the constraint and projector identities and the
differentiated constraint in q, in the oracle's M and J; the uncontacted arm; the singular set; and the argument checks of
nimblephysics_b200.impulse_dynamics_jacobians."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from tests.host_emul.binding_impj import EmulImpjWorld
from tests.test_constrained_forward_dynamics import FEET, LIMBS, _setup
from tests.test_constrained_forward_dynamics_jacobians import _central, _point_form, singular_middle_world
from tests.test_impulse_dynamics import _inputs, oracle_imp
from tests.test_world_jacobian import oracle_point
from tests.util import load_raw, rel_err

ROW_CASES = [("atlas", FEET, False), ("atlas", LIMBS, False), ("atlas", LIMBS, True), ("atlas_sdf", FEET, False), ("free_child", None, True)]


def vjp_rows(ew, s, bodies, T, off, point, e, rho, slots=8):
    """the four blocks assembled from the emulated VJP seeded with e_i on qdot+ and e_r on the impulses, [B, n or m, n] each"""
    B, n, k, r = s.shape[0], ew.n, len(bodies), 3 if point else 6
    m = k * r
    blocks = [np.empty((B, n, n)) for _ in range(2)] + [np.empty((B, m, n)) for _ in range(2)]
    for i in range(n + m):
        gv, gw = np.zeros((B, n)), np.zeros((B, m))
        (gv[:, i] if i < n else gw[:, i - n])[...] = 1.0
        gs, _, _ = ew.impulse_dynamics_backward(s, bodies, T, gv, gw.reshape(B, k, r), off, point=point, e=e, rho=rho, fp64=True, slots=slots)
        o, row = (0, i) if i < n else (2, i - n)
        blocks[o][:, row], blocks[o + 1][:, row] = gs[:, :n], gs[:, n:]
    return blocks


@pytest.mark.parametrize("rho", [0.0, 1e-3])
@pytest.mark.parametrize("e", [0.0, 0.5, 1.0])
@pytest.mark.parametrize("name,names,point", ROW_CASES)
def test_emulated_rows_are_the_vjp_bit_for_bit(name, names, point, e, rho):
    raw, cm, ris, (bodies, T) = _setup(name, names)
    ew = EmulImpjWorld(cm)
    B, k, n = 2, len(ris), raw.ndof
    s = _inputs(raw, B, seed=41).astype(np.float64)
    off = np.random.default_rng(42).uniform(-0.1, 0.1, (B, k, 3))
    out = ew.impulse_dynamics_jacobians(s, bodies, T, off, point=point, e=e, rho=rho, fp64=True)
    v, w = ew.impulse_dynamics(s, bodies, T, off, point=point, e=e, rho=rho, fp64=True)
    assert np.array_equal(out[0], v) and np.array_equal(out[1], w)
    m = k * (3 if point else 6)
    ref = vjp_rows(ew, s, bodies, T, off, point, e, rho)
    for got, want in zip(out[2:4] + tuple(x.reshape(B, m, n) for x in out[4:]), ref):
        # the per-seed code does the VJP's arithmetic (cfd_point_form, mu, g and the dL/dqdot- row, the FD backward, the jpb VJP)
        assert np.array_equal(got, want), rel_err(got, want)


@pytest.mark.parametrize("lanes", [2, 4, 8])
def test_emulated_lane_schedules_and_slot_counts_agree(lanes):
    raw, cm1, ris, (bodies, T) = _setup("atlas", LIMBS)
    e1, ek = EmulImpjWorld(cm1), EmulImpjWorld(_setup("atlas", LIMBS, lanes)[1])
    s = _inputs(raw, 3, seed=lanes)
    off = np.random.default_rng(lanes).uniform(-0.1, 0.1, (3, 4, 3))
    args = dict(e=0.5, rho=1e-4, fp64=True)
    ref = e1.impulse_dynamics_jacobians(s, bodies, T, off, **args)
    for ew, slots in ((ek, 8), (ek, 1), (e1, 1)):
        got = ew.impulse_dynamics_jacobians(s, bodies, T, off, slots=slots, **args)
        for a, b in zip(got, ref):
            assert rel_err(a, b) < 1e-12


@pytest.mark.parametrize("name,names,point,rho", [("free_child", None, True, 0.0), ("atlas", FEET, False, 0.0), ("atlas", FEET, False, 1e-3),
                                                  ("atlas", ["l_foot", "r_hand"], True, 1e-3)])
def test_emulated_blocks_match_oracle_differences(name, names, point, rho):
    raw, cm, ris, (bodies, T) = _setup(name, names)
    ew = EmulImpjWorld(cm)
    k, n, e = len(ris), raw.ndof, 0.5
    s = _inputs(raw, 1, seed=31).astype(np.float64)
    off = np.random.default_rng(32).uniform(-0.1, 0.1, (1, k, 3))
    out = ew.impulse_dynamics_jacobians(s, bodies, T, off, point=point, e=e, rho=rho, fp64=True)
    D = _central(lambda x: np.concatenate([y.reshape(-1) for y in oracle_imp(raw, x, ris, off[0], point, e, rho)]), s[0])
    m = k * (3 if point else 6)
    want = [D[:n, :n], D[:n, n:], D[n:, :n], D[n:, n:]]
    for got, ref in zip([x[0] for x in out[2:4]] + [x[0].reshape(m, n) for x in out[4:]], want):
        assert rel_err(got, ref) < 1e-6, rel_err(got, ref)


@pytest.mark.parametrize("rho", [0.0, 1e-3])
@pytest.mark.parametrize("e", [0.0, 0.5, 1.0])
@pytest.mark.parametrize("names,point", [(FEET, False), (LIMBS, True)])
def test_emulated_closed_forms(names, point, e, rho):
    raw, cm, ris, (bodies, T) = _setup("atlas", names)
    ew = EmulImpjWorld(cm)
    B, k, n = 2, len(ris), raw.ndof
    s = _inputs(raw, B, seed=51).astype(np.float64)
    off = np.random.default_rng(52).uniform(-0.1, 0.1, (k, 3))
    rows = slice(3, 6) if point else slice(0, 6)
    v, imp, dv_dq, dv_dqd, di_dq, di_dqd = ew.impulse_dynamics_jacobians(s, bodies, T, off, point=point, e=e, rho=rho, fp64=True)
    m = k * (3 if point else 6)
    for w in range(B):
        q, qd = s[w, :n], s[w, n:]
        _, _, J, M, _ = oracle_imp(raw, s[w], ris, off, point, e, rho, full=True)
        Mi = np.linalg.inv(M)
        A = J @ Mi @ J.T + rho * np.eye(m)
        P, Pi = dv_dqd[w], di_dqd[w].reshape(m, n)
        dlam_dqd = _point_form(raw, q, ris, off, Pi, point)
        assert rel_err(P, np.eye(n) - (1 + e) * Mi @ J.T @ np.linalg.solve(A, J)) < 1e-9
        assert rel_err(dlam_dqd, -(1 + e) * np.linalg.solve(A, J)) < 1e-9
        # linear in qdot- at fixed q (the 6-D impulses about the origin too: the point p depends on q only)
        assert rel_err(P @ qd, v[w]) < 1e-12 and rel_err(Pi @ qd, imp[w].reshape(-1)) < 1e-12
        if rho == 0.0:
            assert np.abs(J @ P + e * J).max() < 1e-10 * np.abs(J).max()
            if e == 0.0:  # a projector, M-symmetric
                assert np.abs(P @ P - P).max() < 1e-10 * np.abs(P).max()
                assert rel_err(M @ P, (M @ P).T) < 1e-10
        if point or rho == 0.0:
            # J qdot+ = -e J qdot- - rho Lam, differentiated in q: J dv/dq + d(J(q) u)/dq |_(u = qdot+ + e qdot-) = -rho dLam/dq.  With point
            # contacts the impulses are Lam; with 6-D ones rho = 0 drops the term that needs Lam's point form in q.
            u = v[w] + e * qd
            dJu = _central(lambda x: np.concatenate([oracle_point(raw, x, ri, o)[rows] for ri, o in zip(ris, off)]) @ u, q)
            lhs = J @ dv_dq[w] + dJu + rho * di_dq[w].reshape(m, n)
            assert np.abs(lhs).max() < 1e-7 * (np.abs(dJu).max() + np.abs(J @ dv_dq[w]).max())


def test_emulated_uncontacted_arm_keeps_unit_rows():
    """free_child held at its free root only: the arm's columns of Y = (M^-1 J^T)^T are exactly zero, so mu is exactly zero for the arm's
    seeds and their rows of dqdot+/dqdot- are exactly the unit rows"""
    raw, cm, ris, (bodies, T) = _setup("free_child", None)
    ew = EmulImpjWorld(cm)
    n = raw.ndof
    s = _inputs(raw, 3, seed=14)
    for fp64 in (False, True):
        P = ew.impulse_dynamics_jacobians(s, bodies[:1], T[:1], point=True, e=0.5, fp64=fp64)[3]
        for i in range(n - 3, n):
            assert np.array_equal(P[:, i], np.broadcast_to(np.eye(n)[i], (3, n)))


def test_emulated_singular_world_is_nan_and_isolated():
    """the singular world's outputs and blocks are all NaN; the other worlds' are their own single-world results; damping makes it finite"""
    raw, cm, bodies, T, s, _, off = singular_middle_world()
    ew = EmulImpjWorld(cm)
    for fp64 in (False, True):
        out = ew.impulse_dynamics_jacobians(s, bodies, T, off, point=True, e=0.5, fp64=fp64)
        for w in (0, 2):
            one = ew.impulse_dynamics_jacobians(s[w:w + 1], bodies, T, off[w:w + 1], point=True, e=0.5, fp64=fp64)
            for a, b in zip(out, one):
                assert np.isnan(a[1]).all() and np.isfinite(b).all() and np.array_equal(a[w:w + 1], b)
    out = ew.impulse_dynamics_jacobians(s, bodies, T, off, point=True, e=0.5, rho=1e-3, fp64=True)
    assert all(np.isfinite(x).all() for x in out)


def test_emulated_empty_batch():
    raw, cm, ris, (bodies, T) = _setup("atlas", FEET)
    n = raw.ndof
    out = EmulImpjWorld(cm).impulse_dynamics_jacobians(np.zeros((0, 2 * n)), bodies, T, fp64=True)
    assert [x.shape for x in out] == [(0, n), (0, 2, 6)] + [(0, n, n)] * 2 + [(0, 2, 6, n)] * 2


def test_value_errors():
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    n = raw.ndof
    s = torch.zeros(2, 2 * n)
    nodes = world.skeletons[0]._ordered_bodies()
    feet = [b for b in nodes if b.name in FEET]
    f = nb.impulse_dynamics_jacobians
    for e in (-0.1, 1.5, float("nan"), float("inf"), torch.tensor(0.5), "0.5", None, True):
        with pytest.raises(ValueError, match="impulse_dynamics_jacobians"):
            f(world, s, feet, restitution=e)
    for bad in ([], feet + feet[:1], nodes[:5]):
        with pytest.raises(ValueError, match="impulse_dynamics_jacobians"):
            f(world, s, bad)
    other = nb.World.from_raw(raw).skeletons[0]._ordered_bodies()[0]
    with pytest.raises(ValueError, match="impulse_dynamics_jacobians"):
        f(world, s, [other])
    for rho in (-1.0, float("nan"), float("inf"), torch.tensor(0.1)):
        with pytest.raises(ValueError, match="impulse_dynamics_jacobians"):
            f(world, s, feet, damping=rho)
    for off in (torch.zeros(3, 3), torch.zeros(2, 3, 3), torch.zeros(2, 3, dtype=torch.int64)):
        with pytest.raises(ValueError, match="impulse_dynamics_jacobians"):
            f(world, s, feet, offsets=off)
    for bad_s in (torch.zeros(2, 2 * n + 1), torch.zeros(2, n), torch.zeros(2, 2, 2 * n), s.long()):
        with pytest.raises(ValueError, match="impulse_dynamics_jacobians"):
            f(world, bad_s, feet)
    with pytest.raises(ValueError, match="impulse_dynamics_jacobians"):
        f(world, s, feet, mass=torch.zeros(3, world.getMassDims(), dtype=torch.float64))
    gw = nb.World.from_raw(load_raw("atlas_ground"))
    ground = [b for sk in gw.skeletons if not sk.mobile or sk.getNumDofs() == 0 for b in sk._ordered_bodies()]
    with pytest.raises(ValueError, match="impulse_dynamics_jacobians"):
        f(gw, torch.zeros(2, 2 * gw.getNumDofs()), ground[:1])
