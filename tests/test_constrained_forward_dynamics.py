"""Constrained forward dynamics on the CPU: an fp64 oracle composed from the pinned oracles (qdd_free from the step oracle, M from
oracle_M, J and Jdot qdot from the world-Jacobian oracles) with a dense KKT solve, pinned against the closed forms of a free box held at its
origin and at a corner; the host-emulated program (csrc/nb2_cfd.cuh, tests/host_emul/emul_cfd.cpp) against that oracle on the models with
movable nodes, both row-slot counts and every lane schedule; the constraint residual and the round trip through forward dynamics; the
state, tau, offset and per-world-mass VJPs against central differences of the oracle; the singular contact set; and the argument checks of
nimblephysics_b200.constrained_forward_dynamics."""
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import nimblephysics_b200 as nb
from nimblephysics_b200 import modelspec as ms
from oracle.binding import OracleWorld
from tests.host_emul.binding_cfd import EmulCfdWorld
from tests.host_emul.binding_fd import EmulFdWorld
from tests.test_forward_dynamics import fd_inputs, oracle_qdd, per_dof
from tests.test_inverse_dynamics import _compile
from tests.test_mass_matrix import model_raw, oracle_M
from tests.test_per_world_mass import random_masses, raw_at, register
from tests.test_world_jacobian import canon_nodes, oracle_point
from tests.test_world_jacobian_deriv import oracle_point_deriv
from tests.util import load_raw, rel_err

FEET = ["l_foot", "r_foot"]
LIMBS = ["l_foot", "r_foot", "l_hand", "r_hand"]


def oracle_cfd(raw, s, tau, ris, offs=None, point=False, rho=0.0, full=False):
    """fp64 (qdd, wrenches [k, 6 or 3]) of raw bodies `ris` held at offsets `offs` [k, 3]; full: also (J, Jdot qdot, M, lam)."""
    n = raw.ndof
    q, qd = s[:n], s[n:]
    offs = np.zeros((len(ris), 3)) if offs is None else np.asarray(offs, np.float64)
    qf = oracle_qdd(OracleWorld(per_dof(raw)), s, tau)
    M = oracle_M(raw, q)
    rows = slice(3, 6) if point else slice(0, 6)
    J = np.concatenate([oracle_point(raw, q, ri, o)[rows] for ri, o in zip(ris, offs)])
    jd = np.concatenate([oracle_point_deriv(raw, q, qd, ri, o)[rows] for ri, o in zip(ris, offs)]) @ qd
    Mi = np.linalg.inv(M)
    lam = -np.linalg.solve(J @ Mi @ J.T + rho * np.eye(len(J)), J @ qf + jd)
    qdd = qf + Mi @ J.T @ lam
    ow, w = OracleWorld(raw), []
    for i, (ri, o) in enumerate(zip(ris, offs)):
        pos = ow.ik(np.concatenate([q, 0 * q]), [0], [ri], want_jac=False)[0]
        p = pos[3:6] + Rotation.from_rotvec(pos[:3]).as_matrix() @ o
        li = lam[3 * i:3 * i + 3] if point else lam[6 * i:6 * i + 6]
        w.append(li if point else np.concatenate([li[:3] + np.cross(p, li[3:]), li[3:]]))
    return (qdd, np.array(w), J, jd, M, lam) if full else (qdd, np.array(w))


def _ris(raw, names):
    return [list(raw.body_names).index(x) for x in names]


def _box_world(I=(0.3, 0.5, 0.4), m=2.0):
    w = nb.World()
    sk = nb.Skeleton("box")
    _, b = sk.createFreeJointAndBodyNodePair(None)
    b.setMass(m)
    b.setLocalCOM([0.0, 0.0, 0.0])
    b.setMomentOfInertia(*I)
    w.addSkeleton(sk)
    return w, b


def test_oracle_free_box_held_at_its_origin_cancels_gravity_and_the_applied_wrench():
    w, _ = _box_world()
    raw = nb.flatten_world(w)
    s = np.zeros(12)
    tau = np.array([0.3, -0.2, 0.5, 1.0, -2.0, 3.0])
    qdd, wr = oracle_cfd(raw, s, tau, [0])
    g = np.asarray(w.getGravity(), np.float64)
    assert np.abs(qdd).max() < 1e-9
    assert np.abs(wr[0] - -np.concatenate([tau[:3], tau[3:] + 2.0 * g])).max() < 1e-9


def test_oracle_free_box_held_at_a_corner_pivots_about_it():
    Id, m = np.array([0.3, 0.5, 0.4]), 2.0
    w, _ = _box_world(tuple(Id), m)
    raw = nb.flatten_world(w)
    r = np.array([0.2, -0.1, 0.15])  # the corner, from the centre of mass
    qdd, f = oracle_cfd(raw, np.zeros(12), np.zeros(6), [0], [r], point=True)
    g = np.asarray(w.getGravity(), np.float64)
    Ip = np.diag(Id) + m * (r @ r * np.eye(3) - np.outer(r, r))
    alpha = np.linalg.solve(Ip, np.cross(-r, m * g))
    ac = np.cross(r, alpha)
    assert rel_err(qdd[:3], alpha) < 1e-9 and rel_err(qdd[3:], ac) < 1e-9
    assert rel_err(f[0], m * (ac - g)) < 1e-9


CASES = [("atlas", FEET, False), ("atlas", LIMBS, False), ("atlas", LIMBS, True), ("atlas_sdf", FEET, False), ("atlas_sdf", LIMBS, True)]


def _free_child_nodes(raw):
    """one body of each skeleton of the free_child model (the arm has three dofs: it is held at a point)"""
    return [2, raw.nb - 1]


def _setup(name, names, lanes=1):
    raw = model_raw(name)
    ris = _free_child_nodes(raw) if names is None else _ris(raw, names)
    cm = nb.compile_model(raw, lanes=lanes) if lanes == 1 else _compile(raw, lanes)
    return raw, cm, ris, canon_nodes(cm, ris)


@pytest.mark.parametrize("name,names,point", CASES + [("free_child", None, True)])
@pytest.mark.parametrize("fp64", [False, True])
def test_emulated_forward_matches_oracle(name, names, point, fp64):
    raw, cm, ris, (bodies, T) = _setup(name, names)
    ew = EmulCfdWorld(cm)
    B, k = 2, len(ris)
    s, tau = fd_inputs(raw, B, seed=21)
    off = np.random.default_rng(22).uniform(-0.1, 0.1, (B, k, 3))
    qdd, wr = ew.constrained_forward_dynamics(s, tau, bodies, T, off, point=point, fp64=fp64)
    for w in range(B):
        sw, tw, ow = (x if fp64 else x.astype(np.float32).astype(np.float64) for x in (s[w].astype(np.float64), tau[w].astype(np.float64), off[w]))
        rq, rw, J, _, M, _ = oracle_cfd(raw, sw, tw, ris, ow, point, full=True)
        A = J @ np.linalg.solve(M, J.T)
        # fp64: the Richardson error of the Jdot oracle (about 1e-10) bounds the agreement; fp32: 1e-4 scaled by cond(J M^-1 J^T)
        tol = 1e-8 if fp64 else 1e-4 * np.linalg.cond(A)
        assert rel_err(qdd[w], rq) < tol, (w, rel_err(qdd[w], rq), tol)
        assert rel_err(wr[w], rw) < tol, (w, rel_err(wr[w], rw), tol)


@pytest.mark.parametrize("lanes", [2, 4, 8])
def test_emulated_lane_schedules_and_slot_counts_agree(lanes):
    raw, cm1, ris, (bodies, T) = _setup("atlas", LIMBS)
    e1, ek = EmulCfdWorld(cm1), EmulCfdWorld(_compile(raw, lanes))
    s, tau = fd_inputs(raw, 3, seed=lanes)
    rng = np.random.default_rng(lanes)
    gq, gw = rng.normal(size=(3, raw.ndof)), rng.normal(size=(3, 4, 6))
    ref = e1.constrained_forward_dynamics(s, tau, bodies, T, fp64=True) + e1.constrained_forward_dynamics_backward(s, tau, bodies, T, gq, gw, fp64=True)[:3]
    for ew, slots in ((ek, 8), (ek, 1), (e1, 1)):
        got = ew.constrained_forward_dynamics(s, tau, bodies, T, fp64=True, slots=slots) + ew.constrained_forward_dynamics_backward(
            s, tau, bodies, T, gq, gw, fp64=True, slots=slots)[:3]
        for a, b in zip(got, ref):
            assert rel_err(a, b) < 1e-12


@pytest.mark.parametrize("point", [False, True])
def test_emulated_residual_and_round_trip_through_forward_dynamics(point):
    raw, cm, ris, (bodies, T) = _setup("atlas", LIMBS)
    ew, ef = EmulCfdWorld(cm), EmulFdWorld(cm)
    B, n = 3, raw.ndof
    s, tau = fd_inputs(raw, B, seed=5)
    s, tau = s.astype(np.float64), tau.astype(np.float64)
    rho = 1e-3
    qdd, wr = ew.constrained_forward_dynamics(s, tau, bodies, T, point=point, rho=rho, fp64=True)
    for w in range(B):
        rq, rw, J, jd, M, lam = oracle_cfd(raw, s[w], tau[w], ris, point=point, rho=rho, full=True)
        # the residual of the emulated qdd with the oracle's lam (the same lam: the wrenches agree)
        assert rel_err(wr[w], rw) < 1e-8
        assert np.abs(J @ qdd[w] + jd + rho * lam).max() < 1e-7 * max(1.0, np.abs(jd).max())
        back, _ = ef.forward_dynamics(s[w:w + 1], (tau[w] + J.T @ lam)[None], True)
        assert rel_err(back[0], qdd[w]) < 1e-8


def _vjp_oracle(raw, ris, s, tau, off, point, gq, gw, h=1e-5):
    def L(s_, t_, o_):
        q, w = oracle_cfd(raw, s_, t_, ris, o_, point)
        return float(gq @ q + (gw * w).sum())

    def fd(x, f):
        out = np.zeros(x.size)
        for c in range(x.size):
            xp, xm = x.reshape(-1).copy(), x.reshape(-1).copy()
            xp[c] += h
            xm[c] -= h
            out[c] = (f(xp.reshape(x.shape)) - f(xm.reshape(x.shape))) / (2 * h)
        return out.reshape(x.shape)

    return fd(s, lambda x: L(x, tau, off)), fd(tau, lambda x: L(s, x, off)), fd(off, lambda x: L(s, tau, x))


@pytest.mark.parametrize("name,names,point", [("free_child", None, True), ("atlas", FEET, False), ("atlas", ["l_foot", "r_hand"], True)])
def test_emulated_vjp_matches_oracle_differences(name, names, point):
    raw, cm, ris, (bodies, T) = _setup(name, names)
    ew = EmulCfdWorld(cm)
    k, n = len(ris), raw.ndof
    s, tau = fd_inputs(raw, 1, seed=31)
    s, tau = s.astype(np.float64), tau.astype(np.float64)
    off = np.random.default_rng(32).uniform(-0.1, 0.1, (1, k, 3))
    rng = np.random.default_rng(33)
    gq, gw = rng.normal(size=(1, n)), rng.normal(size=(1, k, 3 if point else 6))
    gs, gt, go, _ = ew.constrained_forward_dynamics_backward(s, tau, bodies, T, gq, gw, off, point=point, fp64=True)
    rs, rt, ro = _vjp_oracle(raw, ris, s[0], tau[0], off[0], point, gq[0], gw[0])
    assert rel_err(gs[0], rs) < 1e-6, rel_err(gs[0], rs)
    assert rel_err(gt[0], rt) < 1e-6, rel_err(gt[0], rt)
    assert rel_err(go[0], ro) < 1e-6, rel_err(go[0], ro)


def test_emulated_per_world_mass_vjp_matches_oracle_differences():
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=4)
    B = 2
    Mv = random_masses(world, B, seed=9)
    wi = nb.mass_to_inertia(world, torch.tensor(Mv, dtype=torch.float64)).numpy()
    cm = nb.compile_model(raw, lanes=2)
    ew = EmulCfdWorld(cm)
    ris = _ris(raw, FEET)
    bodies, T = canon_nodes(cm, ris)
    s, tau = fd_inputs(raw, B, seed=5)
    s, tau = s.astype(np.float64), tau.astype(np.float64)
    rng = np.random.default_rng(6)
    gq, gw = rng.normal(size=(B, raw.ndof)), rng.normal(size=(B, 2, 6))
    qdd, _ = ew.constrained_forward_dynamics(s, tau, bodies, T, fp64=True, world_inertia=wi)
    _, _, _, gi = ew.constrained_forward_dynamics_backward(s, tau, bodies, T, gq, gw, fp64=True, world_inertia=wi)
    entries = world._mass_entries()
    for w in range(B):
        rw = raw_at(raw, entries, Mv[w])
        assert rel_err(qdd[w], oracle_cfd(rw, s[w], tau[w], ris)[0]) < 1e-8
        gm = ms.inertia_param_jacobian(rw, cm, entries) @ gi[:, w]

        def loss(mv):
            q, wr = oracle_cfd(raw_at(raw, entries, mv), s[w], tau[w], ris)
            return float(gq[w] @ q + (gw[w] * wr).sum())

        fdm = np.array([(loss(Mv[w] + 1e-6 * e) - loss(Mv[w] - 1e-6 * e)) / 2e-6 for e in np.eye(len(Mv[w]))])
        assert rel_err(gm, fdm) < 1e-6, (gm, fdm)


def test_emulated_singular_set_is_nan_and_damping_regularises_it():
    """cartpole's pole held 6-D: J has rank 2 of 6, so J M^-1 J^T is singular.  rho = 0 gives NaN rows; rho > 0 the oracle's damped solution."""
    raw = load_raw("cartpole")
    cm = nb.compile_model(raw, lanes=1)
    ew = EmulCfdWorld(cm)
    ris = [raw.nb - 1]
    bodies, T = canon_nodes(cm, ris)
    s, tau = fd_inputs(raw, 2, seed=3)
    s, tau = s.astype(np.float64), tau.astype(np.float64)
    for fp64 in (False, True):
        qdd, wr = ew.constrained_forward_dynamics(s, tau, bodies, T, fp64=fp64)
        assert np.isnan(qdd).all() and np.isnan(wr).all()
        gs, gt, go, _ = ew.constrained_forward_dynamics_backward(s, tau, bodies, T, np.ones((2, raw.ndof)), np.ones((2, 1, 6)), fp64=fp64)
        assert np.isnan(gs).all() and np.isnan(gt).all() and np.isnan(go).all()
    qdd, wr = ew.constrained_forward_dynamics(s, tau, bodies, T, rho=1e-2, fp64=True)
    for w in range(2):
        rq, rw = oracle_cfd(raw, s[w], tau[w], ris, rho=1e-2)
        assert rel_err(qdd[w], rq) < 1e-8 and rel_err(wr[w], rw) < 1e-8


def test_value_errors():
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    n = raw.ndof
    s, t = torch.zeros(2, 2 * n), torch.zeros(2, n)
    nodes = world.skeletons[0]._ordered_bodies()
    feet = [b for b in nodes if b.name in FEET]
    f = nb.constrained_forward_dynamics
    for bad in ([], feet + feet[:1], nodes[:5]):
        with pytest.raises(ValueError):
            f(world, s, t, bad)
    other = nb.World.from_raw(raw).skeletons[0]._ordered_bodies()[0]
    with pytest.raises(ValueError):
        f(world, s, t, [other])
    for rho in (-1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            f(world, s, t, feet, damping=rho)
    for off in (torch.zeros(3, 3), torch.zeros(2, 3, 3), torch.zeros(2, 3, dtype=torch.int64)):
        with pytest.raises(ValueError):
            f(world, s, t, feet, offsets=off)
    for bad_s, bad_t in ((torch.zeros(2, 2 * n + 1), t), (s, torch.zeros(3, n)), (s.long(), t), (s, t.long())):
        with pytest.raises(ValueError):
            f(world, bad_s, bad_t, feet)
    with pytest.raises(ValueError):
        f(world, s, t, feet, mass=torch.zeros(3, world.getMassDims(), dtype=torch.float64))
    gw = nb.World.from_raw(load_raw("atlas_ground"))
    ground = [b for sk in gw.skeletons if not sk.mobile or sk.getNumDofs() == 0 for b in sk._ordered_bodies()]
    assert ground
    gn = gw.getNumDofs()
    with pytest.raises(ValueError):
        f(gw, torch.zeros(2, 2 * gn), torch.zeros(2, gn), ground[:1])
