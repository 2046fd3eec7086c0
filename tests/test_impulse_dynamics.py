"""Impulse dynamics on the CPU: an fp64 oracle composed from the pinned oracles (M from oracle_M, J from the world-Jacobian oracle) with a
dense solve, pinned against the closed forms of a free box held 6-D at its origin and struck at a corner; the host-emulated program
(csrc/nb2_imp.cuh, tests/host_emul/emul_imp.cpp) against that oracle on the models with movable nodes, at three restitutions, both
row-slot counts and every lane schedule; the constraint residual, the energy identity, idempotence at e = 0 and an uncontacted tree; the
state, offset and per-world-mass VJPs against central differences of the oracle; and the argument checks of
nimblephysics_b200.impulse_dynamics."""
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import nimblephysics_b200 as nb
from nimblephysics_b200 import modelspec as ms
from oracle.binding import OracleWorld
from tests.host_emul.binding_imp import EmulImpWorld
from tests.test_constrained_forward_dynamics import CASES, FEET, LIMBS, _box_world, _ris, _setup
from tests.test_forward_dynamics import fd_inputs
from tests.test_mass_matrix import oracle_M
from tests.test_per_world_mass import random_masses, raw_at, register
from tests.test_world_jacobian import canon_nodes, oracle_point
from tests.util import load_raw, rel_err

ES = [0.0, 0.5, 1.0]


def oracle_imp(raw, s, ris, offs=None, point=False, e=0.0, rho=0.0, full=False):
    """fp64 (qdot_after, impulses [k, 6 or 3]) of raw bodies `ris` struck at offsets `offs` [k, 3]; full: also (J, M, Lam)."""
    n = raw.ndof
    q, qd = s[:n], s[n:]
    offs = np.zeros((len(ris), 3)) if offs is None else np.asarray(offs, np.float64)
    M = oracle_M(raw, q)
    rows = slice(3, 6) if point else slice(0, 6)
    J = np.concatenate([oracle_point(raw, q, ri, o)[rows] for ri, o in zip(ris, offs)])
    Y = np.linalg.solve(M, J.T)
    lam = -np.linalg.solve(J @ Y + rho * np.eye(len(J)), (1 + e) * J @ qd)
    v = qd + Y @ lam
    ow, w = OracleWorld(raw), []
    for i, (ri, o) in enumerate(zip(ris, offs)):
        pos = ow.ik(np.concatenate([q, 0 * q]), [0], [ri], want_jac=False)[0]
        p = pos[3:6] + Rotation.from_rotvec(pos[:3]).as_matrix() @ o
        li = lam[3 * i:3 * i + 3] if point else lam[6 * i:6 * i + 6]
        w.append(li if point else np.concatenate([li[:3] + np.cross(p, li[3:]), li[3:]]))
    return (v, np.array(w), J, M, lam) if full else (v, np.array(w))


def _inputs(raw, B, seed):
    s, _ = fd_inputs(raw, B, seed)
    return s


@pytest.mark.parametrize("e", ES)
def test_oracle_free_box_held_at_its_origin_reverses_its_momentum(e):
    Id, m = np.array([0.3, 0.5, 0.4]), 2.0
    w, _ = _box_world(tuple(Id), m)
    raw = nb.flatten_world(w)
    rng = np.random.default_rng(1)
    s = np.concatenate([rng.uniform(-0.5, 0.5, 6), rng.uniform(-1, 1, 6)])  # [log R ; p], body twist [omega ; v]
    v, imp = oracle_imp(raw, s, [0], e=e)
    assert np.abs(v + e * s[6:]).max() < 1e-9 * np.abs(s[6:]).max()
    R, p = Rotation.from_rotvec(s[:3]).as_matrix(), s[3:6]
    om, vel = R @ s[6:9], R @ s[9:12]
    h = np.concatenate([R @ np.diag(Id) @ R.T @ om + m * np.cross(p, vel), m * vel])  # spatial momentum about the world origin
    assert rel_err(imp[0], -(1 + e) * h) < 1e-9


@pytest.mark.parametrize("e", ES)
def test_oracle_free_box_struck_at_a_corner_is_the_rigid_body_impact(e):
    Id, m = np.array([0.3, 0.5, 0.4]), 2.0
    w, _ = _box_world(tuple(Id), m)
    raw = nb.flatten_world(w)
    r = np.array([0.2, -0.1, 0.15])
    rng = np.random.default_rng(2)
    s = np.concatenate([np.zeros(6), rng.uniform(-1, 1, 6)])
    om, vel = s[6:9], s[9:12]
    v, imp = oracle_imp(raw, s, [0], [r], point=True, e=e)
    rx = np.array([[0, -r[2], r[1]], [r[2], 0, -r[0]], [-r[1], r[0], 0]])
    Iw = np.diag(Id)
    K = np.eye(3) / m - rx @ np.linalg.solve(Iw, rx)
    lam = -(1 + e) * np.linalg.solve(K, vel + np.cross(om, r))
    assert rel_err(imp[0], lam) < 1e-9
    assert rel_err(v[:3], om + np.linalg.solve(Iw, np.cross(r, lam))) < 1e-9 and rel_err(v[3:], vel + lam / m) < 1e-9


@pytest.mark.parametrize("name,names,point", CASES + [("free_child", None, True)])
@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("e", ES)
def test_emulated_forward_matches_oracle(name, names, point, fp64, e):
    raw, cm, ris, (bodies, T) = _setup(name, names)
    ew = EmulImpWorld(cm)
    B, k = 2, len(ris)
    s = _inputs(raw, B, seed=21)
    off = np.random.default_rng(22).uniform(-0.1, 0.1, (B, k, 3))
    v, imp = ew.impulse_dynamics(s, bodies, T, off, point=point, e=e, fp64=fp64)
    for w in range(B):
        sw, ow = (x if fp64 else x.astype(np.float32).astype(np.float64) for x in (s[w].astype(np.float64), off[w]))
        rv, ri, J, M, _ = oracle_imp(raw, sw, ris, ow, point, e, full=True)
        tol = 1e-8 if fp64 else 1e-4 * np.linalg.cond(J @ np.linalg.solve(M, J.T))
        assert rel_err(v[w], rv) < tol, (w, rel_err(v[w], rv), tol)
        assert rel_err(imp[w], ri) < tol, (w, rel_err(imp[w], ri), tol)


@pytest.mark.parametrize("lanes", [1, 2, 4, 8])
def test_emulated_lane_schedules_and_slot_counts_agree(lanes):
    raw, cm1, ris, (bodies, T) = _setup("atlas", LIMBS)
    e1, ek = EmulImpWorld(cm1), EmulImpWorld(_setup("atlas", LIMBS, lanes)[1])
    s = _inputs(raw, 3, seed=lanes)
    rng = np.random.default_rng(lanes)
    gv, gi = rng.normal(size=(3, raw.ndof)), rng.normal(size=(3, 4, 6))
    args = dict(e=0.5, rho=1e-4, fp64=True)
    ref = e1.impulse_dynamics(s, bodies, T, **args) + e1.impulse_dynamics_backward(s, bodies, T, gv, gi, **args)[:2]
    for slots in (8, 1):
        got = ek.impulse_dynamics(s, bodies, T, slots=slots, **args) + ek.impulse_dynamics_backward(s, bodies, T, gv, gi, slots=slots, **args)[:2]
        for a, b in zip(got, ref):
            assert rel_err(a, b) < 1e-12


@pytest.mark.parametrize("point", [False, True])
@pytest.mark.parametrize("e", ES)
def test_emulated_constraint_energy_and_idempotence(point, e):
    raw, cm, ris, (bodies, T) = _setup("atlas", FEET if not point else LIMBS)
    ew = EmulImpWorld(cm)
    n = raw.ndof
    s = _inputs(raw, 3, seed=5).astype(np.float64)
    rho = 1e-3
    v, imp = ew.impulse_dynamics(s, bodies, T, point=point, e=e, rho=rho, fp64=True)
    v0, _ = ew.impulse_dynamics(s, bodies, T, point=point, e=e, fp64=True)
    for w in range(3):
        _, _, J, M, lam = oracle_imp(raw, s[w], ris, point=point, e=e, rho=rho, full=True)
        qd = s[w, n:]
        # J qdot+ + e J qdot- + rho Lam = 0, with the oracle's Lam (the same Lam: the impulses agree)
        assert np.abs(J @ v[w] + e * J @ qd + rho * lam).max() < 1e-9 * max(1.0, np.abs(J @ qd).max())
        # rho = 0: T+ - T- = -(1 - e^2) / 2 (J qdot-)^T (J M^-1 J^T)^-1 (J qdot-)
        c = J @ qd
        loss = -0.5 * (1 - e * e) * c @ np.linalg.solve(J @ np.linalg.solve(M, J.T), c)
        T0, T1 = 0.5 * qd @ M @ qd, 0.5 * v0[w] @ M @ v0[w]
        assert abs((T1 - T0) - loss) < 1e-9 * T0
        assert T1 <= T0 * (1 + 1e-12)
    if e == 0.0:  # a second impact changes nothing
        s2 = np.concatenate([s[:, :n], v0], 1)
        v2, imp2 = ew.impulse_dynamics(s2, bodies, T, point=point, fp64=True)
        assert np.abs(imp2).max() < 1e-9 * np.abs(ew.impulse_dynamics(s, bodies, T, point=point, fp64=True)[1]).max()
        assert rel_err(v2, v0) < 1e-10


def test_emulated_tree_without_a_contact_keeps_its_velocity_bit_for_bit():
    raw, cm, ris, (bodies, T) = _setup("free_child", None)
    ew = EmulImpWorld(cm)
    s = _inputs(raw, 4, seed=14)
    n = raw.ndof
    arm = slice(n - 3, n)
    for fp64 in (False, True):
        v, _ = ew.impulse_dynamics(s, bodies[:1], T[:1], point=True, e=0.5, fp64=fp64)
        want = s[:, n:].astype(np.float64 if fp64 else np.float32)
        assert np.array_equal(v[:, arm], want[:, arm])


def _num_grad(x, f, h=1e-6):
    out = np.zeros(x.size)
    for c in range(x.size):
        xp, xm = x.reshape(-1).copy(), x.reshape(-1).copy()
        xp[c] += h
        xm[c] -= h
        out[c] = (f(xp.reshape(x.shape)) - f(xm.reshape(x.shape))) / (2 * h)
    return out.reshape(x.shape)


@pytest.mark.parametrize("name,names,point,rho", [("free_child", None, True, 0.0), ("atlas", FEET, False, 0.0), ("atlas", FEET, False, 1e-3),
                                                  ("atlas", ["l_foot", "r_hand"], True, 1e-3)])
def test_emulated_vjp_matches_oracle_differences(name, names, point, rho):
    raw, cm, ris, (bodies, T) = _setup(name, names)
    ew = EmulImpWorld(cm)
    k, n, e = len(ris), raw.ndof, 0.3
    s = _inputs(raw, 1, seed=31).astype(np.float64)
    off = np.random.default_rng(32).uniform(-0.1, 0.1, (1, k, 3))
    rng = np.random.default_rng(33)
    gv, gw = rng.normal(size=(1, n)), rng.normal(size=(1, k, 3 if point else 6))
    gs, go, _ = ew.impulse_dynamics_backward(s, bodies, T, gv, gw, off, point=point, e=e, rho=rho, fp64=True)

    def L(s_, o_):
        v, w = oracle_imp(raw, s_, ris, o_, point, e, rho)
        return float(gv[0] @ v + (gw[0] * w).sum())

    assert rel_err(gs[0], _num_grad(s[0], lambda x: L(x, off[0]), 1e-5)) < 1e-6
    # a 6-D hold constrains the body's twist wherever the point is, and the impulses are about the world origin: the offset gradient
    # is zero there, so it is compared on the scale of the state gradient
    ro = _num_grad(off[0], lambda x: L(s[0], x), 1e-5)
    assert np.abs(go[0] - ro).max() < 1e-6 * max(np.abs(ro).max(), 1e-3 * np.abs(gs[0]).max())


def test_emulated_per_world_mass_vjp_matches_oracle_differences():
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=4)
    B, e = 2, 0.5
    Mv = random_masses(world, B, seed=9)
    wi = nb.mass_to_inertia(world, torch.tensor(Mv, dtype=torch.float64)).numpy()
    cm = nb.compile_model(raw, lanes=2)
    ew = EmulImpWorld(cm)
    ris = _ris(raw, FEET)
    bodies, T = canon_nodes(cm, ris)
    s = _inputs(raw, B, seed=5).astype(np.float64)
    rng = np.random.default_rng(6)
    gv, gw = rng.normal(size=(B, raw.ndof)), rng.normal(size=(B, 2, 6))
    v, _ = ew.impulse_dynamics(s, bodies, T, e=e, fp64=True, world_inertia=wi)
    _, _, gi = ew.impulse_dynamics_backward(s, bodies, T, gv, gw, e=e, fp64=True, world_inertia=wi)
    entries = world._mass_entries()
    for w in range(B):
        rw = raw_at(raw, entries, Mv[w])
        assert rel_err(v[w], oracle_imp(rw, s[w], ris, e=e)[0]) < 1e-8
        gm = ms.inertia_param_jacobian(rw, cm, entries) @ gi[:, w]

        def loss(mv):
            q, wr = oracle_imp(raw_at(raw, entries, mv), s[w], ris, e=e)
            return float(gv[w] @ q + (gw[w] * wr).sum())

        assert rel_err(gm, _num_grad(Mv[w], loss)) < 1e-6


def test_emulated_singular_set_is_nan_and_damping_regularises_it():
    """cartpole's pole held 6-D: J has rank 2 of 6, so J M^-1 J^T is singular.  rho = 0 gives NaN rows; rho > 0 the oracle's damped map."""
    raw = load_raw("cartpole")
    cm = nb.compile_model(raw, lanes=1)
    ew = EmulImpWorld(cm)
    ris = [raw.nb - 1]
    bodies, T = canon_nodes(cm, ris)
    s = _inputs(raw, 2, seed=3).astype(np.float64)
    for fp64 in (False, True):
        v, imp = ew.impulse_dynamics(s, bodies, T, fp64=fp64)
        assert np.isnan(v).all() and np.isnan(imp).all()
        gs, go, gi = ew.impulse_dynamics_backward(s, bodies, T, np.ones((2, raw.ndof)), np.ones((2, 1, 6)), fp64=fp64)
        assert np.isnan(gs).all() and np.isnan(go).all()
    v, imp = ew.impulse_dynamics(s, bodies, T, e=0.5, rho=1e-2, fp64=True)
    for w in range(2):
        rv, ri = oracle_imp(raw, s[w], ris, e=0.5, rho=1e-2)
        assert rel_err(v[w], rv) < 1e-8 and rel_err(imp[w], ri) < 1e-8


def test_value_errors():
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    n = raw.ndof
    s = torch.zeros(2, 2 * n)
    nodes = world.skeletons[0]._ordered_bodies()
    feet = [b for b in nodes if b.name in FEET]
    f = nb.impulse_dynamics
    for e in (-0.1, 1.5, float("nan"), float("inf"), torch.tensor(0.5), "0.5", None, True):
        with pytest.raises(ValueError):
            f(world, s, feet, restitution=e)
    for bad in ([], feet + feet[:1], nodes[:5]):
        with pytest.raises(ValueError):
            f(world, s, bad)
    other = nb.World.from_raw(raw).skeletons[0]._ordered_bodies()[0]
    with pytest.raises(ValueError):
        f(world, s, [other])
    for rho in (-1.0, float("nan"), float("inf"), torch.tensor(0.1)):
        with pytest.raises(ValueError):
            f(world, s, feet, damping=rho)
    for off in (torch.zeros(3, 3), torch.zeros(2, 3, 3), torch.zeros(2, 3, dtype=torch.int64)):
        with pytest.raises(ValueError):
            f(world, s, feet, offsets=off)
    for bad_s in (torch.zeros(2, 2 * n + 1), torch.zeros(2, n), torch.zeros(2, 2, 2 * n), s.long()):
        with pytest.raises(ValueError):
            f(world, bad_s, feet)
    with pytest.raises(ValueError):
        f(world, s, feet, mass=torch.zeros(3, world.getMassDims(), dtype=torch.float64))
    gw = nb.World.from_raw(load_raw("atlas_ground"))
    ground = [b for sk in gw.skeletons if not sk.mobile or sk.getNumDofs() == 0 for b in sk._ordered_bodies()]
    assert ground
    with pytest.raises(ValueError):
        f(gw, torch.zeros(2, 2 * gw.getNumDofs()), ground[:1])
