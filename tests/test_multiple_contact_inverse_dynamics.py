"""Multiple-contact inverse dynamics on the CPU: the fp64 oracle (tests/oracle_id/mcid_oracle.cpp, a KKT solve of the definition) against
contact Jacobians built independently from the step oracle's IKMapping velocity map, its optimality and invariances, its reduction to the
one-body oracle, its dual-number Jacobians against finite differences, the device functions (csrc/nb2_dyn.cuh mcid_*, host build)
against the oracle, mass and guess gradients included, and the argument checks that need no device."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from tests.host_emul.binding_mcid import EmulMcidWorld
from tests.oracle_id.binding_mcid import McidOracle
from tests.test_contact_inverse_dynamics import WELDED, _ik_contact_jacobian
from tests.test_inverse_dynamics import id_inputs
from tests.test_per_world_mass import random_masses, raw_at, register
from tests.util import load_raw, rel_err

FEET = ["l_foot", "r_foot"]
LIMBS = ["l_foot", "r_foot", "l_hand", "r_hand"]


def _bodies(raw, names):
    return [list(raw.body_names).index(n) for n in names]


def _inputs(raw, seed):
    s, vn = id_inputs(raw, 1, seed=seed)
    return s[0].astype(np.float64), vn[0].astype(np.float64)


def _gam_inv(p, w):
    """Gamma(p)^-1 w: a wrench about the origin -> about p"""
    return np.concatenate([w[:3] - np.cross(p, w[3:]), w[3:]])


def _points(ow, s, bodies):
    return [ow.ik(s, [0], [b], want_jac=False)[0][3:6] for b in bodies]


@pytest.mark.parametrize("name,names", [("atlas", FEET), ("atlas", LIMBS), ("atlas", ["l_foot", "r_hand", WELDED]),
                                        ("atlas_sdf", FEET), ("atlas_sdf", LIMBS)])
def test_oracle_satisfies_the_definition(oracle_mod, name, names):
    raw = load_raw(name)
    ow, mo = oracle_mod.OracleWorld(raw), McidOracle(raw)
    s, vn = _inputs(raw, 41)
    bodies = _bodies(raw, names)
    tau_id = mo.inverse_dynamics(s, vn)
    scale = max(1.0, np.abs(tau_id).max())
    g = np.random.default_rng(3).normal(0, 50, (len(bodies), 6))
    for guess in (None, g):
        tau, w = mo.multiple_contact_inverse_dynamics(bodies, s, vn, guess)
        JTw = sum(_ik_contact_jacobian(ow, raw, s, b).T @ w[i] for i, b in enumerate(bodies))
        assert np.abs(tau + JTw - tau_id).max() < 1e-9 * scale
        assert np.abs(tau[:6]).max() < 1e-9 * scale
        # the wrenches sum to the one-body wrench
        _, wc = mo.contact_inverse_dynamics(bodies[0], s, vn)
        assert np.abs(w.sum(0) - wc).max() < 1e-9 * max(1.0, np.abs(wc).max())
        # optimality: Gamma_i^-1 (w_i - g_i) = Gamma_i^T lambda for one lambda, i.e. Gamma_i^-T Gamma_i^-1 (w_i - g_i) is the same for all i
        gi = np.zeros_like(w) if guess is None else guess
        lams = []
        for i, p in enumerate(_points(ow, s, bodies)):
            e = _gam_inv(p, w[i] - gi[i])
            lams.append(np.concatenate([e[:3], e[3:] + np.cross(p, e[:3])]))  # Gamma_i^-T e
        assert max(np.abs(l - lams[0]).max() for l in lams) < 1e-9 * max(1.0, np.abs(w).max())


def test_one_body_is_the_contact_oracle():
    raw = load_raw("atlas")
    mo = McidOracle(raw)
    s, vn = _inputs(raw, 42)
    for b in _bodies(raw, ["l_foot", "r_hand", WELDED]):
        tau, w = mo.multiple_contact_inverse_dynamics([b], s, vn, np.full((1, 6), 7.0))
        tc, wc = mo.contact_inverse_dynamics(b, s, vn)
        assert np.abs(tau - tc).max() < 1e-9 * max(1.0, np.abs(tc).max()) and np.abs(w[0] - wc).max() < 1e-9 * max(1.0, np.abs(wc).max())


def test_consistent_guesses_come_back_unchanged():
    raw = load_raw("atlas")
    mo = McidOracle(raw)
    s, vn = _inputs(raw, 43)
    bodies = _bodies(raw, LIMBS)
    _, W = mo.contact_inverse_dynamics(bodies[0], s, vn)
    g = np.random.default_rng(4).normal(0, 80, (4, 6))
    g[-1] = W - g[:-1].sum(0)
    _, w = mo.multiple_contact_inverse_dynamics(bodies, s, vn, g)
    assert np.abs(w - g).max() < 1e-9 * np.abs(g).max()


def test_the_split_about_each_point_does_not_depend_on_the_origin(oracle_mod):
    raw = load_raw("atlas")
    ow, mo = oracle_mod.OracleWorld(raw), McidOracle(raw)
    s, vn = _inputs(raw, 44)
    bodies = _bodies(raw, LIMBS)
    s2 = s.copy()
    s2[3:6] += [3.0, -2.0, 0.7]  # the free root's translation
    local = []
    for x in (s, s2):
        _, w = mo.multiple_contact_inverse_dynamics(bodies, x, vn)
        local.append(np.array([_gam_inv(p, w[i]) for i, p in enumerate(_points(ow, x, bodies))]))
    assert np.abs(local[0] - local[1]).max() < 1e-9 * np.abs(local[0]).max()


@pytest.mark.parametrize("names", [FEET, ["l_foot", "pelvis", WELDED]])
def test_oracle_jacobians_match_finite_differences(names):
    raw = load_raw("atlas")
    mo = McidOracle(raw)
    n, bodies = raw.ndof, _bodies(raw, names)
    k = len(bodies)
    s, vn = _inputs(raw, 45)
    g = np.random.default_rng(5).normal(0, 30, 6 * k)
    x = np.concatenate([s, vn, g])
    split = lambda x: (x[:2 * n], x[2 * n:3 * n], x[3 * n:])
    tau, w, J = mo.multiple_contact_inverse_dynamics(bodies, *split(x), want_jac=True)
    eps = 1e-6
    Jfd = np.zeros_like(J)
    for c in range(len(x)):
        xp, xm = x.copy(), x.copy()
        xp[c] += eps
        xm[c] -= eps
        tp, wp = mo.multiple_contact_inverse_dynamics(bodies, *split(xp))
        tm, wm = mo.multiple_contact_inverse_dynamics(bodies, *split(xm))
        Jfd[:, c] = (np.concatenate([tp, wp.ravel()]) - np.concatenate([tm, wm.ravel()])) / (2 * eps)
    assert np.abs(J - Jfd).max() < 1e-7 * max(1.0, np.abs(J).max())


def _device_set(cm, bodies):
    return [int(cm.body_owner[b]) for b in bodies], [cm.body_T[b][:3, 3] for b in bodies]


@pytest.mark.parametrize("name,names", [("atlas", FEET), ("atlas", LIMBS), ("atlas", ["r_foot", "l_hand", WELDED]), ("atlas_sdf", LIMBS),
                                        ("atlas", ["l_foot"])])
@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("guessed", [False, True])
def test_emulated_multiple_contact_id_and_vjp_match_oracle(name, names, fp64, guessed):
    raw = load_raw(name)
    cm = nb.compile_model(raw, lanes=2)
    ew, mo = EmulMcidWorld(cm), McidOracle(raw)
    n, B, bodies = raw.ndof, 5, _bodies(raw, names)
    k = len(bodies)
    s, vn = id_inputs(raw, B, seed=51 + k)
    rng = np.random.default_rng(k)
    g = rng.normal(0, 40, (B, k, 6)) if guessed else None
    gt, gw = rng.normal(size=(B, n)), rng.normal(size=(B, k, 6))
    db, dp = _device_set(cm, bodies)
    tau, w, saved = ew.multiple_contact_inverse_dynamics(db, dp, s, vn, g, fp64)
    gs, gn, _, gg = ew.multiple_contact_inverse_dynamics_backward(db, dp, s, saved, w, gt, gw, g, fp64)
    tol = 1e-9 if fp64 else 1e-4
    cast = (lambda a: a.astype(np.float64)) if fp64 else (lambda a: a.astype(np.float32).astype(np.float64))
    for b in range(B):
        gb = cast(g[b]) if guessed else None
        rt, rw, J = mo.multiple_contact_inverse_dynamics(bodies, cast(s[b]), cast(vn[b]), gb, want_jac=True)
        ref = J.T @ np.concatenate([cast(gt[b]), cast(gw[b]).ravel()])
        scale = max(np.linalg.norm(rt), np.linalg.norm(rw))
        assert np.linalg.norm(tau[b] - rt) < tol * scale and np.linalg.norm(w[b] - rw) < tol * scale, b
        assert rel_err(gs[b], ref[:2 * n]) < tol, (b, rel_err(gs[b], ref[:2 * n]))
        assert rel_err(gn[b], ref[2 * n:3 * n]) < tol, (b, rel_err(gn[b], ref[2 * n:3 * n]))
        if k == 1:
            assert not np.any(gg[b])
        else:
            assert rel_err(gg[b].ravel(), ref[3 * n:]) < tol, (b, rel_err(gg[b].ravel(), ref[3 * n:]))


def test_emulated_per_world_mass_gradient_matches_oracle_differences():
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=4)
    B = 3
    M = random_masses(world, B, seed=29)
    wi = nb.mass_to_inertia(world, torch.tensor(M, dtype=torch.float64)).numpy()
    cm = nb.compile_model(raw, lanes=2)
    ew = EmulMcidWorld(cm)
    bodies = _bodies(raw, LIMBS)
    db, dp = _device_set(cm, bodies)
    s, vn = id_inputs(raw, B, seed=25)
    rng = np.random.default_rng(26)
    g = rng.normal(0, 40, (B, 4, 6))
    gt, gw = rng.normal(size=(B, raw.ndof)), rng.normal(size=(B, 4, 6))
    tau, w, saved = ew.multiple_contact_inverse_dynamics(db, dp, s, vn, g, True, world_inertia=wi)
    _, _, gi, _ = ew.multiple_contact_inverse_dynamics_backward(db, dp, s, saved, w, gt, gw, g, True, world_inertia=wi)
    entries = world._mass_entries()
    for b in range(B):
        s64, vn64 = s[b].astype(np.float64), vn[b].astype(np.float64)
        rw = raw_at(raw, entries, M[b])
        rt, rwr = McidOracle(rw).multiple_contact_inverse_dynamics(bodies, s64, vn64, g[b])
        assert rel_err(tau[b], rt) < 1e-9 and rel_err(w[b], rwr) < 1e-9
        gm = nb.modelspec.inertia_param_jacobian(rw, cm, entries) @ gi[:, b]

        def loss(mv):
            t, ww = McidOracle(raw_at(raw, entries, mv)).multiple_contact_inverse_dynamics(bodies, s64, vn64, g[b])
            return float(gt[b] @ t + (gw[b] * ww).sum())

        fd = np.array([(loss(M[b] + 1e-5 * e) - loss(M[b] - 1e-5 * e)) / 2e-5 for e in np.eye(len(M[b]))])
        assert rel_err(gm, fd) < 1e-7, (gm, fd)


def _rows(world, B=2):
    n = world.getNumDofs()
    return torch.zeros(B, 2 * n), torch.zeros(B, n)


def _node(world, name, sk=0):
    return next(b for b in world.skeletons[sk]._ordered_bodies() if b.name == name)


def test_bad_contact_sets_and_shapes_are_refused():
    world = nb.World.from_raw(load_raw("atlas_ground"))
    lf, rf, lh, rh, pel = (_node(world, n) for n in ("l_foot", "r_foot", "l_hand", "r_hand", "pelvis"))
    s, v = _rows(world)
    f = nb.multiple_contact_inverse_dynamics
    with pytest.raises(ValueError, match="0 contact bodies"):
        f(world, s, v, [])
    with pytest.raises(ValueError, match="5 contact bodies"):
        f(world, s, v, [lf, rf, lh, rh, pel])
    with pytest.raises(ValueError, match="appears twice"):
        f(world, s, v, [lf, rf, lf])
    other = nb.World.from_raw(load_raw("atlas"))
    with pytest.raises(ValueError, match="not a body of this world"):
        f(world, s, v, [lf, _node(other, "r_foot")])
    with pytest.raises(ValueError, match="immobile"):
        f(world, s, v, [lf, world.skeletons[1]._ordered_bodies()[0]])
    frozen = nb.World.from_raw(load_raw("atlas"))
    frozen.skeletons[0].setMobile(False)
    with pytest.raises(ValueError, match="immobile"):
        f(frozen, *_rows(frozen), [_node(frozen, "l_foot"), _node(frozen, "r_foot")])
    for name in ("cartpole", "half_cheetah"):
        w2 = nb.World.from_raw(load_raw(name))
        last = w2.getBodyNodeByIndex(w2.getNumBodyNodes() - 1)
        with pytest.raises(ValueError, match="FreeJoint"):
            f(w2, *_rows(w2), [last, last.parent_body])
    two = nb.World.from_raw(load_raw("atlas"))
    sk = nb.Skeleton("box")
    _, box = sk.createFreeJointAndBodyNodePair(None)
    box.setMass(3.0)
    two.addSkeleton(sk)
    with pytest.raises(ValueError, match="different skeletons"):
        f(two, *_rows(two), [_node(two, "l_foot"), box])
    with pytest.raises(ValueError, match="wrench_guesses has shape"):
        f(world, s, v, [lf, rf], wrench_guesses=torch.zeros(2, 3, 6))
    with pytest.raises(ValueError, match="wrench_guesses has shape"):
        f(world, s[0], v[0], [lf, rf], wrench_guesses=torch.zeros(1, 2, 6))
    with pytest.raises(ValueError, match="state has shape"):
        f(world, s[:, 1:], v, [lf, rf])
    with pytest.raises(ValueError, match="next_vel has shape"):
        f(world, s, v[:1], [lf, rf])
