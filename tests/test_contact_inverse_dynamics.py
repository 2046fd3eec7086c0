"""Contact inverse dynamics on the CPU: the fp64 oracle (tests/oracle_id/cid_oracle.cpp) against a contact Jacobian built independently from
the step oracle's IKMapping velocity map, its independence of the contact body, its dual-number Jacobians against finite differences, the
device functions (csrc/nb2_dyn.cuh cid_*, host build) against the oracle, mass gradient included, and the argument checks that need no
device."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from nimblephysics_b200 import modelspec as ms
from tests.host_emul.binding_cid import EmulCidWorld
from tests.oracle_id.binding_cid import CidOracle
from tests.test_inverse_dynamics import id_inputs
from tests.test_per_world_mass import random_masses, raw_at, register
from tests.util import load_raw, rel_err

WELDED = "l_situational_awareness_camera_optical_frame"  # welded (through a camera link) to utorso in the URDF model


def _body(raw, name):
    return list(raw.body_names).index(name)


def _ik_contact_jacobian(ow, raw, s, body):
    """J_c [6, n] from the step oracle's IKMapping: the body's [omega; v_body_origin] in world axes for a unit qdot at fixed q, with the
    linear part shifted to the world origin (v_O = v_P - omega x p)."""
    n = raw.ndof
    J = np.zeros((6, n))
    for j in range(n):
        sj = s.copy()
        sj[n:] = 0.0
        sj[n + j] = 1.0
        pos, vel, _, _ = ow.ik(sj, [0], [body], want_jac=False)
        om, p = vel[:3], pos[3:6]
        J[:3, j] = om
        J[3:, j] = vel[3:6] - np.cross(om, p)
    return J


@pytest.mark.parametrize("name,bodies", [("atlas", ["l_foot", "r_hand", "pelvis", WELDED]), ("atlas_sdf", ["r_foot", "l_hand", "pelvis"])])
def test_oracle_matches_an_independent_contact_jacobian(oracle_mod, name, bodies):
    raw = load_raw(name)
    ow, co = oracle_mod.OracleWorld(raw), CidOracle(raw)
    n = raw.ndof
    s, vn = id_inputs(raw, 1, seed=21)
    s, vn = s[0].astype(np.float64), vn[0].astype(np.float64)
    tau_id = co.inverse_dynamics(s, vn)
    scale = max(1.0, np.abs(tau_id).max())
    for bn in bodies:
        b = _body(raw, bn)
        tau, w = co.contact_inverse_dynamics(b, s, vn)
        J = _ik_contact_jacobian(ow, raw, s, b)
        assert np.abs(tau + J.T @ w - tau_id).max() < 1e-9 * scale, bn
        assert np.abs(tau[:6]).max() < 1e-9 * scale, bn


def test_wrench_does_not_depend_on_the_contact_body():
    raw = load_raw("atlas")
    co = CidOracle(raw)
    n = raw.ndof
    s, vn = id_inputs(raw, 1, seed=22)
    s, vn = s[0].astype(np.float64), vn[0].astype(np.float64)
    tau_id = co.inverse_dynamics(s, vn)
    t1, w1 = co.contact_inverse_dynamics(_body(raw, "l_foot"), s, vn)
    t2, w2 = co.contact_inverse_dynamics(_body(raw, "r_hand"), s, vn)
    assert np.abs(w1 - w2).max() < 1e-9 * max(1.0, np.abs(w1).max())

    def chain_dofs(name):
        out, i = set(), _body(raw, name)
        while raw.parent[i] >= 0:
            out |= set(range(raw.dof_off[i], raw.dof_off[i] + ms.JOINT_NDOF[int(raw.jtype[i])]))
            i = raw.parent[i]
        return out

    off = [d for d in range(6, n) if d not in chain_dofs("l_foot") | chain_dofs("r_hand")]
    assert np.abs(t1[off] - t2[off]).max() < 1e-9 * max(1.0, np.abs(tau_id).max())
    assert np.array_equal(t1[off], tau_id[off])  # J_c has zero columns off the chain


@pytest.mark.parametrize("bn", ["l_foot", "pelvis", WELDED])
def test_oracle_jacobians_match_finite_differences(bn):
    raw = load_raw("atlas")
    co = CidOracle(raw)
    n, b = raw.ndof, _body(raw, bn)
    s, vn = id_inputs(raw, 1, seed=23)
    x = np.concatenate([s[0], vn[0]]).astype(np.float64)
    tau, w, J = co.contact_inverse_dynamics(b, x[:2 * n], x[2 * n:], want_jac=True)
    eps = 1e-6
    Jfd = np.zeros_like(J)
    for c in range(3 * n):
        xp, xm = x.copy(), x.copy()
        xp[c] += eps
        xm[c] -= eps
        tp, wp = co.contact_inverse_dynamics(b, xp[:2 * n], xp[2 * n:])
        tm, wm = co.contact_inverse_dynamics(b, xm[:2 * n], xm[2 * n:])
        Jfd[:, c] = (np.concatenate([tp, wp]) - np.concatenate([tm, wm])) / (2 * eps)
    assert np.abs(J - Jfd).max() < 1e-7 * max(1.0, np.abs(J).max())


@pytest.mark.parametrize("name,bn", [("atlas", "l_foot"), ("atlas", "pelvis"), ("atlas", WELDED), ("atlas_sdf", "r_hand")])
@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("lanes", [1, 4])
def test_emulated_contact_id_and_vjp_match_oracle(name, bn, fp64, lanes):
    raw = load_raw(name)
    try:
        cm = nb.compile_model(raw, lanes=lanes)
    except ValueError:
        pytest.skip(f"no {lanes}-lane schedule for this model")
    ew, co = EmulCidWorld(cm), CidOracle(raw)
    n, B, b = raw.ndof, 5, _body(raw, bn)
    s, vn = id_inputs(raw, B, seed=31 + lanes)
    rng = np.random.default_rng(lanes)
    gt, gw = rng.normal(size=(B, n)), rng.normal(size=(B, 6))
    tau, w, saved = ew.contact_inverse_dynamics(int(cm.body_owner[b]), s, vn, fp64)
    gs, gn, _ = ew.contact_inverse_dynamics_backward(int(cm.body_owner[b]), s, saved, w, gt, gw, fp64)
    tol = 1e-9 if fp64 else 1e-4
    cast = (lambda a: a.astype(np.float64)) if fp64 else (lambda a: a.astype(np.float32).astype(np.float64))
    for k in range(B):
        rt, rw, J = co.contact_inverse_dynamics(b, s[k].astype(np.float64), vn[k].astype(np.float64), want_jac=True)
        g = J.T @ np.concatenate([cast(gt[k]), cast(gw[k])])
        scale = max(np.linalg.norm(rt), np.linalg.norm(rw))
        assert np.linalg.norm(tau[k] - rt) < tol * scale and np.linalg.norm(w[k] - rw) < tol * scale, k
        assert rel_err(gs[k], g[:2 * n]) < tol, (k, rel_err(gs[k], g[:2 * n]))
        assert rel_err(gn[k], g[2 * n:]) < tol, (k, rel_err(gn[k], g[2 * n:]))


def test_emulated_per_world_mass_gradient_matches_oracle_differences():
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=4)
    B = 3
    M = random_masses(world, B, seed=19)
    wi = nb.mass_to_inertia(world, torch.tensor(M, dtype=torch.float64)).numpy()
    cm = nb.compile_model(raw, lanes=2)
    ew = EmulCidWorld(cm)
    b = _body(raw, "r_foot")
    s, vn = id_inputs(raw, B, seed=15)
    rng = np.random.default_rng(16)
    gt, gw = rng.normal(size=(B, raw.ndof)), rng.normal(size=(B, 6))
    tau, w, saved = ew.contact_inverse_dynamics(int(cm.body_owner[b]), s, vn, True, world_inertia=wi)
    _, _, gi = ew.contact_inverse_dynamics_backward(int(cm.body_owner[b]), s, saved, w, gt, gw, True, world_inertia=wi)
    entries = world._mass_entries()
    for k in range(B):
        s64, vn64 = s[k].astype(np.float64), vn[k].astype(np.float64)
        rw = raw_at(raw, entries, M[k])
        rt, rwr = CidOracle(rw).contact_inverse_dynamics(b, s64, vn64)
        assert rel_err(tau[k], rt) < 1e-9 and rel_err(w[k], rwr) < 1e-9
        gm = ms.inertia_param_jacobian(rw, cm, entries) @ gi[:, k]

        def loss(mv):
            t, ww = CidOracle(raw_at(raw, entries, mv)).contact_inverse_dynamics(b, s64, vn64)
            return float(gt[k] @ t + gw[k] @ ww)

        fd = np.array([(loss(M[k] + 1e-5 * e) - loss(M[k] - 1e-5 * e)) / 2e-5 for e in np.eye(len(M[k]))])
        assert rel_err(gm, fd) < 1e-7, (gm, fd)


def _rows(world, B=2):
    n = world.getNumDofs()
    return torch.zeros(B, 2 * n), torch.zeros(B, n)


@pytest.mark.parametrize("name", ["cartpole", "half_cheetah"])
def test_a_root_that_is_not_free_is_refused(name):
    world = nb.World.from_raw(load_raw(name))
    body = world.getBodyNodeByIndex(world.getNumBodyNodes() - 1)
    with pytest.raises(ValueError, match="FreeJoint"):
        nb.contact_inverse_dynamics(world, *_rows(world), body)


def test_bad_bodies_and_shapes_are_refused():
    world = nb.World.from_raw(load_raw("atlas_ground"))
    other = nb.World.from_raw(load_raw("atlas"))
    foot = next(b for b in world.skeletons[0]._ordered_bodies() if b.name == "l_foot")
    s, v = _rows(world)
    with pytest.raises(ValueError, match="not a body of this world"):
        nb.contact_inverse_dynamics(world, s, v, other.getBodyNodeByIndex(27))
    ground = world.skeletons[1]._ordered_bodies()[0]  # welded to the world: nothing moves
    with pytest.raises(ValueError, match="immobile"):
        nb.contact_inverse_dynamics(world, s, v, ground)
    frozen = nb.World.from_raw(load_raw("atlas"))
    frozen.skeletons[0].setMobile(False)
    with pytest.raises(ValueError, match="immobile"):
        nb.contact_inverse_dynamics(frozen, *_rows(frozen), frozen.getBodyNodeByIndex(27))
    with pytest.raises(ValueError, match="state has shape"):
        nb.contact_inverse_dynamics(world, s[:, 1:], v, foot)
    with pytest.raises(ValueError, match="next_vel has shape"):
        nb.contact_inverse_dynamics(world, s, v[:1], foot)
    with pytest.raises(ValueError, match="next_vel has shape"):
        nb.contact_inverse_dynamics(world, s, v[0], foot)
