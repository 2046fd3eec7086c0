"""World Jacobians of body points and of a skeleton's COM on the host: an fp64 oracle built on the step oracle's kinematics (its IKMapping
rows, d vel / d qdot by dual numbers, extended by an offset) pinned against a welded child frame and the oracle's body velocities; the
host-emulated device functions (tests/host_emul/emul_jac.cpp) against that oracle for J, the position, offset and per-world mass VJPs,
on the models of test_mass_matrix; welded and static nodes, exact zeros off the chain; and the argument checks of
nimblephysics_b200.world_jacobian / com_jacobian."""
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import nimblephysics_b200 as nb
from nimblephysics_b200 import modelspec as ms
from nimblephysics_b200.world_jacobian import MAX_NODES
from oracle.binding import OracleWorld
from tests.host_emul.binding_jac import EmulJacWorld
from tests.test_mass_matrix import MODELS, built_world, model_raw, positions
from tests.test_per_world_mass import random_masses, raw_at, register
from tests.util import load_raw, rel_err


def _skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


def oracle_point(raw, q, ri, offset=None, qd=None):
    """fp64 J [6, n] of raw body ri at the point `offset` of its frame: the oracle's spatial IKMapping rows [omega; v_origin] (dual
    numbers in qdot) with v = v_origin + omega x R o.  With qd: also the oracle's [omega; v] of the point at (q, qd)."""
    ow = OracleWorld(raw)
    n = raw.ndof
    pos, vel, _, Jv = ow.ik(np.concatenate([q, np.zeros(n) if qd is None else qd]), [0], [ri])
    r = Rotation.from_rotvec(pos[:3]).as_matrix() @ (np.zeros(3) if offset is None else np.asarray(offset, np.float64))
    J = Jv.copy()
    J[3:] -= _skew(r) @ Jv[:3]
    if qd is None:
        return J
    return J, np.concatenate([vel[:3], vel[3:] + np.cross(vel[:3], r)])


def oracle_com(raw, q, ri, qd=None):
    """fp64 J_com [3, n] of the skeleton of raw body ri (the oracle's COM IKMapping rows)."""
    n = raw.ndof
    _, vel, _, Jv = OracleWorld(raw).ik(np.concatenate([q, np.zeros(n) if qd is None else qd]), [3], [ri])
    return Jv if qd is None else (Jv, vel)


def canon_nodes(cm, ris):
    """raw bodies -> (canonical owners, owner <- body transforms), as world_jacobian.resolve_nodes maps BodyNodes."""
    return np.array([cm.body_owner[r] for r in ris], np.int32), np.stack([np.asarray(cm.body_T[r], np.float64) for r in ris])


def canon_root(cm, ri):
    o = int(cm.body_owner[ri])
    while cm.parent[o] >= 0:
        o = int(cm.parent[o])
    return o


def mobile_nodes(raw, cm):
    mob = [r for r in range(raw.nb) if cm.body_owner[r] >= 0]
    return sorted({mob[0], mob[len(mob) // 2], mob[-1]})


def com_body(raw, cm):
    """the root (a raw body) of the largest skeleton whose root moves, or None (a skeleton fixed to the world has no COM Jacobian)"""
    roots = [r for r in range(raw.nb) if raw.parent[r] < 0 and cm.body_owner[r] >= 0]
    if not roots:
        return None
    return max(roots, key=lambda r: sum(1 for i in range(raw.nb) if raw.skel_id[i] == raw.skel_id[r]))


@pytest.mark.parametrize("name", ["cartpole", "half_cheetah", "atlas"])
def test_oracle_is_the_derivative_of_the_body_velocities(name):
    raw = model_raw(name)
    cm = nb.compile_model(raw, lanes=1)
    q = positions(raw, 1, seed=2)[0].astype(np.float64)
    qd = np.random.default_rng(3).normal(size=raw.ndof)
    o = np.array([0.03, -0.05, 0.11])
    for ri in mobile_nodes(raw, cm):
        J, v = oracle_point(raw, q, ri, o, qd)
        assert rel_err(J @ qd, v) < 1e-12
    rc = com_body(raw, cm)
    if rc is not None:
        Jc, vc = oracle_com(raw, q, rc, qd)
        assert rel_err(Jc @ qd, vc) < 1e-12


def _welded_world(o):
    """free root - revolute - revolute, the last body carrying a welded child frame at translation o, and a static skeleton."""
    w = nb.World()
    w.setTimeStep(1e-3)
    sk = nb.Skeleton("arm")
    j, root = sk.createFreeJointAndBodyNodePair(None)
    p = root
    for k in range(2):
        j, p = sk.createRevoluteJointAndBodyNodePair(p)
        j.setAxis([[0, 0, 1], [0, 1, 0]][k])
        T = nb.Isometry3()
        T.set_translation([0.1, 0.02 * k, 0.3])
        j.setTransformFromParentBodyNode(T)
        p.setMass(1.0 + k)
    j, tip = sk.createWeldJointAndBodyNodePair(p)
    T = nb.Isometry3()
    T.set_translation(list(o))
    j.setTransformFromParentBodyNode(T)
    tip.setMass(0.5)
    w.addSkeleton(sk)
    g = nb.Skeleton("ground")
    g.createWeldJointAndBodyNodePair(None)
    w.addSkeleton(g)
    return w, p, tip


def test_oracle_offset_equals_a_welded_child_frame():
    o = np.array([0.07, -0.04, 0.12])
    w, p, tip = _welded_world(o)
    raw = nb.flatten_world(w)
    q = positions(raw, 1, seed=4)[0].astype(np.float64)
    ris = {id(b): k for k, b in enumerate(b for sk in w.skeletons for b in sk._ordered_bodies())}
    assert rel_err(oracle_point(raw, q, ris[id(p)], o), oracle_point(raw, q, ris[id(tip)])) < 1e-12


@pytest.mark.parametrize("name", MODELS)
@pytest.mark.parametrize("fp64", [False, True])
def test_emulated_forward_matches_oracle(name, fp64):
    raw = model_raw(name)
    cm = nb.compile_model(raw, lanes=1)
    ew = EmulJacWorld(cm)
    B, n = 2, raw.ndof
    q = positions(raw, B, seed=21)
    ris = mobile_nodes(raw, cm)
    bodies, T = canon_nodes(cm, ris)
    off = np.random.default_rng(22).uniform(-0.1, 0.1, (B, len(ris), 3))
    J = ew.world_jacobian(q, bodies, T, off, fp64=fp64)
    J0 = ew.world_jacobian(q, bodies, T, None, fp64=fp64)
    rc = com_body(raw, cm)
    Jc = ew.com_jacobian(q, canon_root(cm, rc), fp64=fp64) if rc is not None else None
    tol = 1e-9 if fp64 else 1e-4
    for w in range(B):
        qw = q[w].astype(np.float64) if fp64 else q[w].astype(np.float32).astype(np.float64)
        for e, ri in enumerate(ris):
            assert rel_err(J[w, e], oracle_point(raw, qw, ri, off[w, e])) < tol, (w, ri)
            assert rel_err(J0[w, e], oracle_point(raw, qw, ri)) < tol, (w, ri)
        if rc is not None:
            assert rel_err(Jc[w], oracle_com(raw, qw, rc)) < tol
    assert J.shape == (B, len(ris), 6, n)


def _on_chain(cm, body):
    cols = np.zeros(cm.ndof, bool)
    j = body
    while j >= 0:
        cols[cm.dof_off[j]:cm.dof_off[j] + (6 if cm.jtype[j] == 3 else 1)] = True
        j = cm.parent[j]
    return cols


@pytest.mark.parametrize("name", ["free_child", "atlas", "limit"])
def test_emulated_exact_zeros_off_the_chain_and_static_nodes(name):
    raw = model_raw(name)
    cm = nb.compile_model(raw, lanes=1)
    ew = EmulJacWorld(cm)
    q = positions(raw, 3, seed=4)
    ris = mobile_nodes(raw, cm)
    bodies, T = canon_nodes(cm, ris)
    bodies = np.concatenate([bodies, [-1]])
    T = np.concatenate([T, np.eye(4)[None]])
    for fp64 in (False, True):
        J = ew.world_jacobian(q, bodies, T, fp64=fp64)
        for e, b in enumerate(bodies[:-1]):
            assert np.all(J[:, e][:, :, ~_on_chain(cm, b)] == 0)
            assert np.all(np.any(J[:, e][:, :, _on_chain(cm, b)] != 0, axis=1))
        assert np.all(J[:, -1] == 0)
        rc = com_body(raw, cm)
        Jc = ew.com_jacobian(q, canon_root(cm, rc), fp64=fp64)
        tree = np.zeros(cm.ndof, bool)
        for i in range(cm.nb):
            r = i
            while cm.parent[r] >= 0:
                r = cm.parent[r]
            if r == canon_root(cm, rc):
                tree |= _on_chain(cm, i)
        assert np.all(Jc[:, :, ~tree] == 0)


def test_emulated_welded_and_static_nodes():
    o = np.array([0.07, -0.04, 0.12])
    w, p, tip = _welded_world(o)
    raw = nb.flatten_world(w)
    cm = nb.compile_model(raw, lanes=1)
    ew = EmulJacWorld(cm)
    ris = {id(b): k for k, b in enumerate(b for sk in w.skeletons for b in sk._ordered_bodies())}
    ground = ris[id(w.skeletons[1]._ordered_bodies()[0])]
    assert cm.body_owner[ground] == -1 and cm.body_owner[ris[id(tip)]] == cm.body_owner[ris[id(p)]]
    q = positions(raw, 2, seed=5).astype(np.float64)
    bodies, T = canon_nodes(cm, [ris[id(tip)], ris[id(p)], ground])
    off = np.zeros((2, 3, 3))
    off[:, 1] = o
    J = ew.world_jacobian(q, bodies, T, off, fp64=True)
    assert rel_err(J[:, 0], J[:, 1]) < 1e-14 and np.all(J[:, 2] == 0)
    for wi in range(2):
        assert rel_err(J[wi, 0], oracle_point(raw, q[wi], ris[id(tip)])) < 1e-12


def _fd(f, x, h):
    return np.array([(f(x + h * e) - f(x - h * e)) / (2 * h) for e in np.eye(len(x))])


@pytest.mark.parametrize("name", ["cartpole", "tree", "half_cheetah", "atlas", "atlas_sdf", "free_child"])
def test_emulated_position_and_offset_vjp_match_oracle_differences(name):
    raw = model_raw(name)
    cm = nb.compile_model(raw, lanes=1)
    ew = EmulJacWorld(cm)
    n, B = raw.ndof, 2
    q = positions(raw, B, seed=31).astype(np.float64)
    ris = mobile_nodes(raw, cm)
    bodies, T = canon_nodes(cm, ris)
    rng = np.random.default_rng(32)
    off = rng.uniform(-0.1, 0.1, (B, len(ris), 3))
    G = rng.normal(size=(B, len(ris), 6, n))
    gp, go = ew.world_jacobian_backward(q, bodies, T, G, off, fp64=True)
    gp32, go32 = ew.world_jacobian_backward(q, bodies, T, G, off, fp64=False)
    rc = com_body(raw, cm)
    Gc = rng.normal(size=(B, 3, n))
    if rc is not None:
        gc, _ = ew.com_jacobian_backward(q, canon_root(cm, rc), Gc, fp64=True)
        gc32, _ = ew.com_jacobian_backward(q, canon_root(cm, rc), Gc, fp64=False)
    for w in range(B):
        loss = lambda x: sum(float(np.sum(G[w, e] * oracle_point(raw, x, ri, off[w, e]))) for e, ri in enumerate(ris))
        fd = _fd(loss, q[w], 1e-6)
        assert rel_err(gp[w], fd) < 1e-7, (w, rel_err(gp[w], fd))
        assert rel_err(gp32[w], gp[w]) < 1e-4
        for e, ri in enumerate(ris):
            lo = lambda o: float(np.sum(G[w, e] * oracle_point(raw, q[w], ri, o)))
            fdo = _fd(lo, off[w, e], 1e-6)
            assert rel_err(go[w, e], fdo) < 1e-7 and rel_err(go32[w, e], go[w, e]) < 1e-4
        if rc is None:
            continue
        lc = lambda x: float(np.sum(Gc[w] * oracle_com(raw, x, rc)))
        fdc = _fd(lc, q[w], 1e-6)
        assert rel_err(gc[w], fdc) < 1e-7, (w, rel_err(gc[w], fdc))
        assert rel_err(gc32[w], gc[w]) < 1e-4


@pytest.mark.parametrize("name", ["half_cheetah", "atlas"])
def test_emulated_per_world_mass_vjp_matches_oracle_differences(name):
    raw = load_raw(name)
    world = register(nb.World.from_raw(raw), step=4)
    B = 2
    mv = random_masses(world, B, seed=9)
    wi = nb.mass_to_inertia(world, torch.tensor(mv, dtype=torch.float64)).numpy()
    cm = nb.compile_model(raw, lanes=1)
    ew = EmulJacWorld(cm)
    q = positions(raw, B, seed=5).astype(np.float64)
    rc = com_body(raw, cm)
    root = canon_root(cm, rc)
    G = np.random.default_rng(6).normal(size=(B, 3, raw.ndof))
    J = ew.com_jacobian(q, root, fp64=True, world_inertia=wi)
    _, gi = ew.com_jacobian_backward(q, root, G, fp64=True, world_inertia=wi)
    entries = world._mass_entries()
    for w in range(B):
        rw = raw_at(raw, entries, mv[w])
        assert rel_err(J[w], oracle_com(rw, q[w], rc)) < 1e-9
        gm = ms.inertia_param_jacobian(rw, cm, entries) @ gi[:, w]
        loss = lambda m: float(np.sum(G[w] * oracle_com(raw_at(raw, entries, m), q[w], rc)))
        fd = _fd(loss, mv[w], 1e-6)
        assert rel_err(gm, fd) < 1e-7, (w, rel_err(gm, fd))


def test_value_errors():
    raw = load_raw("half_cheetah")
    world = register(nb.World.from_raw(raw), step=2)
    other = nb.World.from_raw(raw)
    n, m = raw.ndof, world.getMassDims()
    sk = max(world.skeletons, key=lambda s: s.getNumDofs())
    node = sk._ordered_bodies()[-1]
    for bad in (torch.zeros(n + 1), torch.zeros(2, n - 1), torch.zeros(2, 3, n), torch.zeros(0, n)):
        with pytest.raises(ValueError):
            nb.world_jacobian(world, bad, [node])
        with pytest.raises(ValueError):
            nb.com_jacobian(world, bad, sk)
    q = torch.zeros(2, n)
    for bad_off in (torch.zeros(2), torch.zeros(1, 4), torch.zeros(3, 1, 3), torch.zeros(2, 2, 3)):
        with pytest.raises(ValueError):
            nb.world_jacobian(world, q, [node], bad_off)
    with pytest.raises(ValueError):
        nb.world_jacobian(world, torch.zeros(n), [node], torch.zeros(2, 1, 3))
    with pytest.raises(ValueError):
        nb.world_jacobian(world, q, [])
    with pytest.raises(ValueError):
        nb.world_jacobian(world, q, [node] * (MAX_NODES + 1))
    with pytest.raises(ValueError):
        nb.world_jacobian(world, q, [other.skeletons[-1]._ordered_bodies()[-1]])
    with pytest.raises(ValueError):
        nb.com_jacobian(world, q, max(other.skeletons, key=lambda s: s.getNumDofs()))
    static = [s for s in world.skeletons if s.getNumDofs() == 0]
    if static:
        with pytest.raises(ValueError):
            nb.com_jacobian(world, q, static[0])
    for bad_m in (torch.zeros(m + 1, dtype=torch.float64), torch.zeros(2, m + 1, dtype=torch.float64), torch.zeros(3, m, dtype=torch.float64)):
        with pytest.raises(ValueError):
            nb.com_jacobian(world, q, sk, bad_m)
    with pytest.raises(ValueError):
        nb.com_jacobian(world, torch.zeros(n), sk, torch.zeros(2, m, dtype=torch.float64))
    with pytest.raises(ValueError):
        nb.world_jacobian(nb.World(), torch.zeros(2, 0), [node])
