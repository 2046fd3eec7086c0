"""Mass matrix and its inverse on the host: the oracle's M (columns of inverse-dynamics differences) against the numpy Lagrangian, the
host-emulated device functions (tests/host_emul/emul_mm.cpp) against the oracle for M, M^-1, the position VJP and the per-world mass VJP,
on the reference models, a model whose dofs do not follow the bodies' DFS order (Atlas from SDF), several skeletons, a non-root free joint
and the compiled limits; and the argument checks of nimblephysics_b200.mass_matrix / inverse_mass_matrix."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from tests.host_emul.binding_mm import EmulMmWorld
from tests.oracle_id.binding import IdOracle
from tests.test_inverse_dynamics import _velocity_map, id_inputs
from tests.test_oracle import _tree_world, mass_matrix as lagrangian_M
from tests.test_per_world_mass import random_masses, raw_at, register
from tests.util import load_raw, rel_err


def oracle_M(raw, q):
    """fp64 M(q) from the inverse-dynamics oracle: M e_j = ID(q, 0, dt e_j) - ID(q, 0, 0)."""
    n = raw.ndof
    ow = IdOracle(raw)
    s = np.concatenate([q, np.zeros(n)])
    t0 = ow.inverse_dynamics(s, np.zeros(n))
    return np.stack([ow.inverse_dynamics(s, raw.dt * e) - t0 for e in np.eye(n)], 1)


def _body(sk, kind, parent, k, offset=0.15):
    j, b = getattr(sk, f"create{kind}JointAndBodyNodePair")(parent)
    if kind != "Free":
        j.setAxis([[0, 0, 1], [0, 1, 0], [1, 0, 0]][k % 3])
    T = nb.Isometry3()
    T.set_translation([0.02 * (k % 2), 0.0, offset if parent is not None else 0.0])
    j.setTransformFromParentBodyNode(T)
    b.setMass(1.0 + 0.1 * (k % 7))
    b.setLocalCOM([0.01 * (k % 3), 0.005, 0.07])
    b.setMomentOfInertia(0.02, 0.03, 0.015, 0.001, 0.0005, 0.002)
    return b


def built_world(name):
    """Worlds built for the limits and the tree shapes the loaders do not produce:
    chain64: 64 revolute / prismatic bodies in one chain (NB2_MAX_BODIES); free16: 16 free-floating bodies, 96 dofs (NB2_MAX_DOFS);
    limit: 7 free roots with 54 revolute bodies below them, 61 bodies and 96 dofs (the largest working set of the M^-1 kernel);
    free_child: a free joint below a revolute joint below a free root, and a second skeleton (an arm) beside it."""
    w = nb.World()
    w.setTimeStep(1e-3)
    if name == "chain64":
        sk, p = nb.Skeleton("chain"), None
        for k in range(64):
            p = _body(sk, "Prismatic" if k % 5 == 4 else "Revolute", p, k)
        w.addSkeleton(sk)
    elif name == "free16":
        for k in range(16):
            sk = nb.Skeleton(f"box{k}")
            _body(sk, "Free", None, k)
            w.addSkeleton(sk)
    elif name == "limit":
        for r, m in enumerate([8, 8, 8, 8, 8, 7, 7]):
            sk = nb.Skeleton(f"tree{r}")
            root = p = _body(sk, "Free", None, r)
            for k in range(m):
                p = _body(sk, "Revolute", root if k == m // 2 else p, k)
            w.addSkeleton(sk)
    elif name == "free_child":
        sk = nb.Skeleton("floating")
        root = _body(sk, "Free", None, 0)
        arm = _body(sk, "Revolute", root, 1)
        tip = _body(sk, "Free", arm, 2)
        _body(sk, "Revolute", tip, 3)
        _body(sk, "Prismatic", root, 4)
        w.addSkeleton(sk)
        sk2, p = nb.Skeleton("arm"), None
        for k in range(3):
            p = _body(sk2, "Revolute", p, k)
        w.addSkeleton(sk2)
    else:
        raise KeyError(name)
    return w


def model_raw(name):
    if name == "tree":
        return nb.flatten_world(_tree_world())
    if name in ("chain64", "free16", "limit", "free_child"):
        return nb.flatten_world(built_world(name))
    return load_raw(name)


def positions(raw, B, seed):
    s, _ = id_inputs(raw, B, seed=seed)
    return s[:, :raw.ndof]


@pytest.mark.parametrize("name", ["cartpole", "tree", "half_cheetah", "atlas", "atlas_sdf"])
def test_oracle_M_matches_lagrangian_mechanics(name):
    raw = model_raw(name)
    q = positions(raw, 1, seed=3)[0].astype(np.float64)
    Einv = np.linalg.inv(_velocity_map(raw, q))
    ref = Einv.T @ lagrangian_M(raw, q) @ Einv  # M in the coordinates q, mapped to the joint velocities
    assert rel_err(oracle_M(raw, q), ref) < 2e-5


MODELS = ["cartpole", "tree", "half_cheetah", "atlas", "atlas_sdf", "free_child", "chain64", "free16", "limit"]


@pytest.mark.parametrize("name", MODELS)
@pytest.mark.parametrize("fp64", [False, True])
def test_emulated_forward_matches_oracle(name, fp64):
    raw = model_raw(name)
    ew = EmulMmWorld(nb.compile_model(raw, lanes=1))
    B = 2
    q = positions(raw, B, seed=21)
    M = ew.mass_matrix(q, fp64=fp64)
    Mi = ew.mass_matrix(q, inverse=True, fp64=fp64)
    assert np.array_equal(M, M.transpose(0, 2, 1)) and np.array_equal(Mi, Mi.transpose(0, 2, 1))
    tol = 1e-9 if fp64 else 1e-4
    for w in range(B):
        Mo = oracle_M(raw, q[w].astype(np.float64))
        assert rel_err(M[w], Mo) < tol, (w, rel_err(M[w], Mo))
        assert rel_err(Mi[w], np.linalg.inv(Mo)) < tol, (w, rel_err(Mi[w], np.linalg.inv(Mo)), np.linalg.cond(Mo))


def _blocks(raw):
    """[n, n] True on the dof pairs of one skeleton."""
    world_sk = np.zeros(raw.ndof, int)
    for i in range(raw.nb):
        r = i
        while raw.parent[r] >= 0:
            r = raw.parent[r]
        nd = 6 if raw.jtype[i] == nb.world.FREE else (0 if raw.jtype[i] == nb.world.WELD else 1)
        world_sk[raw.dof_off[i]:raw.dof_off[i] + nd] = r
    return world_sk[:, None] == world_sk[None, :]


@pytest.mark.parametrize("name", ["free_child", "free16"])
def test_emulated_off_block_entries_are_exact_zeros(name):
    raw = model_raw(name)
    ew = EmulMmWorld(nb.compile_model(raw, lanes=1))
    q = positions(raw, 3, seed=4)
    blk = _blocks(raw)
    assert not blk.all()
    for inverse in (False, True):
        out = ew.mass_matrix(q, inverse=inverse, fp64=True)
        assert np.all(out[:, ~blk] == 0)


@pytest.mark.parametrize("name", ["cartpole", "tree", "half_cheetah", "atlas", "atlas_sdf", "free_child"])
@pytest.mark.parametrize("inverse", [False, True])
def test_emulated_position_vjp_matches_oracle_differences(name, inverse):
    raw = model_raw(name)
    ew = EmulMmWorld(nb.compile_model(raw, lanes=1))
    n, B = raw.ndof, 2
    q = positions(raw, B, seed=31).astype(np.float64)
    G = np.random.default_rng(32).normal(size=(B, n, n))
    minv = ew.mass_matrix(q, inverse=True, fp64=True) if inverse else None
    gp, _ = ew.mass_matrix_backward(q, G, minv=minv, fp64=True)
    gp32, _ = ew.mass_matrix_backward(q.astype(np.float32), G.astype(np.float32), minv=None if minv is None else minv.astype(np.float32))
    f = (lambda x: np.linalg.inv(oracle_M(raw, x))) if inverse else (lambda x: oracle_M(raw, x))
    h = 1e-5  # the oracle's M comes from differences of inverse-dynamics forces: a smaller step only adds their rounding
    for w in range(B):
        fd = np.array([(np.sum(G[w] * f(q[w] + h * e)) - np.sum(G[w] * f(q[w] - h * e))) / (2 * h) for e in np.eye(n)])
        assert rel_err(gp[w], fd) < 1e-6, (w, rel_err(gp[w], fd))
        assert rel_err(gp32[w], gp[w]) < 1e-4, (w, rel_err(gp32[w], gp[w]))
        roots = [raw.dof_off[i] for i in range(raw.nb) if raw.parent[i] < 0 and raw.jtype[i] == nb.world.FREE]
        for o in roots:
            assert np.all(gp[w, o:o + 6] == 0)


@pytest.mark.parametrize("name", ["half_cheetah", "atlas"])
@pytest.mark.parametrize("inverse", [False, True])
def test_emulated_per_world_mass_vjp_matches_oracle_differences(name, inverse):
    raw = load_raw(name)
    world = register(nb.World.from_raw(raw), step=4)
    B = 2
    mv = random_masses(world, B, seed=9)
    wi = nb.mass_to_inertia(world, torch.tensor(mv, dtype=torch.float64)).numpy()
    cm = nb.compile_model(raw, lanes=1)
    ew = EmulMmWorld(cm)
    q = positions(raw, B, seed=5).astype(np.float64)
    G = np.random.default_rng(6).normal(size=(B, raw.ndof, raw.ndof))
    minv = ew.mass_matrix(q, inverse=True, fp64=True, world_inertia=wi) if inverse else None
    _, gi = ew.mass_matrix_backward(q, G, minv=minv, fp64=True, world_inertia=wi)
    entries = world._mass_entries()
    f = (lambda r, x: np.linalg.inv(oracle_M(r, x))) if inverse else oracle_M
    from nimblephysics_b200 import modelspec as ms
    for w in range(B):
        rw = raw_at(raw, entries, mv[w])
        gm = ms.inertia_param_jacobian(rw, cm, entries) @ gi[:, w]
        loss = lambda m: float(np.sum(G[w] * f(raw_at(raw, entries, m), q[w])))
        fd = np.array([(loss(mv[w] + 1e-6 * e) - loss(mv[w] - 1e-6 * e)) / 2e-6 for e in np.eye(len(mv[w]))])
        assert rel_err(gm, fd) < 1e-6, (w, rel_err(gm, fd))


def test_emulated_M_does_not_depend_on_a_free_root_pose():
    raw = load_raw("atlas")
    ew = EmulMmWorld(nb.compile_model(raw, lanes=1))
    q = positions(raw, 4, seed=7)
    q2 = q.copy()
    q2[:, :6] = np.random.default_rng(8).uniform(-2, 2, (4, 6))
    for fp64 in (False, True):
        assert np.array_equal(ew.mass_matrix(q, fp64=fp64), ew.mass_matrix(q2, fp64=fp64))


@pytest.mark.parametrize("fn", [nb.mass_matrix, nb.inverse_mass_matrix])
def test_value_errors(fn):
    raw = load_raw("half_cheetah")
    world = register(nb.World.from_raw(raw), step=2)
    n, m = raw.ndof, world.getMassDims()
    for bad in (torch.zeros(n + 1), torch.zeros(2, n - 1), torch.zeros(2, 3, n), torch.zeros(0, n)):
        with pytest.raises(ValueError):
            fn(world, bad)
    with pytest.raises(ValueError):
        fn(world, torch.zeros(2, n), torch.zeros(2, m + 1, dtype=torch.float64))
    with pytest.raises(ValueError):
        fn(world, torch.zeros(2, n), torch.zeros(3, m, dtype=torch.float64))
    with pytest.raises(ValueError):
        fn(world, torch.zeros(n), torch.zeros(2, m, dtype=torch.float64))
    with pytest.raises(ValueError):
        fn(nb.World(), torch.zeros(2, 0))
