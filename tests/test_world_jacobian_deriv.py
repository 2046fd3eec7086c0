"""Time derivatives of the world and COM Jacobians on the host: an fp64 oracle (Richardson-extrapolated central differences of the
Jacobian oracle of test_world_jacobian along the step's position update q (+) t qdot) pinned against the closed form of a planar two-link
arm; the host-emulated device functions (tests/host_emul/emul_jacd.cpp) against that oracle for Jdot, the state, offset and per-world
mass VJPs against central differences of the emulated forward, on the models of test_mass_matrix; exact zeros, linearity in qdot, the
identity between the qdot gradient of <G, Jdot> and the position gradient of <G, J>; and the argument checks of
nimblephysics_b200.world_jacobian_deriv / com_jacobian_deriv."""
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import nimblephysics_b200 as nb
from nimblephysics_b200 import modelspec as ms
from nimblephysics_b200.world_jacobian import MAX_NODES
from tests.host_emul.binding_jacd import EmulJacdWorld
from tests.test_inverse_dynamics import id_inputs
from tests.test_mass_matrix import MODELS, model_raw
from tests.test_per_world_mass import random_masses, raw_at, register
from tests.test_world_jacobian import _on_chain, canon_nodes, canon_root, com_body, mobile_nodes, oracle_com, oracle_point
from tests.util import load_raw, rel_err


def advance(raw, q, qd, t):
    """q (+) t qdot: the step's position update (FreeJoint.cpp:922-929 for every free joint: R exp(t omega), p + t R v), q + t qdot elsewhere."""
    out = q + t * qd
    for i in range(raw.nb):
        if raw.jtype[i] != nb.world.FREE:
            continue
        o = raw.dof_off[i]
        R = Rotation.from_rotvec(q[o:o + 3]).as_matrix()
        out[o:o + 3] = Rotation.from_matrix(R @ Rotation.from_rotvec(t * qd[o:o + 3]).as_matrix()).as_rotvec()
        out[o + 3:o + 6] = q[o + 3:o + 6] + R @ (t * qd[o + 3:o + 6])
    return out


def oracle_deriv(raw, f, q, qd, h=1e-3):
    """d/dt f(q (+) t qdot) at t = 0: central differences at h and h / 2, Richardson-extrapolated (error O(h^4))."""
    D = lambda s: (f(advance(raw, q, qd, s)) - f(advance(raw, q, qd, -s))) / (2 * s)
    return (4 * D(h / 2) - D(h)) / 3


def oracle_point_deriv(raw, q, qd, ri, offset=None):
    return oracle_deriv(raw, lambda x: oracle_point(raw, x, ri, offset), q, qd)


def oracle_com_deriv(raw, q, qd, ri):
    return oracle_deriv(raw, lambda x: oracle_com(raw, x, ri), q, qd)


def states(raw, B, seed):
    s, _ = id_inputs(raw, B, seed=seed)
    return s.astype(np.float64)


def test_oracle_matches_the_planar_two_link_closed_form():
    l1, l2 = 0.7, 0.45
    w = nb.World()
    sk = nb.Skeleton("arm")
    j1, b1 = sk.createRevoluteJointAndBodyNodePair(None)
    j1.setAxis([0, 0, 1])
    j2, b2 = sk.createRevoluteJointAndBodyNodePair(b1)
    j2.setAxis([0, 0, 1])
    T = nb.Isometry3()
    T.set_translation([l1, 0, 0])
    j2.setTransformFromParentBodyNode(T)
    b1.setMass(1.0)
    b2.setMass(2.0)
    w.addSkeleton(sk)
    raw = nb.flatten_world(w)
    for th, thd in (([0.3, -1.1], [0.8, 1.7]), ([2.0, 0.4], [-1.3, 0.6])):
        t1, t12, w1, w12 = th[0], th[0] + th[1], thd[0], thd[0] + thd[1]
        ref = np.zeros((6, 2))
        ref[3] = [-l1 * np.cos(t1) * w1 - l2 * np.cos(t12) * w12, -l2 * np.cos(t12) * w12]
        ref[4] = [-l1 * np.sin(t1) * w1 - l2 * np.sin(t12) * w12, -l2 * np.sin(t12) * w12]
        got = oracle_point_deriv(raw, np.array(th), np.array(thd), 1, [l2, 0, 0])
        assert np.max(np.abs(got - ref)) < 1e-8 * max(1.0, np.max(np.abs(ref))), got - ref


@pytest.mark.parametrize("name", MODELS)
@pytest.mark.parametrize("fp64", [False, True])
def test_emulated_forward_matches_oracle(name, fp64):
    raw = model_raw(name)
    cm = nb.compile_model(raw, lanes=1)
    ew = EmulJacdWorld(cm)
    B, n = 2, raw.ndof
    s = states(raw, B, seed=41)
    ris = mobile_nodes(raw, cm)
    bodies, T = canon_nodes(cm, ris)
    off = np.random.default_rng(42).uniform(-0.1, 0.1, (B, len(ris), 3))
    dJ = ew.world_jacobian_deriv(s, bodies, T, off, fp64=fp64)
    rc = com_body(raw, cm)
    dJc = ew.com_jacobian_deriv(s, canon_root(cm, rc), fp64=fp64) if rc is not None else None
    tol = 1e-8 if fp64 else 1e-4
    for w in range(B):
        sw = s[w] if fp64 else s[w].astype(np.float32).astype(np.float64)
        q, qd = sw[:n], sw[n:]
        for e, ri in enumerate(ris):
            ow = off[w, e] if fp64 else off[w, e].astype(np.float32).astype(np.float64)
            assert rel_err(dJ[w, e], oracle_point_deriv(raw, q, qd, ri, ow)) < tol, (w, ri)
        if rc is not None:
            assert rel_err(dJc[w], oracle_com_deriv(raw, q, qd, rc)) < tol
    assert dJ.shape == (B, len(ris), 6, n)


@pytest.mark.parametrize("name", ["free_child", "atlas", "limit"])
def test_emulated_exact_zeros_and_linearity_in_qdot(name):
    raw = model_raw(name)
    cm = nb.compile_model(raw, lanes=1)
    ew = EmulJacdWorld(cm)
    n = raw.ndof
    s = states(raw, 3, seed=43)
    ris = mobile_nodes(raw, cm)
    bodies, T = canon_nodes(cm, ris)
    bodies = np.concatenate([bodies, [-1]])
    T = np.concatenate([T, np.eye(4)[None]])
    root = canon_root(cm, com_body(raw, cm))
    s0 = s.copy()
    s0[:, n:] = 0
    for fp64 in (False, True):
        dJ = ew.world_jacobian_deriv(s, bodies, T, fp64=fp64)
        for e, b in enumerate(bodies[:-1]):
            assert np.all(dJ[:, e][:, :, ~_on_chain(cm, b)] == 0)
        assert np.all(dJ[:, -1] == 0)
        assert np.all(ew.world_jacobian_deriv(s0, bodies, T, fp64=fp64) == 0)
        assert np.all(ew.com_jacobian_deriv(s0, root, fp64=fp64) == 0)
    # linear in qdot
    rng = np.random.default_rng(44)
    v1, v2 = rng.normal(size=(3, n)), rng.normal(size=(3, n))
    at = lambda v: np.concatenate([s[:, :n], v], 1)
    a, b = 0.7, -1.9
    dJ1, dJ2, dJ12 = (ew.world_jacobian_deriv(at(v), bodies, T, fp64=True) for v in (v1, v2, a * v1 + b * v2))
    assert rel_err(dJ12, a * dJ1 + b * dJ2) < 1e-12
    dC1, dC2, dC12 = (ew.com_jacobian_deriv(at(v), root, fp64=True) for v in (v1, v2, a * v1 + b * v2))
    assert rel_err(dC12, a * dC1 + b * dC2) < 1e-12


def _fd(f, x, h):
    return np.array([(f(x + h * e) - f(x - h * e)) / (2 * h) for e in np.eye(len(x))])


def _fd_rows(f, X, h):
    """central differences of the per-row losses f(X) [B] with respect to each row's own entries X [B, m] -> [B, m]"""
    out = np.empty(X.shape)
    for i in range(X.shape[1]):
        E = np.zeros(X.shape)
        E[:, i] = h
        out[:, i] = (f(X + E) - f(X - E)) / (2 * h)
    return out


@pytest.mark.parametrize("name", ["cartpole", "tree", "half_cheetah", "atlas", "atlas_sdf", "free_child"])
def test_emulated_state_and_offset_vjp_match_differences(name):
    raw = model_raw(name)
    cm = nb.compile_model(raw, lanes=1)
    ew = EmulJacdWorld(cm)
    B = 2
    s = states(raw, B, seed=45)
    ris = mobile_nodes(raw, cm)
    bodies, T = canon_nodes(cm, ris)
    rng = np.random.default_rng(46)
    off = rng.uniform(-0.1, 0.1, (B, len(ris), 3))
    G = rng.normal(size=(B, len(ris), 6, raw.ndof))
    gs, go = ew.world_jacobian_deriv_backward(s, bodies, T, G, off, fp64=True)
    gs32, go32 = ew.world_jacobian_deriv_backward(s, bodies, T, G, off, fp64=False)
    # the worlds are independent: perturbing one entry in every world at once gives each world's difference
    loss = lambda x: np.einsum("bkrn,bkrn->b", G, ew.world_jacobian_deriv(x, bodies, T, off, fp64=True))
    fd = _fd_rows(loss, s, 1e-6)
    lo = lambda o: np.einsum("bkrn,bkrn->b", G, ew.world_jacobian_deriv(s, bodies, T, o.reshape(off.shape), fp64=True))
    fdo = _fd_rows(lo, off.reshape(B, -1), 1e-6).reshape(off.shape)
    for w in range(B):
        assert rel_err(gs[w], fd[w]) < 1e-7, (w, rel_err(gs[w], fd[w]))
        assert rel_err(go[w], fdo[w]) < 1e-7 and rel_err(go32[w], go[w]) < 1e-4
        assert rel_err(gs32[w], gs[w]) < 1e-4
    rc = com_body(raw, cm)
    if rc is None:
        return
    root = canon_root(cm, rc)
    Gc = rng.normal(size=(B, 3, raw.ndof))
    gc, _ = ew.com_jacobian_deriv_backward(s, root, Gc, fp64=True)
    gc32, _ = ew.com_jacobian_deriv_backward(s, root, Gc, fp64=False)
    lc = lambda x: np.einsum("brn,brn->b", Gc, ew.com_jacobian_deriv(x, root, fp64=True))
    fdc = _fd_rows(lc, s, 1e-6)
    for w in range(B):
        assert rel_err(gc[w], fdc[w]) < 1e-7, (w, rel_err(gc[w], fdc[w]))
        assert rel_err(gc32[w], gc[w]) < 1e-4


@pytest.mark.parametrize("name", ["half_cheetah", "atlas"])
def test_emulated_per_world_mass_vjp_matches_differences(name):
    raw = load_raw(name)
    world = register(nb.World.from_raw(raw), step=4)
    B = 2
    mv = random_masses(world, B, seed=47)
    cm = nb.compile_model(raw, lanes=1)
    ew = EmulJacdWorld(cm)
    s = states(raw, B, seed=48)
    rc = com_body(raw, cm)
    root = canon_root(cm, rc)
    G = np.random.default_rng(49).normal(size=(B, 3, raw.ndof))
    wi_of = lambda m: nb.mass_to_inertia(world, torch.tensor(m, dtype=torch.float64)).numpy()
    dJ = ew.com_jacobian_deriv(s, root, fp64=True, world_inertia=wi_of(mv))
    _, gi = ew.com_jacobian_deriv_backward(s, root, G, fp64=True, world_inertia=wi_of(mv))
    entries = world._mass_entries()
    n = raw.ndof
    for w in range(B):
        rw = raw_at(raw, entries, mv[w])
        assert rel_err(dJ[w], oracle_com_deriv(rw, s[w, :n], s[w, n:], rc)) < 1e-8
        gm = ms.inertia_param_jacobian(rw, cm, entries) @ gi[:, w]
        loss = lambda m: float(np.sum(G[w] * ew.com_jacobian_deriv(s[w:w + 1], root, fp64=True, world_inertia=wi_of(m[None]))[0]))
        fd = _fd(loss, mv[w], 1e-6)
        assert rel_err(gm, fd) < 1e-7, (w, rel_err(gm, fd))


@pytest.mark.parametrize("name", [m for m in MODELS if all(j != nb.world.FREE for j in model_raw(m).jtype)])
def test_qdot_gradient_equals_the_jacobian_position_gradient(name):
    """J is a function of q alone and Jdot = sum_j dJ/dq_j qdot_j, so d<G, Jdot>/dqdot = d<G, J>/dq (no free joint: coordinates = tangent)."""
    raw = model_raw(name)
    cm = nb.compile_model(raw, lanes=1)
    ew = EmulJacdWorld(cm)
    B, n = 2, raw.ndof
    s = states(raw, B, seed=50)
    ris = mobile_nodes(raw, cm)
    bodies, T = canon_nodes(cm, ris)
    rng = np.random.default_rng(51)
    off = rng.uniform(-0.1, 0.1, (B, len(ris), 3))
    G = rng.normal(size=(B, len(ris), 6, n))
    gs, _ = ew.world_jacobian_deriv_backward(s, bodies, T, G, off, fp64=True)
    gp, _ = ew.world_jacobian_backward(s[:, :n], bodies, T, G, off, fp64=True)
    assert rel_err(gs[:, n:], gp) < 1e-10
    rc = com_body(raw, cm)
    if rc is not None:
        Gc = rng.normal(size=(B, 3, n))
        gc, _ = ew.com_jacobian_deriv_backward(s, canon_root(cm, rc), Gc, fp64=True)
        gpc, _ = ew.com_jacobian_backward(s[:, :n], canon_root(cm, rc), Gc, fp64=True)
        assert rel_err(gc[:, n:], gpc) < 1e-10


def test_value_errors():
    raw = load_raw("half_cheetah")
    world = register(nb.World.from_raw(raw), step=2)
    other = nb.World.from_raw(raw)
    n, m = raw.ndof, world.getMassDims()
    sk = max(world.skeletons, key=lambda s: s.getNumDofs())
    node = sk._ordered_bodies()[-1]
    for bad in (torch.zeros(n), torch.zeros(2 * n + 1), torch.zeros(2, n), torch.zeros(2, 3, 2 * n), torch.zeros(0, 2 * n)):
        with pytest.raises(ValueError):
            nb.world_jacobian_deriv(world, bad, [node])
        with pytest.raises(ValueError):
            nb.com_jacobian_deriv(world, bad, sk)
    s = torch.zeros(2, 2 * n)
    for bad_off in (torch.zeros(2), torch.zeros(1, 4), torch.zeros(3, 1, 3), torch.zeros(2, 2, 3)):
        with pytest.raises(ValueError):
            nb.world_jacobian_deriv(world, s, [node], bad_off)
    with pytest.raises(ValueError):
        nb.world_jacobian_deriv(world, torch.zeros(2 * n), [node], torch.zeros(2, 1, 3))
    with pytest.raises(ValueError):
        nb.world_jacobian_deriv(world, s, [])
    with pytest.raises(ValueError):
        nb.world_jacobian_deriv(world, s, [node] * (MAX_NODES + 1))
    with pytest.raises(ValueError):
        nb.world_jacobian_deriv(world, s, [other.skeletons[-1]._ordered_bodies()[-1]])
    with pytest.raises(ValueError):
        nb.com_jacobian_deriv(world, s, max(other.skeletons, key=lambda s: s.getNumDofs()))
    static = [x for x in world.skeletons if x.getNumDofs() == 0]
    assert static
    with pytest.raises(ValueError):
        nb.com_jacobian_deriv(world, s, static[0])
    for bad_m in (torch.zeros(m + 1, dtype=torch.float64), torch.zeros(2, m + 1, dtype=torch.float64), torch.zeros(3, m, dtype=torch.float64)):
        with pytest.raises(ValueError):
            nb.com_jacobian_deriv(world, s, sk, bad_m)
    with pytest.raises(ValueError):
        nb.com_jacobian_deriv(world, torch.zeros(2 * n), sk, torch.zeros(2, m, dtype=torch.float64))
    with pytest.raises(ValueError):
        nb.world_jacobian_deriv(nb.World(), torch.zeros(2, 0), [node])
    with pytest.raises(ValueError):
        nb.com_jacobian_deriv(nb.World(), torch.zeros(2, 0), sk)
