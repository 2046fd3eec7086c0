"""Kinetic and potential energy and centroidal momentum on the host: an fp64 numpy oracle (forward kinematics and spatial inertias of
test_oracle, body velocities by Richardson-extrapolated differences along the step's position update) pinned against the closed forms of a
free box and a planar two-link arm; the host-emulated device functions (tests/host_emul/emul_energy.cpp) against that oracle and against
1/2 qdot^T M qdot on the models of test_mass_matrix; the state and per-world mass VJPs against central differences, dT/dqdot = M qdot,
exact zeros off the skeleton; and the argument checks of nimblephysics_b200.energy_and_momentum and the Skeleton methods."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from nimblephysics_b200 import modelspec as ms
from tests.host_emul.binding_energy import EmulEnergyWorld
from tests.test_mass_matrix import MODELS, model_raw, oracle_M
from tests.test_oracle import fk, potential, spatial_G
from tests.test_per_world_mass import random_masses, raw_at, register
from tests.test_world_jacobian import canon_root, com_body
from tests.test_world_jacobian_deriv import _fd, _fd_rows, advance, states
from tests.util import load_raw, rel_err


def body_twists(raw, q, qd, h=1e-3):
    """every raw body's twist [omega ; v] in its own frame: W^-1 dW/dt along q (+) t qdot, Richardson-extrapolated"""
    def D(s):
        Wp, Wm = fk(raw, advance(raw, q, qd, s)), fk(raw, advance(raw, q, qd, -s))
        return [(a - b) / (2 * s) for a, b in zip(Wp, Wm)]
    W0 = fk(raw, q)
    out = []
    for W, d1, d2 in zip(W0, D(h), D(h / 2)):
        dW = np.linalg.inv(W) @ ((4 * d2 - d1) / 3)
        out.append(np.array([dW[2, 1], dW[0, 2], dW[1, 0], dW[0, 3], dW[1, 3], dW[2, 3]]))
    return W0, out


def skeleton_of(raw, rb):
    """(raw bodies, dofs) of the skeleton of raw body rb"""
    bodies = [i for i in range(raw.nb) if raw.skel_id[i] == raw.skel_id[rb] and raw.mobile[i]]
    dofs = [raw.dof_off[i] + k for i in bodies for k in range(ms.JOINT_NDOF[int(raw.jtype[i])])]
    return bodies, dofs


def oracle_energy(raw, q, qd, rb):
    """fp64 (T, U, h [6]) of the skeleton of raw body rb"""
    bodies, dofs = skeleton_of(raw, rb)
    W, Vb = body_twists(raw, q, qd)
    T, A, P, x, mt = 0.0, np.zeros(3), np.zeros(3), np.zeros(3), 0.0
    for i in bodies:
        G = spatial_G(raw, i)
        pb = G @ Vb[i]
        T += 0.5 * Vb[i] @ pb
        R, p = W[i][:3, :3], W[i][:3, 3]
        l = R @ pb[3:]
        A += R @ pb[:3] + np.cross(p, l)
        P += l
        x += raw.mass[i] * (R @ raw.com[i] + p)
        mt += raw.mass[i]
    sub = raw.__class__.__new__(raw.__class__)
    sub.__dict__.update(raw.__dict__)
    sub.mobile = np.array([1 if i in bodies else 0 for i in range(raw.nb)])
    U = potential(sub, q) + sum(0.5 * raw.spring[d] * (q[d] - raw.rest[d]) ** 2 for d in dofs)
    return T, U, np.concatenate([A - np.cross(x / mt, P), P])


def _arm(free=False):
    w = nb.World()
    w.setGravity([0.0, -9.81, 0.3])
    sk = nb.Skeleton("arm")
    if free:
        j, b = sk.createFreeJointAndBodyNodePair(None)
        b.setMass(2.0)
        b.setLocalCOM([0.1, -0.05, 0.2])
        b.setMomentOfInertia(0.3, 0.5, 0.7, 0.01, -0.02, 0.03)
        w.addSkeleton(sk)
        return w, [b]
    j1, b1 = sk.createRevoluteJointAndBodyNodePair(None)
    j1.setAxis([0, 0, 1])
    j2, b2 = sk.createRevoluteJointAndBodyNodePair(b1)
    j2.setAxis([0, 0, 1])
    T = nb.Isometry3()
    T.set_translation([0.7, 0, 0])
    j2.setTransformFromParentBodyNode(T)
    for b, m, c, izz in ((b1, 1.0, 0.35, 0.05), (b2, 2.0, 0.2, 0.08)):
        b.setMass(m)
        b.setLocalCOM([c, 0, 0])
        b.setMomentOfInertia(0.01, 0.02, izz)
    w.addSkeleton(sk)
    return w, [b1, b2]


def test_oracle_matches_the_free_box_closed_form():
    w, (b,) = _arm(free=True)
    raw = nb.flatten_world(w)
    rng = np.random.default_rng(1)
    from scipy.spatial.transform import Rotation
    for _ in range(2):
        q, qd = rng.uniform(-1, 1, 6), rng.uniform(-2, 2, 6)
        R = Rotation.from_rotvec(q[:3]).as_matrix()
        c = np.asarray(b.com)
        Ic = np.asarray(b.moment)  # about the COM
        wb, vb = qd[:3], qd[3:]
        vc = R @ (vb + np.cross(wb, c))
        T, U, h = oracle_energy(raw, q, qd, 0)
        assert abs(T - (0.5 * 2.0 * vc @ vc + 0.5 * wb @ Ic @ wb)) < 1e-9
        assert abs(U - (-2.0 * raw.gravity @ (R @ c + q[3:]))) < 1e-12
        assert np.allclose(h, np.concatenate([R @ Ic @ R.T @ (R @ wb), 2.0 * vc]), atol=1e-9)


def test_oracle_matches_the_planar_two_link_closed_form():
    w, _ = _arm()
    raw = nb.flatten_world(w)
    l1, (m1, c1, i1), (m2, c2, i2) = 0.7, (1.0, 0.35, 0.05), (2.0, 0.2, 0.08)
    g = raw.gravity
    for th, thd in (([0.3, -1.1], [0.8, 1.7]), ([2.0, 0.4], [-1.3, 0.6])):
        t1, t12, w1, w12 = th[0], th[0] + th[1], thd[0], thd[0] + thd[1]
        e = lambda t: np.array([np.cos(t), np.sin(t), 0.0])
        de = lambda t: np.array([-np.sin(t), np.cos(t), 0.0])
        p1, p2 = c1 * e(t1), l1 * e(t1) + c2 * e(t12)
        v1, v2 = c1 * w1 * de(t1), l1 * w1 * de(t1) + c2 * w12 * de(t12)
        T = 0.5 * m1 * v1 @ v1 + 0.5 * m2 * v2 @ v2 + 0.5 * i1 * w1 ** 2 + 0.5 * i2 * w12 ** 2
        U = -g @ (m1 * p1 + m2 * p2)
        c = (m1 * p1 + m2 * p2) / (m1 + m2)
        L = m1 * np.cross(p1 - c, v1) + m2 * np.cross(p2 - c, v2) + np.array([0, 0, i1 * w1 + i2 * w12])
        To, Uo, ho = oracle_energy(raw, np.array(th), np.array(thd), 0)
        assert abs(To - T) < 1e-9 and abs(Uo - U) < 1e-12
        assert np.allclose(ho, np.concatenate([L, m1 * v1 + m2 * v2]), atol=1e-9)


def _setup(name):
    raw = model_raw(name)
    cm = nb.compile_model(raw, lanes=1)
    rb = com_body(raw, cm)
    return raw, cm, rb


@pytest.mark.parametrize("name", MODELS)
@pytest.mark.parametrize("fp64", [False, True])
def test_emulated_forward_matches_oracle(name, fp64):
    raw, cm, rb = _setup(name)
    if rb is None:
        pytest.skip("no skeleton with a moving root")
    ew = EmulEnergyWorld(cm)
    B, n = 2, raw.ndof
    s = states(raw, B, seed=61)
    T, U, h = ew.energy_momentum(s, canon_root(cm, rb), fp64=fp64)
    tol = 1e-9 if fp64 else 1e-4
    _, dofs = skeleton_of(raw, rb)
    for w in range(B):
        sw = s[w] if fp64 else s[w].astype(np.float32).astype(np.float64)
        q, qd = sw[:n], sw[n:]
        To, Uo, ho = oracle_energy(raw, q, qd, rb)
        scale = max(abs(To), abs(Uo), 1.0)
        assert abs(T[w] - To) < tol * scale and abs(U[w] - Uo) < tol * scale, (T[w], To, U[w], Uo)
        assert rel_err(h[w], ho) < tol, rel_err(h[w], ho)
        Mo = oracle_M(raw, q)
        v = np.zeros(n)
        v[dofs] = qd[dofs]
        assert abs(T[w] - 0.5 * v @ Mo @ v) < tol * scale


@pytest.mark.parametrize("name", ["tree", "half_cheetah", "atlas", "atlas_sdf", "free_child", "limit"])
def test_emulated_state_vjp_matches_differences(name):
    raw, cm, rb = _setup(name)
    root = canon_root(cm, rb)
    ew = EmulEnergyWorld(cm)
    B, n = 2, raw.ndof
    s = states(raw, B, seed=62)
    rng = np.random.default_rng(63)
    gT, gU, gh = rng.normal(size=B), rng.normal(size=B), rng.normal(size=(B, 6))
    gs, _ = ew.energy_momentum_backward(s, root, gT, gU, gh, fp64=True)
    gs32, _ = ew.energy_momentum_backward(s, root, gT, gU, gh, fp64=False)

    def loss(x):
        T, U, h = ew.energy_momentum(x, root, fp64=True)
        return gT * T + gU * U + np.einsum("bk,bk->b", gh, h)
    fd = _fd_rows(loss, s, 1e-6)
    for w in range(B):
        assert rel_err(gs[w], fd[w]) < 1e-7, (w, rel_err(gs[w], fd[w]))
        assert rel_err(gs32[w], gs[w]) < 1e-4
    # dT/dqdot = M qdot on the skeleton's dofs, exact zeros elsewhere
    _, dofs = skeleton_of(raw, rb)
    off = np.setdiff1d(np.arange(n), dofs)
    gk, _ = ew.energy_momentum_backward(s, root, np.ones(B), np.zeros(B), np.zeros((B, 6)), fp64=True)
    for w in range(B):
        v = np.zeros(n)
        v[dofs] = s[w, n:][dofs]
        assert rel_err(gk[w, n:], oracle_M(raw, s[w, :n]) @ v) < 1e-9
        assert np.all(gs[w, off] == 0) and np.all(gs[w, n + off] == 0) and np.all(gs32[w, off] == 0)


@pytest.mark.parametrize("name", ["half_cheetah", "atlas"])
def test_emulated_per_world_mass_matches_oracle_and_differences(name):
    raw = load_raw(name)
    world = register(nb.World.from_raw(raw), step=4)
    B, n = 2, raw.ndof
    mv = random_masses(world, B, seed=64)
    cm = nb.compile_model(raw, lanes=1)
    ew = EmulEnergyWorld(cm)
    rb = com_body(raw, cm)
    root = canon_root(cm, rb)
    s = states(raw, B, seed=65)
    rng = np.random.default_rng(66)
    gT, gU, gh = rng.normal(size=B), rng.normal(size=B), rng.normal(size=(B, 6))
    wi_of = lambda m: nb.mass_to_inertia(world, torch.tensor(m, dtype=torch.float64)).numpy()
    T, U, h = ew.energy_momentum(s, root, fp64=True, world_inertia=wi_of(mv))
    _, gi = ew.energy_momentum_backward(s, root, gT, gU, gh, fp64=True, world_inertia=wi_of(mv))
    entries = world._mass_entries()
    for w in range(B):
        rw = raw_at(raw, entries, mv[w])
        To, Uo, ho = oracle_energy(rw, s[w, :n], s[w, n:], rb)
        assert abs(T[w] - To) < 1e-9 * max(1, abs(To)) and abs(U[w] - Uo) < 1e-9 * max(1, abs(Uo)) and rel_err(h[w], ho) < 1e-9
        gm = ms.inertia_param_jacobian(rw, cm, entries) @ gi[:, w]

        def loss(m):
            t, u, hh = ew.energy_momentum(s[w:w + 1], root, fp64=True, world_inertia=wi_of(m[None]))
            return float(gT[w] * t[0] + gU[w] * u[0] + gh[w] @ hh[0])
        fd = _fd(loss, mv[w], 1e-6)
        assert rel_err(gm, fd) < 1e-7, (w, rel_err(gm, fd))


def test_value_errors():
    raw = load_raw("half_cheetah")
    world = register(nb.World.from_raw(raw), step=2)
    other = nb.World.from_raw(raw)
    n, m = raw.ndof, world.getMassDims()
    sk = max(world.skeletons, key=lambda s: s.getNumDofs())
    for bad in (torch.zeros(n), torch.zeros(2 * n + 1), torch.zeros(2, n), torch.zeros(2, 3, 2 * n), torch.zeros(0, 2 * n)):
        with pytest.raises(ValueError):
            nb.energy_and_momentum(world, bad, sk)
    s = torch.zeros(2, 2 * n)
    with pytest.raises(ValueError):
        nb.energy_and_momentum(world, s, max(other.skeletons, key=lambda s: s.getNumDofs()))
    static = [x for x in world.skeletons if x.getNumDofs() == 0]
    assert static
    with pytest.raises(ValueError):
        nb.energy_and_momentum(world, s, static[0])
    for bad_m in (torch.zeros(m + 1, dtype=torch.float64), torch.zeros(2, m + 1, dtype=torch.float64), torch.zeros(3, m, dtype=torch.float64)):
        with pytest.raises(ValueError):
            nb.energy_and_momentum(world, s, sk, bad_m)
    with pytest.raises(ValueError):
        nb.energy_and_momentum(world, torch.zeros(2 * n), sk, torch.zeros(2, m, dtype=torch.float64))
    with pytest.raises(ValueError):
        nb.energy_and_momentum(nb.World(), torch.zeros(2, 0), sk)
    # the Skeleton methods: a skeleton outside any World, and one whose root is welded to it
    for meth in ("computeKineticEnergy", "computePotentialEnergy", "computeLagrangian"):
        with pytest.raises(ValueError):
            getattr(nb.Skeleton("loose"), meth)()
        with pytest.raises(ValueError):
            getattr(static[0], meth)()
