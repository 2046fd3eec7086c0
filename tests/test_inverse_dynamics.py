"""Contact-free inverse dynamics on the CPU: the fp64 oracle (tests/oracle_id, orc_inverse_dynamics) against an independent Lagrangian computation,
its round trip through the oracle's step, its dual-number Jacobians against finite differences, and the device functions
(csrc/nb2_dyn.cuh, host build, reversed lane order for odd worlds) against the oracle, mass gradient included."""
import copy

import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from nimblephysics_b200 import modelspec as ms
from nimblephysics_b200.world import FREE
from tests.host_emul.binding_id import EmulIdWorld
from tests.oracle_id.binding import IdOracle
from tests.test_oracle import _rodrigues, _tree_world, mass_matrix, potential
from tests.test_per_world_mass import random_masses, raw_at, register
from tests.util import load_raw, rel_err, sample_inputs


def _raw(name):
    return nb.flatten_world(_tree_world()) if name == "tree" else load_raw(name)


def id_inputs(raw, B, seed):
    """fp32 states and next velocities one step apart (accelerations of a few units)."""
    s, _, _ = sample_inputs(raw, B, seed=seed)
    rng = np.random.default_rng(seed + 100)
    vn = (s[:, raw.ndof:] + raw.dt * rng.uniform(-5, 5, (B, raw.ndof))).astype(np.float32)
    return s, vn


def _velocity_map(raw, q):
    """E(q): joint velocities = E(q) dq/dt.  Identity but for free joints, whose velocity is the body twist of [exp(phi), p]:
    omega = Jr(phi) dphi/dt, v = R(phi)^T dp/dt."""
    E = np.eye(raw.ndof)
    for i in range(raw.nb):
        if raw.jtype[i] != FREE:
            continue
        o = raw.dof_off[i]
        phi = q[o:o + 3]
        th = np.linalg.norm(phi)
        K = np.array([[0, -phi[2], phi[1]], [phi[2], 0, -phi[0]], [-phi[1], phi[0], 0]])
        E[o:o + 3, o:o + 3] = np.eye(3) - (1 - np.cos(th)) / th**2 * K + (th - np.sin(th)) / th**3 * K @ K
        E[o + 3:o + 6, o + 3:o + 6] = _rodrigues(phi).T
    return E


def lagrangian_id(raw, q, v, vn, h=1e-4):
    """M_q qdd + C_q + dV/dq in the coordinates q (mass matrix from numeric body Jacobians, Christoffel terms, potential gradient),
    mapped to the joint velocities' dual by E^-T, plus the step's spring and damping."""
    n = raw.ndof
    Einv = np.linalg.inv(_velocity_map(raw, q))
    qd = Einv @ v
    dEinv = (np.linalg.inv(_velocity_map(raw, q + 1e-5 * qd)) - np.linalg.inv(_velocity_map(raw, q - 1e-5 * qd))) / 2e-5
    qdd = Einv @ ((vn - v) / raw.dt) + dEinv @ v
    M = mass_matrix(raw, q)
    dM = np.zeros((n, n, n))
    gq = np.zeros(n)
    for k in range(n):
        qp, qm = q.copy(), q.copy()
        qp[k] += h
        qm[k] -= h
        dM[k] = (mass_matrix(raw, qp) - mass_matrix(raw, qm)) / (2 * h)
        gq[k] = (potential(raw, qp) - potential(raw, qm)) / (2 * h)
    C = np.einsum("ikj,i,j->k", dM, qd, qd) - 0.5 * np.einsum("i,kij,j->k", qd, dM, qd)
    return Einv.T @ (M @ qdd + C + gq) + raw.damping * v + raw.spring * (q - raw.rest + v * raw.dt)


@pytest.mark.parametrize("name", ["cartpole", "tree", "half_cheetah", "atlas"])
def test_oracle_id_matches_lagrangian_mechanics(name):
    raw = _raw(name)
    ow = IdOracle(raw)
    s, vn = id_inputs(raw, 1, seed=3)
    s, vn = s[0].astype(np.float64), vn[0].astype(np.float64)
    n = raw.ndof
    tau = ow.inverse_dynamics(s, vn)
    ref = lagrangian_id(raw, s[:n], s[n:], vn)
    assert rel_err(tau, ref) < 2e-5, (tau, ref)


@pytest.mark.parametrize("name", ["cartpole", "tree", "half_cheetah", "atlas"])
def test_oracle_round_trip_through_the_step(oracle_mod, name):
    raw = copy.deepcopy(_raw(name))
    raw.action_map = np.arange(raw.ndof)  # every dof actuated: tau is the action
    ow, io = oracle_mod.OracleWorld(raw), IdOracle(raw)
    s, vn = id_inputs(raw, 3, seed=4)
    for w in range(3):
        s64, vn64 = s[w].astype(np.float64), vn[w].astype(np.float64)
        nxt = ow.step(s64, io.inverse_dynamics(s64, vn64))
        v = s64[raw.ndof:]
        assert np.linalg.norm(nxt[raw.ndof:] - vn64) <= 1e-9 * np.linalg.norm(vn64 - v)


@pytest.mark.parametrize("name", ["cartpole", "half_cheetah", "atlas"])
def test_oracle_id_jacobians_match_finite_differences(name):
    raw = _raw(name)
    ow = IdOracle(raw)
    n = raw.ndof
    s, vn = id_inputs(raw, 1, seed=7)
    x = np.concatenate([s[0], vn[0]]).astype(np.float64)
    _, J = ow.inverse_dynamics(x[:2 * n], x[2 * n:], want_jac=True)
    eps = 1e-6
    Jfd = np.zeros_like(J)
    for c in range(3 * n):
        xp, xm = x.copy(), x.copy()
        xp[c] += eps
        xm[c] -= eps
        Jfd[:, c] = (ow.inverse_dynamics(xp[:2 * n], xp[2 * n:]) - ow.inverse_dynamics(xm[:2 * n], xm[2 * n:])) / (2 * eps)
    assert np.abs(J - Jfd).max() < 1e-7 * max(1.0, np.abs(J).max())


def _compile(raw, lanes):
    try:
        return nb.compile_model(raw, lanes=lanes)
    except ValueError:
        pytest.skip(f"no {lanes}-lane schedule for this model")


@pytest.mark.parametrize("name", ["cartpole", "tree", "half_cheetah", "atlas"])
@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("lanes", [1, 2, 4, 8])
def test_emulated_id_and_vjp_match_oracle(name, fp64, lanes):
    raw = _raw(name)
    ew = EmulIdWorld(_compile(raw, lanes))
    ow = IdOracle(raw)
    n, B = raw.ndof, 5  # two groups of the emulated warp, the second partial
    s, vn = id_inputs(raw, B, seed=11 + lanes)
    gt = np.random.default_rng(lanes).normal(size=(B, n))
    tau, saved = ew.inverse_dynamics(s, vn, fp64)
    gs, gn, _ = ew.inverse_dynamics_backward(s, saved, gt, fp64)
    tol = 1e-9 if fp64 else 1e-4
    for w in range(B):
        rt, J = ow.inverse_dynamics(s[w].astype(np.float64), vn[w].astype(np.float64), want_jac=True)
        g = J.T @ gt[w].astype(np.float32 if not fp64 else np.float64).astype(np.float64)
        assert rel_err(tau[w], rt) < tol, (w, rel_err(tau[w], rt))
        assert rel_err(gs[w], g[:2 * n]) < tol, (w, rel_err(gs[w], g[:2 * n]))
        assert rel_err(gn[w], g[2 * n:]) < tol, (w, rel_err(gn[w], g[2 * n:]))


@pytest.mark.parametrize("name", ["half_cheetah", "atlas"])
def test_emulated_per_world_mass_gradient_matches_oracle_differences(name):
    raw = load_raw(name)
    world = register(nb.World.from_raw(raw), step=4)
    B = 3
    M = random_masses(world, B, seed=9)
    wi = nb.mass_to_inertia(world, torch.tensor(M, dtype=torch.float64)).numpy()
    cm = nb.compile_model(raw, lanes=2)
    ew = EmulIdWorld(cm)
    s, vn = id_inputs(raw, B, seed=5)
    gt = np.random.default_rng(6).normal(size=(B, raw.ndof))
    tau, saved = ew.inverse_dynamics(s, vn, True, world_inertia=wi)
    _, _, gi = ew.inverse_dynamics_backward(s, saved, gt, True, world_inertia=wi)
    entries = world._mass_entries()
    for w in range(B):
        s64, vn64 = s[w].astype(np.float64), vn[w].astype(np.float64)
        rw = raw_at(raw, entries, M[w])
        assert rel_err(tau[w], IdOracle(rw).inverse_dynamics(s64, vn64)) < 1e-9
        gm = ms.inertia_param_jacobian(rw, cm, entries) @ gi[:, w]

        def loss(mv):
            return float(gt[w] @ IdOracle(raw_at(raw, entries, mv)).inverse_dynamics(s64, vn64))

        fd = np.array([(loss(M[w] + 1e-5 * e) - loss(M[w] - 1e-5 * e)) / 2e-5 for e in np.eye(len(M[w]))])
        assert rel_err(gm, fd) < 1e-7, (gm, fd)
