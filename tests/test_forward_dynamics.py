"""Contact-free forward dynamics on the CPU: the forward-dynamics device functions (csrc/nb2_dyn.cuh fd_* and the FD pass 3, host build with
the step harness's groups, scratch poisoning and reversed lane order for odd worlds) against the accelerations of the fp64 step oracle, the
round trip through the emulated inverse dynamics, the VJPs against central differences of the oracle, a reduced action space, and the
argument checks of nimblephysics_b200.forward_dynamics."""
import copy

import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from nimblephysics_b200 import modelspec as ms
from oracle.binding import OracleWorld
from tests.host_emul.binding_fd import EmulFdWorld
from tests.host_emul.binding_id import EmulIdWorld
from tests.test_inverse_dynamics import _compile, id_inputs
from tests.test_mass_matrix import MODELS, model_raw
from tests.test_per_world_mass import random_masses, raw_at, register
from tests.util import load_raw, rel_err


def per_dof(raw):
    """The same model with every dof actuated in dof order: its step oracle's action is tau per dof."""
    r = copy.deepcopy(raw)
    r.action_map = np.arange(raw.ndof)
    return r


def fd_inputs(raw, B, seed):
    """fp32 states and per-dof forces of a few tens of units."""
    s, _ = id_inputs(raw, B, seed=seed)
    tau = np.random.default_rng(seed + 200).uniform(-20, 20, (B, raw.ndof)).astype(np.float32)
    return s, tau


def oracle_qdd(ow, s, tau):
    return ow.step(np.asarray(s, np.float64), np.asarray(tau, np.float64), want_qdd=True)[1]


@pytest.mark.parametrize("name", MODELS)
@pytest.mark.parametrize("fp64", [False, True])
def test_emulated_forward_matches_oracle(name, fp64):
    raw = model_raw(name)
    ew, ow = EmulFdWorld(nb.compile_model(raw, lanes=1)), OracleWorld(per_dof(raw))
    B = 4  # two groups of the emulated warp, the second partial
    s, tau = fd_inputs(raw, B, seed=21)
    qdd, _ = ew.forward_dynamics(s, tau, fp64)
    tol = 1e-9 if fp64 else 1e-4
    for w in range(B):
        ref = oracle_qdd(ow, s[w], tau[w])
        assert rel_err(qdd[w], ref) < tol, (w, rel_err(qdd[w], ref))


@pytest.mark.parametrize("name", ["cartpole", "tree", "half_cheetah", "atlas", "atlas_sdf"])
@pytest.mark.parametrize("lanes", [2, 4, 8])
def test_emulated_lane_schedules_match_one_lane(name, lanes):
    raw = model_raw(name)
    ew1, ewk = EmulFdWorld(nb.compile_model(raw, lanes=1)), EmulFdWorld(_compile(raw, lanes))
    s, tau = fd_inputs(raw, 5, seed=3 + lanes)
    g = np.random.default_rng(lanes).normal(size=(5, raw.ndof))
    q1, sv1 = ew1.forward_dynamics(s, tau, True)
    qk, svk = ewk.forward_dynamics(s, tau, True)
    assert rel_err(qk, q1) < 1e-12
    for a, b in zip(ew1.forward_dynamics_backward(s, sv1, g, True), ewk.forward_dynamics_backward(s, svk, g, True)):
        assert rel_err(a, b) < 1e-12


def test_split_position_and_velocity_rows_read_in_place():
    """The legacy entry's separate pos / vel arrays give the state rows' result bit for bit."""
    raw = load_raw("atlas")
    ew = EmulFdWorld(nb.compile_model(raw, lanes=2))
    s, tau = fd_inputs(raw, 5, seed=8)
    for fp64 in (False, True):
        a, _ = ew.forward_dynamics(s, tau, fp64)
        b, _ = ew.forward_dynamics(s, tau, fp64, split=True)
        assert np.array_equal(a, b)


@pytest.mark.parametrize("name", ["cartpole", "tree", "half_cheetah", "atlas", "atlas_sdf", "free_child"])
def test_emulated_round_trip_through_inverse_dynamics(name):
    raw = model_raw(name)
    cm = nb.compile_model(raw, lanes=1)
    ef, ei = EmulFdWorld(cm), EmulIdWorld(cm)
    s, tau = fd_inputs(raw, 4, seed=5)
    s = s.astype(np.float64)
    qdd, _ = ef.forward_dynamics(s, tau, True)
    vn = s[:, raw.ndof:] + raw.dt * qdd
    back, _ = ei.inverse_dynamics(s, vn, True)
    for w in range(4):
        assert rel_err(back[w], tau[w]) < 1e-9, (w, rel_err(back[w], tau[w]))


@pytest.mark.parametrize("name", ["cartpole", "half_cheetah", "atlas"])
def test_emulated_qdd_is_zero_for_the_bias_force(name):
    """tau = ID(q, qdot, qdot) (the force that keeps the velocity) gives qdd = 0 up to the rounding of M^-1 applied to tau's size."""
    raw = model_raw(name)
    cm = nb.compile_model(raw, lanes=1)
    ef, ei = EmulFdWorld(cm), EmulIdWorld(cm)
    s, _ = fd_inputs(raw, 3, seed=6)
    s = s.astype(np.float64)
    tau, _ = ei.inverse_dynamics(s, s[:, raw.ndof:], True)
    qdd, _ = ef.forward_dynamics(s, tau, True)
    for w in range(3):
        ref = oracle_qdd(OracleWorld(per_dof(raw)), s[w], tau[w] + 1.0)  # the acceleration of a unit force on every dof: the scale of M^-1
        assert np.linalg.norm(qdd[w]) <= 1e-10 * np.linalg.norm(tau[w]) * np.linalg.norm(ref), (w, np.abs(qdd[w]).max())


def _fd_vjp(ow, s, tau, g, h=1e-6):
    """[dL/dstate ; dL/dtau] of L = g . qdd by central differences of the oracle."""
    x = np.concatenate([s, tau]).astype(np.float64)
    n2 = len(s)
    out = np.zeros_like(x)
    for c in range(len(x)):
        xp, xm = x.copy(), x.copy()
        xp[c] += h
        xm[c] -= h
        out[c] = (g @ oracle_qdd(ow, xp[:n2], xp[n2:]) - g @ oracle_qdd(ow, xm[:n2], xm[n2:])) / (2 * h)
    return out


@pytest.mark.parametrize("name", ["cartpole", "tree", "half_cheetah", "atlas", "atlas_sdf", "free_child"])
@pytest.mark.parametrize("fp64", [False, True])
def test_emulated_vjp_matches_oracle_differences(name, fp64):
    raw = model_raw(name)
    ew, ow = EmulFdWorld(nb.compile_model(raw, lanes=1)), OracleWorld(per_dof(raw))
    n, B = raw.ndof, 2
    s, tau = fd_inputs(raw, B, seed=31)
    g = np.random.default_rng(32).normal(size=(B, n))
    _, saved = ew.forward_dynamics(s, tau, fp64)
    gs, gt, _ = ew.forward_dynamics_backward(s, saved, g, fp64)
    tol = 1e-6 if fp64 else 1e-4
    for w in range(B):
        ref = _fd_vjp(ow, s[w], tau[w], g[w])
        assert rel_err(gs[w], ref[:2 * n]) < tol, (w, rel_err(gs[w], ref[:2 * n]))
        assert rel_err(gt[w], ref[2 * n:]) < tol, (w, rel_err(gt[w], ref[2 * n:]))


@pytest.mark.parametrize("name", ["half_cheetah", "atlas"])
def test_emulated_per_world_mass_vjp_matches_oracle_differences(name):
    raw = load_raw(name)
    world = register(nb.World.from_raw(raw), step=4)
    B = 3
    M = random_masses(world, B, seed=9)
    wi = nb.mass_to_inertia(world, torch.tensor(M, dtype=torch.float64)).numpy()
    cm = nb.compile_model(raw, lanes=2)
    ew = EmulFdWorld(cm)
    s, tau = fd_inputs(raw, B, seed=5)
    g = np.random.default_rng(6).normal(size=(B, raw.ndof))
    qdd, saved = ew.forward_dynamics(s, tau, True, world_inertia=wi)
    _, _, gi = ew.forward_dynamics_backward(s, saved, g, True, world_inertia=wi)
    entries = world._mass_entries()
    for w in range(B):
        rw = raw_at(raw, entries, M[w])
        assert rel_err(qdd[w], oracle_qdd(OracleWorld(per_dof(rw)), s[w], tau[w])) < 1e-9
        gm = ms.inertia_param_jacobian(rw, cm, entries) @ gi[:, w]

        def loss(mv):
            return float(g[w] @ oracle_qdd(OracleWorld(per_dof(raw_at(raw, entries, mv))), s[w], tau[w]))

        fd = np.array([(loss(M[w] + 1e-6 * e) - loss(M[w] - 1e-6 * e)) / 2e-6 for e in np.eye(len(M[w]))])
        assert rel_err(gm, fd) < 1e-6, (gm, fd)


def test_reduced_and_reordered_action_space_takes_tau_per_dof():
    """An action space that leaves the free root unactuated and lists the other dofs backwards: tau is still read per dof."""
    raw = load_raw("atlas")
    red = copy.deepcopy(raw)
    red.action_map = np.arange(raw.ndof - 1, 5, -1)
    ew, ref_w = EmulFdWorld(nb.compile_model(red, lanes=1)), EmulFdWorld(nb.compile_model(raw, lanes=1))
    ow = OracleWorld(per_dof(raw))
    s, tau = fd_inputs(raw, 3, seed=12)
    for fp64 in (False, True):
        qdd, _ = ew.forward_dynamics(s, tau, fp64)
        assert np.array_equal(qdd, ref_w.forward_dynamics(s, tau, fp64)[0])
        for w in range(3):
            assert rel_err(qdd[w], oracle_qdd(ow, s[w], tau[w])) < (1e-9 if fp64 else 1e-4)


def test_value_errors():
    raw = load_raw("half_cheetah")
    world = register(nb.World.from_raw(raw), step=2)
    n, m = raw.ndof, world.getMassDims()
    s, t = torch.zeros(2, 2 * n), torch.zeros(2, n)
    for bad_s, bad_t in ((torch.zeros(2, 2 * n + 1), t), (s, torch.zeros(2, n + 1)), (s, torch.zeros(3, n)), (torch.zeros(2 * n), t),
                         (torch.zeros(2, 3, 2 * n), torch.zeros(2, 3, n))):
        with pytest.raises(ValueError):
            nb.forward_dynamics(world, bad_s, bad_t)
    with pytest.raises(ValueError):
        nb.forward_dynamics(world, s, t, torch.zeros(2, m + 1, dtype=torch.float64))
    with pytest.raises(ValueError):
        nb.forward_dynamics(world, s, t, torch.zeros(3, m, dtype=torch.float64))
    with pytest.raises(ValueError):
        nb.forward_dynamics(world, s[0], t[0], torch.zeros(2, m, dtype=torch.float64))
    with pytest.raises(ValueError):
        nb.forward_dynamics(world, s, t, torch.ones(m + 1, dtype=torch.float64))
    with pytest.raises(ValueError):
        nb.ForwardDynamicsLayer.apply(world, s, t, torch.ones(m, dtype=torch.float64), torch.ones(2, raw.nb, 10, dtype=torch.float64))
    with pytest.raises(ValueError):
        nb.forward_dynamics(nb.World(), torch.zeros(2, 0), torch.zeros(2, 0))
