"""The inverse-dynamics and energy regressors on the host (tests/host_emul/emul_reg.cpp): Y pi + tau_passive against the emulated inverse
dynamics at the model's and at per-world inertia tables, Y_T pi and Y_U pi + U_spring against the emulated energies, the fp64 oracle and
1/2 qdot^T M qdot; every row of Y against the emulated ID backward's inertia gradient seeded with e_d; Y P^T against central differences
of the fp64 inverse-dynamics oracle with respect to a mass vector registering every body; the power balance of every parameter column;
the structural zeros; and the argument checks of nimblephysics_b200.inverse_dynamics_regressor / energy_regressor."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from nimblephysics_b200 import modelspec as ms
from tests.host_emul.binding_energy import EmulEnergyWorld
from tests.host_emul.binding_reg import EmulRegWorld
from tests.oracle_id.binding import IdOracle
from tests.test_energy import oracle_energy, skeleton_of
from tests.test_inverse_dynamics import _velocity_map, id_inputs
from tests.test_mass_matrix import MODELS, model_raw, oracle_M
from tests.test_per_world_mass import random_masses, raw_at, register
from tests.test_world_jacobian import canon_root, com_body
from tests.util import load_raw, rel_err


def _world(raw):
    return nb.World.from_raw(raw)


def _tables(raw, cm, B, seed):
    """[(name, [B, nb, 10] table)]: the model's own, and per-world tables from mass_to_inertia of random masses"""
    own = np.broadcast_to(cm.inertia, (B, cm.nb, 10)).copy()
    world = register(_world(raw), step=2)
    M = random_masses(world, B, seed=seed)
    return [("model", own), ("per-world", nb.mass_to_inertia(world, torch.tensor(M, dtype=torch.float64)).numpy())]


def _anc(cm):
    """A[d, j]: dof d's joint is at or above canonical body j"""
    A = np.zeros((cm.ndof, cm.nb), bool)
    for j in range(cm.nb):
        i = j
        while i >= 0:
            o = int(cm.dof_off[i])
            A[o:o + (6 if cm.jtype[i] == 3 else 1), j] = True  # canonical joints: 1 revolute, 2 prismatic, 3 free
            i = int(cm.parent[i])
    return A


@pytest.mark.parametrize("name", MODELS)
@pytest.mark.parametrize("fp64", [False, True])
def test_emulated_id_regressor_reproduces_inverse_dynamics(name, fp64):
    raw = model_raw(name)
    cm = nb.compile_model(raw, lanes=1)
    ew = EmulRegWorld(cm)
    B = 3
    s, vn = id_inputs(raw, B, seed=71)
    Y, tp = ew.id_regressor(s, vn, fp64)
    assert np.isfinite(Y).all() and np.isfinite(tp).all()
    tol = 1e-12 if fp64 else 1e-5
    for kind, pi in _tables(raw, cm, B, seed=72):
        tau, _ = ew.inverse_dynamics(s, vn, fp64, world_inertia=pi)
        got = np.einsum("bdjk,bjk->bd", Y.astype(np.float64), pi) + tp
        for w in range(B):
            assert rel_err(got[w], tau[w]) < tol, (kind, w, rel_err(got[w], tau[w]))
    sd = s.astype(np.float64)
    n = raw.ndof
    assert np.allclose(tp, raw.spring * (sd[:, :n] - raw.rest + sd[:, n:] * raw.dt) + raw.damping * sd[:, n:], rtol=tol, atol=tol)


@pytest.mark.parametrize("name", MODELS)
@pytest.mark.parametrize("fp64", [False, True])
def test_emulated_energy_regressor_reproduces_the_energies(name, fp64):
    raw = model_raw(name)
    cm = nb.compile_model(raw, lanes=1)
    ew = EmulRegWorld(cm)
    B, n = 2, raw.ndof
    s = id_inputs(raw, B, seed=73)[0].astype(np.float64)
    YT, YU, Us = ew.energy_regressor(s, fp64)
    tol = 1e-12 if fp64 else 1e-5
    pi = cm.inertia
    for w in range(B):
        q, qd = s[w, :n], s[w, n:]
        T = float(np.sum(YT[w].astype(np.float64) * pi))
        Tm = 0.5 * qd @ oracle_M(raw, q) @ qd
        assert abs(T - Tm) < max(tol, 1e-9) * max(1.0, abs(Tm)), (w, T, Tm)
        assert abs(Us[w] - 0.5 * np.sum(raw.spring * (q - raw.rest) ** 2)) < tol * max(1.0, abs(Us[w]))
    rb = com_body(raw, cm)
    if rb is None:
        return
    root = canon_root(cm, rb)
    cols = np.array([canon_root(cm, int(cm.orig_body[j])) == root for j in range(cm.nb)])
    _, dofs = skeleton_of(raw, rb)
    Te, Ue, _ = EmulEnergyWorld(cm).energy_momentum(s, root, fp64=fp64)
    for w in range(B):
        q, qd = s[w, :n], s[w, n:]
        T = float(np.sum(YT[w][cols].astype(np.float64) * pi[cols]))
        U = float(np.sum(YU[w][cols].astype(np.float64) * pi[cols])) + 0.5 * np.sum(raw.spring[dofs] * (q[dofs] - raw.rest[dofs]) ** 2)
        scale = max(abs(Te[w]), abs(Ue[w]), 1.0)
        assert abs(T - Te[w]) < tol * scale and abs(U - Ue[w]) < tol * scale, (w, T, Te[w], U, Ue[w])
        To, Uo, _ = oracle_energy(raw, q, qd, rb)
        assert abs(T - To) < max(tol, 1e-9) * scale and abs(U - Uo) < max(tol, 1e-9) * scale, (w, T, To, U, Uo)


@pytest.mark.parametrize("name", MODELS)
def test_emulated_rows_are_the_inverse_dynamics_vjp(name):
    raw = model_raw(name)
    cm = nb.compile_model(raw, lanes=1)
    ew = EmulRegWorld(cm)
    n = raw.ndof
    s, vn = id_inputs(raw, 1, seed=74)
    Y, _ = ew.id_regressor(s, vn, True)
    S, V = np.repeat(s, n, 0), np.repeat(vn, n, 0)  # world d: the seed e_d
    _, saved = ew.inverse_dynamics(S, V, True)
    _, _, gi = ew.inverse_dynamics_backward(S, saved, np.eye(n), True)
    G = gi.T.reshape(n, cm.nb, 10)
    scale = np.abs(Y[0]).max(axis=(1, 2))
    err = np.abs(G - Y[0]).max(axis=(1, 2))
    assert np.all(err <= 1e-12 * np.maximum(scale, 1.0)), err.max()


@pytest.mark.parametrize("name", ["half_cheetah", "atlas"])
def test_emulated_regressor_matches_oracle_mass_differences(name):
    """Every raw body registered INERTIA_FULL: Y P^T against central differences of the fp64 oracle's tau with respect to the mass vector."""
    raw = load_raw(name)
    world = _world(raw)
    for sk in world.skeletons:
        for b in sk._ordered_bodies():
            world.tuneMass(b, ms.INERTIA_FULL)
    entries = world._mass_entries()
    cm = nb.compile_model(raw, lanes=1)
    ew = EmulRegWorld(cm)
    s, vn = id_inputs(raw, 2, seed=75)
    Y, _ = ew.id_regressor(s, vn, True)
    m0 = np.concatenate([ms._mass_entry_value(ms.INERTIA_FULL, raw.mass[bi], raw.com[bi], raw.moment[bi]) for bi, _ in entries])
    P = ms.inertia_param_jacobian(raw, cm, entries)
    for w in range(2):
        s64, vn64 = s[w].astype(np.float64), vn[w].astype(np.float64)
        J = Y[w].reshape(raw.ndof, -1) @ P.T
        fd = np.zeros_like(J)
        for c in range(len(m0)):
            mp, mm = m0.copy(), m0.copy()
            mp[c] += 1e-5
            mm[c] -= 1e-5
            fd[:, c] = (IdOracle(raw_at(raw, entries, mp)).inverse_dynamics(s64, vn64)
                        - IdOracle(raw_at(raw, entries, mm)).inverse_dynamics(s64, vn64)) / 2e-5
        assert np.abs(J - fd).max() < 1e-7 * max(1.0, np.abs(fd).max()), np.abs(J - fd).max()


@pytest.mark.parametrize("name", ["tree", "half_cheetah", "atlas"])
def test_emulated_power_balance_of_every_parameter_column(name):
    """d/dt (Y_T + Y_U)[j, k] along (qdot, qddot) = sum_d qdot_d Y[d, j, k] with v' = qdot + dt qddot, by fp64 central differences."""
    raw = model_raw(name)
    cm = nb.compile_model(raw, lanes=1)
    ew = EmulRegWorld(cm)
    n, B = raw.ndof, 3
    s = id_inputs(raw, B, seed=76)[0].astype(np.float64)
    qdd = np.random.default_rng(77).uniform(-5, 5, (B, n))
    Y, _ = ew.id_regressor(s, s[:, n:] + raw.dt * qdd, True)
    h = 1e-5
    for w in range(B):
        q, qd = s[w, :n], s[w, n:]
        qr = np.linalg.solve(_velocity_map(raw, q), qd)
        E = lambda t: sum(ew.energy_regressor(np.concatenate([q + t * qr, qd + t * qdd[w]])[None], True)[:2])[0]
        lhs = (E(h) - E(-h)) / (2 * h)
        rhs = np.einsum("d,djk->jk", qd, Y[w])
        assert np.abs(lhs - rhs).max() < 1e-7 * max(1.0, np.abs(rhs).max()), np.abs(lhs - rhs).max()


@pytest.mark.parametrize("name", ["tree", "half_cheetah", "atlas", "free16"])
@pytest.mark.parametrize("lanes", [2, 4, 8])
def test_emulated_lane_schedules_agree(name, lanes):
    """the kinematics stages run on the model's lane schedule (the device takes the widest): every schedule gives the same bits"""
    raw = model_raw(name)
    try:
        cm = nb.compile_model(raw, lanes=lanes)
    except ValueError:
        pytest.skip(f"no {lanes}-lane schedule for this model")
    s, vn = id_inputs(raw, 3, seed=79)
    one, many = EmulRegWorld(nb.compile_model(raw, lanes=1)), EmulRegWorld(cm)
    for fp64 in (False, True):
        for a, b in zip(one.id_regressor(s, vn, fp64) + one.energy_regressor(s, fp64), many.id_regressor(s, vn, fp64) + many.energy_regressor(s, fp64)):
            assert np.array_equal(a, b)


@pytest.mark.parametrize("name", MODELS)
def test_emulated_structural_zeros(name):
    raw = model_raw(name)
    cm = nb.compile_model(raw, lanes=1)
    ew = EmulRegWorld(cm)
    s, vn = id_inputs(raw, 2, seed=78)
    A = _anc(cm)
    for fp64 in (False, True):
        Y, _ = ew.id_regressor(s, vn, fp64)
        assert np.all(Y[:, ~A] == 0)
        assert np.all(np.abs(Y[:, A]).max(axis=-1) > 0)


def test_emulated_empty_batch():
    raw = load_raw("atlas")
    ew = EmulRegWorld(nb.compile_model(raw, lanes=1))
    n = raw.ndof
    Y, tp = ew.id_regressor(np.zeros((0, 2 * n)), np.zeros((0, n)), True)
    YT, YU, Us = ew.energy_regressor(np.zeros((0, 2 * n)), True)
    assert Y.shape == (0, n, ew.cm.nb, 10) and tp.shape == (0, n) and YT.shape == YU.shape == (0, ew.cm.nb, 10) and Us.shape == (0,)


def test_value_errors():
    raw = load_raw("half_cheetah")
    world = _world(raw)
    n = raw.ndof
    for bad_s, bad_v in ((torch.zeros(n), torch.zeros(n)), (torch.zeros(2, 2 * n + 1), torch.zeros(2, n)), (torch.zeros(2, 2 * n), torch.zeros(2, n + 1)),
                         (torch.zeros(2, 2 * n), torch.zeros(3, n)), (torch.zeros(2, 2 * n), torch.zeros(n)), (torch.zeros(2, 3, 2 * n), torch.zeros(2, 3, n))):
        with pytest.raises(ValueError):
            nb.inverse_dynamics_regressor(world, bad_s, bad_v)
    for bad in (torch.zeros(n), torch.zeros(2, 2 * n + 1), torch.zeros(2, 3, 2 * n), torch.zeros(())):
        with pytest.raises(ValueError):
            nb.energy_regressor(world, bad)
    with pytest.raises(ValueError):
        nb.inverse_dynamics_regressor(nb.World(), torch.zeros(2, 0), torch.zeros(2, 0))
    with pytest.raises(ValueError):
        nb.energy_regressor(nb.World(), torch.zeros(2, 0))
