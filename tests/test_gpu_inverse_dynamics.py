"""Contact-free inverse dynamics on the GPU (nb2_inverse_dynamics / _backward through nimblephysics_b200.inverse_dynamics) against
the fp64 oracle: tau, state / next-velocity / per-world mass gradients at partial-group batch sizes, lane schedules, the round trip
through the step, isolation between worlds, and a world with collision pairs."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from nimblephysics_b200 import modelspec as ms
from tests.oracle_id.binding import IdOracle
from tests.test_inverse_dynamics import id_inputs
from tests.test_per_world_mass import random_masses, raw_at, register
from tests.util import contact_inputs, load_raw, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _check_worlds(B):
    return sorted({0, B // 2, B - 1})


@pytest.mark.parametrize("name", ["cartpole", "half_cheetah", "atlas"])
@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("B", [1, 3, 33, 4099])
def test_id_and_gradients_match_oracle(name, fp64, B):
    raw = load_raw(name)
    world = register(nb.World.from_raw(raw), step=3)
    world._contacts_disabled = True
    n, dt = raw.ndof, torch.float64 if fp64 else torch.float32
    M = random_masses(world, B, seed=B)
    s, vn = id_inputs(raw, B, seed=B + 1)
    gt = np.random.default_rng(B).normal(size=(B, n))
    st = torch.tensor(s, dtype=dt, device=DEV, requires_grad=True)
    vt = torch.tensor(vn, dtype=dt, device=DEV, requires_grad=True)
    mass = torch.tensor(M, dtype=torch.float64, device=DEV, requires_grad=True)
    tau = nb.inverse_dynamics(world, st, vt, mass)
    assert tau.shape == (B, n) and tau.dtype == dt
    tau.backward(torch.tensor(gt, dtype=dt, device=DEV))
    tau, gs, gv, gm = (x.detach().cpu().numpy() for x in (tau, st.grad, vt.grad, mass.grad))
    gt = gt.astype(np.float64) if fp64 else gt.astype(np.float32).astype(np.float64)
    tol = 1e-9 if fp64 else 1e-4
    entries = world._mass_entries()
    for w in _check_worlds(B):
        s64, vn64 = s[w].astype(np.float64), vn[w].astype(np.float64)
        ow = IdOracle(raw_at(raw, entries, M[w]))
        rt, J = ow.inverse_dynamics(s64, vn64, want_jac=True)
        g = J.T @ gt[w]
        assert rel_err(tau[w], rt) < tol and rel_err(gs[w], g[:2 * n]) < tol and rel_err(gv[w], g[2 * n:]) < tol, w

        def loss(mv):  # tau is affine in the mass and diagonal entries and quadratic in the COM: central differences are exact
            return float(gt[w] @ IdOracle(raw_at(raw, entries, mv)).inverse_dynamics(s64, vn64))

        fd = np.array([(loss(M[w] + 1e-3 * e) - loss(M[w] - 1e-3 * e)) / 2e-3 for e in np.eye(len(M[w]))])
        assert rel_err(gm[w], fd) < tol, (w, rel_err(gm[w], fd))


def test_shared_mass_gradient_sums_over_the_batch():
    raw = load_raw("half_cheetah")
    world = register(nb.World.from_raw(raw), step=2)
    world._contacts_disabled = True
    B = 33
    s, vn = id_inputs(raw, B, seed=2)
    gt = np.random.default_rng(3).normal(size=(B, raw.ndof))
    m0 = world.getMasses().copy()
    mass = torch.tensor(m0, dtype=torch.float64, device=DEV, requires_grad=True)
    st, vt = (torch.tensor(x, dtype=torch.float64, device=DEV) for x in (s, vn))
    nb.inverse_dynamics(world, st, vt, mass).backward(torch.tensor(gt, device=DEV))
    entries = world._mass_entries()

    def loss(mv):
        ow = IdOracle(raw_at(raw, entries, mv))
        return sum(float(gt[w] @ ow.inverse_dynamics(s[w].astype(np.float64), vn[w].astype(np.float64))) for w in range(B))

    fd = np.array([(loss(m0 + 1e-3 * e) - loss(m0 - 1e-3 * e)) / 2e-3 for e in np.eye(len(m0))])
    assert rel_err(mass.grad.cpu().numpy(), fd) < 1e-9


@pytest.mark.parametrize("name", ["half_cheetah", "atlas"])
def test_every_lane_schedule_gives_the_same_tau(name):
    raw = load_raw(name)
    world = nb.World.from_raw(raw)
    world._contacts_disabled = True
    dm = nb.device_model_for(world)
    s, vn = id_inputs(raw, 4099, seed=5)
    st, vt = torch.tensor(s, device=DEV), torch.tensor(vn, device=DEV)
    out = {}
    try:
        for c in dm.schedules:
            dm.set_lanes(c.lanes)
            out[c.lanes] = nb.inverse_dynamics(world, st, vt).cpu().numpy()
    finally:
        dm.set_lanes(0)
    assert len(out) > 1
    ref = out[1]
    for k, t in out.items():
        assert max(rel_err(t[w], ref[w]) for w in range(len(t))) < 2e-6, k


@pytest.mark.parametrize("name", ["cartpole", "half_cheetah", "atlas"])
def test_round_trip_through_the_step(name):
    raw = load_raw(name)
    world = nb.World.from_raw(raw)
    world._contacts_disabled = True
    n = raw.ndof
    world.setActionSpace(range(n))
    s, vn = id_inputs(raw, 256, seed=8)
    st, vt = torch.tensor(s, device=DEV), torch.tensor(vn, device=DEV)
    nxt = nb.timestep(world, st, nb.inverse_dynamics(world, st, vt))[:, n:]
    dv = (vt - st[:, n:]).norm(dim=1)
    assert ((nxt - vt).norm(dim=1) <= 1e-3 * dv).all(), ((nxt - vt).norm(dim=1) / dv).max().item()
    # fp64: forward dynamics of the returned force is the acceleration a = (v' - qdot) / dt
    s64, v64 = st.double(), vt.double()
    tau = nb.inverse_dynamics(world, s64, v64)
    acc = nb.device_model_for(world).forward_dynamics(s64[:, :n], s64[:, n:], tau)
    a = (v64 - s64[:, n:]) / raw.dt
    assert ((acc - a).norm(dim=1) <= 1e-9 * a.norm(dim=1)).all(), ((acc - a).norm(dim=1) / a.norm(dim=1)).max().item()


def test_worlds_are_independent():
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=3)
    world._contacts_disabled = True
    B = 96
    M = random_masses(world, B, seed=1)
    s, vn = id_inputs(raw, B, seed=9)
    gt = torch.tensor(np.random.default_rng(4).normal(size=(B, raw.ndof)), dtype=torch.float32, device=DEV)

    def run(s, vn, M):
        st = torch.tensor(s, device=DEV, requires_grad=True)
        vt = torch.tensor(vn, device=DEV, requires_grad=True)
        mass = torch.tensor(M, device=DEV, requires_grad=True)
        tau = nb.inverse_dynamics(world, st, vt, mass)
        tau.backward(gt)
        return [x.detach().cpu().numpy() for x in (tau, st.grad, vt.grad, mass.grad)]

    r0 = run(s, vn, M)
    s2, vn2, M2 = s.copy(), vn.copy(), M.copy()
    s2[40] += 0.1
    vn2[40] -= 0.2
    M2[40] *= 1.3
    r1 = run(s2, vn2, M2)
    keep = np.arange(B) != 40
    assert all(np.array_equal(x[keep], y[keep]) for x, y in zip(r0, r1))
    assert not np.array_equal(r0[0][40], r1[0][40])


def test_single_world_and_contact_world():
    """A 1-D state gives a 1-D tau and leaves the World's state alone; a world with collision pairs gets the contact-free tau of its
    tree and its LCP cache is not touched."""
    raw = load_raw("half_cheetah")
    world = nb.World.from_raw(raw)
    assert nb.device_model_for(world).has_contacts
    B = 16
    cs, ca = contact_inputs(raw, "half_cheetah", B, seed=5)
    nb.reset_contact_cache(world)
    nb.timestep(world, torch.tensor(cs, device=DEV), torch.tensor(ca, device=DEV))
    cache = nb.contact_cache(world, B, DEV)
    before = {k: v.clone() for k, v in cache.items() if torch.is_tensor(v)}
    n = raw.ndof
    vn = (cs[:, n:] + raw.dt * np.random.default_rng(1).uniform(-5, 5, (B, n))).astype(np.float32)
    tau = nb.inverse_dynamics(world, torch.tensor(cs, device=DEV, dtype=torch.float64), torch.tensor(vn, device=DEV, dtype=torch.float64))
    assert world._lcp_cache is cache and all(torch.equal(before[k], cache[k]) for k in before)
    ow = IdOracle(raw)
    for w in range(B):
        assert rel_err(tau[w].cpu().numpy(), ow.inverse_dynamics(cs[w].astype(np.float64), vn[w].astype(np.float64))) < 1e-9
    state0 = world.getState().copy()
    t1 = nb.inverse_dynamics(world, torch.tensor(cs[3], device=DEV), torch.tensor(vn[3], device=DEV))
    assert t1.shape == (n,) and np.array_equal(world.getState(), state0)
    assert rel_err(t1.cpu().numpy(), tau[3].cpu().numpy()) < 1e-4
