"""Contact inverse dynamics on the GPU (nb2_contact_inverse_dynamics / _backward through nimblephysics_b200.contact_inverse_dynamics) against
the fp64 oracle: tau, wrench, state / next-velocity / per-world and shared mass gradients at partial-block batch sizes; dofs off the chain
bit-identical to inverse_dynamics; and the round trip through a single-support contact step of Atlas on the ground."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from tests.oracle_id.binding_cid import CidOracle
from tests.test_inverse_dynamics import id_inputs
from tests.test_per_world_mass import random_masses, raw_at, register
from tests.util import load_raw, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _node(world, name):
    return next(b for sk in world.skeletons for b in sk._ordered_bodies() if b.name == name)


def _raw_index(raw, name):
    return list(raw.body_names).index(name)


@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("B", [1, 3, 33, 4099])
def test_contact_id_and_gradients_match_oracle(fp64, B):
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=3)
    world._contacts_disabled = True
    n, dt = raw.ndof, torch.float64 if fp64 else torch.float32
    M = random_masses(world, B, seed=B)
    s, vn = id_inputs(raw, B, seed=B + 2)
    rng = np.random.default_rng(B)
    gt, gw = rng.normal(size=(B, n)), rng.normal(size=(B, 6))
    st = torch.tensor(s, dtype=dt, device=DEV, requires_grad=True)
    vt = torch.tensor(vn, dtype=dt, device=DEV, requires_grad=True)
    mass = torch.tensor(M, dtype=torch.float64, device=DEV, requires_grad=True)
    tau, w = nb.contact_inverse_dynamics(world, st, vt, _node(world, "l_foot"), mass)
    assert tau.shape == (B, n) and w.shape == (B, 6) and tau.dtype == dt and w.dtype == dt
    torch.autograd.backward([tau, w], [torch.tensor(gt, dtype=dt, device=DEV), torch.tensor(gw, dtype=dt, device=DEV)])
    tau, w, gs, gv, gm = (x.detach().cpu().numpy() for x in (tau, w, st.grad, vt.grad, mass.grad))
    cast = (lambda a: a.astype(np.float64)) if fp64 else (lambda a: a.astype(np.float32).astype(np.float64))
    tol = 1e-9 if fp64 else 1e-4
    entries = world._mass_entries()
    b = _raw_index(raw, "l_foot")
    for k in sorted({0, B // 2, B - 1}):
        s64, vn64 = s[k].astype(np.float64), vn[k].astype(np.float64)
        co = CidOracle(raw_at(raw, entries, M[k]))
        rt, rw, J = co.contact_inverse_dynamics(b, s64, vn64, want_jac=True)
        g = J.T @ np.concatenate([cast(gt[k]), cast(gw[k])])
        scale = max(np.linalg.norm(rt), np.linalg.norm(rw))
        assert np.linalg.norm(tau[k] - rt) < tol * scale and np.linalg.norm(w[k] - rw) < tol * scale, k
        assert rel_err(gs[k], g[:2 * n]) < tol and rel_err(gv[k], g[2 * n:]) < tol, k

        def loss(mv):  # tau and the wrench are affine in the masses and quadratic in the COM: central differences are exact
            t, ww = CidOracle(raw_at(raw, entries, mv)).contact_inverse_dynamics(b, s64, vn64)
            return float(cast(gt[k]) @ t + cast(gw[k]) @ ww)

        fd = np.array([(loss(M[k] + 1e-3 * e) - loss(M[k] - 1e-3 * e)) / 2e-3 for e in np.eye(len(M[k]))])
        assert rel_err(gm[k], fd) < tol, (k, rel_err(gm[k], fd))


def test_shared_mass_gradient_sums_over_the_batch():
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=5)
    world._contacts_disabled = True
    B = 33
    s, vn = id_inputs(raw, B, seed=12)
    rng = np.random.default_rng(13)
    gt, gw = rng.normal(size=(B, raw.ndof)), rng.normal(size=(B, 6))
    m0 = world.getMasses().copy()
    mass = torch.tensor(m0, dtype=torch.float64, device=DEV, requires_grad=True)
    st, vt = (torch.tensor(x, dtype=torch.float64, device=DEV) for x in (s, vn))
    tau, w = nb.contact_inverse_dynamics(world, st, vt, _node(world, "r_hand"), mass)
    torch.autograd.backward([tau, w], [torch.tensor(gt, device=DEV), torch.tensor(gw, device=DEV)])
    entries, b = world._mass_entries(), _raw_index(raw, "r_hand")

    def loss(mv):
        co = CidOracle(raw_at(raw, entries, mv))
        out = 0.0
        for k in range(B):
            t, ww = co.contact_inverse_dynamics(b, s[k].astype(np.float64), vn[k].astype(np.float64))
            out += float(gt[k] @ t + gw[k] @ ww)
        return out

    fd = np.array([(loss(m0 + 1e-3 * e) - loss(m0 - 1e-3 * e)) / 2e-3 for e in np.eye(len(m0))])
    assert rel_err(mass.grad.cpu().numpy(), fd) < 1e-9


@pytest.mark.parametrize("fp64", [False, True])
def test_dofs_off_the_chain_are_those_of_inverse_dynamics(fp64):
    """Atlas plus a second free-floating body: only the stance leg's dofs differ from inverse_dynamics (the root rows are 0); the other
    limbs and the other skeleton are bit-identical."""
    world = nb.World.from_raw(load_raw("atlas"))
    sk = nb.Skeleton("box")
    _, box = sk.createFreeJointAndBodyNodePair(None)
    box.setMass(3.0)
    box.setMomentOfInertia(0.2, 0.3, 0.4)
    world.addSkeleton(sk)
    world._contacts_disabled = True
    raw = nb.flatten_world(world)
    n, B, dt = raw.ndof, 257, torch.float64 if fp64 else torch.float32
    s, vn = id_inputs(raw, B, seed=3)
    st, vt = torch.tensor(s, dtype=dt, device=DEV), torch.tensor(vn, dtype=dt, device=DEV)
    tid = nb.inverse_dynamics(world, st, vt).cpu().numpy()
    tau, w = nb.contact_inverse_dynamics(world, st, vt, _node(world, "l_foot"))
    tau = tau.cpu().numpy()
    chain, i = set(range(6)), _raw_index(raw, "l_foot")
    while raw.parent[i] >= 0:
        chain |= {int(raw.dof_off[i])}
        i = raw.parent[i]
    off = [d for d in range(n) if d not in chain]
    assert len(off) == n - len(chain) and n - 6 in off
    assert np.array_equal(tau[:, off], tid[:, off])
    assert not np.any(tau[:, :6])
    # the box's wrench is its own: naming it gives its six inverse-dynamics entries in world axes, and the robot's dofs unchanged
    tb, wb = nb.contact_inverse_dynamics(world, st, vt, box)
    tb = tb.cpu().numpy()
    assert np.array_equal(tb[:, :n - 6], tid[:, :n - 6]) and not np.any(tb[:, n - 6:])
    assert not torch.equal(wb, w)


def _single_support_inputs(raw, B, seed):
    """Atlas on the ground (the contact_inputs pose: feet 6-10 mm into the ground) with the left leg bent (hip -0.6, knee 1.2, ankle -0.6:
    the left sole 11 cm above the right one), joint noise, and random joint torques inside the force limits; 0 on the root."""
    rng = np.random.default_rng(seed)
    n, na = raw.ndof, len(raw.action_map)
    q = np.zeros((B, n))
    q[:, 0] = -0.5 * np.pi
    q[:, 4] = -0.01 + rng.uniform(-0.004, 0.0, B)
    q[:, 6:] = rng.normal(0, 0.01, (B, n - 6))
    names = list(raw.body_names)
    for bn, val in (("l_uleg", -0.6), ("l_lleg", 1.2), ("l_talus", -0.6)):
        q[:, raw.dof_off[names.index(bn)]] += val
    v = rng.normal(0, 0.05, (B, n))
    lim = np.minimum(np.minimum(-np.asarray(raw.force_lo), np.asarray(raw.force_hi)), 20.0)[np.asarray(raw.action_map)]
    a = rng.uniform(-0.5, 0.5, (B, na)) * lim
    a[:, np.asarray(raw.action_map) < 6] = 0.0
    return np.concatenate([q, v], 1).astype(np.float32), a.astype(np.float32)


def test_single_support_round_trip_through_the_contact_step():
    """One contact step with the left foot lifted; contact inverse dynamics (fp64) of its output with the right foot as the contact body
    returns the applied joint torques.  The step's rows are fp32: the tolerance is the first-order effect of rounding v' to fp32
    (|d tau / d v'| |v'| 2^-24, from the oracle's Jacobian), which 1/dt amplifies."""
    raw = load_raw("atlas_ground")
    world = nb.World.from_raw(raw)
    n, B = raw.ndof, 64
    s, a = _single_support_inputs(raw, B, seed=7)
    st, at = torch.tensor(s, device=DEV), torch.tensor(a, device=DEV)
    nb.reset_contact_cache(world)
    nxt = nb.timestep(world, st, at).cpu().numpy()
    for k in range(B):
        cs = world.getLastCollisionResult(k).getContacts()
        assert cs and all({c.bodyNodeA, c.bodyNodeB} == {"r_foot", "ground_link"} for c in cs), k
    vnext = nxt[:, n:]
    tau, _ = nb.contact_inverse_dynamics(world, st.double(), torch.tensor(vnext, dtype=torch.float64, device=DEV), _node(world, "r_foot"))
    tau = tau.cpu().numpy()
    applied = np.zeros((B, n))
    applied[:, np.asarray(raw.action_map)] = a
    co, b = CidOracle(raw), _raw_index(raw, "r_foot")
    worst = 0.0
    for k in range(B):
        _, _, J = co.contact_inverse_dynamics(b, s[k].astype(np.float64), vnext[k].astype(np.float64), want_jac=True)
        bound = np.abs(J[:n, 2 * n:]) @ (np.abs(vnext[k].astype(np.float64)) * 2.0**-24)
        err = np.abs(tau[k, 6:] - applied[k, 6:])
        worst = max(worst, float(np.max(err / (bound[6:] + 1e-300))))
        assert np.all(err <= 4.0 * bound[6:] + 1e-9), (k, np.max(err / bound[6:]))
    print(f"[single support] worst |tau - applied| / (fp32 rounding bound of v') = {worst:.3f}")
