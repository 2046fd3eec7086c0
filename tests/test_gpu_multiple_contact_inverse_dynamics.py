"""Multiple-contact inverse dynamics on the GPU (nb2_multiple_contact_inverse_dynamics / _backward through
nimblephysics_b200.multiple_contact_inverse_dynamics) against the fp64 oracle: tau, wrenches, state / next-velocity / guess / per-world and
shared mass gradients at partial-block batch sizes; dofs off the chains bit-identical to inverse_dynamics; one body equal to
contact_inverse_dynamics; and the round trip through a double-support contact step of Atlas on the ground."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from tests.oracle_id.binding import IdOracle
from tests.oracle_id.binding_mcid import McidOracle
from tests.test_contact_inverse_dynamics import _ik_contact_jacobian
from tests.test_inverse_dynamics import id_inputs
from tests.test_per_world_mass import random_masses, raw_at, register
from tests.util import contact_inputs, load_raw, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
SETS = {2: ["l_foot", "r_foot"], 4: ["l_foot", "r_foot", "l_hand", "r_hand"]}


def _node(world, name):
    return next(b for sk in world.skeletons for b in sk._ordered_bodies() if b.name == name)


def _raw_index(raw, name):
    return list(raw.body_names).index(name)


@pytest.mark.parametrize("k", [2, 4])
@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("B", [1, 3, 33, 4099])
def test_multiple_contact_id_and_gradients_match_oracle(k, fp64, B):
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=3)
    world._contacts_disabled = True
    n, dt = raw.ndof, torch.float64 if fp64 else torch.float32
    M = random_masses(world, B, seed=B + k)
    s, vn = id_inputs(raw, B, seed=B + 7)
    rng = np.random.default_rng(B + k)
    g = rng.normal(0, 40, (B, k, 6))
    gt, gw = rng.normal(size=(B, n)), rng.normal(size=(B, k, 6))
    st = torch.tensor(s, dtype=dt, device=DEV, requires_grad=True)
    vt = torch.tensor(vn, dtype=dt, device=DEV, requires_grad=True)
    gd = torch.tensor(g, dtype=dt, device=DEV, requires_grad=True)
    mass = torch.tensor(M, dtype=torch.float64, device=DEV, requires_grad=True)
    tau, w = nb.multiple_contact_inverse_dynamics(world, st, vt, [_node(world, x) for x in SETS[k]], mass, gd)
    assert tau.shape == (B, n) and w.shape == (B, k, 6) and tau.dtype == dt and w.dtype == dt
    torch.autograd.backward([tau, w], [torch.tensor(gt, dtype=dt, device=DEV), torch.tensor(gw, dtype=dt, device=DEV)])
    tau, w, gs, gv, gg, gm = (x.detach().cpu().numpy() for x in (tau, w, st.grad, vt.grad, gd.grad, mass.grad))
    cast = (lambda a: a.astype(np.float64)) if fp64 else (lambda a: a.astype(np.float32).astype(np.float64))
    tol = 1e-9 if fp64 else 1e-4
    entries = world._mass_entries()
    bodies = [_raw_index(raw, x) for x in SETS[k]]
    for b in sorted({0, B // 2, B - 1}):
        s64, vn64, g64 = cast(s[b]), cast(vn[b]), cast(g[b])
        mo = McidOracle(raw_at(raw, entries, M[b]))
        rt, rw, J = mo.multiple_contact_inverse_dynamics(bodies, s64, vn64, g64, want_jac=True)
        ref = J.T @ np.concatenate([cast(gt[b]), cast(gw[b]).ravel()])
        scale = max(np.linalg.norm(rt), np.linalg.norm(rw))
        assert np.linalg.norm(tau[b] - rt) < tol * scale and np.linalg.norm(w[b] - rw) < tol * scale, b
        assert rel_err(gs[b], ref[:2 * n]) < tol and rel_err(gv[b], ref[2 * n:3 * n]) < tol, b
        assert rel_err(gg[b].ravel(), ref[3 * n:]) < tol, (b, rel_err(gg[b].ravel(), ref[3 * n:]))

        def loss(mv):  # affine in the masses and quadratic in the COM: central differences are exact
            t, ww = McidOracle(raw_at(raw, entries, mv)).multiple_contact_inverse_dynamics(bodies, s64, vn64, g64)
            return float(cast(gt[b]) @ t + (cast(gw[b]) * ww).sum())

        fd = np.array([(loss(M[b] + 1e-3 * e) - loss(M[b] - 1e-3 * e)) / 2e-3 for e in np.eye(len(M[b]))])
        assert rel_err(gm[b], fd) < tol, (b, rel_err(gm[b], fd))


def test_shared_mass_gradient_sums_over_the_batch():
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=5)
    world._contacts_disabled = True
    B, names = 33, SETS[4]
    s, vn = id_inputs(raw, B, seed=14)
    rng = np.random.default_rng(15)
    gt, gw = rng.normal(size=(B, raw.ndof)), rng.normal(size=(B, 4, 6))
    m0 = world.getMasses().copy()
    mass = torch.tensor(m0, dtype=torch.float64, device=DEV, requires_grad=True)
    st, vt = (torch.tensor(x, dtype=torch.float64, device=DEV) for x in (s, vn))
    tau, w = nb.multiple_contact_inverse_dynamics(world, st, vt, [_node(world, x) for x in names], mass)
    torch.autograd.backward([tau, w], [torch.tensor(gt, device=DEV), torch.tensor(gw, device=DEV)])
    entries, bodies = world._mass_entries(), [_raw_index(raw, x) for x in names]

    def loss(mv):
        mo = McidOracle(raw_at(raw, entries, mv))
        out = 0.0
        for b in range(B):
            t, ww = mo.multiple_contact_inverse_dynamics(bodies, s[b].astype(np.float64), vn[b].astype(np.float64))
            out += float(gt[b] @ t + (gw[b] * ww).sum())
        return out

    fd = np.array([(loss(m0 + 1e-3 * e) - loss(m0 - 1e-3 * e)) / 2e-3 for e in np.eye(len(m0))])
    assert rel_err(mass.grad.cpu().numpy(), fd) < 1e-9


@pytest.mark.parametrize("fp64", [False, True])
def test_dofs_off_the_chains_are_those_of_inverse_dynamics(fp64):
    """Atlas plus a second free-floating body, both feet and the left hand as contact bodies: the dofs off the three chains (the right arm,
    the head, the other skeleton) are bit-identical to inverse_dynamics and the root rows are 0."""
    world = nb.World.from_raw(load_raw("atlas"))
    sk = nb.Skeleton("box")
    _, box = sk.createFreeJointAndBodyNodePair(None)
    box.setMass(3.0)
    box.setMomentOfInertia(0.2, 0.3, 0.4)
    world.addSkeleton(sk)
    world._contacts_disabled = True
    raw = nb.flatten_world(world)
    n, B, dt = raw.ndof, 257, torch.float64 if fp64 else torch.float32
    s, vn = id_inputs(raw, B, seed=5)
    st, vt = torch.tensor(s, dtype=dt, device=DEV), torch.tensor(vn, dtype=dt, device=DEV)
    tid = nb.inverse_dynamics(world, st, vt).cpu().numpy()
    names = ["l_foot", "r_foot", "l_hand"]
    tau, _ = nb.multiple_contact_inverse_dynamics(world, st, vt, [_node(world, x) for x in names])
    tau = tau.cpu().numpy()
    chains = set(range(6))
    for x in names:
        i = _raw_index(raw, x)
        while raw.parent[i] >= 0:
            chains |= {int(raw.dof_off[i])}
            i = raw.parent[i]
    off = [d for d in range(n) if d not in chains]
    assert n - 6 in off and int(raw.dof_off[_raw_index(raw, "r_hand")]) in off
    assert np.array_equal(tau[:, off], tid[:, off])
    assert not np.any(tau[:, :6])


@pytest.mark.parametrize("fp64", [False, True])
def test_one_body_is_contact_inverse_dynamics(fp64):
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    world._contacts_disabled = True
    dt, B = torch.float64 if fp64 else torch.float32, 33
    s, vn = id_inputs(raw, B, seed=8)
    for name in ("l_foot", "r_hand"):
        body = _node(world, name)
        st1, vt1 = (torch.tensor(x, dtype=dt, device=DEV, requires_grad=True) for x in (s, vn))
        st2, vt2 = (torch.tensor(x, dtype=dt, device=DEV, requires_grad=True) for x in (s, vn))
        g = torch.full((B, 1, 6), 5.0, dtype=dt, device=DEV, requires_grad=True)
        t1, w1 = nb.contact_inverse_dynamics(world, st1, vt1, body)
        t2, w2 = nb.multiple_contact_inverse_dynamics(world, st2, vt2, [body], wrench_guesses=g)
        assert torch.equal(t1, t2) and torch.equal(w1, w2[:, 0])
        gt, gw = torch.randn_like(t1), torch.randn_like(w1)
        torch.autograd.backward([t1, w1], [gt, gw])
        torch.autograd.backward([t2, w2], [gt, gw[:, None]])
        assert torch.equal(st1.grad, st2.grad) and torch.equal(vt1.grad, vt2.grad) and not torch.any(g.grad)


def _double_support_inputs(raw, B, seed):
    """Atlas on the ground with both feet 6-10 mm into it (the contact_inputs pose), joint noise, and random joint torques inside the
    force limits (at most 10 N m); 0 on the root."""
    s, _ = contact_inputs(raw, "atlas_ground", B, seed=seed)
    rng = np.random.default_rng(seed + 1)
    amap = np.asarray(raw.action_map)
    lim = np.minimum(np.minimum(-np.asarray(raw.force_lo), np.asarray(raw.force_hi)), 20.0)[amap]
    a = rng.uniform(-0.5, 0.5, (B, len(amap))) * lim
    a[:, amap < 6] = 0.0
    return s, a.astype(np.float32)


def test_double_support_round_trip_through_the_contact_step(oracle_mod):
    """One contact step with both feet on the ground.  In the oracle, the feet's wrenches w_true are the least-squares solution of
    A w = tau_ID - applied, A = [J_l^T J_r^T], over every dof; its residual is within the fp32 rounding of v'.  The fp64 layer with w_true
    as guesses returns w_true and the applied joint torques.  The tolerance is the first-order effect of rounding v' to fp32,
    |d out / d v'| |v'| 2^-24, which 1/dt amplifies, with d out / d v' the derivative of the whole chain from the oracle's Jacobians: the
    residual (I - A A^+) d tau_ID / d v' (the projection mixes the root and leg rows, whose bounds differ by orders of magnitude), and for
    the layer's outputs its v' columns plus its guess columns times d w_true / d v' = A^+ d tau_ID / d v'."""
    raw = load_raw("atlas_ground")
    world = nb.World.from_raw(raw)
    n, B = raw.ndof, 64
    s, a = _double_support_inputs(raw, B, seed=9)
    st, at = torch.tensor(s, device=DEV), torch.tensor(a, device=DEV)
    nb.reset_contact_cache(world)
    vnext = nb.timestep(world, st, at).cpu().numpy()[:, n:]
    for b in range(B):
        cs = world.getLastCollisionResult(b).getContacts()
        feet = {c.bodyNodeA for c in cs} | {c.bodyNodeB for c in cs}
        assert feet == {"l_foot", "r_foot", "ground_link"}, (b, feet)
    applied = np.zeros((B, n))
    applied[:, np.asarray(raw.action_map)] = a
    ow, io, mo = oracle_mod.OracleWorld(raw), IdOracle(raw), McidOracle(raw)
    feet = [_raw_index(raw, "l_foot"), _raw_index(raw, "r_foot")]
    w_true, dw_true = np.zeros((B, 2, 6)), np.zeros((B, 12, n))
    worst = {"residual": 0.0, "tau": 0.0, "wrench": 0.0}
    for b in range(B):
        s64, v64 = s[b].astype(np.float64), vnext[b].astype(np.float64)
        dv = np.abs(v64) * 2.0**-24
        tau_id, Jid = io.inverse_dynamics(s64, v64, want_jac=True)
        A = np.concatenate([_ik_contact_jacobian(ow, raw, s64, f).T for f in feet], axis=1)  # [n, 12]
        Ap = np.linalg.pinv(A)
        w = Ap @ (tau_id - applied[b])
        w_true[b] = w.reshape(2, 6)
        dw_true[b] = Ap @ Jid[:, 2 * n:]
        res = np.abs(A @ w - (tau_id - applied[b]))
        bound = np.abs((np.eye(n) - A @ Ap) @ Jid[:, 2 * n:]) @ dv
        worst["residual"] = max(worst["residual"], float(np.max(res / (bound + 1e-300))))
        assert np.all(res <= 4.0 * bound + 1e-9), (b, np.max(res / bound))
    wt = torch.tensor(w_true, device=DEV)
    tau, wr = nb.multiple_contact_inverse_dynamics(world, st.double(), torch.tensor(vnext, dtype=torch.float64, device=DEV),
                                                   [_node(world, "l_foot"), _node(world, "r_foot")], wrench_guesses=wt)
    tau, wr = tau.cpu().numpy(), wr.cpu().numpy()
    for b in range(B):
        _, _, J = mo.multiple_contact_inverse_dynamics(feet, s[b].astype(np.float64), vnext[b].astype(np.float64), w_true[b], want_jac=True)
        D = J[:, 2 * n:3 * n] + J[:, 3 * n:] @ dw_true[b]
        D[n:] -= dw_true[b]
        bound = np.abs(D) @ (np.abs(vnext[b].astype(np.float64)) * 2.0**-24)
        et, ew = np.abs(tau[b, 6:] - applied[b, 6:]), np.abs(wr[b] - w_true[b]).ravel()
        worst["tau"] = max(worst["tau"], float(np.max(et / (bound[6:n] + 1e-300))))
        worst["wrench"] = max(worst["wrench"], float(np.max(ew / (bound[n:] + 1e-300))))
        assert np.all(et <= 4.0 * bound[6:n] + 1e-9), (b, np.max(et / bound[6:n]))
        assert np.all(ew <= 4.0 * bound[n:] + 1e-9), (b, np.max(ew / bound[n:]))
    print("[double support] worst ratio to the fp32 rounding bound of v': " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))
