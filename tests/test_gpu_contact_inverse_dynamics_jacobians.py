"""Dense Jacobians of contact inverse dynamics on the GPU (nb2_multiple_contact_inverse_dynamics_jacobians through
nimblephysics_b200.contact_inverse_dynamics_jacobians / multiple_contact_inverse_dynamics_jacobians): against the dual-number oracle at
partial-block batch sizes, outputs equal to the layers', against autograd's Jacobian of the layers, rows off the chains equal to
inverse_dynamics_jacobians's, the identities of the definition (world_jacobian, mass_matrix, the one-body wrench, the guess blocks,
affinity in next_vel), per-world masses, guard bands, B = 0 and the 1-D state."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from nimblephysics_b200 import modelspec as ms
from tests.oracle_id.binding_mcid import McidOracle
from tests.test_gpu_multiple_contact_inverse_dynamics import SETS
from tests.test_inverse_dynamics import id_inputs
from tests.test_per_world_mass import random_masses, raw_at, register
from tests.util import load_raw, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAMES = {1: ["l_foot"], 2: SETS[2], 4: SETS[4]}


def _world(step=3):
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=step)
    world._contacts_disabled = True
    return raw, world


def _node(world, name):
    return next(b for sk in world.skeletons for b in sk._ordered_bodies() if b.name == name)


def _raw_index(raw, name):
    return list(raw.body_names).index(name)


def _call(world, st, vt, names, mass=None, guess=None):
    """The multiple-contact call with its blocks flattened to the oracle's rows: (tau, w, [T_q, T_qdot, T_v', T_g, W_q, W_qdot, W_v', W_g])
    with T_g [B, n, 6k], W_* [B, 6k, n], W_g [B, 6k, 6k]."""
    out = nb.multiple_contact_inverse_dynamics_jacobians(world, st, vt, [_node(world, x) for x in names], mass, guess)
    B, n, k = st.shape[0], st.shape[1] // 2, len(names)
    T = [out[2], out[3], out[4], out[5].reshape(B, n, 6 * k)]
    W = [x.reshape(B, 6 * k, -1) for x in out[6:]]
    return out[0], out[1], T + W


@pytest.mark.parametrize("k", [1, 2, 4])
@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("B", [1, 3, 33, 4099])
def test_blocks_match_oracle_and_outputs_are_the_layers(k, fp64, B):
    raw, world = _world()
    n, dt = raw.ndof, torch.float64 if fp64 else torch.float32
    s, vn = id_inputs(raw, B, seed=B + 11 * k)
    g = np.random.default_rng(B + k).normal(0, 40, (B, k, 6))
    st, vt, gd = (torch.tensor(a, dtype=dt, device=DEV) for a in (s, vn, g))
    tau, w, blocks = _call(world, st, vt, NAMES[k], guess=gd)
    for x in [tau, w] + blocks:
        assert x.dtype == dt and x.shape[0] == B and not x.requires_grad
    rt, rw = nb.multiple_contact_inverse_dynamics(world, st, vt, [_node(world, x) for x in NAMES[k]], wrench_guesses=gd)
    assert torch.equal(tau, rt) and torch.equal(w, rw)
    blocks = [x.cpu().numpy() for x in blocks]
    tau, w = tau.cpu().numpy(), w.cpu().numpy()
    cast = (lambda a: a.astype(np.float64)) if fp64 else (lambda a: a.astype(np.float32).astype(np.float64))
    tol = 1e-9 if fp64 else 1e-4
    # the position blocks carry the inverse-dynamics position block, whose rotation-derivative terms cancel to a smaller block and are rounded
    # differently by the device's fused multiply-adds: on Atlas in fp64 that block alone lands up to 3.4e-9 from the oracle (DESIGN.md §6l),
    # and after the contact split, which cancels further, the tau position block up to 1.05e-7 (§6s)
    pos = lambda b: max(tol, 1e-6) if b in (0, 4) else tol
    mo = McidOracle(raw)
    bodies = [_raw_index(raw, x) for x in NAMES[k]]
    for b in sorted({0, B // 2, B - 1}):
        ot, ow, J = mo.multiple_contact_inverse_dynamics(bodies, cast(s[b]), cast(vn[b]), cast(g[b]), want_jac=True)
        scale = max(np.linalg.norm(ot), np.linalg.norm(ow))
        assert np.linalg.norm(tau[b] - ot) < tol * scale and np.linalg.norm(w[b] - ow) < tol * scale, b
        cols = (slice(0, n), slice(n, 2 * n), slice(2 * n, 3 * n), slice(3 * n, None))
        refs = [J[:n, c] for c in cols] + [J[n:, c] for c in cols]
        for i, (got, ref) in enumerate(zip(blocks, refs)):
            if k == 1 and i in (3, 7):
                assert not np.any(got[b]), (b, i)  # one body: the guess is not read
            else:
                assert rel_err(got[b], ref) < pos(i), (b, i, rel_err(got[b], ref))


def _autograd_blocks(f, st, vt, gd):
    """Per-world diagonal blocks of torch.autograd.functional.jacobian of f(state, next_vel, guess) -> (tau, w)."""
    Jt, Jw = torch.autograd.functional.jacobian(f, (st, vt, gd))
    idx = torch.arange(st.shape[0], device=st.device)
    return [Jt[0][idx, :, idx], Jt[1][idx, :, idx], Jt[2][idx, :, idx]], [Jw[0][idx, ..., idx, :], Jw[1][idx, ..., idx, :], Jw[2][idx, ..., idx, :, :]]


@pytest.mark.parametrize("k", [1, 2, 4])
@pytest.mark.parametrize("fp64", [False, True])
def test_blocks_equal_autograd_of_the_layer(k, fp64):
    raw, world = _world()
    n, B, dt = raw.ndof, 3, torch.float64 if fp64 else torch.float32
    s, vn = id_inputs(raw, B, seed=31 + k)
    g = np.random.default_rng(32).normal(0, 40, (B, k, 6))
    st, vt, gd = (torch.tensor(a, dtype=dt, device=DEV) for a in (s, vn, g))
    nodes = [_node(world, x) for x in NAMES[k]]
    out = nb.multiple_contact_inverse_dynamics_jacobians(world, st, vt, nodes, wrench_guesses=gd)
    (Ts, Tv, Tg), (Ws, Wv, Wg) = _autograd_blocks(lambda a, b, c: nb.multiple_contact_inverse_dynamics(world, a, b, nodes, wrench_guesses=c),
                                                  st, vt, gd)
    tol = 1e-10 if fp64 else 1e-4
    pairs = ((out[2], Ts[:, :, :n]), (out[3], Ts[:, :, n:]), (out[4], Tv), (out[5], Tg), (out[6], Ws[..., :n]), (out[7], Ws[..., n:]),
             (out[8], Wv), (out[9], Wg))
    for i, (got, ref) in enumerate(pairs):
        assert got.shape == ref.shape, (i, got.shape, ref.shape)
        assert rel_err(got.cpu().numpy(), ref.cpu().numpy()) < tol or (k == 1 and i in (3, 7) and not got.any() and not ref.any()), (
            i, rel_err(got.cpu().numpy(), ref.cpu().numpy()))


def _chain_dofs(raw, names):
    out = set()
    for name in names:
        i = _raw_index(raw, name)
        while raw.parent[i] >= 0:
            out |= set(range(raw.dof_off[i], raw.dof_off[i] + ms.JOINT_NDOF[int(raw.jtype[i])]))
            i = raw.parent[i]
    return out


@pytest.mark.parametrize("k", [1, 2, 4])
@pytest.mark.parametrize("fp64", [False, True])
def test_rows_off_the_chains_are_inverse_dynamics_rows_and_root_rows_are_zero(k, fp64):
    """Off the chains a row is the inverse-dynamics row: the same stage functions on the same seed, bit for bit on the host
    (tests/test_contact_inverse_dynamics_jacobians.py); the two kernels are compiled apart and the device rounds them apart (§6s).  With the
    feet and hands every dof below the root is on a chain."""
    raw, world = _world()
    n, B, dt = raw.ndof, 33, torch.float64 if fp64 else torch.float32
    s, vn = id_inputs(raw, B, seed=41 + k)
    st, vt = torch.tensor(s, dtype=dt, device=DEV), torch.tensor(vn, dtype=dt, device=DEV)
    out = nb.multiple_contact_inverse_dynamics_jacobians(world, st, vt, [_node(world, x) for x in NAMES[k]])
    ref = nb.inverse_dynamics_jacobians(world, st, vt)
    off = [d for d in range(6, n) if d not in _chain_dofs(raw, NAMES[k])]
    assert bool(off) == (k < 4)
    assert torch.equal(out[0][:, off], ref[0][:, off])
    tol = 1e-8 if fp64 else 1e-4  # the position block's cancelling terms, fused differently by the two kernels, as against the oracle
    for a, b in zip(out[2:5], ref[1:]):
        assert rel_err(a[:, off].cpu().numpy(), b[:, off].cpu().numpy()) < tol, rel_err(a[:, off].cpu().numpy(), b[:, off].cpu().numpy())
    for a in out[2:6]:
        assert not bool(a[:, :6].any())


def _origin_jacobians(world, raw, oracle_mod, st, names):
    """J_i [B, k, 6, n] of the bodies about the world origin: world_jacobian at the body origins p_i, the linear rows shifted by -omega x p_i
    with p_i from the fp64 step oracle."""
    n = raw.ndof
    J = nb.world_jacobian(world, st[:, :n], [_node(world, x) for x in names])
    ow = oracle_mod.OracleWorld(raw)
    s = st.cpu().numpy()
    p = torch.tensor(np.array([[ow.ik(s[b], [0], [_raw_index(raw, x)], want_jac=False)[0][3:6] for x in names] for b in range(len(s))]),
                     dtype=st.dtype, device=DEV)
    Jo = J.clone()
    Jo[:, :, 3:] = J[:, :, 3:] - torch.cross(J[:, :, :3], p[..., None].expand_as(J[:, :, :3]), dim=2)
    return Jo


@pytest.mark.parametrize("k", [2, 4])
def test_identities_of_the_definition(oracle_mod, k):
    raw, world = _world()
    n, B = raw.ndof, 5
    s, vn = id_inputs(raw, B, seed=51 + k)
    g = np.random.default_rng(52).normal(0, 40, (B, k, 6))
    st, vt, gd = (torch.tensor(a, dtype=torch.float64, device=DEV) for a in (s, vn, g))
    names = NAMES[k]
    tau, w, Tq, Tqd, Tn, Tg, Wq, Wqd, Wn, Wg = nb.multiple_contact_inverse_dynamics_jacobians(world, st, vt, [_node(world, x) for x in names],
                                                                                              wrench_guesses=gd)
    _, Iq, Iqd, In = nb.inverse_dynamics_jacobians(world, st, vt)
    Jo = _origin_jacobians(world, raw, oracle_mod, st, names)
    JT = lambda W: torch.einsum("bkcn,bkcj->bnj", Jo, W)  # sum_i J_i^T dW_i
    # tau + sum_i J_i^T w_i = tau_ID, J_i independent of qdot and next_vel
    for T, W, ref in ((Tqd, Wqd, Iqd), (Tn, Wn, In)):
        assert rel_err((T + JT(W)).cpu().numpy(), ref.cpu().numpy()) < 1e-9
    Mdt = nb.mass_matrix(world, st[:, :n]) / raw.dt
    assert rel_err((Tn + JT(Wn)).cpu().numpy(), Mdt.cpu().numpy()) < 1e-9
    # the wrenches sum to the one-body wrench
    one = nb.contact_inverse_dynamics_jacobians(world, st, vt, _node(world, names[0]))
    for W, ref in ((Wq, one[5]), (Wqd, one[6]), (Wn, one[7])):
        assert rel_err(W.sum(1).cpu().numpy(), ref.cpu().numpy()) < 1e-9
    # the guesses only move load between the bodies
    Wgs = Wg.reshape(B, k, 6, 6 * k)
    assert Wgs.sum(1).abs().max().item() < 1e-9 * Wgs.abs().max().item()
    assert rel_err(Tg.reshape(B, n, 6 * k).cpu().numpy(), (-torch.einsum("bkcn,bkcj->bnj", Jo, Wgs)).cpu().numpy()) < 1e-9
    # tau and w are affine in next_vel
    z = torch.zeros_like(vt)
    t0, w0 = nb.multiple_contact_inverse_dynamics(world, st, z, [_node(world, x) for x in names], wrench_guesses=gd)
    assert rel_err(tau.cpu().numpy(), (t0 + torch.einsum("bij,bj->bi", Tn, vt)).cpu().numpy()) < 1e-9
    assert rel_err(w.cpu().numpy(), (w0 + torch.einsum("bkcj,bj->bkc", Wn, vt)).cpu().numpy()) < 1e-9


@pytest.mark.parametrize("fp64", [False, True])
def test_one_body_through_the_multiple_contact_call_is_the_contact_call(fp64):
    raw, world = _world()
    n, B, dt = raw.ndof, 33, torch.float64 if fp64 else torch.float32
    s, vn = id_inputs(raw, B, seed=61)
    st, vt = torch.tensor(s, dtype=dt, device=DEV), torch.tensor(vn, dtype=dt, device=DEV)
    for name in ("l_foot", "r_hand", "pelvis"):
        one = nb.contact_inverse_dynamics_jacobians(world, st, vt, _node(world, name))
        multi = nb.multiple_contact_inverse_dynamics_jacobians(world, st, vt, [_node(world, name)], wrench_guesses=torch.ones(B, 1, 6, dtype=dt, device=DEV))
        assert [tuple(x.shape) for x in one] == [(B, n), (B, 6)] + [(B, n, n)] * 3 + [(B, 6, n)] * 3
        ct, cw = nb.contact_inverse_dynamics(world, st, vt, _node(world, name))
        assert torch.equal(one[0], ct) and torch.equal(one[1], cw)
        for a, b in zip(one, [multi[0], multi[1][:, 0]] + list(multi[2:5]) + [x[:, 0] for x in multi[6:9]]):
            assert torch.equal(a, b), name
        assert not bool(multi[5].any()) and not bool(multi[9].any())


def test_per_world_mass_is_set_masses_per_world():
    raw, world = _world()
    n, B, k = raw.ndof, 5, 4
    M = torch.tensor(random_masses(world, B, seed=71), dtype=torch.float64, device=DEV)
    s, vn = id_inputs(raw, B, seed=72)
    g = np.random.default_rng(73).normal(0, 40, (B, k, 6))
    st, vt, gd = (torch.tensor(a, dtype=torch.float64, device=DEV) for a in (s, vn, g))
    nodes = [_node(world, x) for x in NAMES[k]]
    pw = nb.multiple_contact_inverse_dynamics_jacobians(world, st, vt, nodes, M, gd)
    p1 = nb.contact_inverse_dynamics_jacobians(world, st, vt, nodes[0], M)
    for w in range(B):
        r = nb.multiple_contact_inverse_dynamics_jacobians(world, st[w:w + 1], vt[w:w + 1], nodes, M[w], gd[w:w + 1])
        r1 = nb.contact_inverse_dynamics_jacobians(world, st[w:w + 1], vt[w:w + 1], nodes[0], M[w])
        for a, b in zip(pw + p1, r + r1):
            assert rel_err(a[w].cpu().numpy(), b[0].cpu().numpy()) < 1e-12, w
    # and the layer's own per-world outputs
    lt, lw = nb.multiple_contact_inverse_dynamics(world, st, vt, nodes, M, gd)
    assert torch.equal(pw[0], lt) and torch.equal(pw[1], lw)


@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("B", [1, 33, 4099])
def test_kernel_writes_only_its_own_rows(fp64, B):
    """Every output sits inside a buffer with guard bands on both sides: the bands keep their bits, with and without per-world inertia and
    guesses, with one body and four."""
    raw, world = _world()
    dm = nb.device_model_for(world)
    dt = torch.float64 if fp64 else torch.float32
    prec = nb.engine.FP64 if fp64 else nb.engine.FP32
    n, G = raw.ndof, 4096
    s, vn = id_inputs(raw, B, seed=81)
    st, vt = torch.tensor(s, dtype=dt, device=DEV), torch.tensor(vn, dtype=dt, device=DEV)
    wi = nb.mass_to_inertia(world, torch.tensor(random_masses(world, B, seed=82), dtype=torch.float64, device=DEV))
    wi = wi.reshape(B, -1).t().contiguous()
    cm = dm.cm

    def guarded(numel):
        buf = torch.full((numel + 2 * G,), 12345.0, dtype=dt, device=DEV)
        return buf, buf[G:G + numel]

    stream = torch.cuda.current_stream().cuda_stream
    for k in (1, 4):
        raws = [_raw_index(raw, x) for x in NAMES[k]]
        bodies, points = [int(cm.body_owner[r]) for r in raws], [cm.body_T[r][:3, 3] for r in raws]
        m = 6 * k
        gd = torch.tensor(np.random.default_rng(83).normal(0, 40, (B, k, 6)), dtype=dt, device=DEV)
        for w, g in ((None, None), (wi, gd)):
            bufs = [guarded(B * n), guarded(B * m)] + [guarded(B * n * n) for _ in range(3)] + [guarded(B * n * m)] + [
                guarded(B * m * n) for _ in range(3)] + [guarded(B * m * m)]
            o = [x.data_ptr() for _, x in bufs]
            dm.multiple_contact_inverse_dynamics_jacobians_device(B, bodies, points, st.data_ptr(), vt.data_ptr(), None if g is None else g.data_ptr(),
                                                                  o[0], o[1], o[2:], stream, prec, wi_ptr=None if w is None else w.data_ptr())
            torch.cuda.synchronize()
            for i, (buf, out) in enumerate(bufs):
                assert bool((buf[:G] == 12345.0).all()) and bool((buf[-G:] == 12345.0).all()), (k, i)
                assert bool(torch.isfinite(out).all()) and not bool((out == 12345.0).any()), (k, i)


def test_empty_batch_and_single_row():
    raw, world = _world()
    n, B = raw.ndof, 16
    s, vn = id_inputs(raw, B, seed=91)
    st, vt = torch.tensor(s, dtype=torch.float64, device=DEV), torch.tensor(vn, dtype=torch.float64, device=DEV)
    nodes = [_node(world, x) for x in NAMES[2]]
    g = torch.tensor(np.random.default_rng(92).normal(0, 40, (B, 2, 6)), device=DEV)
    full = nb.multiple_contact_inverse_dynamics_jacobians(world, st, vt, nodes, wrench_guesses=g)
    one = nb.multiple_contact_inverse_dynamics_jacobians(world, st[3], vt[3], nodes, wrench_guesses=g[3])
    assert [tuple(x.shape) for x in one] == [(n,), (2, 6), (n, n), (n, n), (n, n), (n, 2, 6), (2, 6, n), (2, 6, n), (2, 6, n), (2, 6, 2, 6)]
    for a, b in zip(one, full):
        assert torch.equal(a, b[3])
    c1 = nb.contact_inverse_dynamics_jacobians(world, st[3], vt[3], nodes[0])
    assert [tuple(x.shape) for x in c1] == [(n,), (6,), (n, n), (n, n), (n, n), (6, n), (6, n), (6, n)]
    empty = nb.multiple_contact_inverse_dynamics_jacobians(world, torch.zeros(0, 2 * n, device=DEV), torch.zeros(0, n, device=DEV), nodes)
    assert [tuple(x.shape) for x in empty] == [(0, n), (0, 2, 6), (0, n, n), (0, n, n), (0, n, n), (0, n, 2, 6), (0, 2, 6, n), (0, 2, 6, n),
                                               (0, 2, 6, n), (0, 2, 6, 2, 6)]
    assert all(x.dtype == torch.float32 for x in empty)
    e1 = nb.contact_inverse_dynamics_jacobians(world, torch.zeros(0, 2 * n, device=DEV), torch.zeros(0, n, device=DEV), nodes[0])
    assert [tuple(x.shape) for x in e1] == [(0, n), (0, 6)] + [(0, n, n)] * 3 + [(0, 6, n)] * 3
    assert not any(x.requires_grad for x in nb.multiple_contact_inverse_dynamics_jacobians(world, st.clone().requires_grad_(True), vt, nodes))
