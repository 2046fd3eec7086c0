"""The inverse-dynamics and energy regressors on the GPU (nb2_inverse_dynamics_regressor / nb2_energy_regressor through
nimblephysics_b200.inverse_dynamics_regressor / energy_regressor): against the host emulation at partial-block batch sizes, against
inverse_dynamics with a per-world inertia table and energy_and_momentum through their defining identities, against autograd's Jacobian of
InverseDynamicsLayer with respect to that table; guard bands, the untouched LCP cache, B = 0 and the 1-D state; and the recovery of
per-world inertia tables and masses by least squares on data generated with forward_dynamics."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from nimblephysics_b200 import modelspec as ms
from nimblephysics_b200.inverse_dynamics import ForwardDynamicsLayer, InverseDynamicsLayer
from tests.host_emul.binding_reg import EmulRegWorld
from tests.test_energy import skeleton_of
from tests.test_gpu_forward_dynamics import _check_worlds, _world
from tests.test_inverse_dynamics import id_inputs
from tests.test_mass_matrix import MODELS, model_raw
from tests.test_per_world_mass import random_masses, register
from tests.test_world_jacobian import canon_root, com_body
from tests.util import contact_inputs, load_raw, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _tables(world, B, seed):
    """per-world canonical inertia tables [B, nb, 10] (fp64, on the device) from random masses of a registered copy of `world`"""
    reg = register(nb.World.from_raw(nb.flatten_world(world)), step=2)
    return nb.mass_to_inertia(reg, torch.tensor(random_masses(reg, B, seed=seed), dtype=torch.float64, device=DEV))


def _check(name, raw, world, B, fp64, worlds):
    n = raw.ndof
    dt = torch.float64 if fp64 else torch.float32
    s, vn = id_inputs(raw, B, seed=B + 81)
    st, vt = torch.tensor(s, dtype=dt, device=DEV), torch.tensor(vn, dtype=dt, device=DEV)
    Y, tp = nb.inverse_dynamics_regressor(world, st, vt)
    YT, YU, Us = nb.energy_regressor(world, st)
    cm = nb.device_model_for(world).cm
    assert Y.dtype == tp.dtype == YT.dtype == YU.dtype == Us.dtype == dt
    assert tuple(Y.shape) == (B, n, cm.nb, 10) and tuple(tp.shape) == (B, n) and tuple(YT.shape) == tuple(YU.shape) == (B, cm.nb, 10)
    tol = 1e-12 if fp64 else 1e-5
    # the host emulation, world by world
    ew = EmulRegWorld(nb.compile_model(raw, lanes=1))
    eY, etp = ew.id_regressor(s[worlds], vn[worlds], fp64)
    eT, eU, eS = ew.energy_regressor(s[worlds], fp64)
    for k, w in enumerate(worlds):
        for got, ref in ((Y[w], eY[k]), (tp[w], etp[k]), (YT[w], eT[k]), (YU[w], eU[k])):
            assert rel_err(got.cpu().numpy(), ref) < tol, (w, rel_err(got.cpu().numpy(), ref))
        assert abs(float(Us[w]) - float(eS[k])) <= tol * max(1.0, abs(float(eS[k])))
    # the definition: inverse_dynamics at the model's table and at per-world tables (the device ID rounds in another order: 1e-11 in fp64).
    # No step schedule of the 64-body chain fits shared memory in fp64, so inverse_dynamics runs it in fp32 only: compared there at 3e-5.
    own = torch.tensor(cm.inertia, device=DEV).expand(B, cm.nb, 10).contiguous()
    id64 = fp64 and name != "chain64"
    si, vi = (st.float(), vt.float()) if fp64 and not id64 else (st, vt)
    for pi in (own, _tables(world, B, seed=B + 82)):
        tau = InverseDynamicsLayer.apply(world, si, vi, None, pi).double()
        got = torch.einsum("bdjk,bjk->bd", Y.double(), pi) + tp.double()
        err = ((got - tau).norm(dim=1) / tau.norm(dim=1).clamp_min(1e-30)).max().item()
        assert err < (1e-11 if id64 else 3e-5), err
    # energy_and_momentum of the largest skeleton with a moving root: its columns, its springs
    rb = com_body(raw, cm)
    if rb is None:
        return
    sk = world.skeletons[int(raw.skel_id[rb])]
    T, U, _ = nb.energy_and_momentum(world, st, sk)
    root = canon_root(cm, rb)
    cols = torch.tensor([canon_root(cm, int(cm.orig_body[j])) == root for j in range(cm.nb)], device=DEV)
    _, dofs = skeleton_of(raw, rb)
    pi = own * cols[None, :, None]
    sd = st.double()
    spring = 0.5 * (torch.tensor(raw.spring[dofs], device=DEV) * (sd[:, dofs] - torch.tensor(raw.rest[dofs], device=DEV)) ** 2).sum(1)
    Tg = torch.einsum("bjk,bjk->b", YT.double(), pi)
    Ug = torch.einsum("bjk,bjk->b", YU.double(), pi) + spring
    scale = torch.maximum(T.double().abs(), U.double().abs()).clamp_min(1.0)
    etol = 1e-11 if fp64 else 1e-5
    assert ((Tg - T.double()).abs() / scale).max().item() < etol
    assert ((Ug - U.double()).abs() / scale).max().item() < etol


@pytest.mark.parametrize("name", ["atlas", "atlas_sdf"])
@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("B", [1, 3, 33, 4099])
def test_atlas(name, fp64, B):
    _check(name, load_raw(name), _world(name), B, fp64, _check_worlds(B))


@pytest.mark.parametrize("name", [m for m in MODELS if m not in ("atlas", "atlas_sdf")])
def test_other_models_fp64(name):
    _check(name, model_raw(name), _world(name), 5, True, list(range(5)))


@pytest.mark.parametrize("name", ["cartpole", "tree", "half_cheetah", "atlas", "free_child", "free16"])
def test_regressor_is_autograds_jacobian_of_the_layer(name):
    raw, world = model_raw(name), _world(name)
    B = 2
    s, vn = id_inputs(raw, B, seed=83)
    st, vt = torch.tensor(s, dtype=torch.float64, device=DEV), torch.tensor(vn, dtype=torch.float64, device=DEV)
    pi = _tables(world, B, seed=84)
    J = torch.autograd.functional.jacobian(lambda p: InverseDynamicsLayer.apply(world, st, vt, None, p), pi)  # [B, n, B, nb, 10]
    idx = torch.arange(B, device=DEV)
    J = J[idx, :, idx]
    Y, _ = nb.inverse_dynamics_regressor(world, st, vt)
    assert rel_err(Y.cpu().numpy(), J.cpu().numpy()) < 1e-10, rel_err(Y.cpu().numpy(), J.cpu().numpy())


@pytest.mark.parametrize("name", ["atlas", "half_cheetah_contact"])
@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("B", [1, 33, 4099])
def test_kernels_write_only_their_own_rows(name, fp64, B):
    """Every output sits inside a NaN-filled buffer with guard bands on both sides: the bands stay NaN and every output word is written.
    half_cheetah_contact: the half-cheetah with its ground contacts enabled (a model whose device schedules carry contact data)."""
    raw = load_raw(name.replace("_contact", ""))
    world = nb.World.from_raw(raw) if name.endswith("_contact") else _world(name)
    dm = nb.device_model_for(world)
    dt = torch.float64 if fp64 else torch.float32
    prec = nb.engine.FP64 if fp64 else nb.engine.FP32
    n, nb_, G = raw.ndof, dm.cm.nb, 4096
    s, vn = id_inputs(raw, B, seed=85)
    st, vt = torch.tensor(s, dtype=dt, device=DEV), torch.tensor(vn, dtype=dt, device=DEV)

    def guarded(numel):
        buf = torch.full((numel + 2 * G,), float("nan"), dtype=dt, device=DEV)
        return buf, buf[G:G + numel]

    stream = torch.cuda.current_stream().cuda_stream
    bufs = [guarded(B * n * nb_ * 10), guarded(B * n)]
    dm.inverse_dynamics_regressor_device(B, st.data_ptr(), vt.data_ptr(), *(o.data_ptr() for _, o in bufs), stream, prec)
    ebufs = [guarded(B * nb_ * 10), guarded(B * nb_ * 10), guarded(B)]
    dm.energy_regressor_device(B, st.data_ptr(), *(o.data_ptr() for _, o in ebufs), stream, prec)
    torch.cuda.synchronize()
    for buf, out in bufs + ebufs:
        assert bool(buf[:G].isnan().all()) and bool(buf[-G:].isnan().all())
        assert bool(torch.isfinite(out).all())


def test_contact_world_cache_empty_batch_and_single_row():
    raw = load_raw("half_cheetah")
    world = nb.World.from_raw(raw)
    assert nb.device_model_for(world).has_contacts
    n, B = raw.ndof, 16
    cs, ca = contact_inputs(raw, "half_cheetah", B, seed=5)
    nb.reset_contact_cache(world)
    nb.timestep(world, torch.tensor(cs, device=DEV), torch.tensor(ca, device=DEV))
    cache = nb.contact_cache(world, B, DEV)
    before = {k: v.clone() for k, v in cache.items() if torch.is_tensor(v)}
    st = torch.tensor(cs, device=DEV, dtype=torch.float64)
    vt = torch.tensor(np.random.default_rng(1).uniform(-1, 1, (B, n)), device=DEV)
    full_id = nb.inverse_dynamics_regressor(world, st, vt)
    full_e = nb.energy_regressor(world, st)
    # bit for bit: the workspace `ws` is uninitialised memory and may hold NaN patterns, which torch.equal never calls equal
    bits = lambda t: t.view({8: torch.int64, 4: torch.int32, 2: torch.int16, 1: torch.uint8}[t.element_size()])
    assert world._lcp_cache is cache and all(torch.equal(bits(before[k]), bits(cache[k])) for k in before)
    nbod = nb.device_model_for(world).cm.nb
    one_id, one_e = nb.inverse_dynamics_regressor(world, st[3], vt[3]), nb.energy_regressor(world, st[3])
    assert [tuple(r.shape) for r in one_id] == [(n, nbod, 10), (n,)] and [tuple(r.shape) for r in one_e] == [(nbod, 10), (nbod, 10), ()]
    for a, b in zip(one_id + one_e, full_id + full_e):
        assert torch.equal(a, b[3])
    e_id = nb.inverse_dynamics_regressor(world, torch.zeros(0, 2 * n, device=DEV), torch.zeros(0, n, device=DEV))
    e_e = nb.energy_regressor(world, torch.zeros(0, 2 * n, device=DEV))
    assert [tuple(r.shape) for r in e_id] == [(0, n, nbod, 10), (0, n)] and [tuple(r.shape) for r in e_e] == [(0, nbod, 10), (0, nbod, 10), (0,)]
    assert all(r.dtype == torch.float32 for r in e_id + e_e)
    sg = st.clone().requires_grad_(True)
    assert not any(r.requires_grad for r in nb.inverse_dynamics_regressor(world, sg, vt) + nb.energy_regressor(world, sg))


@pytest.mark.parametrize("name", ["cartpole", "half_cheetah"])
def test_least_squares_recovers_tables_and_masses(name):
    """fp64 data at per-world true tables: random states and torques, v' = qdot + dt qdd with qdd from forward_dynamics at that table.
    Least squares on the stacked rows predicts held-out torques of the true table; restricted to a mass vector of INERTIA_MASS entries
    (the table is affine in it) it returns the true masses."""
    raw = load_raw(name)
    world = nb.World.from_raw(raw)
    world._contacts_disabled = True
    owner = nb.compile_model(raw).body_owner
    for k, b in enumerate(b for sk in world.skeletons for b in sk._ordered_bodies()):
        if owner[k] >= 0:  # bodies that move (a body welded to the world has no regressor columns)
            world.tuneMass(b, ms.INERTIA_MASS)
    W, K, H, n = 4, 40, 10, raw.ndof  # worlds, fitting samples and held-out samples per world
    m0 = torch.tensor(world.getMasses(), dtype=torch.float64, device=DEV)
    m_true = m0 * torch.tensor(np.random.default_rng(86).uniform(0.6, 1.6, (W, m0.numel())), device=DEV)
    pi_true = nb.mass_to_inertia(world, m_true)                                 # [W, nb, 10]
    rng = np.random.default_rng(87)
    s = torch.tensor(np.concatenate([rng.uniform(-0.5, 0.5, (W * (K + H), n)), rng.uniform(-2, 2, (W * (K + H), n))], 1), device=DEV)
    tau = torch.tensor(rng.uniform(-5, 5, (W * (K + H), n)), device=DEV)
    pi_rows = pi_true.repeat_interleave(K + H, 0)
    qdd = ForwardDynamicsLayer.apply(world, s, tau, None, pi_rows)
    Y, tp = nb.inverse_dynamics_regressor(world, s, s[:, n:] + raw.dt * qdd)
    P = nb.device_model_for(world).cm.nb * 10
    A = Y.reshape(W, K + H, n, P)
    b = (tau - tp).reshape(W, K + H, n)
    Af, bf = A[:, :K].reshape(W, K * n, P), b[:, :K].reshape(W, K * n)
    pi_hat = torch.linalg.lstsq(Af.cpu(), bf.cpu().unsqueeze(-1), driver="gelsd").solution.squeeze(-1).to(DEV)
    Ah = A[:, K:].reshape(W, H * n, P)
    ref = torch.einsum("wrp,wp->wr", Ah, pi_true.reshape(W, P))
    assert ((torch.einsum("wrp,wp->wr", Ah, pi_hat) - ref).norm(dim=1) / ref.norm(dim=1)).max().item() < 1e-9
    # the mass vector: table = base + Pm^T m, Pm = d table / d mass (constant for INERTIA_MASS entries)
    Pm = torch.tensor(ms.inertia_param_jacobian(nb.flatten_world(world), nb.device_model_for(world).cm, world._mass_entries()), device=DEV)
    base = nb.mass_to_inertia(world, m0[None]).reshape(P) - Pm.t() @ m0
    Am = Af @ Pm.t()
    bm = bf - torch.einsum("wrp,p->wr", Af, base)
    m_hat = torch.linalg.lstsq(Am.cpu(), bm.cpu().unsqueeze(-1)).solution.squeeze(-1).to(DEV)
    assert ((m_hat - m_true).abs() / m_true.abs()).max().item() < 1e-8, (m_hat, m_true)
