"""Dense Jacobians of contact-free inverse and forward dynamics on the GPU (nb2_inverse_dynamics_jacobians / nb2_forward_dynamics_jacobians
through nimblephysics_b200.inverse_dynamics_jacobians / forward_dynamics_jacobians): against the dual-number oracle at partial-block batch
sizes, against autograd's Jacobian of inverse_dynamics / forward_dynamics, against mass_matrix / inverse_mass_matrix, against central
differences along random directions, guard bands, the untouched LCP cache, per-world masses, B = 0 and the 1-D state."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from tests.oracle_id.binding import IdOracle
from tests.test_dynamics_jacobians import fd_tol, oracle_fd_blocks, oracle_id_blocks
from tests.test_forward_dynamics import fd_inputs
from tests.test_gpu_forward_dynamics import _check_worlds, _world
from tests.test_inverse_dynamics import id_inputs
from tests.test_mass_matrix import MODELS, model_raw
from tests.test_per_world_mass import random_masses, register
from tests.util import contact_inputs, load_raw, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _check_against_oracle(raw, world, B, fp64, worlds):
    n = raw.ndof
    dt = torch.float64 if fp64 else torch.float32
    s, vn = id_inputs(raw, B, seed=B + 1)
    _, tau = fd_inputs(raw, B, seed=B + 2)
    st = torch.tensor(s, dtype=dt, device=DEV)
    gid = nb.inverse_dynamics_jacobians(world, st, torch.tensor(vn, dtype=dt, device=DEV))
    gfd = nb.forward_dynamics_jacobians(world, st, torch.tensor(tau, dtype=dt, device=DEV))
    for r in gid + gfd:
        assert r.dtype == dt and r.shape[0] == B and r.shape[-1] == n
    gid = [r.cpu().numpy() for r in gid]
    gfd = [r.cpu().numpy() for r in gfd]
    ow = IdOracle(raw)
    # the position blocks (k = 1) sum rotation-derivative terms of the size of |M a + C| that cancel to a smaller block, and the device's
    # fused multiply-adds round those terms differently from the host: on Atlas in fp64 they land up to 3.4e-9 (ID) and, after the solve
    # with M, 2.9e-8 (FD) from the oracle.  The blocks' definition, autograd through the layers, is checked at 1e-10 below.
    pos = lambda k, tol: max(tol, 1e-7) if fp64 and k == 1 else tol
    for w in worlds:
        for k, ref in enumerate(oracle_id_blocks(ow, n, s[w], vn[w])):
            assert rel_err(gid[k][w], ref) < pos(k, 1e-9 if fp64 else 1e-4), (w, k, rel_err(gid[k][w], ref))
        tol = fd_tol(ow, n, s[w], fp64)
        for k, ref in enumerate(oracle_fd_blocks(ow, n, raw.dt, s[w], tau[w])):
            assert rel_err(gfd[k][w], ref) < pos(k, tol), (w, k, rel_err(gfd[k][w], ref))


@pytest.mark.parametrize("name", ["atlas", "atlas_sdf"])
@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("B", [1, 3, 33, 4099])
def test_atlas_matches_oracle(name, fp64, B):
    _check_against_oracle(load_raw(name), _world(name), B, fp64, _check_worlds(B))


@pytest.mark.parametrize("name", [m for m in MODELS if m not in ("atlas", "atlas_sdf")])
@pytest.mark.parametrize("fp64", [False, True])
def test_other_models_match_oracle(name, fp64):
    """fp64 on every model (the 64-body chain included: the Jacobians do not inherit forward_dynamics's shared-memory refusal), fp32 on
    half_cheetah and limit."""
    if not fp64 and name not in ("half_cheetah", "limit"):
        pytest.skip("fp32 is checked on half_cheetah and limit")
    _check_against_oracle(model_raw(name), _world(name), 5, fp64, range(5))


def _autograd_blocks(f, world, st, x):
    """Per-world diagonal blocks of torch.autograd.functional.jacobian of f(world, state, x): (d/dstate [B, n, 2n], d/dx [B, n, n])."""
    Js, Jx = torch.autograd.functional.jacobian(lambda a, b: f(world, a, b), (st, x))
    idx = torch.arange(st.shape[0], device=st.device)
    return Js[idx, :, idx], Jx[idx, :, idx]


@pytest.mark.parametrize("name", [m for m in MODELS if m != "chain64"] + ["chain64_fp32"])
def test_blocks_equal_autograd_of_the_layers(name):
    """autograd's Jacobian runs the layers' VJP once per output row; forward_dynamics refuses the 64-body chain in fp64 (no step schedule
    fits shared memory), so that model is compared in fp32 only (its fp64 blocks are checked against the oracle above)."""
    fp64 = not name.endswith("_fp32")
    name = name.replace("_fp32", "")
    raw, world = model_raw(name), _world(name)
    n, B = raw.ndof, 3
    dt = torch.float64 if fp64 else torch.float32
    s, vn = id_inputs(raw, B, seed=61)
    _, tau = fd_inputs(raw, B, seed=62)
    st, vt, tt = (torch.tensor(a, dtype=dt, device=DEV) for a in (s, vn, tau))
    tol = 1e-10 if fp64 else 1e-4
    for f, fj, x in ((nb.inverse_dynamics, nb.inverse_dynamics_jacobians, vt), (nb.forward_dynamics, nb.forward_dynamics_jacobians, tt)):
        out, J1, J2, J3 = fj(world, st, x)
        Js, Jx = _autograd_blocks(f, world, st, x)
        assert rel_err(out.cpu().numpy(), f(world, st, x).cpu().numpy()) < tol
        for got, ref in ((J1, Js[:, :, :n]), (J2, Js[:, :, n:]), (J3, Jx)):
            assert rel_err(got.cpu().numpy(), ref.cpu().numpy()) < tol, (f.__name__, rel_err(got.cpu().numpy(), ref.cpu().numpy()))


@pytest.mark.parametrize("name", ["cartpole", "half_cheetah", "atlas", "free16", "chain64"])
def test_force_and_velocity_blocks_are_the_mass_matrix_and_its_inverse(name):
    raw, world = model_raw(name), _world(name)
    n, B = raw.ndof, 33
    s, vn = id_inputs(raw, B, seed=63)
    _, tau = fd_inputs(raw, B, seed=64)
    st = torch.tensor(s, dtype=torch.float64, device=DEV)
    Jn = nb.inverse_dynamics_jacobians(world, st, torch.tensor(vn, dtype=torch.float64, device=DEV))[3]
    Jt = nb.forward_dynamics_jacobians(world, st, torch.tensor(tau, dtype=torch.float64, device=DEV))[3]
    assert rel_err(Jn.cpu().numpy(), (nb.mass_matrix(world, st[:, :n]) / raw.dt).cpu().numpy()) < 1e-12
    assert rel_err(Jt.cpu().numpy(), nb.inverse_mass_matrix(world, st[:, :n]).cpu().numpy()) < 1e-9


@pytest.mark.parametrize("name", ["half_cheetah", "atlas", "free_child"])
def test_linearisation_matches_central_differences(name):
    raw, world = model_raw(name), _world(name)
    n, B, h = raw.ndof, 4, 1e-6
    s, vn = id_inputs(raw, B, seed=65)
    _, tau = fd_inputs(raw, B, seed=66)
    st, vt, tt = (torch.tensor(a, dtype=torch.float64, device=DEV) for a in (s, vn, tau))
    rng = np.random.default_rng(67)
    ds = torch.tensor(rng.normal(size=(B, 2 * n)), device=DEV)
    dx = torch.tensor(rng.normal(size=(B, n)), device=DEV)
    for f, fj, x in ((nb.inverse_dynamics, nb.inverse_dynamics_jacobians, vt), (nb.forward_dynamics, nb.forward_dynamics_jacobians, tt)):
        _, J1, J2, J3 = fj(world, st, x)
        lin = (torch.einsum("bij,bj->bi", J1, ds[:, :n]) + torch.einsum("bij,bj->bi", J2, ds[:, n:]) + torch.einsum("bij,bj->bi", J3, dx))
        cd = (f(world, st + h * ds, x + h * dx) - f(world, st - h * ds, x - h * dx)) / (2 * h)
        # the outputs reach 1e4 here: a central difference with h = 1e-6 carries about 1e-16 * 1e4 / 1e-6 = 1e-6 of rounding
        assert rel_err(lin.cpu().numpy(), cd.cpu().numpy()) < 1e-6, (f.__name__, rel_err(lin.cpu().numpy(), cd.cpu().numpy()))


def test_per_world_mass_is_set_masses_per_world():
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=3)
    world._contacts_disabled = True
    n, B = raw.ndof, 5
    M = torch.tensor(random_masses(world, B, seed=68), dtype=torch.float64, device=DEV)
    s, vn = id_inputs(raw, B, seed=69)
    _, tau = fd_inputs(raw, B, seed=70)
    st, vt, tt = (torch.tensor(a, dtype=torch.float64, device=DEV) for a in (s, vn, tau))
    pid = nb.inverse_dynamics_jacobians(world, st, vt, M)
    pfd = nb.forward_dynamics_jacobians(world, st, tt, M)
    for w in range(B):
        rid = nb.inverse_dynamics_jacobians(world, st[w:w + 1], vt[w:w + 1], M[w])
        rfd = nb.forward_dynamics_jacobians(world, st[w:w + 1], tt[w:w + 1], M[w])
        for a, b in zip(pid + pfd, rid + rfd):
            assert rel_err(a[w].cpu().numpy(), b[0].cpu().numpy()) < 1e-12, w


@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("B", [1, 33, 4099])
def test_kernels_write_only_their_own_rows(fp64, B):
    """Every output sits inside a buffer with guard bands on both sides: the bands keep their bits, with and without per-world inertia."""
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=3)
    world._contacts_disabled = True
    dm = nb.device_model_for(world)
    dt = torch.float64 if fp64 else torch.float32
    prec = nb.engine.FP64 if fp64 else nb.engine.FP32
    n, G = raw.ndof, 4096
    s, vn = id_inputs(raw, B, seed=71)
    st, vt = torch.tensor(s, dtype=dt, device=DEV), torch.tensor(vn, dtype=dt, device=DEV)
    wi = nb.mass_to_inertia(world, torch.tensor(random_masses(world, B, seed=72), dtype=torch.float64, device=DEV))
    wi = wi.reshape(B, -1).t().contiguous()

    def guarded(numel):
        buf = torch.full((numel + 2 * G,), 12345.0, dtype=dt, device=DEV)
        return buf, buf[G:G + numel]

    stream = torch.cuda.current_stream().cuda_stream
    for w in (None, wi):
        for run in (dm.inverse_dynamics_jacobians_device, dm.forward_dynamics_jacobians_device):
            bufs = [guarded(B * n)] + [guarded(B * n * n) for _ in range(3)]
            run(B, st.data_ptr(), vt.data_ptr(), *(o.data_ptr() for _, o in bufs), stream, prec, wi_ptr=None if w is None else w.data_ptr())
            torch.cuda.synchronize()
            for buf, out in bufs:
                assert bool((buf[:G] == 12345.0).all()) and bool((buf[-G:] == 12345.0).all())
                assert bool(torch.isfinite(out).all()) and not bool((out == 12345.0).any())


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
    x = torch.tensor(np.random.default_rng(1).uniform(-20, 20, (B, n)), device=DEV)
    full = [fn(world, st, x) for fn in (nb.inverse_dynamics_jacobians, nb.forward_dynamics_jacobians)]
    assert world._lcp_cache is cache and all(torch.equal(before[k], cache[k]) for k in before)
    for fn, ref in zip((nb.inverse_dynamics_jacobians, nb.forward_dynamics_jacobians), full):
        one = fn(world, st[3], x[3])
        assert [tuple(r.shape) for r in one] == [(n,), (n, n), (n, n), (n, n)]
        for a, b in zip(one, ref):
            assert torch.equal(a, b[3])
        empty = fn(world, torch.zeros(0, 2 * n, device=DEV), torch.zeros(0, n, device=DEV))
        assert [tuple(r.shape) for r in empty] == [(0, n), (0, n, n), (0, n, n), (0, n, n)]
        assert all(r.dtype == torch.float32 for r in empty)
        assert not any(r.requires_grad for r in fn(world, st.clone().requires_grad_(True), x))
