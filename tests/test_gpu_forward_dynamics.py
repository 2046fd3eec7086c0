"""Contact-free forward dynamics on the GPU (nb2_forward_dynamics_batch / _backward through nimblephysics_b200.forward_dynamics) against
the fp64 step oracle's accelerations at partial-group batch sizes; gradcheck of every input; the backward identity against the
inverse-dynamics backward; consistency with inverse_mass_matrix, inverse_dynamics, timestep, the legacy nb2_forward_dynamics and the COM
Jacobians; a world with collision pairs, B = 0, a single row and a reduced action space."""
import copy

import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from oracle.binding import OracleWorld
from tests.test_forward_dynamics import fd_inputs, oracle_qdd, per_dof
from tests.test_mass_matrix import MODELS, built_world, model_raw
from tests.test_oracle import _tree_world
from tests.test_per_world_mass import random_masses, register
from tests.util import contact_inputs, load_raw, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _world(name):
    if name == "tree":
        return _tree_world()
    if name in ("chain64", "free16", "limit", "free_child"):
        return built_world(name)
    w = nb.World.from_raw(load_raw(name))
    w._contacts_disabled = True
    return w


def _check_worlds(B):
    return sorted({0, 1 % B, B // 2, B - 1})


@pytest.mark.parametrize("name", ["atlas", "atlas_sdf"])
@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("B", [1, 3, 33, 4099])
def test_atlas_matches_oracle(name, fp64, B):
    raw = load_raw(name)
    world = _world(name)
    dt = torch.float64 if fp64 else torch.float32
    s, tau = fd_inputs(raw, B, seed=B)
    qdd = nb.forward_dynamics(world, torch.tensor(s, dtype=dt, device=DEV), torch.tensor(tau, dtype=dt, device=DEV))
    assert qdd.shape == (B, raw.ndof) and qdd.dtype == dt
    qdd = qdd.cpu().numpy()
    ow = OracleWorld(per_dof(raw))
    for w in _check_worlds(B):
        assert rel_err(qdd[w], oracle_qdd(ow, s[w], tau[w])) < (1e-9 if fp64 else 1e-4), w


# chain64 has only the one-lane schedule (more lanes do not shorten a chain), whose fp64 working set of one warp (32 worlds) exceeds the
# 227 KB of shared memory of the step's launch family: it runs in fp32 here (the host emulation checks it in fp64, and the legacy entry's
# global-memory path below runs it in fp64)
@pytest.mark.parametrize("name", [m for m in MODELS if m not in ("atlas", "atlas_sdf")])
def test_other_models_match_oracle(name):
    raw = model_raw(name)
    world = _world(name)
    fp64 = name != "chain64"
    dt = torch.float64 if fp64 else torch.float32
    s, tau = fd_inputs(raw, 5, seed=7)
    qdd = nb.forward_dynamics(world, torch.tensor(s, dtype=dt, device=DEV), torch.tensor(tau, dtype=dt, device=DEV))
    ow = OracleWorld(per_dof(raw))
    for w in range(5):
        assert rel_err(qdd[w].cpu().numpy(), oracle_qdd(ow, s[w], tau[w])) < (1e-9 if fp64 else 1e-4), w


def test_legacy_entry_runs_a_model_outside_the_shared_memory_envelope():
    """The 64-body chain in fp64 fits no schedule's shared memory: nb2_forward_dynamics_batch refuses it (NB2_ERR_UNSUPPORTED, as the fp64
    step does), while the legacy pointer-style entry keeps accepting it through its global-memory path."""
    raw = model_raw("chain64")
    world = _world("chain64")
    dm = nb.device_model_for(world)
    n, B = raw.ndof, 67
    s, tau = fd_inputs(raw, B, seed=15)
    st, tt = torch.tensor(s, dtype=torch.float64, device=DEV), torch.tensor(tau, dtype=torch.float64, device=DEV)
    with pytest.raises(nb.engine._cabi.Nb2Error, match="shared memory"):
        nb.forward_dynamics(world, st, tt)
    acc = dm.forward_dynamics(st[:, :n], st[:, n:], tt).cpu().numpy()
    ow = OracleWorld(per_dof(raw))
    for w in (0, 1, 33, B - 1):
        assert rel_err(acc[w], oracle_qdd(ow, s[w], tau[w])) < 1e-9, w
    # the same accelerations as the fp32 batch path, to its precision
    a32 = nb.forward_dynamics(world, st.float(), tt.float()).double().cpu().numpy()
    assert rel_err(a32, acc) < 1e-4


def test_gradcheck_state_tau_mass_and_world_inertia():
    raw = load_raw("half_cheetah")
    world = register(nb.World.from_raw(raw), step=3)
    world._contacts_disabled = True
    B = 3
    s, tau = fd_inputs(raw, B, seed=2)
    st = torch.tensor(s, dtype=torch.float64, device=DEV, requires_grad=True)
    tt = torch.tensor(tau, dtype=torch.float64, device=DEV, requires_grad=True)
    mass = torch.tensor(random_masses(world, B, seed=3), dtype=torch.float64, device=DEV, requires_grad=True)
    # the accelerations reach 1e4 here: a central difference with eps = 1e-6 carries about 1e-16 * 1e4 / 1e-6 = 1e-6 of rounding
    assert torch.autograd.gradcheck(lambda a, b, m: nb.forward_dynamics(world, a, b, m), (st, tt, mass), eps=1e-6, atol=1e-4, rtol=1e-5)
    wi = nb.mass_to_inertia(world, mass.detach()).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda a, b, i: nb.ForwardDynamicsLayer.apply(world, a, b, None, i), (st, tt, wi), eps=1e-6, atol=1e-4,
                                    rtol=1e-5)


def test_shared_mass_gradient_is_the_sum_of_the_per_world_ones():
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=2)
    world._contacts_disabled = True
    B = 9
    s, tau = fd_inputs(raw, B, seed=4)
    st, tt = torch.tensor(s, dtype=torch.float64, device=DEV), torch.tensor(tau, dtype=torch.float64, device=DEV)
    G = torch.tensor(np.random.default_rng(5).normal(size=(B, raw.ndof)), device=DEV)
    m0 = torch.tensor(random_masses(world, 1, seed=6)[0], dtype=torch.float64, device=DEV)
    m1 = m0.clone().requires_grad_(True)
    (nb.forward_dynamics(world, st, tt, m1) * G).sum().backward()
    m2 = m0.repeat(B, 1).requires_grad_(True)
    (nb.forward_dynamics(world, st, tt, m2) * G).sum().backward()
    assert rel_err(m1.grad.cpu().numpy(), m2.grad.sum(0).cpu().numpy()) < 1e-12


@pytest.mark.parametrize("name", ["half_cheetah", "atlas", "free_child"])
def test_backward_identity_with_the_inverse_dynamics_backward(name):
    """dL/dqdot = -(g_qdot + g_v') and dL/dq = -g_q of inverse_dynamics's backward seeded with lambda = M^-1 g at v' = qdot + dt qdd."""
    raw = model_raw(name)
    world = _world(name)
    n, B = raw.ndof, 5
    s, tau = fd_inputs(raw, B, seed=10)
    st = torch.tensor(s, dtype=torch.float64, device=DEV, requires_grad=True)
    tt = torch.tensor(tau, dtype=torch.float64, device=DEV, requires_grad=True)
    g = torch.tensor(np.random.default_rng(11).normal(size=(B, n)), device=DEV)
    qdd = nb.forward_dynamics(world, st, tt)
    gs, gt = torch.autograd.grad(qdd, (st, tt), g)
    lam = torch.einsum("bij,bj->bi", nb.inverse_mass_matrix(world, st.detach()[:, :n]), g)
    s2 = st.detach().clone().requires_grad_(True)
    vn = (st.detach()[:, n:] + raw.dt * qdd.detach()).requires_grad_(True)
    gis, giv = torch.autograd.grad(nb.inverse_dynamics(world, s2, vn), (s2, vn), lam)
    assert rel_err(gt.cpu().numpy(), lam.cpu().numpy()) < 1e-10
    assert rel_err(gs[:, :n].cpu().numpy(), (-gis[:, :n]).cpu().numpy()) < 1e-10
    assert rel_err(gs[:, n:].cpu().numpy(), (-(gis[:, n:] + giv)).cpu().numpy()) < 1e-10


@pytest.mark.parametrize("name", ["cartpole", "half_cheetah", "atlas"])
def test_consistency_with_inverse_dynamics_and_the_mass_matrix(name):
    raw = load_raw(name)
    world = _world(name)
    n, B = raw.ndof, 64
    s, tau = fd_inputs(raw, B, seed=12)
    st, tt = torch.tensor(s, dtype=torch.float64, device=DEV), torch.tensor(tau, dtype=torch.float64, device=DEV)
    qd = st[:, n:]
    qdd = nb.forward_dynamics(world, st, tt)
    dense = torch.einsum("bij,bj->bi", nb.inverse_mass_matrix(world, st[:, :n]), tt - nb.inverse_dynamics(world, st, qd))
    assert ((qdd - dense).norm(dim=1) <= 1e-9 * dense.norm(dim=1)).all()
    # round trips: ID(state, qdot + dt FD(state, tau)) = tau, FD(state, ID(state, v')) = (v' - qdot) / dt
    back = nb.inverse_dynamics(world, st, qd + raw.dt * qdd)
    assert ((back - tt).norm(dim=1) <= 1e-9 * tt.norm(dim=1)).all()
    vn = qd + raw.dt * torch.tensor(np.random.default_rng(13).uniform(-5, 5, (B, n)), device=DEV)
    a = nb.forward_dynamics(world, st, nb.inverse_dynamics(world, st, vn))
    ref = (vn - qd) / raw.dt
    assert ((a - ref).norm(dim=1) <= 1e-9 * ref.norm(dim=1)).all()
    # the legacy pointer-style entry runs the same kernel
    legacy = nb.device_model_for(world).forward_dynamics(st[:, :n], qd, tt)
    assert ((legacy - qdd).norm(dim=1) <= 1e-10 * qdd.norm(dim=1)).all()


@pytest.mark.parametrize("name", ["cartpole", "half_cheetah", "atlas"])
def test_step_applies_the_forward_dynamics(name):
    raw = load_raw(name)
    world = _world(name)
    n = raw.ndof
    world.setActionSpace(range(n))
    s, tau = fd_inputs(raw, 256, seed=14)
    st, tt = torch.tensor(s, device=DEV), torch.tensor(tau, device=DEV)
    vplus = nb.timestep(world, st, tt)[:, n:]
    ref = (st[:, n:] + raw.dt * nb.forward_dynamics(world, st.double(), tt.double())).float()
    dv = (vplus - st[:, n:]).norm(dim=1)
    assert ((vplus - ref).norm(dim=1) <= 1e-3 * dv + 1e-6).all(), ((vplus - ref).norm(dim=1) / dv).max().item()


@pytest.mark.parametrize("name", ["atlas", "atlas_sdf"])
def test_com_of_a_floating_robot_accelerates_with_gravity(name):
    raw = load_raw(name)
    world = _world(name)
    n, B = raw.ndof, 7
    s, tau = fd_inputs(raw, B, seed=19)
    st = torch.tensor(s, dtype=torch.float64, device=DEV)
    sk = max(world.skeletons, key=lambda k: k.getNumDofs())
    o = sk._dof_offset_in_world()[1]
    assert sk._ordered_bodies()[0].parent_joint.jtype == nb.world.FREE
    tt = torch.tensor(tau, dtype=torch.float64, device=DEV)
    tt[:, o:o + 6] = 0
    qdd = nb.forward_dynamics(world, st, tt)
    acc = torch.einsum("brn,bn->br", nb.com_jacobian(world, st[:, :n], sk), qdd) + \
        torch.einsum("brn,bn->br", nb.com_jacobian_deriv(world, st, sk), st[:, n:])
    g = np.asarray(raw.gravity, np.float64)
    for w in range(B):
        assert rel_err(acc[w].cpu().numpy(), g) < 1e-9, (w, acc[w])


def test_contact_world_single_row_empty_batch_and_reduced_action_space():
    raw = load_raw("half_cheetah")
    world = nb.World.from_raw(raw)
    assert nb.device_model_for(world).has_contacts
    n, B = raw.ndof, 16
    cs, ca = contact_inputs(raw, "half_cheetah", B, seed=5)
    nb.reset_contact_cache(world)
    nb.timestep(world, torch.tensor(cs, device=DEV), torch.tensor(ca, device=DEV))
    cache = nb.contact_cache(world, B, DEV)
    before = {k: v.clone() for k, v in cache.items() if torch.is_tensor(v)}
    tau = np.random.default_rng(1).uniform(-20, 20, (B, n))
    qdd = nb.forward_dynamics(world, torch.tensor(cs, device=DEV, dtype=torch.float64), torch.tensor(tau, device=DEV))
    assert world._lcp_cache is cache and all(torch.equal(before[k], cache[k]) for k in before)
    ow = OracleWorld(per_dof(raw))
    for w in range(B):
        assert rel_err(qdd[w].cpu().numpy(), oracle_qdd(ow, cs[w], tau[w])) < 1e-9
    state0 = world.getState().copy()
    q1 = nb.forward_dynamics(world, torch.tensor(cs[3], device=DEV), torch.tensor(tau[3], device=DEV, dtype=torch.float32))
    assert q1.shape == (n,) and q1.dtype == torch.float32 and np.array_equal(world.getState(), state0)
    assert rel_err(q1.cpu().numpy(), qdd[3].cpu().numpy()) < 1e-4
    assert nb.forward_dynamics(world, torch.zeros(0, 2 * n, device=DEV), torch.zeros(0, n, device=DEV)).shape == (0, n)
    # a reduced, reordered action space: tau is still per dof
    red = copy.deepcopy(load_raw("atlas"))
    red.action_map = np.arange(red.ndof - 1, 5, -1)
    wr, wf = nb.World.from_raw(red), _world("atlas")
    s, t = fd_inputs(red, 33, seed=2)
    args = (torch.tensor(s, dtype=torch.float64, device=DEV), torch.tensor(t, dtype=torch.float64, device=DEV))
    assert torch.equal(nb.forward_dynamics(wr, *args), nb.forward_dynamics(wf, *args))


def test_c_abi_empty_batch_and_bad_arguments():
    from nimblephysics_b200 import _cabi
    dm = nb.device_model_for(_world("cartpole"))
    L = _cabi.lib()
    x = torch.zeros(4, device=DEV, dtype=torch.float64)
    p = x.data_ptr()
    assert L.nb2_forward_dynamics_batch(dm.handle, 0, p, p, None, p, None, 1, None) == 0
    assert L.nb2_forward_dynamics_backward(dm.handle, 0, p, None, p, p, p, p, None, 1, None) == 0
    assert L.nb2_forward_dynamics_batch(dm.handle, 1, None, p, None, p, None, 1, None) != 0
    assert L.nb2_forward_dynamics_backward(dm.handle, 1, p, None, None, p, p, p, None, 1, None) != 0


@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("B", [1, 33, 4099])
def test_kernels_write_only_their_own_rows(fp64, B):
    """Every output of both kernels sits inside a buffer with guard bands on both sides: the bands keep their bits, on every lane
    schedule the batch picks and on the per-world inertia path."""
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=3)
    world._contacts_disabled = True
    dm = nb.device_model_for(world)
    dt = torch.float64 if fp64 else torch.float32
    prec = nb.engine.FP64 if fp64 else nb.engine.FP32
    n, G = raw.ndof, 4096
    s, tau = fd_inputs(raw, B, seed=16)
    st, tt = torch.tensor(s, dtype=dt, device=DEV), torch.tensor(tau, dtype=dt, device=DEV)
    wi = nb.mass_to_inertia(world, torch.tensor(random_masses(world, B, seed=17), dtype=torch.float64, device=DEV))
    wi = wi.reshape(B, -1).t().contiguous()
    g = torch.randn((B, n), dtype=dt, device=DEV)

    def guarded(numel, dtype):
        buf = torch.full((numel + 2 * G,), 12345.0, dtype=dtype, device=DEV)
        return buf, buf[G:G + numel]

    stream = torch.cuda.current_stream().cuda_stream
    for w in (None, wi):
        qb, qdd = guarded(B * n, dt)
        sb, saved = guarded(dm.saved_words * B, dt)
        dm.forward_dynamics_device(B, st.data_ptr(), tt.data_ptr(), qdd.data_ptr(), saved.data_ptr(), stream, prec,
                                   wi_ptr=None if w is None else w.data_ptr())
        gsb, gs = guarded(B * 2 * n, dt)
        gtb, gt = guarded(B * n, dt)
        gib, gi = guarded(10 * dm.cm.nb * B, torch.float64)
        dm.forward_dynamics_backward_device(B, st.data_ptr(), saved.data_ptr(), g.data_ptr(), gs.data_ptr(), gt.data_ptr(), stream, prec,
                                            ginertia_ptr=gi.data_ptr(), wi_ptr=None if w is None else w.data_ptr())
        torch.cuda.synchronize()
        for buf in (qb, sb, gsb, gtb, gib):
            assert bool((buf[:G] == 12345.0).all()) and bool((buf[-G:] == 12345.0).all())
        for out in (qdd, gs, gt, gi):
            assert bool(torch.isfinite(out).all()) and not bool((out == 12345.0).any())
