"""Energy and momentum on the GPU (nb2_energy_momentum and its backward through nimblephysics_b200.energy_and_momentum) against the
fp64 oracle of test_energy and the host emulation at partial-block batch sizes; against mass_matrix, com_jacobian and the IKMapping COM
entry; the power balance dE/dt = qdot^T tau - qdot^T D qdot - dt qdot^T K qdot and the momentum rate of a floating robot through
forward_dynamics; gradcheck, per-world and shared masses; guard bands, B = 0, the 1-D state and the Skeleton mirrors."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from tests.host_emul.binding_energy import EmulEnergyWorld
from tests.test_energy import oracle_energy, skeleton_of
from tests.test_inverse_dynamics import _velocity_map, id_inputs
from tests.test_mass_matrix import MODELS, built_world, model_raw
from tests.test_oracle import _tree_world
from tests.test_per_world_mass import random_masses, register
from tests.test_world_jacobian import canon_root, com_body
from tests.util import load_raw, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _world(name):
    if name == "tree":
        return _tree_world()
    if name in ("chain64", "free16", "limit", "free_child"):
        return built_world(name)
    return nb.World.from_raw(load_raw(name))


def _skeleton(world, raw, rb):
    """the Skeleton of raw body rb"""
    return world.skeletons[int(raw.skel_id[rb])]


def _check(raw, s, T, U, h, rb, ws, tol):
    n = raw.ndof
    for w in ws:
        To, Uo, ho = oracle_energy(raw, s[w, :n], s[w, n:], rb)
        scale = max(abs(To), abs(Uo), 1.0)
        assert abs(T[w] - To) < tol * scale and abs(U[w] - Uo) < tol * scale, (w, T[w], To, U[w], Uo)
        assert rel_err(h[w], ho) < tol, (w, rel_err(h[w], ho))


@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("B", [1, 3, 33, 4099])
@pytest.mark.parametrize("name", ["atlas", "atlas_sdf"])
def test_atlas_matches_oracle_and_emulation(name, B, fp64):
    raw = load_raw(name)
    world = nb.World.from_raw(raw)
    cm = nb.compile_model(raw, lanes=1)
    rb = com_body(raw, cm)
    dt = torch.float64 if fp64 else torch.float32
    s, _ = id_inputs(raw, B, seed=B)
    s = s.astype(np.float64) if fp64 else s
    T, U, h = nb.energy_and_momentum(world, torch.tensor(s, dtype=dt, device=DEV), _skeleton(world, raw, rb))
    assert T.shape == (B,) and U.shape == (B,) and h.shape == (B, 6) and T.dtype == dt
    T, U, h = (x.cpu().numpy() for x in (T, U, h))
    _check(raw, s.astype(np.float64), T, U, h, rb, sorted({0, B // 2, B - 1}), 1e-9 if fp64 else 1e-4)
    Te, Ue, he = EmulEnergyWorld(cm).energy_momentum(s, canon_root(cm, rb), fp64=fp64)
    tol = 1e-12 if fp64 else 1e-5
    assert rel_err(T, Te) < tol and rel_err(U, Ue) < tol and rel_err(h, he) < tol


@pytest.mark.parametrize("name", [m for m in MODELS if m not in ("atlas", "atlas_sdf")])
def test_other_models_against_the_oracle(name):
    raw = model_raw(name)
    cm = nb.compile_model(raw, lanes=1)
    rb = com_body(raw, cm)
    if rb is None:
        pytest.skip("no skeleton with a moving root")
    world = _world(name)
    s, _ = id_inputs(raw, 5, seed=7)
    s = s.astype(np.float64)
    T, U, h = (x.cpu().numpy() for x in nb.energy_and_momentum(world, torch.tensor(s, device=DEV), _skeleton(world, raw, rb)))
    _check(raw, s, T, U, h, rb, [0, 4], 1e-9)


def test_against_mass_matrix_com_jacobian_and_the_ik_com_entry():
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    sk = _skeleton(world, raw, com_body(raw, nb.compile_model(raw, lanes=1)))
    n, B = raw.ndof, 9
    s, _ = id_inputs(raw, B, seed=13)
    st = torch.tensor(s, dtype=torch.float64, device=DEV, requires_grad=True)
    T, U, h = nb.energy_and_momentum(world, st, sk)
    q, qd = st.detach()[:, :n], st.detach()[:, n:]
    M = nb.mass_matrix(world, q)
    assert rel_err(T.detach().cpu().numpy(), (0.5 * torch.einsum("bi,bij,bj->b", qd, M, qd)).cpu().numpy()) < 1e-12
    mt = float(np.sum(raw.mass[skeleton_of(raw, com_body(raw, nb.compile_model(raw, lanes=1)))[0]]))
    Jc = nb.com_jacobian(world, q, sk)
    assert rel_err(h[:, 3:].detach().cpu().numpy(), (mt * torch.einsum("brn,bn->br", Jc, qd)).cpu().numpy()) < 1e-12
    # the momentum matrix's linear rows, one VJP each, are m_tot J_com
    for r in range(3):
        (g,) = torch.autograd.grad(h[:, 3 + r].sum(), st, retain_graph=True)
        assert rel_err(g[:, n:].cpu().numpy(), (mt * Jc[:, r]).cpu().numpy()) < 1e-12
    # gravity part of U (Atlas has no springs) against the IKMapping COM entry, which computes in fp32
    assert not np.any(raw.spring)
    ik = nb.IKMapping(world)
    ik.addSkeletonCOM(sk)
    com = nb.map_to_pos(world, ik, st.detach()).double()
    g = torch.tensor(raw.gravity, dtype=torch.float64, device=DEV)
    assert rel_err(U.detach().cpu().numpy(), (-mt * com @ g).cpu().numpy()) < 1e-5


def _q_rate(raw, q, qd):
    """dq/dt of the step's position update (free joints: Rdot = R [omega]x, pdot = R v)"""
    return np.linalg.solve(_velocity_map(raw, q), qd)


def _energy_grads(world, sk, st, which):
    """d(sum of the chosen outputs)/d state, [B, 2n]"""
    x = st.clone().requires_grad_(True)
    out = which(*nb.energy_and_momentum(world, x, sk))
    (g,) = torch.autograd.grad(out, x)
    return g.cpu().numpy()


@pytest.mark.parametrize("name", ["tree", "half_cheetah", "atlas"])
def test_power_balance(name):
    """dE/dt along the contact-free motion (qddot from forward_dynamics) is the power of tau, the damping and the springs' implicit
    dt-term.  Free-joint dofs carry no spring on these models (checked), where the spring energy is not a function of the motion alone.
    (Cartpole's skeleton root is welded to the world, so it has no energy_and_momentum; 'tree' has a spring and a damper.)"""
    raw = model_raw(name)
    world = _world(name)
    world._contacts_disabled = True
    cm = nb.compile_model(raw, lanes=1)
    rb = com_body(raw, cm)
    sk = _skeleton(world, raw, rb)
    _, dofs = skeleton_of(raw, rb)
    for i in range(raw.nb):
        if raw.jtype[i] == nb.world.FREE:
            o = raw.dof_off[i]
            assert not np.any(raw.spring[o:o + 6])
    n, B = raw.ndof, 4
    s, _ = id_inputs(raw, B, seed=23)
    s = s.astype(np.float64)
    tau = np.random.default_rng(24).uniform(-5, 5, (B, n))
    st = torch.tensor(s, device=DEV)
    qdd = nb.forward_dynamics(world, st, torch.tensor(tau, device=DEV)).cpu().numpy()
    gE = _energy_grads(world, sk, st, lambda T, U, h: (T + U).sum())
    for w in range(B):
        q, qd = s[w, :n], s[w, n:]
        lhs_terms = np.concatenate([gE[w, :n] * _q_rate(raw, q, qd), gE[w, n:] * qdd[w]])
        v = qd[dofs]
        rhs_terms = np.concatenate([v * tau[w, dofs], -raw.damping[dofs] * v * v, -raw.dt * raw.spring[dofs] * v * v])
        scale = max(np.abs(lhs_terms).max(), np.abs(rhs_terms).max())
        assert abs(lhs_terms.sum() - rhs_terms.sum()) < 1e-9 * scale, (w, lhs_terms.sum(), rhs_terms.sum(), scale)
    if name == "tree":
        assert np.any(raw.spring[dofs]) and np.any(raw.damping[dofs])


def test_momentum_rate_of_a_floating_robot():
    """tau = 0 on the free root (no spring or damping there): the linear momentum changes at m_tot g, the angular momentum about the COM
    not at all.  hdot = dh/d[q ; qdot] . [q_rate ; qddot], the six rows by one VJP each."""
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    world._contacts_disabled = True
    rb = com_body(raw, nb.compile_model(raw, lanes=1))
    sk = _skeleton(world, raw, rb)
    assert raw.jtype[rb] == nb.world.FREE
    o = raw.dof_off[rb]
    assert not np.any(raw.spring[o:o + 6]) and not np.any(raw.damping[o:o + 6])
    n, B = raw.ndof, 4
    s, _ = id_inputs(raw, B, seed=29)
    s = s.astype(np.float64)
    tau = np.random.default_rng(30).uniform(-20, 20, (B, n))
    tau[:, o:o + 6] = 0
    st = torch.tensor(s, device=DEV)
    qdd = nb.forward_dynamics(world, st, torch.tensor(tau, device=DEV)).cpu().numpy()
    rows = [_energy_grads(world, sk, st, lambda T, U, h, r=r: h[:, r].sum()) for r in range(6)]
    mt = float(np.sum(raw.mass[skeleton_of(raw, rb)[0]]))
    for w in range(B):
        rate = np.concatenate([_q_rate(raw, s[w, :n], s[w, n:]), qdd[w]])
        terms = np.stack([rows[r][w] * rate for r in range(6)])
        hdot = terms.sum(1)
        scale = np.abs(terms).max()
        assert np.abs(hdot[:3]).max() < 1e-9 * scale, (w, hdot[:3], scale)
        assert np.abs(hdot[3:] - mt * raw.gravity).max() < 1e-9 * max(scale, mt * np.abs(raw.gravity).max()), (w, hdot[3:])


def test_gradcheck_and_masses():
    raw = load_raw("half_cheetah")
    world = register(nb.World.from_raw(raw), step=2)
    sk = max(world.skeletons, key=lambda s: s.getNumDofs())
    n, B = raw.ndof, 3
    s, _ = id_inputs(raw, B, seed=31)
    st = torch.tensor(s, dtype=torch.float64, device=DEV, requires_grad=True)
    assert torch.autograd.gradcheck(lambda x: nb.energy_and_momentum(world, x, sk), (st,))
    mB = torch.tensor(random_masses(world, B, seed=32), device=DEV, requires_grad=True)
    assert torch.autograd.gradcheck(lambda x, m: nb.energy_and_momentum(world, x, sk, m), (st, mB))
    # a per-world mass gives world w the result of setMasses(mass[w])
    outB = nb.energy_and_momentum(world, st.detach(), sk, mB.detach())
    m0 = world.getMasses().copy()
    for w in range(B):
        world.setMasses(mB[w].detach().cpu().numpy())
        ref = nb.energy_and_momentum(world, st.detach()[w:w + 1], sk)
        for a, b in zip(outB, ref):
            assert rel_err(a[w:w + 1].cpu().numpy(), b.cpu().numpy()) < 1e-13
    world.setMasses(m0)
    # a 1-D mass (shared by the batch) gets the per-world gradients summed
    G = torch.randn(B, 8, dtype=torch.float64, device=DEV)
    loss = lambda T, U, h: (torch.cat([T[:, None], U[:, None], h], 1) * G).sum()
    m1 = torch.tensor(m0, device=DEV, requires_grad=True)
    loss(*nb.energy_and_momentum(world, st.detach(), sk, m1)).backward()
    m2 = torch.tensor(m0, device=DEV).repeat(B, 1).requires_grad_(True)
    loss(*nb.energy_and_momentum(world, st.detach(), sk, m2)).backward()
    assert rel_err(m1.grad.cpu().numpy(), m2.grad.sum(0).cpu().numpy()) < 1e-12


@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("B", [1, 33, 4099])
def test_kernels_write_only_their_own_rows(fp64, B):
    """Every output and gradient row sits inside a buffer with guard bands on both sides: the bands keep their bits, with and without
    per-world inertia; B = 0 validates and writes nothing."""
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=3)
    dm = nb.device_model_for(world)
    root = canon_root(dm.cm, com_body(raw, dm.cm))
    dt = torch.float64 if fp64 else torch.float32
    prec = nb.engine.FP64 if fp64 else nb.engine.FP32
    n, nb_, G = raw.ndof, dm.cm.nb, 4096
    s, _ = id_inputs(raw, B, seed=71)
    st = torch.tensor(s, dtype=dt, device=DEV)
    wi = nb.mass_to_inertia(world, torch.tensor(random_masses(world, B, seed=72), dtype=torch.float64, device=DEV))
    wi = wi.reshape(B, -1).t().contiguous()
    grads = [torch.randn(k, dtype=dt, device=DEV) for k in (B, B, 6 * B)]

    def guarded(numel, dtype=dt):
        buf = torch.full((numel + 2 * G,), 12345.0, dtype=dtype, device=DEV)
        return buf, buf[G:G + numel]

    stream = torch.cuda.current_stream().cuda_stream
    for w in (None, wi):
        wp = None if w is None else w.data_ptr()
        fwd = [guarded(B), guarded(B), guarded(6 * B)]
        dm.energy_momentum_device(B, st.data_ptr(), root, *(o.data_ptr() for _, o in fwd), stream, prec, wi_ptr=wp)
        bwd = [guarded(2 * B * n), guarded(10 * nb_ * B, torch.float64)]
        dm.energy_momentum_backward_device(B, st.data_ptr(), root, *(g.data_ptr() for g in grads), bwd[0][1].data_ptr(), stream, prec,
                                           ginertia_ptr=bwd[1][1].data_ptr(), wi_ptr=wp)
        torch.cuda.synchronize()
        for buf, out in fwd + bwd:
            assert bool((buf[:G] == 12345.0).all()) and bool((buf[-G:] == 12345.0).all())
            assert bool(torch.isfinite(out).all()) and not bool((out == 12345.0).any())
    empty = [guarded(0)[0] for _ in range(3)]  # an empty tensor's data_ptr() is NULL: hand the kernels real buffers
    dm.energy_momentum_device(0, st.data_ptr(), root, *(buf.data_ptr() for buf in empty), stream, prec)
    dm.energy_momentum_backward_device(0, st.data_ptr(), root, *(g.data_ptr() for g in grads), empty[0].data_ptr(), stream, prec)
    torch.cuda.synchronize()
    assert all(bool((buf == 12345.0).all()) for buf in empty)


def test_single_row_and_mirrors():
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    sk = _skeleton(world, raw, com_body(raw, nb.compile_model(raw, lanes=1)))
    n, B = raw.ndof, 5
    s, _ = id_inputs(raw, B, seed=37)
    st = torch.tensor(s, dtype=torch.float64, device=DEV)
    full = nb.energy_and_momentum(world, st, sk)
    one = nb.energy_and_momentum(world, st[2], sk)
    assert [tuple(x.shape) for x in one] == [(), (), (6,)]
    for a, b in zip(one, full):
        assert torch.equal(a, b[2])
    world.setState(s[2].astype(np.float64))
    T, U = sk.computeKineticEnergy(), sk.computePotentialEnergy()
    assert isinstance(T, float) and T == float(full[0][2]) and U == float(full[1][2])
    assert sk.computeLagrangian() == T - U
