"""Constrained forward dynamics on the GPU (nb2_constrained_forward_dynamics / _backward through
nimblephysics_b200.constrained_forward_dynamics): Atlas at partial-block batch sizes in both precisions against the fp64 oracle and the
host emulation; the other models in fp64; gradcheck of every differentiable input; the round trip through multiple-contact inverse
dynamics; the composed route through inverse_mass_matrix, world_jacobian, world_jacobian_deriv and forward_dynamics; trees without a
contact; guard bands, B = 0, the 1-D state, the untouched LCP cache and a singular contact set."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from tests.host_emul.binding_cfd import EmulCfdWorld
from tests.test_constrained_forward_dynamics import FEET, LIMBS, _free_child_nodes, oracle_cfd
from tests.test_forward_dynamics import fd_inputs
from tests.test_mass_matrix import built_world, model_raw
from tests.test_per_world_mass import random_masses, register
from tests.test_world_jacobian import canon_nodes
from tests.util import contact_inputs, load_raw, rel_err
from nimblephysics_b200.world_jacobian import resolve_nodes

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _nodes(world, names):
    bodies = [b for sk in world.skeletons for b in sk._ordered_bodies()]
    return [next(b for b in bodies if b.name == x) for x in names]


def _world(name):
    return built_world(name) if name in ("free_child", "chain64") else nb.World.from_raw(load_raw(name))


@pytest.mark.parametrize("name", ["atlas", "atlas_sdf"])
@pytest.mark.parametrize("names,point", [(FEET, False), (LIMBS, False), (LIMBS, True)])
@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("B", [1, 3, 33, 4099])
def test_atlas_matches_oracle_and_emulation(name, names, point, fp64, B):
    raw = load_raw(name)
    world = nb.World.from_raw(raw)
    cm = nb.device_model_for(world).cm
    ris = [list(raw.body_names).index(x) for x in names]
    bodies, T = canon_nodes(cm, ris)
    dt = torch.float64 if fp64 else torch.float32
    s, tau = fd_inputs(raw, B, seed=B)
    off = np.random.default_rng(B).uniform(-0.1, 0.1, (len(ris), 3))
    qdd, wr = nb.constrained_forward_dynamics(world, torch.tensor(s, dtype=dt, device=DEV), torch.tensor(tau, dtype=dt, device=DEV),
                                              _nodes(world, names), torch.tensor(off, dtype=dt, device=DEV), point_contacts=point)
    assert qdd.dtype == dt and qdd.shape == (B, raw.ndof) and wr.shape == (B, len(ris), 3 if point else 6)
    qdd, wr = qdd.cpu().numpy(), wr.cpu().numpy()
    rows = sorted({0, B // 2, B - 1})
    eq, ew = EmulCfdWorld(cm).constrained_forward_dynamics(s[rows], tau[rows], bodies, T, off, point=point, fp64=fp64)
    cast = (lambda a: a.astype(np.float64)) if fp64 else (lambda a: a.astype(np.float32).astype(np.float64))
    for i, w in enumerate(rows):
        rq, rw, J, _, M, _ = oracle_cfd(raw, cast(s[w]), cast(tau[w]), ris, cast(off), point, full=True)
        tol = 1e-8 if fp64 else 1e-4 * np.linalg.cond(J @ np.linalg.solve(M, J.T))
        assert rel_err(qdd[w], eq[i]) < min(tol, 1e-10 if fp64 else 1.0) and rel_err(wr[w], ew[i]) < min(tol, 1e-10 if fp64 else 1.0)
        assert rel_err(qdd[w], rq) < tol and rel_err(wr[w], rw) < tol, (w, rel_err(qdd[w], rq), rel_err(wr[w], rw))


@pytest.mark.parametrize("name", ["free_child", "chain64"])
def test_other_models_fp64(name):
    raw = model_raw(name)
    world = _world(name)
    cm = nb.device_model_for(world).cm
    flat = [b for sk in world.skeletons for b in sk._ordered_bodies()]
    ris = _free_child_nodes(raw) if name == "free_child" else [raw.nb - 1]
    point = True  # the arm of free_child has three dofs
    B = 2
    s, tau = fd_inputs(raw, B, seed=21)
    off = np.random.default_rng(22).uniform(-0.1, 0.1, (B, len(ris), 3))
    qdd, wr = nb.constrained_forward_dynamics(world, torch.tensor(s, dtype=torch.float64, device=DEV), torch.tensor(tau, dtype=torch.float64, device=DEV),
                                              [flat[r] for r in ris], torch.tensor(off, device=DEV), point_contacts=point)
    for w in range(B):
        rq, rw = oracle_cfd(raw, s[w].astype(np.float64), tau[w].astype(np.float64), ris, off[w], point)
        assert rel_err(qdd[w].cpu().numpy(), rq) < 1e-8 and rel_err(wr[w].cpu().numpy(), rw) < 1e-8


@pytest.mark.parametrize("point", [False, True])
def test_gradcheck(point):
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=6)
    n, B, names = raw.ndof, 2, FEET
    s, tau = fd_inputs(raw, B, seed=3)
    st = torch.tensor(s, dtype=torch.float64, device=DEV, requires_grad=True)
    tt = torch.tensor(tau, dtype=torch.float64, device=DEV, requires_grad=True)
    off = torch.tensor(np.random.default_rng(4).uniform(-0.1, 0.1, (B, 2, 3)), device=DEV, requires_grad=True)
    nodes = _nodes(world, names)
    f = lambda a, b, o: nb.constrained_forward_dynamics(world, a, b, nodes, o, point_contacts=point, damping=1e-4)
    assert torch.autograd.gradcheck(f, (st, tt, off), eps=1e-6, atol=1e-5, rtol=1e-4)
    M = torch.tensor(random_masses(world, B, seed=5), device=DEV, requires_grad=True)
    g = lambda m: nb.constrained_forward_dynamics(world, st.detach(), tt.detach(), nodes, off.detach(), point_contacts=point, mass=m)
    assert torch.autograd.gradcheck(g, (M,), eps=1e-6, atol=1e-5, rtol=1e-4)
    # a 1-D mass is set on the World (setMasses), which gradcheck's in-place perturbation bypasses: its gradient is the sum of the
    # per-world ones at the same masses
    m1 = M[0].detach().clone().requires_grad_(True)
    mB = M[0].detach().repeat(B, 1).requires_grad_(True)
    y1, yB = g(m1), g(mB)
    seeds = [torch.randn_like(y) for y in y1]
    torch.autograd.backward(list(y1), seeds)
    torch.autograd.backward(list(yB), seeds)
    assert rel_err(m1.grad.cpu().numpy(), mB.grad.sum(0).cpu().numpy()) < 1e-10
    wi = nb.mass_to_inertia(world, M.detach()).to(DEV).requires_grad_(True)
    h = lambda w: nb.ConstrainedForwardDynamicsLayer.apply(world, st.detach(), tt.detach(), None, w, None, *resolve_nodes(world, nodes),
                                                           point, 0.0)
    assert torch.autograd.gradcheck(h, (wi,), eps=1e-6, atol=1e-5, rtol=1e-4)


def test_round_trip_through_multiple_contact_inverse_dynamics():
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    n, B = raw.ndof, 8
    s, tau = fd_inputs(raw, B, seed=11)
    tau[:, :6] = 0
    st, tt = torch.tensor(s, dtype=torch.float64, device=DEV), torch.tensor(tau, dtype=torch.float64, device=DEV)
    feet = _nodes(world, FEET)
    qdd, wr = nb.constrained_forward_dynamics(world, st, tt, feet)
    back, w2 = nb.multiple_contact_inverse_dynamics(world, st, st[:, n:] + raw.dt * qdd, feet, wrench_guesses=wr)
    assert rel_err(back[:, 6:].cpu().numpy(), tau[:, 6:]) < 1e-8 and float(back[:, :6].abs().max()) < 1e-8 * float(tt.abs().max())
    assert rel_err(w2.cpu().numpy(), wr.cpu().numpy()) < 1e-8


def test_composed_route_outputs_and_gradients():
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    n, B = raw.ndof, 4
    s, tau = fd_inputs(raw, B, seed=12)
    nodes = _nodes(world, LIMBS)
    rng = np.random.default_rng(13)
    gq, gw = torch.tensor(rng.normal(size=(B, n)), device=DEV), torch.tensor(rng.normal(size=(B, 4, 3)), device=DEV)
    off = torch.tensor(rng.uniform(-0.1, 0.1, (4, 3)), device=DEV)

    def route(fused):
        st = torch.tensor(s, dtype=torch.float64, device=DEV, requires_grad=True)
        tt = torch.tensor(tau, dtype=torch.float64, device=DEV, requires_grad=True)
        o = off.clone().requires_grad_(True)
        if fused:
            qdd, wr = nb.constrained_forward_dynamics(world, st, tt, nodes, o)
        else:
            q = st[:, :n]
            Minv = nb.inverse_mass_matrix(world, q)
            J = nb.world_jacobian(world, q, nodes, o).reshape(B, 24, n)
            Jd = nb.world_jacobian_deriv(world, st, nodes, o).reshape(B, 24, n)
            qf = nb.forward_dynamics(world, st, tt)
            A = J @ Minv @ J.transpose(1, 2)
            c = (J @ qf[..., None] + Jd @ st[:, n:, None])[..., 0]
            lam = -torch.linalg.solve(A, c)
            qdd = qf + (Minv @ J.transpose(1, 2) @ lam[..., None])[..., 0]
            wr = lam.reshape(B, 4, 6)
        wr = wr[..., 3:]  # the forces: the same in both conventions
        torch.autograd.backward([qdd, wr], [gq, gw])
        return [x.detach() for x in (qdd, wr, st.grad, tt.grad, o.grad)]

    for a, b in zip(route(True), route(False)):
        assert rel_err(a.cpu().numpy(), b.cpu().numpy()) < 1e-8


def test_trees_without_a_contact_follow_forward_dynamics():
    raw = model_raw("free_child")
    world = built_world("free_child")
    flat = [b for sk in world.skeletons for b in sk._ordered_bodies()]
    s, tau = fd_inputs(raw, 6, seed=14)
    st, tt = torch.tensor(s, dtype=torch.float64, device=DEV), torch.tensor(tau, dtype=torch.float64, device=DEV)
    qdd, _ = nb.constrained_forward_dynamics(world, st, tt, [flat[2]])
    ref = nb.forward_dynamics(world, st, tt)
    arm = slice(raw.ndof - 3, raw.ndof)
    assert rel_err(qdd[:, arm].cpu().numpy(), ref[:, arm].cpu().numpy()) < 1e-12


@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("B", [1, 33, 4099])
def test_kernels_write_only_their_own_rows(fp64, B):
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    dm = nb.device_model_for(world)
    dt = torch.float64 if fp64 else torch.float32
    prec = nb.engine.FP64 if fp64 else nb.engine.FP32
    n, nb_, G = raw.ndof, dm.cm.nb, 4096
    bodies, T12 = resolve_nodes(world, _nodes(world, FEET))  # regular in fp32 at these states (24 fp32 rows flag a few worlds singular)
    s, tau = fd_inputs(raw, B, seed=15)
    st, tt = torch.tensor(s, dtype=dt, device=DEV), torch.tensor(tau, dtype=dt, device=DEV)

    def guarded(numel, dtype=dt):
        buf = torch.full((numel + 2 * G,), float("nan"), dtype=dtype, device=DEV)
        return buf, buf[G:G + numel]

    stream = torch.cuda.current_stream().cuda_stream
    fw = [guarded(B * n), guarded(B * 12)]
    dm.constrained_forward_dynamics_device(B, st.data_ptr(), tt.data_ptr(), bodies, T12, None, False, False, 0.0, fw[0][1].data_ptr(),
                                           fw[1][1].data_ptr(), stream, prec)
    gq, gw = torch.ones(B, n, dtype=dt, device=DEV), torch.ones(B, 12, dtype=dt, device=DEV)
    bw = [guarded(B * 2 * n), guarded(B * n), guarded(B * 6), guarded(10 * nb_ * B, torch.float64)]
    dm.constrained_forward_dynamics_backward_device(B, st.data_ptr(), tt.data_ptr(), bodies, T12, None, False, False, 0.0, gq.data_ptr(), gw.data_ptr(),
                                                    *(o.data_ptr() for _, o in bw[:3]), stream, prec, ginertia_ptr=bw[3][1].data_ptr())
    torch.cuda.synchronize()
    for buf, out in fw + bw:
        assert bool(buf[:G].isnan().all()) and bool(buf[-G:].isnan().all())
        assert bool(torch.isfinite(out).all())


def test_contact_world_cache_empty_batch_single_row_and_singular_isolation():
    raw = load_raw("half_cheetah")
    world = nb.World.from_raw(raw)
    n, B = raw.ndof, 16
    cs, ca = contact_inputs(raw, "half_cheetah", B, seed=5)
    nb.reset_contact_cache(world)
    nb.timestep(world, torch.tensor(cs, device=DEV), torch.tensor(ca, device=DEV))
    cache = nb.contact_cache(world, B, DEV)
    before = {k: v.clone() for k, v in cache.items() if torch.is_tensor(v)}
    st = torch.tensor(cs, device=DEV, dtype=torch.float64)
    tt = torch.tensor(np.random.default_rng(1).uniform(-5, 5, (B, n)), device=DEV)
    node = [b for sk in world.skeletons for b in sk._ordered_bodies() if sk.mobile][-1]
    full = nb.constrained_forward_dynamics(world, st, tt, [node], damping=1e-3)  # the planar model: damping makes the set regular
    bits = lambda t: t.view({8: torch.int64, 4: torch.int32, 2: torch.int16, 1: torch.uint8}[t.element_size()])
    assert world._lcp_cache is cache and all(torch.equal(bits(before[k]), bits(cache[k])) for k in before)
    one = nb.constrained_forward_dynamics(world, st[3], tt[3], [node], damping=1e-3)
    assert one[0].shape == (n,) and one[1].shape == (1, 6) and bool(torch.isfinite(full[0]).all())
    assert torch.equal(one[0], full[0][3]) and torch.equal(one[1], full[1][3])
    e = nb.constrained_forward_dynamics(world, torch.zeros(0, 2 * n, device=DEV), torch.zeros(0, n, device=DEV), [node])
    assert e[0].shape == (0, n) and e[1].shape == (0, 1, 6)
    # cartpole's pole held 6-D is singular at rho = 0 in every world: NaN rows and gradients; rho > 0 regularises it
    craw = load_raw("cartpole")
    cw = nb.World.from_raw(craw)
    pole = [b for sk in cw.skeletons for b in sk._ordered_bodies()][-1]
    s, tau = fd_inputs(craw, 33, seed=2)
    sc = torch.tensor(s, dtype=torch.float64, device=DEV, requires_grad=True)
    q, w = nb.constrained_forward_dynamics(cw, sc, torch.tensor(tau, dtype=torch.float64, device=DEV), [pole])
    assert bool(q.isnan().all()) and bool(w.isnan().all())
    (q.sum() + w.sum()).backward()
    assert bool(sc.grad.isnan().all())
    q2, w2 = nb.constrained_forward_dynamics(cw, sc.detach(), torch.tensor(tau, dtype=torch.float64, device=DEV), [pole], damping=1e-2)
    assert bool(torch.isfinite(q2).all()) and bool(torch.isfinite(w2).all())
