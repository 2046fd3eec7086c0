"""Impulse dynamics on the GPU (nb2_impulse_dynamics / _backward through nimblephysics_b200.impulse_dynamics): Atlas at partial-block batch
sizes in both precisions against the fp64 oracle and the host emulation; the other models in fp64; gradcheck of every differentiable
input; the relation to constrained forward dynamics; the composed route through mass_matrix, world_jacobian and a torch solve; momentum and
energy through energy_and_momentum; B = 0, the 1-D state, the untouched LCP cache and a singular contact set."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from tests.host_emul.binding_imp import EmulImpWorld
from tests.test_constrained_forward_dynamics import FEET, LIMBS, _free_child_nodes
from tests.test_energy import skeleton_of
from tests.test_forward_dynamics import fd_inputs
from tests.test_impulse_dynamics import ES, oracle_imp
from tests.test_mass_matrix import built_world, model_raw
from tests.test_oracle import fk
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
    s, _ = fd_inputs(raw, B, seed=B)
    off = np.random.default_rng(B).uniform(-0.1, 0.1, (len(ris), 3))
    e = ES[B % 3]
    v, imp = nb.impulse_dynamics(world, torch.tensor(s, dtype=dt, device=DEV), _nodes(world, names), torch.tensor(off, dtype=dt, device=DEV),
                                 point_contacts=point, restitution=e)
    assert v.dtype == dt and v.shape == (B, raw.ndof) and imp.shape == (B, len(ris), 3 if point else 6)
    v, imp = v.cpu().numpy(), imp.cpu().numpy()
    rows = sorted({0, B // 2, B - 1})
    ev, ei = EmulImpWorld(cm).impulse_dynamics(s[rows], bodies, T, off, point=point, e=e, fp64=fp64)
    cast = (lambda a: a.astype(np.float64)) if fp64 else (lambda a: a.astype(np.float32).astype(np.float64))
    for i, w in enumerate(rows):
        rv, ri, J, M, _ = oracle_imp(raw, cast(s[w]), ris, cast(off), point, e, full=True)
        tol = 1e-8 if fp64 else 1e-4 * np.linalg.cond(J @ np.linalg.solve(M, J.T))
        assert rel_err(v[w], ev[i]) < min(tol, 1e-10 if fp64 else 1.0) and rel_err(imp[w], ei[i]) < min(tol, 1e-10 if fp64 else 1.0)
        assert rel_err(v[w], rv) < tol and rel_err(imp[w], ri) < tol, (w, rel_err(v[w], rv), rel_err(imp[w], ri))


@pytest.mark.parametrize("name", ["free_child", "chain64"])
def test_other_models_fp64(name):
    raw = model_raw(name)
    world = _world(name)
    flat = [b for sk in world.skeletons for b in sk._ordered_bodies()]
    ris = _free_child_nodes(raw) if name == "free_child" else [raw.nb - 1]
    B = 2
    s, _ = fd_inputs(raw, B, seed=21)
    off = np.random.default_rng(22).uniform(-0.1, 0.1, (B, len(ris), 3))
    v, imp = nb.impulse_dynamics(world, torch.tensor(s, dtype=torch.float64, device=DEV), [flat[r] for r in ris], torch.tensor(off, device=DEV),
                                 point_contacts=True, restitution=0.5)
    for w in range(B):
        rv, ri = oracle_imp(raw, s[w].astype(np.float64), ris, off[w], True, 0.5)
        assert rel_err(v[w].cpu().numpy(), rv) < 1e-8 and rel_err(imp[w].cpu().numpy(), ri) < 1e-8


@pytest.mark.parametrize("point", [False, True])
def test_gradcheck(point):
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=6)
    B, names = 2, FEET
    s, _ = fd_inputs(raw, B, seed=3)
    st = torch.tensor(s, dtype=torch.float64, device=DEV, requires_grad=True)
    off = torch.tensor(np.random.default_rng(4).uniform(-0.1, 0.1, (B, 2, 3)), device=DEV, requires_grad=True)
    nodes = _nodes(world, names)
    f = lambda a, o: nb.impulse_dynamics(world, a, nodes, o, point_contacts=point, restitution=0.4, damping=1e-4)
    assert torch.autograd.gradcheck(f, (st, off), eps=1e-6, atol=1e-5, rtol=1e-4)
    M = torch.tensor(random_masses(world, B, seed=5), device=DEV, requires_grad=True)
    g = lambda m: nb.impulse_dynamics(world, st.detach(), nodes, off.detach(), point_contacts=point, restitution=0.4, mass=m)
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
    h = lambda w: nb.ImpulseDynamicsLayer.apply(world, st.detach(), None, w, None, *resolve_nodes(world, nodes), point, 0.4, 0.0)
    assert torch.autograd.gradcheck(h, (wi,), eps=1e-6, atol=1e-5, rtol=1e-4)


@pytest.mark.parametrize("point", [False, True])
def test_relation_to_constrained_forward_dynamics(point):
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    n, B, e = raw.ndof, 8, 0.3
    s, _ = fd_inputs(raw, B, seed=11)
    st = torch.tensor(s, dtype=torch.float64, device=DEV)
    nodes = _nodes(world, LIMBS)
    off = torch.tensor(np.random.default_rng(12).uniform(-0.1, 0.1, (4, 3)), device=DEV)
    v, imp = nb.impulse_dynamics(world, st, nodes, off, point_contacts=point, restitution=e, damping=1e-3)
    q, qd = st[:, :n], st[:, n:]
    s0 = torch.cat([q, torch.zeros_like(qd)], 1)
    tau = (1 + e) * (nb.mass_matrix(world, q) @ qd[..., None])[..., 0]
    a1, w1 = nb.constrained_forward_dynamics(world, s0, tau, nodes, off, point_contacts=point, damping=1e-3)
    a0, w0 = nb.constrained_forward_dynamics(world, s0, torch.zeros_like(tau), nodes, off, point_contacts=point, damping=1e-3)
    assert rel_err((v + e * qd).cpu().numpy(), (a1 - a0).cpu().numpy()) < 1e-8
    assert rel_err(imp.cpu().numpy(), (w1 - w0).cpu().numpy()) < 1e-8


def test_composed_route_outputs_and_gradients():
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    n, B, e = raw.ndof, 4, 0.5
    s, _ = fd_inputs(raw, B, seed=12)
    nodes = _nodes(world, LIMBS)
    rng = np.random.default_rng(13)
    gv, gw = torch.tensor(rng.normal(size=(B, n)), device=DEV), torch.tensor(rng.normal(size=(B, 4, 3)), device=DEV)
    off = torch.tensor(rng.uniform(-0.1, 0.1, (4, 3)), device=DEV)

    def route(fused):
        st = torch.tensor(s, dtype=torch.float64, device=DEV, requires_grad=True)
        o = off.clone().requires_grad_(True)
        if fused:
            v, imp = nb.impulse_dynamics(world, st, nodes, o, restitution=e)
        else:
            q, qd = st[:, :n], st[:, n:]
            M = nb.mass_matrix(world, q)
            J = nb.world_jacobian(world, q, nodes, o).reshape(B, 24, n)
            Y = torch.linalg.solve(M, J.transpose(1, 2))
            lam = -torch.linalg.solve(J @ Y, (1 + e) * (J @ qd[..., None]))
            v = qd + (Y @ lam)[..., 0]
            imp = lam[..., 0].reshape(B, 4, 6)
        imp = imp[..., 3:]  # the linear impulses: the same in both conventions
        torch.autograd.backward([v, imp], [gv, gw])
        return [x.detach() for x in (v, imp, st.grad, o.grad)]

    fused, comp = route(True), route(False)
    for a, b in zip(fused[:3], comp[:3]):
        assert rel_err(a.cpu().numpy(), b.cpu().numpy()) < 1e-8
    # 6-D holds fix the bodies' twists wherever the points are: the offset gradient is zero up to rounding, on the state gradient's scale
    assert float((fused[3] - comp[3]).abs().max()) < 1e-8 * float(comp[2].abs().max())


def _com(raw, q, rb):
    bodies, _ = skeleton_of(raw, rb)
    W = fk(raw, q)
    mt = sum(raw.mass[i] for i in bodies)
    return sum(raw.mass[i] * (W[i][:3, :3] @ raw.com[i] + W[i][:3, 3]) for i in bodies) / mt


@pytest.mark.parametrize("e", ES)
def test_momentum_and_energy(e):
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    n, B = raw.ndof, 6
    s, _ = fd_inputs(raw, B, seed=17)
    st = torch.tensor(s, dtype=torch.float64, device=DEV)
    names = FEET
    nodes = _nodes(world, names)
    v, imp = nb.impulse_dynamics(world, st, nodes, restitution=e)
    after = torch.cat([st[:, :n], v], 1)
    sk = nodes[0].skeleton
    T0, _, h0 = nb.energy_and_momentum(world, st, sk)
    T1, _, h1 = nb.energy_and_momentum(world, after, sk)
    rb = list(raw.body_names).index(names[0])
    ris = [list(raw.body_names).index(x) for x in names]
    for w in range(B):
        c = _com(raw, s[w, :n].astype(np.float64), rb)
        iw = imp[w].cpu().numpy()
        want = np.concatenate([(iw[:, :3] - np.cross(c, iw[:, 3:])).sum(0), iw[:, 3:].sum(0)])  # the impulses about the COM
        assert rel_err((h1[w] - h0[w]).cpu().numpy(), want) < 1e-8
        _, _, J, M, _ = oracle_imp(raw, s[w].astype(np.float64), ris, full=True)
        cq = J @ s[w, n:].astype(np.float64)
        loss = -0.5 * (1 - e * e) * cq @ np.linalg.solve(J @ np.linalg.solve(M, J.T), cq)
        assert abs(float(T1[w] - T0[w]) - loss) < 1e-9 * float(T0[w])
    if e == 1.0:
        assert rel_err(T1.cpu().numpy(), T0.cpu().numpy()) < 1e-12
    else:
        assert bool((T1 < T0).all())


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
    node = [b for sk in world.skeletons for b in sk._ordered_bodies() if sk.mobile][-1]
    full = nb.impulse_dynamics(world, st, [node], restitution=0.2, damping=1e-3)  # the planar model: damping makes the set regular
    bits = lambda t: t.view({8: torch.int64, 4: torch.int32, 2: torch.int16, 1: torch.uint8}[t.element_size()])
    assert world._lcp_cache is cache and all(torch.equal(bits(before[k]), bits(cache[k])) for k in before)
    one = nb.impulse_dynamics(world, st[3], [node], restitution=0.2, damping=1e-3)
    assert one[0].shape == (n,) and one[1].shape == (1, 6) and bool(torch.isfinite(full[0]).all())
    assert torch.equal(one[0], full[0][3]) and torch.equal(one[1], full[1][3])
    e0 = nb.impulse_dynamics(world, torch.zeros(0, 2 * n, device=DEV), [node])
    assert e0[0].shape == (0, n) and e0[1].shape == (0, 1, 6)
    # two 6-D holds on one chain (Atlas's left foot and shin) are singular at rho = 0: NaN rows and gradients; rho > 0 regularises them
    araw = load_raw("atlas")
    aw = nb.World.from_raw(araw)
    s, _ = fd_inputs(araw, 33, seed=2)
    nodes = _nodes(aw, ["l_foot", "l_lleg"])
    sc = torch.tensor(s, dtype=torch.float64, device=DEV, requires_grad=True)
    v, imp = nb.impulse_dynamics(aw, sc, nodes, restitution=0.5)
    assert bool(v.isnan().all()) and bool(imp.isnan().all())
    (v.sum() + imp.sum()).backward()
    assert bool(sc.grad.isnan().all())
    v2, imp2 = nb.impulse_dynamics(aw, sc.detach(), nodes, restitution=0.5, damping=1e-2)
    assert bool(torch.isfinite(v2).all()) and bool(torch.isfinite(imp2).all())
