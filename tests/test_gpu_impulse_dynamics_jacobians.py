"""Dense Jacobians of impulse dynamics on the GPU (nb2_impulse_dynamics_jacobians through nimblephysics_b200.impulse_dynamics_jacobians):
Atlas at partial-block batch sizes in both precisions against the host emulation, with qdot+ and the impulses bit-identical to
impulse_dynamics; the other models in fp64; the blocks against autograd's Jacobian of impulse_dynamics; the qdot- blocks against
inverse_mass_matrix and world_jacobian and the position block against the constraint differentiated through world_jacobian; per-world and
1-D masses, offsets and damping; guard bands, the singular world, B = 0 and the 1-D state."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from nimblephysics_b200._cabi import Nb2Error
from nimblephysics_b200.world_jacobian import resolve_nodes
from tests.host_emul.binding_impj import EmulImpjWorld
from tests.test_constrained_forward_dynamics import FEET, LIMBS, _free_child_nodes
from tests.test_constrained_forward_dynamics_jacobians import singular_middle_world
from tests.test_impulse_dynamics import _inputs, oracle_imp
from tests.test_mass_matrix import built_world, model_raw
from tests.test_per_world_mass import random_masses, register
from tests.test_world_jacobian import canon_nodes
from tests.util import load_raw, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
E = 0.5
f_j = nb.impulse_dynamics_jacobians


def _nodes(world, names):
    bodies = [b for sk in world.skeletons for b in sk._ordered_bodies()]
    return [next(b for b in bodies if b.name == x) for x in names]


def _bits(t):
    return t.view(torch.int64 if t.element_size() == 8 else torch.int32)


def _np(xs):
    return [x.detach().cpu().numpy() for x in xs]


@pytest.mark.parametrize("name", ["atlas", "atlas_sdf"])
@pytest.mark.parametrize("names,point", [(FEET, False), (LIMBS, False), (LIMBS, True)])
@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("B", [1, 3, 33, 4099])
def test_atlas_matches_emulation_and_forward(name, names, point, fp64, B):
    raw = load_raw(name)
    world = nb.World.from_raw(raw)
    cm = nb.device_model_for(world).cm
    ris = [list(raw.body_names).index(x) for x in names]
    bodies, T = canon_nodes(cm, ris)
    dt = torch.float64 if fp64 else torch.float32
    s = _inputs(raw, B, seed=B)
    off = np.random.default_rng(B).uniform(-0.1, 0.1, (len(ris), 3))
    args = (world, torch.tensor(s, dtype=dt, device=DEV), _nodes(world, names), torch.tensor(off, dtype=dt, device=DEV))
    out = f_j(*args, point_contacts=point, restitution=E)
    n, k, r = raw.ndof, len(ris), 3 if point else 6
    assert [tuple(x.shape) for x in out] == [(B, n), (B, k, r)] + [(B, n, n)] * 2 + [(B, k, r, n)] * 2 and all(x.dtype == dt for x in out)
    v, w = nb.impulse_dynamics(*args, point_contacts=point, restitution=E)
    assert torch.equal(_bits(out[0]), _bits(v)) and torch.equal(_bits(out[1]), _bits(w))  # NaN rows of singular worlds included
    out = _np(out)
    rows = sorted({0, B // 2, B - 1})
    emu = EmulImpjWorld(cm).impulse_dynamics_jacobians(s[rows], bodies, T, off, point=point, e=E, fp64=fp64)
    cast = (lambda a: a.astype(np.float64)) if fp64 else (lambda a: a.astype(np.float32).astype(np.float64))
    for i, wi in enumerate(rows):
        _, _, J, M, _ = oracle_imp(raw, cast(s[wi]), ris, cast(off), point, E, full=True)
        tol = 1e-9 if fp64 else min(1e-4 * np.linalg.cond(J @ np.linalg.solve(M, J.T)), 1.0)
        for a, b in zip(out[2:], emu[2:]):
            assert rel_err(a[wi], b[i]) < tol, (wi, rel_err(a[wi], b[i]), tol)


@pytest.mark.parametrize("name", ["free_child", "chain64"])
def test_other_models_fp64(name):
    raw = model_raw(name)
    world = built_world(name)
    cm = nb.device_model_for(world).cm
    flat = [b for sk in world.skeletons for b in sk._ordered_bodies()]
    ris = _free_child_nodes(raw) if name == "free_child" else [raw.nb - 1]
    bodies, T = canon_nodes(cm, ris)
    B = 2
    s = _inputs(raw, B, seed=21)
    off = np.random.default_rng(22).uniform(-0.1, 0.1, (B, len(ris), 3))
    args = (world, torch.tensor(s, dtype=torch.float64, device=DEV), [flat[x] for x in ris], torch.tensor(off, device=DEV))
    try:
        out = f_j(*args, point_contacts=True, restitution=E)
    except Nb2Error as e:  # a working set beyond shared memory even at one row slot
        assert name == "chain64" and "does not fit in shared memory" in str(e)
        return
    emu = EmulImpjWorld(cm).impulse_dynamics_jacobians(s, bodies, T, off, point=True, e=E, fp64=True)
    for a, b in zip(_np(out), emu):
        assert rel_err(a, b) < 1e-10


def _autograd_blocks(world, st, nodes, off, point, e=E, rho=0.0, mass=None):
    """the four blocks of torch.autograd.functional.jacobian of impulse_dynamics, per world (its diagonal over the batch)"""
    B, n = st.shape[0], st.shape[1] // 2
    f = lambda s_: nb.impulse_dynamics(world, s_, nodes, off, point_contacts=point, restitution=e, damping=rho, mass=mass)
    vs, ws = torch.autograd.functional.jacobian(f, st)
    ar = torch.arange(B)
    vs, ws = vs[ar, :, ar], ws[ar, :, :, ar]
    return [vs[..., :n], vs[..., n:], ws[..., :n], ws[..., n:]]


@pytest.mark.parametrize("names,point", [(FEET, False), (["l_foot", "r_hand"], True)])
@pytest.mark.parametrize("fp64", [False, True])
def test_blocks_match_autograd(names, point, fp64):
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    dt = torch.float64 if fp64 else torch.float32
    st = torch.tensor(_inputs(raw, 3, seed=71), dtype=dt, device=DEV)
    off = torch.tensor(np.random.default_rng(72).uniform(-0.1, 0.1, (3, len(names), 3)), dtype=dt, device=DEV)
    nodes = _nodes(world, names)
    out = f_j(world, st, nodes, off, point_contacts=point, restitution=E)
    ref = _autograd_blocks(world, st, nodes, off, point)
    for a, b in zip(_np(out[2:]), _np(ref)):
        assert rel_err(a, b) < (1e-10 if fp64 else 1e-4), rel_err(a, b)


@pytest.mark.parametrize("rho", [0.0, 1e-3])
@pytest.mark.parametrize("names,point", [(FEET, False), (LIMBS, True)])
def test_velocity_blocks_against_inverse_mass_matrix_and_world_jacobian(rho, names, point):
    """dv/dqdot- = I - (1 + e) M^-1 J^T A^-1 J; for point contacts also dLam/dqdot- = -(1 + e) A^-1 J (a 6-D impulse is about the origin)"""
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    n, B = raw.ndof, 4
    st = torch.tensor(_inputs(raw, B, seed=81), dtype=torch.float64, device=DEV)
    nodes = _nodes(world, names)
    out = f_j(world, st, nodes, point_contacts=point, restitution=E, damping=rho)
    Mi = nb.inverse_mass_matrix(world, st[:, :n])
    J = nb.world_jacobian(world, st[:, :n], nodes)[:, :, 3:] if point else nb.world_jacobian(world, st[:, :n], nodes)
    J = J.reshape(B, -1, n)
    A = J @ Mi @ J.transpose(1, 2) + rho * torch.eye(J.shape[1], dtype=torch.float64, device=DEV)
    ref = torch.eye(n, dtype=torch.float64, device=DEV) - (1 + E) * Mi @ J.transpose(1, 2) @ torch.linalg.solve(A, J)
    assert rel_err(out[3].cpu().numpy(), ref.cpu().numpy()) < 1e-9
    if point:
        assert rel_err(out[5].reshape(B, -1, n).cpu().numpy(), (-(1 + E) * torch.linalg.solve(A, J)).cpu().numpy()) < 1e-9


@pytest.mark.parametrize("rho", [0.0, 1e-3])
def test_position_block_satisfies_the_differentiated_constraint(rho):
    """J dv/dq + d(J(q) u)/dq |_(u = qdot+ + e qdot-) = -rho dLam/dq, with the second term from autograd through world_jacobian (point
    contacts: Lam is the returned impulse)"""
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    n, B = raw.ndof, 2
    st = torch.tensor(_inputs(raw, B, seed=91), dtype=torch.float64, device=DEV)
    nodes = _nodes(world, LIMBS)
    off = torch.tensor(np.random.default_rng(92).uniform(-0.1, 0.1, (4, 3)), device=DEV)
    out = f_j(world, st, nodes, off, point_contacts=True, restitution=E, damping=rho)
    u = out[0] + E * st[:, n:]
    dv_dq, dlam_dq = out[2], out[4].reshape(B, 12, n)

    def c(q):
        return (nb.world_jacobian(world, q, nodes, off)[:, :, 3:].reshape(B, 12, n) @ u[..., None])[..., 0]

    dc = torch.autograd.functional.jacobian(c, st[:, :n])
    dc = dc[torch.arange(B), :, torch.arange(B)]
    J = nb.world_jacobian(world, st[:, :n], nodes, off)[:, :, 3:].reshape(B, 12, n)
    res = J @ dv_dq + dc + rho * dlam_dq
    scale = float(dc.abs().max() + (J @ dv_dq).abs().max())
    assert float(res.abs().max()) < 1e-9 * scale


def test_per_world_masses_offsets_and_damping():
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=6)
    B = 3
    st = torch.tensor(_inputs(raw, B, seed=101), dtype=torch.float64, device=DEV)
    off = torch.tensor(np.random.default_rng(102).uniform(-0.1, 0.1, (B, 2, 3)), device=DEV)
    nodes = _nodes(world, FEET)
    Mv = torch.tensor(random_masses(world, B, seed=103), device=DEV)
    for mass in (Mv, Mv[1]):
        out = f_j(world, st, nodes, off, restitution=E, damping=1e-3, mass=mass)
        v, w = nb.impulse_dynamics(world, st, nodes, off, restitution=E, damping=1e-3, mass=mass)
        assert torch.equal(out[0], v) and torch.equal(out[1], w)
        ref = _autograd_blocks(world, st, nodes, off, False, E, 1e-3, mass)
        for a, b in zip(_np(out[2:]), _np(ref)):
            assert rel_err(a, b) < 1e-10


@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("B", [1, 33, 4099])
def test_kernel_writes_only_its_own_rows(fp64, B):
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    dm = nb.device_model_for(world)
    dt = torch.float64 if fp64 else torch.float32
    prec = nb.engine.FP64 if fp64 else nb.engine.FP32
    n, G = raw.ndof, 4096
    bodies, T12 = resolve_nodes(world, _nodes(world, FEET))
    st = torch.tensor(_inputs(raw, B, seed=15), dtype=dt, device=DEV)

    def guarded(numel):
        buf = torch.full((numel + 2 * G,), float("nan"), dtype=dt, device=DEV)
        return buf, buf[G:G + numel]

    bufs = [guarded(B * n), guarded(B * 12)] + [guarded(B * n * n) for _ in range(2)] + [guarded(B * 12 * n) for _ in range(2)]
    dm.impulse_dynamics_jacobians_device(B, st.data_ptr(), bodies, T12, None, False, False, E, 0.0, bufs[0][1].data_ptr(), bufs[1][1].data_ptr(),
                                         [o.data_ptr() for _, o in bufs[2:]], torch.cuda.current_stream().cuda_stream, prec)
    torch.cuda.synchronize()
    for buf, out in bufs:
        assert bool(buf[:G].isnan().all()) and bool(buf[-G:].isnan().all())
        assert bool(torch.isfinite(out).all())


def test_singular_world_empty_batch_and_single_row():
    raw, _, _, _, s, _, off = singular_middle_world()
    world = built_world("free_child")
    node = [b for sk in world.skeletons for b in sk._ordered_bodies()][raw.nb - 1]
    st, ot = (torch.tensor(x, dtype=torch.float64, device=DEV) for x in (s, off))
    out = f_j(world, st, [node], ot, point_contacts=True, restitution=E)
    for w in (0, 2):
        one = f_j(world, st[w:w + 1], [node], ot[w:w + 1], point_contacts=True, restitution=E)
        for a, b in zip(out, one):
            assert bool(a[1].isnan().all()) and bool(torch.isfinite(b).all()) and torch.equal(a[w:w + 1], b)
    assert all(bool(torch.isfinite(x).all()) for x in f_j(world, st, [node], ot, point_contacts=True, restitution=E, damping=1e-3))
    n = raw.ndof
    e = f_j(world, torch.zeros(0, 2 * n, device=DEV), [node], point_contacts=True)
    assert [tuple(x.shape) for x in e] == [(0, n), (0, 1, 3)] + [(0, n, n)] * 2 + [(0, 1, 3, n)] * 2
    single = f_j(world, st[2], [node], ot[2], point_contacts=True, restitution=E)
    assert [tuple(x.shape) for x in single] == [(n,), (1, 3)] + [(n, n)] * 2 + [(1, 3, n)] * 2
    for a, b in zip(single, out):
        assert torch.equal(a, b[2])
