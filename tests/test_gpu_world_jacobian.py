"""World Jacobians on the GPU (nb2_world_jacobian / nb2_com_jacobian and their backwards through nimblephysics_b200.world_jacobian /
com_jacobian) against the fp64 oracle of test_world_jacobian at partial-block batch sizes; gradcheck to positions, offsets and mass;
consistency with map_to_vel, the IK COM entry, IKMapping.getRealVelToMappedVelJac and contact_inverse_dynamics; a world with collision
pairs; the reference-named mirrors."""
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import nimblephysics_b200 as nb
from oracle.binding import OracleWorld
from tests.test_inverse_dynamics import id_inputs
from tests.test_mass_matrix import built_world, model_raw
from tests.test_per_world_mass import random_masses, raw_at, register
from tests.test_world_jacobian import oracle_com, oracle_point
from tests.util import contact_inputs, load_raw, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
ATLAS_NODES = ["l_foot", "r_foot", "l_hand", "r_hand"]


def _nodes(world, names):
    by = {b.name: b for sk in world.skeletons for b in sk._ordered_bodies()}
    return [by[k] for k in names]


def _raw_index(raw, name):
    return list(raw.body_names).index(name)


def _robot(world):
    return max(world.skeletons, key=lambda s: s.getNumDofs())


@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("B", [1, 3, 33, 4099])
def test_forward_matches_oracle(fp64, B):
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    n, dt = raw.ndof, torch.float64 if fp64 else torch.float32
    s, _ = id_inputs(raw, B, seed=B)
    q = torch.tensor(s[:, :n], dtype=dt, device=DEV)
    off = torch.tensor(np.random.default_rng(B).uniform(-0.1, 0.1, (B, 4, 3)), dtype=dt, device=DEV)
    J = nb.world_jacobian(world, q, _nodes(world, ATLAS_NODES), off)
    J0 = nb.world_jacobian(world, q, _nodes(world, ATLAS_NODES))
    Jc = nb.com_jacobian(world, q, _robot(world))
    assert J.shape == (B, 4, 6, n) and J.dtype == dt and Jc.shape == (B, 3, n) and Jc.dtype == dt
    J, J0, Jc, off = (x.cpu().numpy() for x in (J, J0, Jc, off))
    tol = 1e-9 if fp64 else 1e-4
    cast = (lambda a: a.astype(np.float64)) if fp64 else (lambda a: a.astype(np.float32).astype(np.float64))
    root = _raw_index(raw, _robot(world)._ordered_bodies()[0].name)
    for w in sorted({0, B // 2, B - 1}):
        qw = cast(s[w, :n])
        for e, name in enumerate(ATLAS_NODES):
            ri = _raw_index(raw, name)
            assert rel_err(J[w, e], oracle_point(raw, qw, ri, off[w, e].astype(np.float64))) < tol, (w, name)
            assert rel_err(J0[w, e], oracle_point(raw, qw, ri)) < tol, (w, name)
        assert rel_err(Jc[w], oracle_com(raw, qw, root)) < tol


@pytest.mark.parametrize("name", ["free_child", "chain64", "free16", "limit"])
def test_compiled_limits_against_the_oracle(name):
    raw = model_raw(name)
    world = built_world(name)
    n, B = raw.ndof, 33
    s, _ = id_inputs(raw, B, seed=17)
    nodes = [sk._ordered_bodies()[-1] for sk in world.skeletons]
    index = {id(b): k for k, b in enumerate(b for sk in world.skeletons for b in sk._ordered_bodies())}  # body names repeat across skeletons
    J = nb.world_jacobian(world, torch.tensor(s[:, :n], dtype=torch.float64, device=DEV), nodes).cpu().numpy()
    for w in (0, B - 1):
        for e, b in enumerate(nodes):
            assert rel_err(J[w, e], oracle_point(raw, s[w, :n].astype(np.float64), index[id(b)])) < 1e-9


def test_gradcheck_fp64():
    raw = load_raw("half_cheetah")
    world = register(nb.World.from_raw(raw), step=2)
    n, B = raw.ndof, 2
    s, _ = id_inputs(raw, B, seed=3)
    sk = _robot(world)
    nodes = [sk._ordered_bodies()[-1], sk._ordered_bodies()[len(sk._ordered_bodies()) // 2]]
    q = torch.tensor(s[:, :n], dtype=torch.float64, device=DEV, requires_grad=True)
    o1 = torch.tensor(np.random.default_rng(1).uniform(-0.1, 0.1, (2, 3)), device=DEV, requires_grad=True)
    oB = torch.tensor(np.random.default_rng(2).uniform(-0.1, 0.1, (B, 2, 3)), device=DEV, requires_grad=True)
    assert torch.autograd.gradcheck(lambda x, o: nb.world_jacobian(world, x, nodes, o), (q, o1))
    assert torch.autograd.gradcheck(lambda x, o: nb.world_jacobian(world, x, nodes, o), (q, oB))
    mB = torch.tensor(random_masses(world, B, seed=4), device=DEV, requires_grad=True)
    assert torch.autograd.gradcheck(lambda x, m: nb.com_jacobian(world, x, sk, m), (q, mB))
    # a 1-D mass goes through setMasses, which gradcheck's in-place perturbations bypass: central differences of the oracle instead,
    # summed over the batch
    m0 = world.getMasses().copy()
    m1 = torch.tensor(m0, device=DEV, requires_grad=True)
    G = np.random.default_rng(5).normal(size=(B, 3, n))
    (nb.com_jacobian(world, q.detach(), sk, m1) * torch.tensor(G, device=DEV)).sum().backward()
    entries, root = world._mass_entries(), _raw_index(raw, sk._ordered_bodies()[0].name)
    loss = lambda m: sum(float(np.sum(G[w] * oracle_com(raw_at(raw, entries, m), s[w, :n].astype(np.float64), root))) for w in range(B))
    fd = np.array([(loss(m0 + 1e-6 * e) - loss(m0 - 1e-6 * e)) / 2e-6 for e in np.eye(len(m0))])
    assert rel_err(m1.grad.cpu().numpy(), fd) < 1e-7


def test_per_world_mass_gradient_matches_oracle():
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=3)
    n, B = raw.ndof, 3
    s, _ = id_inputs(raw, B, seed=7)
    mv = random_masses(world, B, seed=8)
    G = np.random.default_rng(9).normal(size=(B, 3, n))
    m0 = world.getMasses().copy()
    mass = torch.tensor(mv, device=DEV, requires_grad=True)
    q = torch.tensor(s[:, :n], dtype=torch.float64, device=DEV)
    (nb.com_jacobian(world, q, _robot(world), mass) * torch.tensor(G, device=DEV)).sum().backward()
    assert np.array_equal(world.getMasses(), m0)
    entries = world._mass_entries()
    root = _raw_index(raw, _robot(world)._ordered_bodies()[0].name)
    for w in range(B):
        loss = lambda m: float(np.sum(G[w] * oracle_com(raw_at(raw, entries, m), s[w, :n].astype(np.float64), root)))
        fd = np.array([(loss(mv[w] + 1e-6 * e) - loss(mv[w] - 1e-6 * e)) / 2e-6 for e in np.eye(len(mv[w]))])
        assert rel_err(mass.grad[w].cpu().numpy(), fd) < 1e-7


def test_consistent_with_map_to_vel_and_the_ik_com_entry():
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    n, B = raw.ndof, 65
    s, _ = id_inputs(raw, B, seed=11)
    st = torch.tensor(s, dtype=torch.float32, device=DEV)
    nodes = _nodes(world, ATLAS_NODES)
    ik = nb.IKMapping(world)
    for b in nodes:
        ik.addSpatialBodyNode(b)
    ik.addSkeletonCOM(_robot(world))
    v = nb.map_to_vel(world, ik, st)
    J = nb.world_jacobian(world, st[:, :n], nodes)
    Jc = nb.com_jacobian(world, st[:, :n], _robot(world))
    qd = st[:, n:]
    mine = torch.cat([torch.einsum("bkrn,bn->bkr", J, qd).reshape(B, -1), torch.einsum("brn,bn->br", Jc, qd)], 1)
    assert rel_err(mine.cpu().numpy(), v.cpu().numpy()) < 1e-5
    world.setState(s[0].astype(np.float64))
    ref = ik.getRealVelToMappedVelJac()
    rows = torch.cat([J[0].reshape(-1, n), Jc[0]]).double().cpu().numpy()
    assert rel_err(rows, ref) < 1e-5


def test_contact_inverse_dynamics_identity():
    """With offsets that put each foot's point at the world origin, J_c^T wrench = tau_ID - tau of contact_inverse_dynamics (DESIGN §6f)."""
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    world._contacts_disabled = True
    n, B = raw.ndof, 5
    s, vn = id_inputs(raw, B, seed=13)
    st = torch.tensor(s, dtype=torch.float64, device=DEV)
    vt = torch.tensor(vn, dtype=torch.float64, device=DEV)
    ow = OracleWorld(raw)
    for name in ("l_foot", "r_foot"):
        node = _nodes(world, [name])[0]
        off = np.zeros((B, 1, 3))
        for w in range(B):
            pos, _, _, _ = ow.ik(s[w].astype(np.float64), [0], [_raw_index(raw, name)], want_jac=False)
            off[w, 0] = -Rotation.from_rotvec(pos[:3]).as_matrix().T @ pos[3:]
        Jc = nb.world_jacobian(world, st[:, :n], [node], torch.tensor(off, device=DEV))[:, 0]
        tau, wr = nb.contact_inverse_dynamics(world, st, vt, node)
        tid = nb.inverse_dynamics(world, st, vt)
        lhs = torch.einsum("brn,br->bn", Jc, wr)
        assert rel_err(lhs.cpu().numpy(), (tid - tau).cpu().numpy()) < 1e-10


def test_world_with_collision_pairs_keeps_the_lcp_cache_and_mirrors():
    raw = load_raw("half_cheetah")
    world = nb.World.from_raw(raw)
    n, B = raw.ndof, 4
    cs, ca = contact_inputs(raw, "half_cheetah", B, seed=13)
    nb.timestep(world, torch.tensor(cs, device=DEV), torch.tensor(ca, device=DEV))  # fills the LCP cache
    cache = world._lcp_cache
    before = {k: v.clone() for k, v in cache.items() if torch.is_tensor(v)}
    sk = _robot(world)
    node = sk._ordered_bodies()[-1]
    q = torch.tensor(cs[:, :n], dtype=torch.float64, device=DEV)
    nb.world_jacobian(world, q, [node])
    assert world._lcp_cache is cache and all(torch.equal(cache[k], v) for k, v in before.items())

    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    sk = _robot(world)
    node = _nodes(world, ["l_hand"])[0]
    q = torch.tensor(np.asarray(world.getPositions(), np.float64), device=DEV)
    o = np.array([0.05, 0.1, -0.02])
    w, off = sk._dof_offset_in_world()
    k = sk.getNumDofs()
    J = nb.world_jacobian(world, q, [node], torch.tensor(o[None], device=DEV))[0].cpu().numpy()[:, off:off + k]
    Jc = nb.com_jacobian(world, q, sk).cpu().numpy()[:, off:off + k]
    assert np.array_equal(sk.getWorldJacobian(node, o), J) and sk.getWorldJacobian(node, o).dtype == np.float64
    assert np.array_equal(sk.getLinearJacobian(node, o), J[3:]) and np.array_equal(sk.getCOMLinearJacobian(), Jc)
    J0 = nb.world_jacobian(world, q, [node])[0].cpu().numpy()[:, off:off + k]
    assert np.array_equal(sk.getAngularJacobian(node), J0[:3])
