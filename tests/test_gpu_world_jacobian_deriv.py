"""Time derivatives of the world Jacobians on the GPU (nb2_world_jacobian_deriv / nb2_com_jacobian_deriv and their backwards through
nimblephysics_b200.world_jacobian_deriv / com_jacobian_deriv) against the fp64 oracle of test_world_jacobian_deriv at partial-block batch
sizes; gradcheck to both halves of the state, offsets and mass; the COM acceleration of a free-floating robot equal to gravity through
the mass matrix and inverse dynamics; the point acceleration against differences of world_jacobian along the motion; a world with
collision pairs; the reference-named mirrors."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from tests.test_inverse_dynamics import id_inputs
from tests.test_mass_matrix import built_world, model_raw
from tests.test_per_world_mass import random_masses, register
from tests.test_world_jacobian_deriv import advance, oracle_com_deriv, oracle_point_deriv
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
    st = torch.tensor(s, dtype=dt, device=DEV)
    off = torch.tensor(np.random.default_rng(B).uniform(-0.1, 0.1, (B, 4, 3)), dtype=dt, device=DEV)
    dJ = nb.world_jacobian_deriv(world, st, _nodes(world, ATLAS_NODES), off)
    dJc = nb.com_jacobian_deriv(world, st, _robot(world))
    assert dJ.shape == (B, 4, 6, n) and dJ.dtype == dt and dJc.shape == (B, 3, n) and dJc.dtype == dt
    dJ, dJc, off = (x.cpu().numpy() for x in (dJ, dJc, off))
    tol = 1e-8 if fp64 else 1e-4
    cast = (lambda a: a.astype(np.float64)) if fp64 else (lambda a: a.astype(np.float32).astype(np.float64))
    root = _raw_index(raw, _robot(world)._ordered_bodies()[0].name)
    for w in sorted({0, B // 2, B - 1}):
        sw = cast(s[w])
        for e, name in enumerate(ATLAS_NODES):
            ref = oracle_point_deriv(raw, sw[:n], sw[n:], _raw_index(raw, name), off[w, e].astype(np.float64))
            assert rel_err(dJ[w, e], ref) < tol, (w, name)
        assert rel_err(dJc[w], oracle_com_deriv(raw, sw[:n], sw[n:], root)) < tol


@pytest.mark.parametrize("name", ["atlas_sdf", "free_child", "chain64", "free16", "limit"])
def test_other_models_against_the_oracle(name):
    raw = model_raw(name)
    world = nb.World.from_raw(raw) if name == "atlas_sdf" else built_world(name)
    n, B = raw.ndof, 33
    s, _ = id_inputs(raw, B, seed=17)
    nodes = [sk._ordered_bodies()[-1] for sk in world.skeletons if sk.getNumDofs() > 0]
    index = {id(b): k for k, b in enumerate(b for sk in world.skeletons for b in sk._ordered_bodies())}  # body names repeat across skeletons
    dJ = nb.world_jacobian_deriv(world, torch.tensor(s, dtype=torch.float64, device=DEV), nodes).cpu().numpy()
    # the oracle divides the rounding of its J (about 1e-11 relative at the end of the 64-link chain) by its step h = 1e-3: its error
    # there grows as 1/h (2.7e-8 at h = 2e-3, 5.8e-8 at 1e-3, 1.2e-7 at 5e-4 in world 32), so 1e-7 is the oracle's resolution
    tol = 1e-7 if name == "chain64" else 1e-8
    for w in (0, B - 1):
        sw = s[w].astype(np.float64)
        for e, b in enumerate(nodes):
            assert rel_err(dJ[w, e], oracle_point_deriv(raw, sw[:n], sw[n:], index[id(b)])) < tol


def test_gradcheck_fp64():
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=3)
    n, B = raw.ndof, 2
    s, _ = id_inputs(raw, B, seed=3)
    sk = _robot(world)
    nodes = _nodes(world, ["l_foot", "r_hand"])
    st = torch.tensor(s, dtype=torch.float64, device=DEV, requires_grad=True)
    o1 = torch.tensor(np.random.default_rng(1).uniform(-0.1, 0.1, (2, 3)), device=DEV, requires_grad=True)
    oB = torch.tensor(np.random.default_rng(2).uniform(-0.1, 0.1, (B, 2, 3)), device=DEV, requires_grad=True)
    assert torch.autograd.gradcheck(lambda x, o: nb.world_jacobian_deriv(world, x, nodes, o), (st, o1))
    assert torch.autograd.gradcheck(lambda x, o: nb.world_jacobian_deriv(world, x, nodes, o), (st, oB))
    mB = torch.tensor(random_masses(world, B, seed=4), device=DEV, requires_grad=True)
    assert torch.autograd.gradcheck(lambda x, m: nb.com_jacobian_deriv(world, x, sk, m), (st, mB))
    # a 1-D mass (setMasses, shared by the batch) gets the per-world gradients summed
    m0 = torch.tensor(world.getMasses().copy(), device=DEV)
    G = torch.randn(B, 3, n, dtype=torch.float64, device=DEV)
    m1 = m0.clone().requires_grad_(True)
    (nb.com_jacobian_deriv(world, st.detach(), sk, m1) * G).sum().backward()
    m2 = m0.repeat(B, 1).requires_grad_(True)
    (nb.com_jacobian_deriv(world, st.detach(), sk, m2) * G).sum().backward()
    assert rel_err(m1.grad.cpu().numpy(), m2.grad.sum(0).cpu().numpy()) < 1e-12


@pytest.mark.parametrize("name", ["atlas", "atlas_sdf"])
def test_com_of_a_floating_robot_accelerates_with_gravity(name):
    """qddot = M^-1 (tau - inverse_dynamics(q, qdot, qdot)), tau = 0 on the free root: no external wrench but gravity, so
    J_com qddot + Jdot_com qdot = g in every world (DESIGN §6h, §6j)."""
    raw = load_raw(name)
    world = nb.World.from_raw(raw)
    world._contacts_disabled = True
    n, B = raw.ndof, 7
    s, _ = id_inputs(raw, B, seed=19)
    st = torch.tensor(s, dtype=torch.float64, device=DEV)
    q, qd = st[:, :n], st[:, n:]
    sk = _robot(world)
    root = sk._ordered_bodies()[0]
    o = sk._dof_offset_in_world()[1]
    assert root.parent_joint.jtype == nb.world.FREE
    tau = torch.tensor(np.random.default_rng(20).uniform(-20, 20, (B, n)), device=DEV)
    tau[:, o:o + 6] = 0
    qdd = torch.einsum("bij,bj->bi", nb.inverse_mass_matrix(world, q), tau - nb.inverse_dynamics(world, st, qd))
    acc = torch.einsum("brn,bn->br", nb.com_jacobian(world, q, sk), qdd) + torch.einsum("brn,bn->br", nb.com_jacobian_deriv(world, st, sk), qd)
    g = np.asarray(raw.gravity, np.float64)
    for w in range(B):
        assert rel_err(acc[w].cpu().numpy(), g) < 1e-9, (w, acc[w])


def test_point_acceleration_matches_differences_along_the_motion():
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    n, B, h = raw.ndof, 3, 1e-4
    s, _ = id_inputs(raw, B, seed=23)
    s = s.astype(np.float64)
    nodes = _nodes(world, ATLAS_NODES)
    st = torch.tensor(s, device=DEV)
    qd = st[:, n:]
    dJ = nb.world_jacobian_deriv(world, st, nodes)
    mine = torch.einsum("bkrn,bn->bkr", dJ, qd).cpu().numpy()
    at = lambda t: torch.tensor(np.stack([advance(raw, s[w, :n], s[w, n:], t) for w in range(B)]), device=DEV)
    Jq = lambda t: torch.einsum("bkrn,bn->bkr", nb.world_jacobian(world, at(t), nodes), qd).cpu().numpy()
    fd = (Jq(h) - Jq(-h)) / (2 * h)
    assert rel_err(mine, fd) < 1e-6


def test_world_with_collision_pairs_keeps_the_lcp_cache_and_mirrors():
    raw = load_raw("half_cheetah")
    world = nb.World.from_raw(raw)
    n, B = raw.ndof, 4
    cs, ca = contact_inputs(raw, "half_cheetah", B, seed=13)
    nb.timestep(world, torch.tensor(cs, device=DEV), torch.tensor(ca, device=DEV))  # fills the LCP cache
    cache = world._lcp_cache
    before = {k: v.clone() for k, v in cache.items() if torch.is_tensor(v)}
    sk = _robot(world)
    st = torch.tensor(cs, dtype=torch.float64, device=DEV)
    nb.world_jacobian_deriv(world, st, [sk._ordered_bodies()[-1]])
    nb.com_jacobian_deriv(world, st, sk)
    assert world._lcp_cache is cache and all(torch.equal(cache[k], v) for k, v in before.items())

    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    s, _ = id_inputs(raw, 1, seed=29)
    world.setState(s[0].astype(np.float64))
    sk = _robot(world)
    node = _nodes(world, ["l_hand"])[0]
    st = torch.tensor(np.concatenate([world.getPositions(), world.getVelocities()]).astype(np.float64), device=DEV)
    o = np.array([0.05, 0.1, -0.02])
    w, off = sk._dof_offset_in_world()
    k = sk.getNumDofs()
    dJ = nb.world_jacobian_deriv(world, st, [node], torch.tensor(o[None], device=DEV))[0].cpu().numpy()[:, off:off + k]
    dJc = nb.com_jacobian_deriv(world, st, sk).cpu().numpy()[:, off:off + k]
    assert np.any(dJ != 0)
    assert np.array_equal(sk.getJacobianClassicDeriv(node, o), dJ) and sk.getJacobianClassicDeriv(node, o).dtype == np.float64
    assert np.array_equal(sk.getLinearJacobianDeriv(node, o), dJ[3:]) and np.array_equal(sk.getCOMLinearJacobianDeriv(), dJc)
    dJ0 = nb.world_jacobian_deriv(world, st, [node])[0].cpu().numpy()[:, off:off + k]
    assert np.array_equal(sk.getAngularJacobianDeriv(node), dJ0[:3])
