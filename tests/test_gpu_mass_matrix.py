"""Mass matrix and its inverse on the GPU (nb2_mass_matrix / nb2_inverse_mass_matrix and their backwards through
nimblephysics_b200.mass_matrix / inverse_mass_matrix) against the fp64 inverse-dynamics oracle: M e_j = ID(q, 0, dt e_j) - ID(q, 0, 0),
M^-1 = inv(M); position and per-world mass gradients against central differences of the oracle; exact symmetry; a free root's pose;
consistency with inverse_dynamics and nb2_forward_dynamics; a world with collision pairs."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from tests.oracle_id.binding import IdOracle
from tests.test_inverse_dynamics import id_inputs
from tests.test_mass_matrix import _blocks, built_world, model_raw, oracle_M
from tests.test_per_world_mass import random_masses, raw_at, register
from tests.util import contact_inputs, load_raw, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _worlds(B):
    return sorted({0, B // 2, B - 1})


@pytest.mark.parametrize("name", ["cartpole", "half_cheetah", "atlas", "atlas_sdf"])
@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("B", [1, 3, 33, 4099])
def test_forward_matches_oracle_and_is_symmetric(name, fp64, B):
    raw = load_raw(name)
    world = nb.World.from_raw(raw)
    n, dt = raw.ndof, torch.float64 if fp64 else torch.float32
    s, _ = id_inputs(raw, B, seed=B)
    q = torch.tensor(s[:, :n], dtype=dt, device=DEV)
    M = nb.mass_matrix(world, q)
    Mi = nb.inverse_mass_matrix(world, q)
    assert M.shape == (B, n, n) and Mi.shape == (B, n, n) and M.dtype == dt
    assert torch.equal(M, M.transpose(1, 2)) and torch.equal(Mi, Mi.transpose(1, 2))
    M, Mi = M.cpu().numpy(), Mi.cpu().numpy()
    tol = 1e-9 if fp64 else 1e-4
    for w in _worlds(B):
        Mo = oracle_M(raw, s[w, :n].astype(np.float64) if fp64 else s[w, :n].astype(np.float32).astype(np.float64))
        assert rel_err(M[w], Mo) < tol, (w, rel_err(M[w], Mo))
        assert rel_err(Mi[w], np.linalg.inv(Mo)) < tol, (w, rel_err(Mi[w], np.linalg.inv(Mo)), np.linalg.cond(Mo))


@pytest.mark.parametrize("name", ["cartpole", "half_cheetah", "atlas", "atlas_sdf"])
@pytest.mark.parametrize("inverse", [False, True])
def test_position_and_per_world_mass_gradients(name, inverse):
    raw = load_raw(name)
    world = register(nb.World.from_raw(raw), step=3)
    n, B = raw.ndof, 3
    s, _ = id_inputs(raw, B, seed=7)
    q0 = s[:, :n].astype(np.float64)
    mv = random_masses(world, B, seed=8)
    rng = np.random.default_rng(9)
    G = rng.normal(size=(B, n, n))
    q = torch.tensor(q0, device=DEV, requires_grad=True)
    mass = torch.tensor(mv, device=DEV, requires_grad=True)
    m0 = world.getMasses().copy()
    out = (nb.inverse_mass_matrix if inverse else nb.mass_matrix)(world, q, mass)
    (out * torch.tensor(G, device=DEV)).sum().backward()
    assert np.array_equal(world.getMasses(), m0)
    gq, gm = q.grad.cpu().numpy(), mass.grad.cpu().numpy()
    entries = world._mass_entries()
    f = (lambda r, x: np.linalg.inv(oracle_M(r, x))) if inverse else oracle_M
    for w in range(B):
        rw = raw_at(raw, entries, mv[w])
        loss = lambda x: float(np.sum(G[w] * f(rw, x)))
        hq, h = 1e-5, 1e-6  # the oracle's M comes from differences of inverse-dynamics forces: a smaller q-step only adds their rounding
        fd = np.array([(loss(q0[w] + hq * e) - loss(q0[w] - hq * e)) / (2 * hq) for e in np.eye(n)])
        assert rel_err(gq[w], fd) < 1e-6, (w, rel_err(gq[w], fd))
        lm = lambda m: float(np.sum(G[w] * f(raw_at(raw, entries, m), q0[w])))
        fdm = np.array([(lm(mv[w] + h * e) - lm(mv[w] - h * e)) / (2 * h) for e in np.eye(len(mv[w]))])  # M^-1 is not quadratic in the mass
        assert rel_err(gm[w], fdm) < 1e-6, (w, rel_err(gm[w], fdm))


def test_gradcheck_fp64():
    raw = load_raw("cartpole")
    world = nb.World.from_raw(raw)
    s, _ = id_inputs(raw, 2, seed=3)
    q = torch.tensor(s[:, :raw.ndof], dtype=torch.float64, device=DEV, requires_grad=True)
    assert torch.autograd.gradcheck(lambda x: nb.mass_matrix(world, x), (q,))
    assert torch.autograd.gradcheck(lambda x: nb.inverse_mass_matrix(world, x), (q,))


def test_shared_mass_gradient_sums_over_the_batch():
    raw = load_raw("half_cheetah")
    world = register(nb.World.from_raw(raw), step=2)
    B, n = 5, raw.ndof
    s, _ = id_inputs(raw, B, seed=2)
    m0 = world.getMasses().copy()
    mass = torch.tensor(m0, device=DEV, requires_grad=True)
    q = torch.tensor(s[:, :n], dtype=torch.float64, device=DEV)
    G = np.random.default_rng(4).normal(size=(B, n, n))
    (nb.mass_matrix(world, q, mass) * torch.tensor(G, device=DEV)).sum().backward()
    entries = world._mass_entries()
    loss = lambda m: sum(float(np.sum(G[w] * oracle_M(raw_at(raw, entries, m), s[w, :n].astype(np.float64)))) for w in range(B))
    fd = np.array([(loss(m0 + 1e-4 * e) - loss(m0 - 1e-4 * e)) / 2e-4 for e in np.eye(len(m0))])
    assert rel_err(mass.grad.cpu().numpy(), fd) < 1e-6


@pytest.mark.parametrize("fp64", [False, True])
def test_free_root_pose_does_not_change_M_and_gets_no_gradient(fp64):
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    n, dt = raw.ndof, torch.float64 if fp64 else torch.float32
    s, _ = id_inputs(raw, 8, seed=5)
    q = torch.tensor(s[:, :n], dtype=dt, device=DEV)
    q2 = q.clone()
    q2[:, :6] = torch.tensor(np.random.default_rng(6).uniform(-2, 2, (8, 6)), dtype=dt, device=DEV)
    assert torch.equal(nb.mass_matrix(world, q), nb.mass_matrix(world, q2))
    for f in (nb.mass_matrix, nb.inverse_mass_matrix):
        qq = q2.clone().requires_grad_(True)
        (f(world, qq) * torch.randn(8, n, n, dtype=dt, device=DEV)).sum().backward()
        assert torch.all(qq.grad[:, :6] == 0)


@pytest.mark.parametrize("name", ["half_cheetah", "atlas"])
def test_consistent_with_inverse_dynamics_and_forward_dynamics(name):
    raw = load_raw(name)
    world = nb.World.from_raw(raw)
    world._contacts_disabled = True
    n, B = raw.ndof, 33
    s, vn = id_inputs(raw, B, seed=11)
    st = torch.tensor(s, dtype=torch.float64, device=DEV)
    vt = torch.tensor(vn, dtype=torch.float64, device=DEV)
    q, qd = st[:, :n], st[:, n:]
    M = nb.mass_matrix(world, q)
    Mi = nb.inverse_mass_matrix(world, q)
    bias = nb.inverse_dynamics(world, st, qd)
    lhs = nb.inverse_dynamics(world, st, vt) - bias
    rhs = torch.einsum("bij,bj->bi", M, vt - qd) / raw.dt
    assert rel_err(lhs.cpu().numpy(), rhs.cpu().numpy()) < 1e-9
    tau = torch.tensor(np.random.default_rng(12).uniform(-20, 20, (B, n)), dtype=torch.float64, device=DEV)
    dm = nb.device_model_for(world)
    if dm.na == dm.ndof:
        acc = dm.forward_dynamics(q, qd, tau)
        ref = torch.einsum("bij,bj->bi", Mi, tau - bias)
        assert rel_err(acc.cpu().numpy(), ref.cpu().numpy()) < 1e-9


def test_world_with_collision_pairs_gives_its_trees_M_and_keeps_the_lcp_cache():
    raw = load_raw("half_cheetah")
    world = nb.World.from_raw(raw)
    free = nb.World.from_raw(raw)
    free._contacts_disabled = True
    n, B = raw.ndof, 4
    cs, ca = contact_inputs(raw, "half_cheetah", B, seed=13)
    nb.timestep(world, torch.tensor(cs, device=DEV), torch.tensor(ca, device=DEV))  # fills the LCP cache
    cache = world._lcp_cache
    assert cache is not None
    before = {k: v.clone() for k, v in cache.items() if torch.is_tensor(v)}
    q = torch.tensor(cs[:, :n], dtype=torch.float64, device=DEV)
    assert torch.equal(nb.mass_matrix(world, q), nb.mass_matrix(free, q))
    assert torch.equal(nb.inverse_mass_matrix(world, q), nb.inverse_mass_matrix(free, q))
    assert world._lcp_cache is cache and all(torch.equal(cache[k], v) for k, v in before.items())


@pytest.mark.parametrize("name", ["free_child", "chain64", "free16", "limit"])
@pytest.mark.parametrize("fp64", [False, True])
def test_compiled_limits_several_skeletons_and_a_non_root_free_joint(name, fp64):
    """The largest models the step accepts (64 bodies; 96 dofs; 61 bodies with 96 dofs, the largest M^-1 working set), exact zeros off the
    skeletons' blocks, and a free joint below another joint, against the oracle; the position gradient against central differences."""
    raw = model_raw(name)
    world = built_world(name)
    n, B, dt = raw.ndof, 33, torch.float64 if fp64 else torch.float32
    s, _ = id_inputs(raw, B, seed=17)
    q = torch.tensor(s[:, :n], dtype=dt, device=DEV, requires_grad=True)
    M = nb.mass_matrix(world, q)
    Mi = nb.inverse_mass_matrix(world, q)
    blk = _blocks(raw)
    assert torch.all(M[:, ~torch.tensor(blk, device=DEV)] == 0) and torch.all(Mi[:, ~torch.tensor(blk, device=DEV)] == 0)
    assert torch.equal(M, M.transpose(1, 2)) and torch.equal(Mi, Mi.transpose(1, 2))
    G = torch.randn(B, n, n, dtype=dt, device=DEV, generator=torch.Generator(DEV).manual_seed(1))
    (gM,) = torch.autograd.grad((M * G).sum(), q)
    (gI,) = torch.autograd.grad((Mi * G).sum(), q)
    tol = 1e-9 if fp64 else 1e-4
    for w in (0, B - 1):
        qw = q[w].detach().cpu().numpy().astype(np.float64)
        Mo = oracle_M(raw, qw)
        assert rel_err(M[w].detach().cpu().numpy(), Mo) < tol and rel_err(Mi[w].detach().cpu().numpy(), np.linalg.inv(Mo)) < tol
    if fp64 and name in ("free_child", "limit"):
        Gw, h = G[0].cpu().numpy(), 1e-5
        qw = q[0].detach().cpu().numpy()
        for g, f in ((gM, oracle_M), (gI, lambda r, x: np.linalg.inv(oracle_M(r, x)))):
            fd = np.array([(np.sum(Gw * f(raw, qw + h * e)) - np.sum(Gw * f(raw, qw - h * e))) / (2 * h) for e in np.eye(n)])
            assert rel_err(g[0].cpu().numpy(), fd) < 1e-6


def test_reference_named_mirrors():
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    M = world.getMassMatrix()
    Mo = oracle_M(raw, np.asarray(world.getPositions(), dtype=np.float64))
    assert M.dtype == np.float64 and rel_err(M, Mo) < 1e-9
    assert rel_err(world.getInvMassMatrix(), np.linalg.inv(Mo)) < 1e-9
    sk = world.skeletons[-1]
    k = sk.getNumDofs()
    off = n0 = world.getNumDofs() - k
    assert rel_err(sk.getMassMatrix(), Mo[off:off + k, off:off + k]) < 1e-9 and n0 >= 0
    assert rel_err(sk.getInvMassMatrix(), np.linalg.inv(Mo)[off:off + k, off:off + k]) < 1e-9
