"""Dense Jacobians of contact-free inverse and forward dynamics on the CPU: the stage functions of csrc/nb2_djac.cuh (host build, poisoned
working set, reversed lane and slot orders) against the dual-number Jacobian of the inverse-dynamics oracle, against the emulated VJPs of
inverse_dynamics / forward_dynamics seeded with the identity, across lane schedules and row-slot counts, with per-world masses, and the
argument checks of nimblephysics_b200.inverse_dynamics_jacobians / forward_dynamics_jacobians."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from tests.host_emul.binding_djac import EmulDjacWorld
from tests.host_emul.binding_fd import EmulFdWorld
from tests.host_emul.binding_id import EmulIdWorld
from tests.oracle_id.binding import IdOracle
from tests.test_forward_dynamics import fd_inputs
from tests.test_inverse_dynamics import _compile, id_inputs
from tests.test_mass_matrix import MODELS, model_raw
from tests.test_per_world_mass import random_masses, raw_at, register
from tests.util import load_raw, rel_err


def oracle_id_blocks(ow, n, s, vn):
    """(tau, dtau/dq, dtau/dqdot, dtau/dv') of the oracle in fp64."""
    tau, J = ow.inverse_dynamics(np.asarray(s, np.float64), np.asarray(vn, np.float64), want_jac=True)
    return tau, J[:, :n], J[:, n:2 * n], J[:, 2 * n:]


def oracle_fd_blocks(ow, n, dt, s, tau):
    """(qdd, dqdd/dq, dqdd/dqdot, dqdd/dtau) of the oracle by the implicit-function theorem.  ID is affine in v', so
    v' = qdot + A_v'^-1 (tau - ID(q, qdot, qdot)) exactly, and at that v' with A = dID/d[q; qdot; v']:
        dqdd/dtau = A_v'^-1 / dt ,  dqdd/dq = -A_v'^-1 A_q / dt ,  dqdd/dqdot = -(A_v'^-1 A_qdot + I) / dt = -A_v'^-1 (A_qdot + A_v') / dt .
    The last form is the one evaluated: A_qdot + A_v' cancels the -M/dt of A_qdot in one fp64 sum, where A_v'^-1 A_qdot + I would cancel
    after a solve and lose the condition number of M times 1/dt in digits."""
    s = np.asarray(s, np.float64)
    v = s[n:]
    t0, _, _, Av = oracle_id_blocks(ow, n, s, v)
    vn = v + np.linalg.solve(Av, np.asarray(tau, np.float64) - t0)
    _, Aq, Aqd, Av = oracle_id_blocks(ow, n, s, vn)
    Ai = np.linalg.inv(Av)
    return (vn - v) / dt, -Ai @ Aq / dt, -Ai @ (Aqd + Av) / dt, Ai / dt


def fd_tol(ow, n, s, fp64):
    """Tolerance of the FD blocks against oracle_fd_blocks.  Both sides solve with M (the oracle explicitly, the kernels through the
    articulated inertias), so each carries a rounding of eps cond(M) times a factor that grows with the sums over n dofs: cond(M) is 6e4 on
    Atlas and 5e5 on the 64-link chain, where the fp64 blocks differ by up to about 7 and 40 eps cond(M)."""
    if not fp64:
        return 1e-4
    return max(1e-9, 1000 * np.finfo(np.float64).eps * np.linalg.cond(oracle_id_blocks(ow, n, s, np.asarray(s, np.float64)[n:])[3]))


@pytest.mark.parametrize("name", MODELS)
@pytest.mark.parametrize("fp64", [False, True])
def test_emulated_id_jacobians_match_oracle(name, fp64):
    raw = model_raw(name)
    n, B = raw.ndof, 2  # the odd world runs its lanes in reverse
    ew, ow = EmulDjacWorld(nb.compile_model(raw, lanes=1)), IdOracle(raw)
    s, vn = id_inputs(raw, B, seed=41)
    got = ew.dynamics_jacobians(s, vn, False, fp64)
    tol = 1e-9 if fp64 else 1e-4
    for w in range(B):
        for k, ref in enumerate(oracle_id_blocks(ow, n, s[w], vn[w])):
            assert rel_err(got[k][w], ref) < tol, (w, k, rel_err(got[k][w], ref))


@pytest.mark.parametrize("name", MODELS)
@pytest.mark.parametrize("fp64", [False, True])
def test_emulated_fd_jacobians_match_oracle(name, fp64):
    raw = model_raw(name)
    n, B = raw.ndof, 2
    ew, ow = EmulDjacWorld(nb.compile_model(raw, lanes=1)), IdOracle(raw)
    s, tau = fd_inputs(raw, B, seed=43)
    got = ew.dynamics_jacobians(s, tau, True, fp64)
    for w in range(B):
        tol = fd_tol(ow, n, s[w], fp64)
        for k, ref in enumerate(oracle_fd_blocks(ow, n, raw.dt, s[w], tau[w])):
            assert rel_err(got[k][w], ref) < tol, (w, k, rel_err(got[k][w], ref))


@pytest.mark.parametrize("name", ["cartpole", "tree", "half_cheetah", "atlas", "free_child", "limit"])
@pytest.mark.parametrize("fp64", [False, True])
def test_rows_are_the_emulated_vjps_seeded_with_the_identity(name, fp64):
    """Row i of each block is the existing inverse_dynamics / forward_dynamics VJP with grad = e_i: the same stage functions, the same bits."""
    raw = model_raw(name)
    n, B = raw.ndof, 3
    cm = nb.compile_model(raw, lanes=1)
    ew, ei, ef = EmulDjacWorld(cm), EmulIdWorld(cm), EmulFdWorld(cm)
    s, vn = id_inputs(raw, B, seed=45)
    _, tau = fd_inputs(raw, B, seed=46)
    tau_j, Jq, Jv, Jn = ew.dynamics_jacobians(s, vn, False, fp64)
    qdd_j, Fq, Fv, Ft = ew.dynamics_jacobians(s, tau, True, fp64)
    tau_e, saved_id = ei.inverse_dynamics(s, vn, fp64)
    qdd_e, saved_fd = ef.forward_dynamics(s, tau, fp64)
    assert np.array_equal(tau_j, tau_e) and np.array_equal(qdd_j, qdd_e)
    for i in range(n):
        seed = np.zeros((B, n))
        seed[:, i] = 1
        gs, gn, _ = ei.inverse_dynamics_backward(s, saved_id, seed, fp64)
        assert np.array_equal(Jq[:, i], gs[:, :n]) and np.array_equal(Jv[:, i], gs[:, n:]) and np.array_equal(Jn[:, i], gn), i
        gs, gt, _ = ef.forward_dynamics_backward(s, saved_fd, seed, fp64)
        assert np.array_equal(Fq[:, i], gs[:, :n]) and np.array_equal(Fv[:, i], gs[:, n:]) and np.array_equal(Ft[:, i], gt), i


@pytest.mark.parametrize("name", ["cartpole", "tree", "half_cheetah", "atlas", "atlas_sdf"])
@pytest.mark.parametrize("lanes", [2, 4, 8])
def test_lane_schedules_and_row_slots_agree(name, lanes):
    raw = model_raw(name)
    ew1, ewk = EmulDjacWorld(nb.compile_model(raw, lanes=1)), EmulDjacWorld(_compile(raw, lanes))
    s, vn = id_inputs(raw, 3, seed=47 + lanes)
    _, tau = fd_inputs(raw, 3, seed=48 + lanes)
    for fd, x in ((False, vn), (True, tau)):
        ref = ew1.dynamics_jacobians(s, x, fd, True, slots=32)
        for slots in (4, 8, 16, 32):
            got = ewk.dynamics_jacobians(s, x, fd, True, slots=slots)
            for a, b in zip(got, ref):
                assert rel_err(a, b) < 1e-12, (fd, slots, rel_err(a, b))


@pytest.mark.parametrize("name", ["half_cheetah", "atlas"])
def test_per_world_mass_is_set_masses_per_world(name):
    raw = load_raw(name)
    world = register(nb.World.from_raw(raw), step=4)
    n, B = raw.ndof, 3
    M = random_masses(world, B, seed=19)
    wi = nb.mass_to_inertia(world, torch.tensor(M, dtype=torch.float64)).numpy()
    ew = EmulDjacWorld(nb.compile_model(raw, lanes=2))
    s, vn = id_inputs(raw, B, seed=21)
    _, tau = fd_inputs(raw, B, seed=22)
    gid = ew.dynamics_jacobians(s, vn, False, True, world_inertia=wi)
    gfd = ew.dynamics_jacobians(s, tau, True, True, world_inertia=wi)
    entries = world._mass_entries()
    for w in range(B):
        ow = IdOracle(raw_at(raw, entries, M[w]))
        for k, ref in enumerate(oracle_id_blocks(ow, n, s[w], vn[w])):
            assert rel_err(gid[k][w], ref) < 1e-9, (w, k)
        for k, ref in enumerate(oracle_fd_blocks(ow, n, raw.dt, s[w], tau[w])):
            assert rel_err(gfd[k][w], ref) < 1e-9, (w, k)


@pytest.mark.parametrize("fn", [nb.inverse_dynamics_jacobians, nb.forward_dynamics_jacobians])
def test_value_errors(fn):
    raw = load_raw("half_cheetah")
    world = register(nb.World.from_raw(raw), step=2)
    n, m = raw.ndof, world.getMassDims()
    s, x = torch.zeros(2, 2 * n), torch.zeros(2, n)
    for bad_s, bad_x in ((torch.zeros(2, 2 * n + 1), x), (s, torch.zeros(2, n + 1)), (s, torch.zeros(3, n)), (torch.zeros(2 * n), x),
                         (torch.zeros(2, 3, 2 * n), torch.zeros(2, 3, n))):
        with pytest.raises(ValueError):
            fn(world, bad_s, bad_x)
    for bad_m in (torch.zeros(2, m + 1, dtype=torch.float64), torch.zeros(3, m, dtype=torch.float64), torch.ones(m + 1, dtype=torch.float64)):
        with pytest.raises(ValueError):
            fn(world, s, x, bad_m)
    with pytest.raises(ValueError):
        fn(world, s[0], x[0], torch.zeros(2, m, dtype=torch.float64))
    with pytest.raises(ValueError, match="degrees of freedom"):
        fn(nb.World(), torch.zeros(2, 0), torch.zeros(2, 0))
