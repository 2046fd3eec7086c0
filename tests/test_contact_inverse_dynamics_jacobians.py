"""Dense Jacobians of contact inverse dynamics on the CPU: the stage functions of csrc/nb2_mcidj.cuh (host build, poisoned working set,
reversed lane and slot orders) against the dual-number Jacobian of the multiple-contact oracle, against the emulated VJPs of
contact_inverse_dynamics / multiple_contact_inverse_dynamics seeded with the identity, across lane schedules and row-slot counts, with
per-world masses, and the argument checks of nimblephysics_b200.contact_inverse_dynamics_jacobians /
multiple_contact_inverse_dynamics_jacobians."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from nimblephysics_b200 import modelspec as ms
from tests.host_emul.binding_djac import EmulDjacWorld
from tests.host_emul.binding_mcid import EmulMcidWorld
from tests.host_emul.binding_mcidj import EmulMcidjWorld
from tests.oracle_id.binding_mcid import McidOracle
from tests.test_contact_inverse_dynamics import WELDED
from tests.test_inverse_dynamics import _compile, id_inputs
from tests.test_per_world_mass import random_masses, raw_at, register
from tests.util import load_raw, rel_err

FEET = ["l_foot", "r_foot"]
LIMBS = ["l_foot", "r_foot", "l_hand", "r_hand"]
CASES = [("atlas", ["l_foot"]), ("atlas", ["r_hand"]), ("atlas", [WELDED]), ("atlas", FEET), ("atlas", LIMBS), ("atlas_sdf", ["r_foot"]),
         ("atlas_sdf", FEET), ("atlas_sdf", LIMBS)]


def _bodies(raw, names):
    return [list(raw.body_names).index(n) for n in names]


def _device_set(cm, bodies):
    return [int(cm.body_owner[b]) for b in bodies], [cm.body_T[b][:3, 3] for b in bodies]


def _blocks(J, n, k):
    """The oracle's d[tau; w]/d[q; qdot; v'; g] [n + 6k, 3n + 6k] as the emulation's eight blocks (T_q, T_qdot, T_v', T_g, W_q, ...)."""
    cols = (slice(0, n), slice(n, 2 * n), slice(2 * n, 3 * n), slice(3 * n, 3 * n + 6 * k))
    return [J[:n, c] for c in cols] + [J[n:, c] for c in cols]


@pytest.mark.parametrize("name,names", CASES)
@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("guessed", [False, True])
def test_emulated_blocks_match_oracle(name, names, fp64, guessed):
    raw = load_raw(name)
    cm = nb.compile_model(raw, lanes=2)
    ew, mo = EmulMcidjWorld(cm), McidOracle(raw)
    bodies = _bodies(raw, names)
    n, k, B = raw.ndof, len(bodies), 2  # the odd world runs its lanes in reverse
    s, vn = id_inputs(raw, B, seed=71 + k)
    g = np.random.default_rng(k).normal(0, 40, (B, k, 6)) if guessed else None
    db, dp = _device_set(cm, bodies)
    got = ew.contact_jacobians(db, dp, s, vn, g, fp64)
    tol = 1e-9 if fp64 else 1e-4
    cast = (lambda a: a.astype(np.float64)) if fp64 else (lambda a: a.astype(np.float32).astype(np.float64))
    for w in range(B):
        rt, rw, J = mo.multiple_contact_inverse_dynamics(bodies, cast(s[w]), cast(vn[w]), cast(g[w]) if guessed else None, want_jac=True)
        assert rel_err(got[0][w], rt) < tol and rel_err(got[1][w], rw) < tol, w
        for b, ref in enumerate(_blocks(J, n, k)):
            if k == 1 and b in (3, 7):
                assert not np.any(got[2 + b][w]) and np.abs(ref).max() < 1e-12, (w, b)  # one body: the guess is not read
            else:
                assert rel_err(got[2 + b][w], ref) < tol, (w, b, rel_err(got[2 + b][w], ref))


@pytest.mark.parametrize("names", [["l_foot"], [WELDED], FEET, LIMBS])
@pytest.mark.parametrize("fp64", [False, True])
def test_rows_are_the_emulated_layer_vjps_seeded_with_the_identity(names, fp64):
    """Row i of each block is the existing layer's VJP with the seed e_i: the contact VJP's seed, the inverse-dynamics backward and the
    contact VJP's direct term, the same stage functions in the same order, the same bits."""
    raw = load_raw("atlas")
    cm = nb.compile_model(raw, lanes=2)
    ej, el = EmulMcidjWorld(cm), EmulMcidWorld(cm)
    bodies = _bodies(raw, names)
    n, k, B = raw.ndof, len(bodies), 3
    m = 6 * k
    s, vn = id_inputs(raw, B, seed=81 + k)
    g = np.random.default_rng(82).normal(0, 40, (B, k, 6))
    db, dp = _device_set(cm, bodies)
    tau, w, Tq, Tqd, Tn, Tg, Wq, Wqd, Wn, Wg = ej.contact_jacobians(db, dp, s, vn, g, fp64)
    tau_e, w_e, saved = el.multiple_contact_inverse_dynamics(db, dp, s, vn, g, fp64)
    assert np.array_equal(tau, tau_e) and np.array_equal(w, w_e)
    for i in range(n + m):
        seed = np.zeros((B, n + m))
        seed[:, i] = 1
        gs, gn, _, gg = el.multiple_contact_inverse_dynamics_backward(db, dp, s, saved, w_e, seed[:, :n], seed[:, n:].reshape(B, k, 6), g, fp64)
        q, qd, nv, gu = (Tq, Tqd, Tn, Tg) if i < n else (Wq, Wqd, Wn, Wg)
        r = i if i < n else i - n
        assert np.array_equal(q[:, r], gs[:, :n]) and np.array_equal(qd[:, r], gs[:, n:]) and np.array_equal(nv[:, r], gn), i
        assert np.array_equal(gu[:, r], gg.reshape(B, m)), i
    # a seed on the free root's rows is dropped: the six root rows of every tau block are exactly zero
    for blk in (Tq, Tqd, Tn, Tg):
        assert not np.any(blk[:, :6])


@pytest.mark.parametrize("names", [["l_foot"], ["r_hand"], FEET])
@pytest.mark.parametrize("fp64", [False, True])
def test_rows_off_the_chains_are_the_inverse_dynamics_rows(names, fp64):
    """A seed on a dof off the union of the chains reaches the inverse-dynamics backward as e_i and the direct term adds zeros: those rows
    are inverse_dynamics_jacobians's (csrc/nb2_djac.cuh) bit for bit."""
    raw = load_raw("atlas")
    cm = nb.compile_model(raw, lanes=2)
    bodies = _bodies(raw, names)
    n, B = raw.ndof, 3
    s, vn = id_inputs(raw, B, seed=87)
    got = EmulMcidjWorld(cm).contact_jacobians(*_device_set(cm, bodies), s, vn, None, fp64)
    ref = EmulDjacWorld(cm).dynamics_jacobians(s, vn, False, fp64)
    chain = set()
    for b in bodies:
        while raw.parent[b] >= 0:
            chain |= set(range(raw.dof_off[b], raw.dof_off[b] + ms.JOINT_NDOF[int(raw.jtype[b])]))
            b = raw.parent[b]
    off = [d for d in range(6, n) if d not in chain]
    assert off
    assert np.array_equal(got[0][:, off], ref[0][:, off])
    for a, r in zip(got[2:5], ref[1:]):
        assert np.array_equal(a[:, off], r[:, off])


@pytest.mark.parametrize("names", [["r_foot"], FEET, LIMBS])
@pytest.mark.parametrize("lanes", [1, 4, 8])
def test_lane_schedules_and_row_slots_agree(names, lanes):
    raw = load_raw("atlas")
    bodies = _bodies(raw, names)
    k = len(bodies)
    cm1, cmk = nb.compile_model(raw, lanes=2), _compile(raw, lanes)
    s, vn = id_inputs(raw, 3, seed=91 + lanes)
    g = np.random.default_rng(92).normal(0, 40, (3, k, 6))
    ref = EmulMcidjWorld(cm1).contact_jacobians(*_device_set(cm1, bodies), s, vn, g, True, slots=32)
    ewk = EmulMcidjWorld(cmk)
    first = None
    for slots in (4, 8, 16, 32):
        got = ewk.contact_jacobians(*_device_set(cmk, bodies), s, vn, g, True, slots=slots)
        if first is None:
            first = got
        for a, b, c in zip(got, first, ref):
            assert np.array_equal(a, b), slots  # the same schedule: the rounds give the same bits
            assert rel_err(a, c) < 1e-12, (slots, rel_err(a, c))  # another schedule sums in another order


def test_per_world_mass_is_set_masses_per_world():
    raw = load_raw("atlas")
    world = register(nb.World.from_raw(raw), step=4)
    n, B = raw.ndof, 3
    M = random_masses(world, B, seed=23)
    wi = nb.mass_to_inertia(world, torch.tensor(M, dtype=torch.float64)).numpy()
    cm = nb.compile_model(raw, lanes=2)
    entries = world._mass_entries()
    for names in (["l_foot"], LIMBS):
        bodies = _bodies(raw, names)
        k = len(bodies)
        s, vn = id_inputs(raw, B, seed=24 + k)
        g = np.random.default_rng(25).normal(0, 40, (B, k, 6))
        got = EmulMcidjWorld(cm).contact_jacobians(*_device_set(cm, bodies), s, vn, g, True, world_inertia=wi)
        for w in range(B):
            mo = McidOracle(raw_at(raw, entries, M[w]))
            rt, rw, J = mo.multiple_contact_inverse_dynamics(bodies, s[w].astype(np.float64), vn[w].astype(np.float64), g[w], want_jac=True)
            assert rel_err(got[0][w], rt) < 1e-9 and rel_err(got[1][w], rw) < 1e-9, w
            for b, ref in enumerate(_blocks(J, n, k)):
                if k > 1 or b not in (3, 7):
                    assert rel_err(got[2 + b][w], ref) < 1e-9, (names, w, b)


def _node(world, name, sk=0):
    return next(b for b in world.skeletons[sk]._ordered_bodies() if b.name == name)


def test_value_errors():
    world = register(nb.World.from_raw(load_raw("atlas_ground")), step=4)
    n, md = world.getNumDofs(), world.getMassDims()
    lf, rf, lh, rh, pel = (_node(world, x) for x in ("l_foot", "r_foot", "l_hand", "r_hand", "pelvis"))
    s, v = torch.zeros(2, 2 * n), torch.zeros(2, n)
    one, multi = nb.contact_inverse_dynamics_jacobians, nb.multiple_contact_inverse_dynamics_jacobians
    for f, body in ((one, lf), (multi, [lf, rf])):
        for bad_s, bad_v, what in ((s[:, 1:], v, "state has shape"), (s, v[:1], "next_vel has shape"), (s, v[0], "next_vel has shape")):
            with pytest.raises(ValueError, match=what):
                f(world, bad_s, bad_v, body)
        for bad_m in (torch.zeros(2, md + 1, dtype=torch.float64), torch.zeros(3, md, dtype=torch.float64), torch.ones(md + 1, dtype=torch.float64)):
            with pytest.raises(ValueError):
                f(world, s, v, body, bad_m)
        with pytest.raises(ValueError):
            f(world, s[0], v[0], body, torch.zeros(2, md, dtype=torch.float64))
    other = nb.World.from_raw(load_raw("atlas"))
    with pytest.raises(ValueError, match="not a body of this world"):
        one(world, s, v, _node(other, "l_foot"))
    with pytest.raises(ValueError, match="immobile"):
        one(world, s, v, world.skeletons[1]._ordered_bodies()[0])
    hc = nb.World.from_raw(load_raw("half_cheetah"))
    last = hc.getBodyNodeByIndex(hc.getNumBodyNodes() - 1)
    with pytest.raises(ValueError, match="FreeJoint"):
        one(hc, torch.zeros(2, 2 * hc.getNumDofs()), torch.zeros(2, hc.getNumDofs()), last)
    with pytest.raises(ValueError, match="FreeJoint"):
        multi(hc, torch.zeros(2, 2 * hc.getNumDofs()), torch.zeros(2, hc.getNumDofs()), [last, last.parent_body])
    with pytest.raises(ValueError, match="0 contact bodies"):
        multi(world, s, v, [])
    with pytest.raises(ValueError, match="5 contact bodies"):
        multi(world, s, v, [lf, rf, lh, rh, pel])
    with pytest.raises(ValueError, match="appears twice"):
        multi(world, s, v, [lf, rf, lf])
    with pytest.raises(ValueError, match="immobile"):
        multi(world, s, v, [lf, world.skeletons[1]._ordered_bodies()[0]])
    two = nb.World.from_raw(load_raw("atlas"))
    sk = nb.Skeleton("box")
    _, box = sk.createFreeJointAndBodyNodePair(None)
    box.setMass(3.0)
    two.addSkeleton(sk)
    with pytest.raises(ValueError, match="different skeletons"):
        multi(two, torch.zeros(2, 2 * two.getNumDofs()), torch.zeros(2, two.getNumDofs()), [_node(two, "l_foot"), box])
    with pytest.raises(ValueError, match="wrench_guesses has shape"):
        multi(world, s, v, [lf, rf], wrench_guesses=torch.zeros(2, 3, 6))
    with pytest.raises(ValueError, match="wrench_guesses has shape"):
        multi(world, s[0], v[0], [lf, rf], wrench_guesses=torch.zeros(1, 2, 6))
    with pytest.raises(ValueError, match="multiple_contact_inverse_dynamics_jacobians"):
        multi(world, s, v, [lf, lf])
    with pytest.raises(ValueError, match="contact_inverse_dynamics_jacobians"):
        one(world, s[:, 1:], v, lf)
