"""Per-world masses on the CPU: the mass-vector -> per-world canonical inertia map (modelspec.mass_to_inertia) against
World.setMasses + the canonical compile, and the device functions (csrc/nb2_dyn.cuh, host build) stepping every world
of a batch with its own inertia table against the fp64 oracle built at that world's masses."""
import copy

import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from nimblephysics_b200 import modelspec as ms
from oracle import binding as ob
from tests.host_emul.binding import EmulWorld
from tests.host_emul.binding_pw import EmulWorldPW
from tests.util import contact_inputs, load_raw, rel_err, sample_inputs

KINDS = [ms.INERTIA_MASS, ms.INERTIA_COM, ms.INERTIA_DIAGONAL, ms.INERTIA_OFF_DIAGONAL, ms.INERTIA_FULL]


def register(world, step=3):
    """tuneMass on every `step`-th body of the largest skeleton (the robot, not the ground), cycling through the supported entry types."""
    bodies = max(world.skeletons, key=lambda sk: sk.getNumBodyNodes())._ordered_bodies()
    for k, b in enumerate(bodies[::step]):
        world.tuneMass(b, KINDS[k % len(KINDS)])
    return world


def random_masses(world, B, seed):
    """[B, getMassDims()] around the current values; inertia tensors stay positive definite."""
    rng = np.random.default_rng(seed)
    rows = []
    for _ in range(B):
        parts = []
        for b, kind, _, _ in world._wrt_mass:
            v = ms._mass_entry_value(kind, b.mass, b.com, world._mom6(b))
            d = float(np.mean(np.diag(b.moment)))
            if kind == ms.INERTIA_MASS:
                v = v * rng.uniform(0.7, 1.4)
            elif kind == ms.INERTIA_COM:
                v = v + rng.uniform(-0.02, 0.02, 3)
            elif kind == ms.INERTIA_DIAGONAL:
                v = v * rng.uniform(0.8, 1.25, 3)
            elif kind == ms.INERTIA_OFF_DIAGONAL:
                v = v + rng.uniform(-0.05, 0.05, 3) * d
            else:
                v = np.concatenate([v[:1] * rng.uniform(0.7, 1.4), v[1:4] + rng.uniform(-0.02, 0.02, 3), v[4:7] * rng.uniform(0.9, 1.1, 3),
                                    v[7:] + rng.uniform(-0.03, 0.03, 3) * d])
            parts.append(v)
        rows.append(np.concatenate(parts))
    return np.array(rows)


def raw_at(raw, entries, mvec):
    """RawModel with the mass vector applied (WrtMassBodyNodyEntry::set), the reference for world w."""
    r = copy.deepcopy(raw)
    k = 0
    for bi, kind in entries:
        d = ms.WRT_MASS_DIMS[kind]
        r.mass[bi], r.com[bi], r.moment[bi] = ms._apply_mass_entry(kind, mvec[k:k + d], r.mass[bi], r.com[bi], r.moment[bi])
        k += d
    return r


def tree_world():
    from tests.test_oracle import _tree_world

    return _tree_world()


@pytest.mark.parametrize("which", ["atlas", "tree"])
def test_mass_to_inertia_matches_set_masses_and_its_jacobian(which):
    world = nb.World.from_raw(load_raw("atlas")) if which == "atlas" else tree_world()
    register(world, step=3 if which == "atlas" else 1)
    kinds = {t for _, t, _, _ in world._wrt_mass}
    assert kinds == set(KINDS) or which == "tree"
    m_before = world.getMasses().copy()
    B = 4
    M = random_masses(world, B, seed=3)
    mt = torch.tensor(M, dtype=torch.float64)
    wi = nb.mass_to_inertia(world, mt)
    assert wi.shape[0] == B and wi.shape[2] == 10 and wi.dtype == torch.float64
    assert np.array_equal(world.getMasses(), m_before)  # the World is not modified
    entries = world._mass_entries()
    for w in range(B):
        w2 = copy.deepcopy(world)
        w2._device_model = None
        w2.setMasses(M[w])
        raw2 = nb.flatten_world(w2)
        cm2 = nb.compile_model(raw2)
        got = wi[w].numpy()
        assert np.abs(got - cm2.inertia).max() <= 1e-13 * np.abs(cm2.inertia).max()
        J = torch.autograd.functional.jacobian(lambda x: nb.mass_to_inertia(world, x[None])[0].reshape(-1), mt[w].clone()).numpy()
        P = ms.inertia_param_jacobian(raw2, cm2, entries)
        assert np.abs(J.T - P).max() <= 1e-10 * max(np.abs(P).max(), 1.0)


def test_mass_to_inertia_rejects_bad_shapes_and_follows_body_edits():
    world = register(nb.World.from_raw(load_raw("cartpole")), step=1)
    with pytest.raises(ValueError):
        nb.mass_to_inertia(world, torch.zeros(3, world.getMassDims() + 1, dtype=torch.float64))
    m = torch.tensor(world.getMasses()[None], dtype=torch.float64)
    a = nb.mass_to_inertia(world, m)
    world.skeletons[0]._ordered_bodies()[1].setMass(2.0)  # registered for its COM: its mass is a fixed parameter of the map
    b = nb.mass_to_inertia(world, m)
    assert not torch.equal(a, b)
    assert np.abs(b[0].numpy() - nb.compile_model(nb.flatten_world(world)).inertia).max() < 1e-13


def test_per_world_mass_shape_errors():
    """A 2-D mass needs a batched state with as many rows; both are rejected before anything runs."""
    raw = load_raw("cartpole")
    world = register(nb.World.from_raw(raw), step=1)
    m = torch.tensor(world.getMasses(), dtype=torch.float64)
    s, a, _ = sample_inputs(raw, 3, seed=1)
    with pytest.raises(ValueError):
        nb.timestep(world, torch.tensor(s[0]), torch.tensor(a[0]), m[None])
    with pytest.raises(ValueError):
        nb.timestep(world, torch.tensor(s), torch.tensor(a), m[None].repeat(2, 1))
    with pytest.raises(ValueError):
        nb.rollout_fused(world, torch.tensor(s), torch.tensor(a)[None], mass=m)


def _per_world(name, B, seed):
    raw = load_raw(name)
    world = register(nb.World.from_raw(raw), step=4)
    M = random_masses(world, B, seed)
    wi = nb.mass_to_inertia(world, torch.tensor(M, dtype=torch.float64)).numpy()
    return raw, world, M, wi


@pytest.mark.parametrize("name", ["half_cheetah", "atlas"])
@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("lanes", [1, 2, 4, 8])
def test_emulated_per_world_step_matches_oracle(oracle_mod, name, fp64, lanes):
    B = 4
    raw, world, M, wi = _per_world(name, B, seed=11 + lanes)
    cm = nb.compile_model(raw, lanes=lanes)
    ew = EmulWorldPW(cm)
    s, a, g = sample_inputs(raw, B, seed=31)
    nxt, saved = ew.forward(s, a, fp64, world_inertia=wi)
    gs, ga, gi = ew.backward(s, a, saved, g, fp64, want_inertia_grad=True, world_inertia=wi)
    entries = world._mass_entries()
    for w in range(B):
        rw = raw_at(raw, entries, M[w])
        ow = oracle_mod.OracleWorld(rw)
        s64, a64, g64 = s[w].astype(np.float64), a[w].astype(np.float64), g[w].astype(np.float64)
        rgs, rga = ow.backprop(s64, a64, g64)
        assert rel_err(nxt[w], ow.step(s64, a64)) < 1e-4
        assert rel_err(gs[w], rgs) < 1e-4 and rel_err(ga[w], rga) < 1e-4
        if fp64 and w < 2:
            gm = ms.inertia_param_jacobian(rw, cm, entries) @ gi[:, w].astype(np.float64)

            def loss(mv):
                return float(g64 @ oracle_mod.OracleWorld(raw_at(raw, entries, mv)).step(s64, a64))

            fd = np.array([(loss(M[w] + 1e-5 * e) - loss(M[w] - 1e-5 * e)) / 2e-5 for e in np.eye(len(M[w]))])
            assert rel_err(gm, fd) < 2e-5, (gm, fd)


@pytest.mark.parametrize("name", ["half_cheetah", "atlas_ground"])
def test_emulated_per_world_contact_step_matches_oracle(oracle_mod, name):
    B = 4
    raw, world, M, wi = _per_world(name, B, seed=5)
    cm = nb.compile_model(raw)
    ew = EmulWorldPW(cm)
    s, a = contact_inputs(raw, name, B, seed=3)
    g = np.random.default_rng(2).normal(size=(B, 2 * raw.ndof)).astype(np.float32)
    r = ew.forward_contact(s, a, reverse=True, world_inertia=wi)
    gs, ga, gi = ew.backward_contact(s, a, r["saved"], r["crec"], g, want_inertia_grad=True, reverse=True, world_inertia=wi)
    entries = world._mass_entries()
    rows = 0
    for w in range(B):
        rw = raw_at(raw, entries, M[w])
        ow = ob.OracleContactWorld(rw)
        s64, a64, g64 = s[w].astype(np.float64), a[w].astype(np.float64), g[w].astype(np.float64)
        ro = ow.step_contact(s64, a64)
        assert r["m"][w] == ro["m"] and np.array_equal(r["labels"][w][: ro["m"]], ro["mapping"])
        rows += ro["m"]
        assert rel_err(r["next"][w], ro["next_state"]) < 1e-4
        rgs, rga, rc = ow.backprop_contact(s64, a64, g64)
        assert rc >= 0 and rel_err(gs[w], rgs) < 1e-4 and rel_err(ga[w], rga) < 1e-4
        if w < 2:
            gm = ms.inertia_param_jacobian(rw, cm, entries) @ gi[:, w].astype(np.float64)

            def loss(mv):
                return float(g64 @ ob.OracleContactWorld(raw_at(raw, entries, mv)).step_contact(s64, a64)["next_state"])

            fd = np.array([(loss(M[w] + 1e-5 * e) - loss(M[w] - 1e-5 * e)) / 2e-5 for e in np.eye(len(M[w]))])
            assert rel_err(gm, fd) < 2e-5, (gm, fd)
    assert rows > 0


@pytest.mark.parametrize("lanes", [1, 2, 4, 8])
def test_emulated_replicated_model_inertia_is_bit_identical(lanes):
    """The model's own table, replicated per world, reproduces the shared-table path (the plain harness) bit for bit."""
    raw = load_raw("atlas")
    cm = nb.compile_model(raw, lanes=lanes)
    ew, ewp = EmulWorld(cm), EmulWorldPW(cm)
    B = 5
    wi = np.broadcast_to(cm.inertia, (B, cm.nb, 10))
    s, a, g = sample_inputs(raw, B, seed=8)
    for fp64 in (False, True):
        n0, sv0 = ew.forward(s, a, fp64)
        n1, sv1 = ewp.forward(s, a, fp64, world_inertia=wi)
        assert np.array_equal(n0, n1) and np.array_equal(sv0, sv1)
        r0 = ew.backward(s, a, sv0, g, fp64, want_inertia_grad=True)
        r1 = ewp.backward(s, a, sv1, g, fp64, want_inertia_grad=True, world_inertia=wi)
        assert all(np.array_equal(x, y) for x, y in zip(r0, r1))


@pytest.mark.parametrize("name", ["half_cheetah", "atlas_ground"])
def test_emulated_replicated_model_inertia_is_bit_identical_with_contacts(name):
    raw = load_raw(name)
    cm = nb.compile_model(raw)
    ew, ewp = EmulWorld(cm), EmulWorldPW(cm)
    B = 4
    wi = np.broadcast_to(cm.inertia, (B, cm.nb, 10))
    s, a = contact_inputs(raw, name, B, seed=6)
    g = np.random.default_rng(4).normal(size=(B, 2 * raw.ndof)).astype(np.float32)
    r0 = ew.forward_contact(s, a, reverse=True, small_mc=2)
    r1 = ewp.forward_contact(s, a, reverse=True, small_mc=2, world_inertia=wi)
    assert all(np.array_equal(r0[k], r1[k]) for k in r0)
    b0 = ew.backward_contact(s, a, r0["saved"], r0["crec"], g, want_inertia_grad=True, reverse=True, small_mc=2)
    b1 = ewp.backward_contact(s, a, r1["saved"], r1["crec"], g, want_inertia_grad=True, reverse=True, small_mc=2, world_inertia=wi)
    assert all(np.array_equal(x, y) for x, y in zip(b0, b1))
