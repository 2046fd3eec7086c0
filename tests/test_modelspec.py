"""Host logic: loaders -> RawModel -> CanonModel invariants (no GPU)."""
import os

import numpy as np
import pytest

import nimblephysics_b200 as nb
from nimblephysics_b200.modelspec import T_from_12
from tests.util import load_raw


def test_fixture_shapes():
    atlas = load_raw("atlas")
    assert atlas.ndof == 33 and atlas.nb == 34  # 28 moving links + 6 welded camera links (contact-free: no ground body)
    hc = load_raw("half_cheetah")
    assert hc.ndof == 9 and hc.dt == pytest.approx(0.002) and tuple(hc.gravity) == (0.0, -9.81, 0.0)
    cp = load_raw("cartpole")
    assert cp.ndof == 2 and cp.nb == 3


def test_raw_json_roundtrip():
    for name in ("cartpole", "half_cheetah", "atlas", "atlas_ground"):
        raw = load_raw(name)
        raw2 = nb.flatten_world(nb.World.from_raw(raw))
        for k, v in raw.__dict__.items():
            v2 = getattr(raw2, k)
            if isinstance(v, np.ndarray):
                assert np.array_equal(v, v2), (name, k)


@pytest.mark.parametrize("name", ["cartpole", "half_cheetah", "atlas", "atlas_ground", "atlas_sdf"])
def test_canonical_model_invariants(name):
    raw = load_raw(name)
    cm = nb.compile_model(raw)
    assert cm.ndof == raw.ndof
    assert all(cm.parent[i] < i for i in range(cm.nb))  # parents first (DFS pre-order)
    assert sorted(int(cm.dof_off[i]) + k for i in range(cm.nb) for k in range(6 if cm.jtype[i] == 3 else 1)) == list(range(cm.ndof))
    # every Xtree is a rigid transform
    for i in range(cm.nb):
        R = T_from_12(cm.Xtree[i])[:3, :3]
        assert np.allclose(R @ R.T, np.eye(3), atol=1e-12) and np.linalg.det(R) == pytest.approx(1.0)
    # total mass is preserved by weld folding (static bodies excluded)
    static = [i for i in range(raw.nb) if not raw.mobile[i]]
    moving_mass = sum(raw.mass[i] for i in range(raw.nb) if i not in static)
    # bodies welded to the world inside a mobile skeleton are static too
    assert cm.inertia[:, 0].sum() <= moving_mass + 1e-9
    _check_slots_and_schedule(cm)


def _check_slots_and_schedule(cm):
    # accumulator-slot discipline: a handoff body's parent is i-1; every other child owns ONE private slot inside the
    # parent's block [slot_self, slot_self + slot_count)
    used = set()
    for i in range(cm.nb):
        p = int(cm.parent[i])
        if cm.flags[i] & 1:
            assert p == i - 1
        elif p >= 0:
            sl = int(cm.slot_parent[i])
            assert cm.flags[p] & 4 and cm.slot_self[p] <= sl < cm.slot_self[p] + cm.slot_count[p]
            assert sl not in used and 0 <= sl < cm.nslots
            used.add(sl)
    assert len(used) == cm.nslots == int(cm.slot_count.sum())
    # schedule: trunk + limbs partition the bodies; the trunk is ancestor-closed; a limb body's parent is in the trunk
    # or swept by the same lane; register handoff never crosses a range
    owner, rng = {}, {}
    rid = 0
    for (lo, hi) in cm.trunk_ranges:
        for i in range(lo, hi):
            assert i not in owner
            owner[i], rng[i] = -1, rid
        rid += 1
    assert len(cm.limb_ranges) == cm.lanes
    for lane, rs in enumerate(cm.limb_ranges):
        assert len(rs) <= 8
        for (lo, hi) in rs:
            for i in range(lo, hi):
                assert i not in owner
                owner[i], rng[i] = lane, rid
            rid += 1
    assert sorted(owner) == list(range(cm.nb)) and len(cm.trunk_ranges) <= 8
    for i in range(cm.nb):
        p = int(cm.parent[i])
        if p >= 0:
            assert owner[p] in (-1, owner[i])
            if cm.flags[i] & 1:
                assert rng[p] == rng[i]


@pytest.mark.parametrize("name", ["cartpole", "half_cheetah", "atlas"])
@pytest.mark.parametrize("lanes", [2, 4, 8])
def test_cooperative_schedule(name, lanes):
    cm = nb.compile_model(load_raw(name), lanes=lanes)
    _check_slots_and_schedule(cm)
    if name == "atlas" and lanes == 4:  # the four limbs run side by side: sequential depth 4 + 6 instead of 28 bodies
        assert sum(hi - lo for lo, hi in cm.trunk_ranges) + max(sum(hi - lo for lo, hi in rs) for rs in cm.limb_ranges) <= 12


def test_builder_surface_matches_reference_example():
    """python/new_examples/cartpole.py:12-46 builds its cartpole through these calls."""
    world = nb.World()
    world.setGravity([0, -9.81, 0])
    cartpole = nb.Skeleton()
    rail, cart = cartpole.createPrismaticJointAndBodyNodePair()
    rail.setAxis([1, 0, 0])
    cart.createShapeNode(nb.BoxShape([.5, .1, .1])).createVisualAspect().setColor([0.5, 0.5, 0.5])
    rail.setPositionUpperLimit(0, 10)
    rail.setPositionLowerLimit(0, -10)
    rail.setControlForceUpperLimit(0, 10)
    rail.setControlForceLowerLimit(0, -10)
    pj, pole = cartpole.createRevoluteJointAndBodyNodePair(cart)
    pj.setAxis([0, 0, 1])
    pj.setControlForceUpperLimit(0, 0)
    pj.setControlForceLowerLimit(0, 0)
    off = nb.Isometry3()
    off.set_translation([0, -0.5, 0])
    pj.setTransformFromChildBodyNode(off)
    world.addSkeleton(cartpole)
    world.setTimeStep(world.getTimeStep() * 10)
    assert world.getStateSize() == 4 and world.getActionSize() == 2 and world.getTimeStep() == pytest.approx(1e-2)
    with pytest.raises(ValueError):
        world.setState(np.zeros(3))  # reference prints + ignores (World.cpp:2027-2033); we raise (documented)
    cm = nb.compile_model(nb.flatten_world(world))
    assert cm.nb == 2 and list(cm.jtype) == [2, 1]


def test_urdf_loader_reproduces_the_cartpole_fixture():
    """tests/golden/loader/cartpole.urdf describes the robot of tests/golden/models/cartpole.json: loading it (DartLoader rules: a root
    link named `world` welds the tree to the ground, joints sorted by name, continuous joints unlimited) gives the stored model."""
    import json
    from tests.util import MODELS, ROOT
    w = nb.loadWorld(os.path.join(ROOT, "tests", "golden", "loader", "cartpole.urdf"))
    w.setGravity([0, -9.81, 0])
    assert json.loads(nb.flatten_world(w).to_json()) == json.load(open(os.path.join(MODELS, "cartpole.json")))


@pytest.mark.skipif(not os.environ.get("NB2_REFERENCE_DATA"), reason="NB2_REFERENCE_DATA does not name the reference's data/ directory")
def test_fixtures_are_current_with_reference_files():
    import json
    from tests.util import MODELS
    w = nb.loadWorld(os.path.join(os.environ["NB2_REFERENCE_DATA"], "skel", "half_cheetah.skel"))
    fresh = json.loads(nb.flatten_world(w).to_json())
    stored = json.load(open(os.path.join(MODELS, "half_cheetah.json")))
    assert fresh == stored


def test_world_mass_vector_api():
    """World::tuneMass / getMasses / setMasses (World.cpp:1013-1053, 1821-1825; WithRespectToMass.cpp:44-185)."""
    from nimblephysics_b200 import modelspec as ms

    w = nb.World.from_raw(load_raw("half_cheetah"))
    bodies = w.getSkeleton(0)._ordered_bodies() if w.getSkeleton(0).isMobile() else w.getSkeleton(1)._ordered_bodies()
    b0, b1 = bodies[1], bodies[2]
    assert w.getMassDims() == 0 and w.getMasses().shape == (0,)
    w.tuneMass(b0, ms.INERTIA_MASS, [10.0], [0.1])
    w.tuneMass(b1, ms.INERTIA_FULL)
    assert w.getMassDims() == 11
    v = w.getMasses()
    assert v[0] == b0.mass and v[1] == b1.mass and np.allclose(v[2:5], b1.com)
    mom_before = b0.moment.copy()
    v2 = v.copy()
    v2[0] *= 2.0
    w.setMasses(v2)
    assert b0.mass == v2[0] and np.allclose(b0.moment, 2.0 * mom_before)  # Inertia::setMass keeps the dimensions
    assert np.allclose(w.getMasses(), v2)
    assert w.getMassUpperLimits()[0] == 10.0 and w.getMassLowerLimits()[0] == 0.1
    with pytest.raises(ValueError):
        w.setMasses(np.zeros(3))


def test_legacy_world_and_skeleton_accessors():
    """Calls the reference's examples make on World / Skeleton (python/new_examples/atlas.py:14-36, cartpole.py):
    setPosition before stepping, control-force limit vectors, body lookup by world index, setAction / getAction."""
    w = nb.World.from_raw(load_raw("atlas"))
    atlas = w.getSkeleton(0)
    n = w.getNumDofs()
    assert atlas.getNumDofs() == n and w.getNumBodyNodes() == atlas.getNumBodyNodes()
    assert w.getBodyNodeByIndex(0) is atlas._ordered_bodies()[0] and w.getBodyNodeByIndex(10 ** 6) is None
    atlas.setPosition(0, -0.5 * np.pi)          # before any state exists: becomes the initial pose
    atlas.setPosition(4, -0.01)
    st = w.getState()
    assert st[0] == pytest.approx(-0.5 * np.pi) and st[4] == pytest.approx(-0.01) and np.all(st[n:] == 0)
    atlas.setPosition(7, 0.25)                   # with a state: edits it in place
    assert w.getState()[7] == 0.25 and atlas.getPositions()[7] == 0.25
    atlas.setVelocity(3, 1.5)
    assert w.getVelocities()[3] == 1.5
    v0 = w._version
    atlas.setControlForceUpperLimits(np.full(n, 7.0))
    atlas.setControlForceLowerLimits(np.full(n, -7.0))
    assert w._version > v0                       # limits are part of the device model: it is rebuilt lazily
    raw = nb.flatten_world(w)
    assert np.all(raw.force_hi == 7.0) and np.all(raw.force_lo == -7.0)
    w.setAction(np.arange(w.getActionSize(), dtype=float))
    assert w.getAction()[3] == 3.0
    with pytest.raises(ValueError):
        w.setAction(np.zeros(3))


def test_world_clone_and_new_model_flags_roundtrip():
    """World::clone gives an independent copy (model, state, action, tunable-mass registrations); the self-collision and limit-enforcement flags
    survive flatten -> JSON -> from_raw."""
    import json

    w = nb.World.from_raw(load_raw("half_cheetah"))
    arm = w.getSkeleton(1)
    arm.enableSelfCollisionCheck()
    j = next(b.parent_joint for b in arm._ordered_bodies() if b.parent_joint.getNumDofs() == 1)
    j.setPositionLimitEnforced(True)
    w.setState(np.linspace(-0.2, 0.3, w.getStateSize()))
    w.setAction(np.ones(w.getActionSize()))
    body = arm._ordered_bodies()[3]
    w.tuneMass(body, 0, upperBound=[5.0], lowerBound=[0.1])
    c = w.clone()
    assert np.allclose(c.getState(), w.getState()) and np.allclose(c.getAction(), w.getAction())
    assert c.getSkeleton(1).isEnabledSelfCollisionCheck() and not c.getSkeleton(1).isEnabledAdjacentBodyCheck()
    assert sum(b.parent_joint.isPositionLimitEnforced() for b in c.getSkeleton(1)._ordered_bodies()) == 1
    assert c.getMassDims() == 1 and np.allclose(c.getMasses(), w.getMasses())
    c.setState(np.zeros(c.getStateSize()))
    assert not np.allclose(c.getState(), w.getState())          # independent
    c.setMasses([3.0])
    assert not np.allclose(c.getMasses(), w.getMasses())
    raw2 = nb.RawModel.from_json(nb.flatten_world(w).to_json())
    assert raw2.self_collision.sum() > 0 and raw2.limit_enforced.sum() == 1
    old = json.loads(nb.flatten_world(w).to_json()); old.pop("self_collision"); old.pop("adjacent_check"); old.pop("limit_enforced")
    raw3 = nb.RawModel.from_json(json.dumps(old))                 # a fixture written before these fields existed
    assert raw3.self_collision.sum() == 0 and raw3.limit_enforced.sum() == 0
