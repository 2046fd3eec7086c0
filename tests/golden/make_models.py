"""Generates tests/golden/models/*.json (flattened RawModel fixtures) from the reference's data files.
Needs a nimblephysics source tree; the JSON fixtures are committed, so tests never need it.
  NB2_REFERENCE_DATA=<nimblephysics>/data python tests/golden/make_models.py
Sources (read-only inputs, SURVEY §8c): data/urdf/cartpole.urdf, data/skel/half_cheetah.skel,
data/sdf/atlas/atlas_v3_box_colliders.urdf, data/sdf/atlas/ground.urdf, data/sdf/atlas/atlas_v3_no_head.sdf."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", ".."))
import nimblephysics_b200 as nb  # noqa: E402

REF = os.environ.get("NB2_REFERENCE_DATA") or sys.exit("set NB2_REFERENCE_DATA to the data/ directory of a nimblephysics source tree")
OUT = os.path.join(os.path.dirname(__file__), "models")


def main():
    os.makedirs(OUT, exist_ok=True)
    # config 1: cartpole (2 DoF), y-up gravity as in unittests/comprehensive/test_Cartpole.cpp:56-65
    w = nb.loadWorld(f"{REF}/urdf/cartpole.urdf")
    w.setGravity([0, -9.81, 0])
    nb.flatten_world(w).save(f"{OUT}/cartpole.json")
    # config 2: Atlas, contact-free (python/nimblephysics_benchmarks/atlas_bench.py:12-27 without the ground)
    w = nb.World()
    w.setGravity([0, -9.81, 0])
    w.loadSkeleton(f"{REF}/sdf/atlas/atlas_v3_box_colliders.urdf")
    nb.flatten_world(w).save(f"{OUT}/atlas.json")
    # config 4: Atlas + ground
    w.loadSkeleton(f"{REF}/sdf/atlas/ground.urdf")
    nb.flatten_world(w).save(f"{OUT}/atlas_ground.json")
    # config 3: half-cheetah + ground
    w = nb.loadWorld(f"{REF}/skel/half_cheetah.skel")
    nb.flatten_world(w).save(f"{OUT}/half_cheetah.json")
    # the SDF description of the same robot (28 links, no welded camera links): exercises the SDF loader
    w = nb.World()
    w.setGravity([0, -9.81, 0])
    w.loadSkeleton(f"{REF}/sdf/atlas/atlas_v3_no_head.sdf")
    nb.flatten_world(w).save(f"{OUT}/atlas_sdf.json")
    print("wrote", sorted(os.listdir(OUT)))


if __name__ == "__main__":
    main()
