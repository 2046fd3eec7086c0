"""Dev: cost of per-world masses on the flagship workload.  Atlas contact-free fwd+bwd, B worlds (default 4096), INERTIA_MASS
registered on every body and a different mass vector per world: nb2_step_forward_pw / nb2_step_backward_pw with a device-resident
[10*nb, B] inertia table and per-world dL/d(inertia), against the shared-table path (the bench.py headline) on the same inputs, the
two timed alternately in one process.  Prints one JSON line with the card's name and power limit.
    python scripts/dev/bench_per_world_mass.py [--batch B] [--steps K] [--rounds R]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", ".."))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import nimblephysics_b200 as nb  # noqa: E402
from bench import make_inputs  # noqa: E402
from nimblephysics_b200.engine import FP32  # noqa: E402
from nimblephysics_b200.modelspec import INERTIA_MASS  # noqa: E402
from tests.util import load_raw  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU (no CPU fallback)"
    B, dev = args.batch, torch.device("cuda")
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    world._contacts_disabled = True
    for sk in world.skeletons:
        for b in sk._ordered_bodies():
            world.tuneMass(b, INERTIA_MASS)
    dm = nb.device_model_for(world)
    rng = np.random.default_rng(77)
    mass = torch.tensor(world.getMasses()[None] * rng.uniform(0.8, 1.25, (B, world.getMassDims())), device=dev)
    wi = nb.mass_to_inertia(world, mass).reshape(B, -1).t().contiguous()   # [10*nb, B] fp64, the kernels' layout
    s, a, g = (torch.tensor(x, device=dev) for x in make_inputs(raw, B, 555))
    nxt, gs, ga = torch.empty_like(s), torch.empty_like(s), torch.empty_like(a)
    sv = torch.empty((dm.saved_words, B), device=dev)
    gi = torch.empty((10 * dm.cm.nb, B), device=dev)
    stream = torch.cuda.current_stream().cuda_stream

    def step(per_world):
        w = wi.data_ptr() if per_world else None
        dm.forward_device(B, s.data_ptr(), a.data_ptr(), nxt.data_ptr(), sv.data_ptr(), stream, FP32, wi_ptr=w)
        dm.backward_device(B, s.data_ptr(), a.data_ptr(), sv.data_ptr(), g.data_ptr(), gs.data_ptr(), ga.data_ptr(), stream, FP32,
                           gi.data_ptr() if per_world else None, wi_ptr=w)

    def timed(per_world):
        for _ in range(20):
            step(per_world)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(args.steps):
            step(per_world)
        e1.record()
        torch.cuda.synchronize()
        return B * args.steps / (e0.elapsed_time(e1) * 1e-3)

    rates = {"shared_table": [], "per_world": []}
    for _ in range(args.rounds):
        rates["shared_table"].append(timed(False))
        rates["per_world"].append(timed(True))
    gpu = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps({"batch": B, "steps": args.steps, "mass_dims": world.getMassDims(), "unit": "world-steps/s", "gpu": gpu, **rates}))


if __name__ == "__main__":
    main()
