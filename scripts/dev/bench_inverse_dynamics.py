"""Dev: contact-free inverse dynamics against the step on the flagship model.  Atlas, fp32, B worlds (default 4096 and 65536): ID
forward + backward (nb2_inverse_dynamics / _backward, tau and the state / next-velocity gradients) and the step's forward + backward
(nb2_step_forward / _backward, the bench.py headline) on the same states, next_vel = the step's next velocity, the two timed
alternately in one process with CUDA events.  Prints one JSON line with the card's name, power limit and maximum SM clock.
    python scripts/dev/bench_inverse_dynamics.py [--batch B ...] [--steps K] [--rounds R]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", ".."))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import nimblephysics_b200 as nb  # noqa: E402
from bench import make_inputs  # noqa: E402
from nimblephysics_b200.engine import FP32  # noqa: E402
from tests.util import load_raw  # noqa: E402


def measure(dm, raw, B, steps, rounds):
    dev = torch.device("cuda")
    n = raw.ndof
    s, a, g = (torch.tensor(x, device=dev) for x in make_inputs(raw, B, 555))
    nxt, gs, ga = torch.empty_like(s), torch.empty_like(s), torch.empty_like(a)
    sv = torch.empty((dm.saved_words, B), device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    dm.forward_device(B, s.data_ptr(), a.data_ptr(), nxt.data_ptr(), sv.data_ptr(), stream, FP32)
    vn = nxt[:, n:].contiguous()
    tau, gt, gv = torch.empty((B, n), device=dev), torch.randn((B, n), device=dev), torch.empty((B, n), device=dev)
    sv2 = torch.empty_like(sv)

    def step():
        dm.forward_device(B, s.data_ptr(), a.data_ptr(), nxt.data_ptr(), sv.data_ptr(), stream, FP32)
        dm.backward_device(B, s.data_ptr(), a.data_ptr(), sv.data_ptr(), g.data_ptr(), gs.data_ptr(), ga.data_ptr(), stream, FP32)

    def inv():
        dm.inverse_dynamics_device(B, s.data_ptr(), vn.data_ptr(), tau.data_ptr(), sv2.data_ptr(), stream, FP32)
        dm.inverse_dynamics_backward_device(B, s.data_ptr(), sv2.data_ptr(), gt.data_ptr(), gs.data_ptr(), gv.data_ptr(), stream, FP32)

    def timed(f):
        for _ in range(20):
            f()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(steps):
            f()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / steps  # microseconds per fwd+bwd

    us = {"step_fwd_bwd_us": [], "id_fwd_bwd_us": []}
    for _ in range(rounds):
        us["step_fwd_bwd_us"].append(round(timed(step), 2))
        us["id_fwd_bwd_us"].append(round(timed(inv), 2))
    lanes = {"step": [dm.lanes_for(B, False), dm.lanes_for(B, True)]}
    return {"batch": B, **us, "lanes_step_fwd_bwd": lanes["step"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[4096, 65536])
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU (no CPU fallback)"
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    world._contacts_disabled = True
    dm = nb.device_model_for(world)
    rows = [measure(dm, raw, B, args.steps, args.rounds) for B in args.batch]
    gpu = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"model": "atlas", "precision": "fp32", "steps": args.steps, "gpu": gpu, "results": rows}))


if __name__ == "__main__":
    main()
