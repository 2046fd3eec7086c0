"""Dev: contact inverse dynamics against plain inverse dynamics on the flagship model.  Atlas, fp32, B worlds (default 4096 and 65536):
contact ID forward + backward with contact body l_foot (nb2_contact_inverse_dynamics / _backward, tau, wrench and the state /
next-velocity gradients), multiple-contact ID forward + backward with both feet (nb2_multiple_contact_inverse_dynamics / _backward, no
guesses) and ID forward + backward (nb2_inverse_dynamics / _backward) on the same states, the three timed alternately in one process
with CUDA events.  Prints one JSON line with the card's name, power limit and maximum SM clock.
    python scripts/dev/bench_contact_inverse_dynamics.py [--batch B ...] [--steps K] [--rounds R]"""
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
from nimblephysics_b200.inverse_dynamics import contact_body_index, contact_body_indices  # noqa: E402
from tests.util import load_raw  # noqa: E402


def measure(world, dm, raw, B, steps, rounds):
    dev = torch.device("cuda")
    n = raw.ndof
    foot = next(b for sk in world.skeletons for b in sk._ordered_bodies() if b.name == "l_foot")
    body = int(dm.cm.body_owner[contact_body_index(world, foot)])
    feet = contact_body_indices(world, [b for sk in world.skeletons for b in sk._ordered_bodies() if b.name in ("l_foot", "r_foot")])
    fbodies, fpoints = [int(dm.cm.body_owner[r]) for r in feet], [dm.cm.body_T[r][:3, 3] for r in feet]
    s, a, _ = (torch.tensor(x, device=dev) for x in make_inputs(raw, B, 555))
    nxt = torch.empty_like(s)
    stream = torch.cuda.current_stream().cuda_stream
    dm.forward_device(B, s.data_ptr(), a.data_ptr(), nxt.data_ptr(), None, stream, FP32)
    vn = nxt[:, n:].contiguous()
    sv = torch.empty((dm.saved_words, B), device=dev)
    tau, w = torch.empty((B, n), device=dev), torch.empty((B, 6), device=dev)
    gt, gw, seed = torch.randn((B, n), device=dev), torch.randn((B, 6), device=dev), torch.empty((B, n), device=dev)
    gs, gv = torch.empty_like(s), torch.empty((B, n), device=dev)
    w2, gw2 = torch.empty((B, 2, 6), device=dev), torch.randn((B, 2, 6), device=dev)

    def inv():
        dm.inverse_dynamics_device(B, s.data_ptr(), vn.data_ptr(), tau.data_ptr(), sv.data_ptr(), stream, FP32)
        dm.inverse_dynamics_backward_device(B, s.data_ptr(), sv.data_ptr(), gt.data_ptr(), gs.data_ptr(), gv.data_ptr(), stream, FP32)

    def cinv():
        dm.contact_inverse_dynamics_device(B, body, s.data_ptr(), vn.data_ptr(), tau.data_ptr(), w.data_ptr(), sv.data_ptr(), stream, FP32)
        dm.contact_inverse_dynamics_backward_device(B, body, s.data_ptr(), sv.data_ptr(), w.data_ptr(), gt.data_ptr(), gw.data_ptr(), seed.data_ptr(),
                                                    gs.data_ptr(), gv.data_ptr(), stream, FP32)

    def mcinv():
        dm.multiple_contact_inverse_dynamics_device(B, fbodies, fpoints, s.data_ptr(), vn.data_ptr(), None, tau.data_ptr(), w2.data_ptr(),
                                                    sv.data_ptr(), stream, FP32)
        dm.multiple_contact_inverse_dynamics_backward_device(B, fbodies, fpoints, s.data_ptr(), sv.data_ptr(), w2.data_ptr(), None, gt.data_ptr(),
                                                             gw2.data_ptr(), seed.data_ptr(), gs.data_ptr(), gv.data_ptr(), stream, FP32)

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

    us = {"id_fwd_bwd_us": [], "contact_id_fwd_bwd_us": [], "two_contact_id_fwd_bwd_us": []}
    for _ in range(rounds):
        us["id_fwd_bwd_us"].append(round(timed(inv), 2))
        us["contact_id_fwd_bwd_us"].append(round(timed(cinv), 2))
        us["two_contact_id_fwd_bwd_us"].append(round(timed(mcinv), 2))
    return {"batch": B, **us}


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
    rows = [measure(world, dm, raw, B, args.steps, args.rounds) for B in args.batch]
    gpu = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"model": "atlas", "precision": "fp32", "contact_body": "l_foot", "contact_bodies": ["l_foot", "r_foot"], "steps": args.steps, "gpu": gpu, "results": rows}))


if __name__ == "__main__":
    main()
