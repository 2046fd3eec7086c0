"""Times the dense Jacobians of constrained forward dynamics (nb2_constrained_forward_dynamics_jacobians) on Atlas against the replicated
route (every world copied n + m times, one constrained_forward_dynamics forward and one backward seeded with the identity rows) and one plain
constrained_forward_dynamics forward, for scale: feet held 6-D (12 rows) and feet and hands (24 rows), B in {4096, 65536}, fp32 and fp64.
CUDA events, the routes alternated over several rounds in one process; peak memory per call; the fp32 blocks against the fp64 ones; the card,
its power limit and SM clock read in the same run.  A route that runs out of device memory is recorded as such.  Prints one JSON line per
configuration and a summary line; --out also writes the whole result to a JSON file."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import nimblephysics_b200 as nb  # noqa: E402
from tests.test_forward_dynamics import fd_inputs  # noqa: E402
from tests.util import load_raw  # noqa: E402

SETS = {12: ["l_foot", "r_foot"], 24: ["l_foot", "r_foot", "l_hand", "r_hand"]}
BLOCKS = ["dqdd_dq", "dqdd_dqdot", "dqdd_dtau", "dwrench_dq", "dwrench_dqdot", "dwrench_dtau"]


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()


def replicated(world, st, tt, nodes):
    """the blocks by autograd: each world copied n + m times, one forward, one backward seeded with the identity rows"""
    B, n, m = tt.shape[0], tt.shape[1], 6 * len(nodes)
    R = n + m
    sr = st.repeat_interleave(R, 0).requires_grad_(True)
    tr = tt.repeat_interleave(R, 0).requires_grad_(True)
    q, w = nb.constrained_forward_dynamics(world, sr, tr, nodes)
    eye = torch.eye(R, dtype=st.dtype, device=st.device).repeat(B, 1)
    gs, gt = torch.autograd.grad([q, w], [sr, tr], [eye[:, :n], eye[:, n:].reshape(B * R, len(nodes), 6)])
    return gs.reshape(B, R, 2 * n), gt.reshape(B, R, n)


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / reps, (torch.cuda.max_memory_allocated() - base) / 2**20


def rel_rows(x, ref):
    """per-world norm-wise relative error of x against ref (worlds finite in both): (worst, median, worlds left out)"""
    e = ((x.double() - ref).flatten(1).norm(dim=1) / ref.flatten(1).norm(dim=1).clamp_min(1e-30)).cpu().numpy()
    ok = np.isfinite(e)
    return {"worst": float(e[ok].max()), "median": float(np.median(e[ok])), "nan_worlds": int((~ok).sum())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the result to this JSON file")
    ap.add_argument("--sizes", default="4096,65536")
    args = ap.parse_args()
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    flat = {b.name: b for sk in world.skeletons for b in sk._ordered_bodies()}
    res = {"card": card(), "rows": []}
    for B in [int(x) for x in args.sizes.split(",")]:
        s, tau = fd_inputs(raw, B, seed=1)
        for m, names in SETS.items():
            nodes = [flat[x] for x in names]
            out64 = None
            for dt in (torch.float64, torch.float32):
                st = torch.tensor(s, dtype=dt, device="cuda")
                tt = torch.tensor(tau, dtype=dt, device="cuda")
                routes = {"new": lambda: nb.constrained_forward_dynamics_jacobians(world, st, tt, nodes),
                          "replicated": lambda: replicated(world, st, tt, nodes)}

                def cfd_fwd():
                    with torch.no_grad():
                        return nb.constrained_forward_dynamics(world, st, tt, nodes)

                routes["cfd_fwd"] = cfd_fwd
                times, mem, failed = {k: [] for k in routes}, {}, {}
                for k, f in routes.items():  # warm-up of every shape; a route that does not fit is recorded, not timed
                    try:
                        f()
                    except torch.cuda.OutOfMemoryError:
                        failed[k] = "out of device memory"
                    torch.cuda.empty_cache()
                reps = 1 if B > 10000 else 5
                for _ in range(args.rounds):
                    for k, f in routes.items():
                        if k not in failed:
                            t, mb = timed(f, reps)
                            times[k].append(t)
                            mem[k] = mb
                out = nb.constrained_forward_dynamics_jacobians(world, st, tt, nodes)
                row = {"B": B, "rows": m, "dtype": str(dt).replace("torch.", ""),
                       "us_median": {k: float(np.median(v)) for k, v in times.items() if v},
                       "us_min": {k: float(np.min(v)) for k, v in times.items() if v}, "peak_MiB": mem, "failed": failed}
                if dt == torch.float64:
                    out64 = out
                    if "replicated" not in failed:  # the new blocks against the replicated route's, rows in the same layout
                        gs, gt = replicated(world, st, tt, nodes)
                        n = tt.shape[1]
                        new_rows = torch.cat([torch.cat(out[2:5], 2), torch.cat([x.reshape(B, m, n) for x in out[5:]], 2)], 1)
                        row["new_vs_replicated_fp64"] = rel_rows(new_rows, torch.cat([gs, gt], 2).double())
                        del gs, gt
                else:
                    row["fp32_vs_fp64"] = {name: rel_rows(a, b) for name, a, b in zip(["qdd", "wrench"] + BLOCKS, out, out64)}
                res["rows"].append(row)
                print(json.dumps(row), flush=True)
                del out
                torch.cuda.empty_cache()
    res["card_after"] = card()
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)
    print(json.dumps({"card": res["card"], "card_after": res["card_after"]}))


if __name__ == "__main__":
    main()
