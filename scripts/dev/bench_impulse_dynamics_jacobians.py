"""Times the dense Jacobians of impulse dynamics (nb2_impulse_dynamics_jacobians) on Atlas against the replicated route (every world copied
n + m times, one impulse_dynamics forward and one backward seeded with the identity rows) and one plain impulse_dynamics forward, for scale:
feet held 6-D (12 rows) and feet and hands (24 rows), B in {4096, 65536}, fp32 and fp64, restitution 0.5.  CUDA events, the routes
alternated over several rounds in one process; peak memory per call; the fp32 blocks against the fp64 ones; the card, its power limit and
SM clock read in the same run.  A route that runs out of device memory is recorded as such.  Prints one JSON line per configuration and a
summary line; --out also writes the whole result to a JSON file."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import nimblephysics_b200 as nb  # noqa: E402
from scripts.dev.bench_constrained_dynamics_jacobians import SETS, card, rel_rows, timed  # noqa: E402
from tests.test_forward_dynamics import fd_inputs  # noqa: E402
from tests.util import load_raw  # noqa: E402

E = 0.5
BLOCKS = ["dv_dq", "dv_dqdot", "dimp_dq", "dimp_dqdot"]


def replicated(world, st, nodes):
    """the blocks by autograd: each world copied n + m times, one forward, one backward seeded with the identity rows"""
    B, n, k = st.shape[0], st.shape[1] // 2, len(nodes)
    R = n + 6 * k
    sr = st.repeat_interleave(R, 0).requires_grad_(True)
    v, w = nb.impulse_dynamics(world, sr, nodes, restitution=E)
    eye = torch.eye(R, dtype=st.dtype, device=st.device).repeat(B, 1)
    (gs,) = torch.autograd.grad([v, w], [sr], [eye[:, :n], eye[:, n:].reshape(B * R, k, 6)])
    return gs.reshape(B, R, 2 * n)


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
        s, _ = fd_inputs(raw, B, seed=1)
        for m, names in SETS.items():
            nodes = [flat[x] for x in names]
            out64 = None
            for dt in (torch.float64, torch.float32):
                st = torch.tensor(s, dtype=dt, device="cuda")

                def imp_fwd():
                    with torch.no_grad():
                        return nb.impulse_dynamics(world, st, nodes, restitution=E)

                routes = {"new": lambda: nb.impulse_dynamics_jacobians(world, st, nodes, restitution=E),
                          "replicated": lambda: replicated(world, st, nodes), "imp_fwd": imp_fwd}
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
                out = nb.impulse_dynamics_jacobians(world, st, nodes, restitution=E)
                row = {"B": B, "rows": m, "dtype": str(dt).replace("torch.", ""),
                       "us_median": {k: float(np.median(v)) for k, v in times.items() if v},
                       "us_min": {k: float(np.min(v)) for k, v in times.items() if v}, "peak_MiB": mem, "failed": failed}
                if dt == torch.float64:
                    out64 = out
                    if "replicated" not in failed:  # the new blocks against the replicated route's, rows in the same layout
                        gs = replicated(world, st, nodes)
                        n = st.shape[1] // 2
                        new_rows = torch.cat([torch.cat(out[2:4], 2), torch.cat([x.reshape(B, m, n) for x in out[4:]], 2)], 1)
                        row["new_vs_replicated_fp64"] = rel_rows(new_rows, gs.double())
                        del gs
                else:
                    row["fp32_vs_fp64"] = {name: rel_rows(a, b) for name, a, b in zip(["qdot_after", "impulses"] + BLOCKS, out, out64)}
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
