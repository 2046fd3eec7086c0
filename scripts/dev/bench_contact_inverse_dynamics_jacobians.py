"""Times the dense Jacobians of contact inverse dynamics (nb2_multiple_contact_inverse_dynamics_jacobians) on Atlas against the replicated
route (every world copied n + 6k times, one multiple_contact_inverse_dynamics forward and one backward seeded with the identity rows) and
one inverse_dynamics_jacobians call, for scale: k = 1 (l_foot), 2 (the feet) and 4 (feet and hands), B in {4096, 65536}, fp32 and fp64.
CUDA events, the routes alternated over several rounds in one process; peak memory per call; the fp32 blocks against the fp64 ones; the
card, its power limit and SM clock read in the same run.  A route that runs out of device memory is recorded as such.  Prints one JSON line
per configuration and a summary line; --out also writes the whole result to a JSON file."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import nimblephysics_b200 as nb  # noqa: E402
from scripts.dev.bench_constrained_dynamics_jacobians import card, rel_rows, timed  # noqa: E402
from tests.test_inverse_dynamics import id_inputs  # noqa: E402
from tests.util import load_raw  # noqa: E402

SETS = {1: ["l_foot"], 2: ["l_foot", "r_foot"], 4: ["l_foot", "r_foot", "l_hand", "r_hand"]}
BLOCKS = ["dtau_dq", "dtau_dqdot", "dtau_dnext_vel", "dw_dq", "dw_dqdot", "dw_dnext_vel"]


def replicated(world, st, vt, nodes):
    """the [q, qdot, next_vel] blocks by autograd: each world copied n + 6k times, one forward, one backward seeded with the identity rows"""
    B, n, k = st.shape[0], st.shape[1] // 2, len(nodes)
    R = n + 6 * k
    sr = st.repeat_interleave(R, 0).requires_grad_(True)
    vr = vt.repeat_interleave(R, 0).requires_grad_(True)
    tau, w = nb.multiple_contact_inverse_dynamics(world, sr, vr, nodes)
    eye = torch.eye(R, dtype=st.dtype, device=st.device).repeat(B, 1)
    gs, gv = torch.autograd.grad([tau, w], [sr, vr], [eye[:, :n], eye[:, n:].reshape(B * R, k, 6)])
    return torch.cat([gs, gv], 1).reshape(B, R, 3 * n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the result to this JSON file")
    ap.add_argument("--sizes", default="4096,65536")
    args = ap.parse_args()
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    world._contacts_disabled = True
    flat = {b.name: b for sk in world.skeletons for b in sk._ordered_bodies()}
    res = {"card": card(), "rows": []}
    for B in [int(x) for x in args.sizes.split(",")]:
        s, vn = id_inputs(raw, B, seed=1)
        for k, names in SETS.items():
            nodes = [flat[x] for x in names]
            out64 = None
            for dt in (torch.float64, torch.float32):
                st = torch.tensor(s, dtype=dt, device="cuda")
                vt = torch.tensor(vn, dtype=dt, device="cuda")
                routes = {"new": lambda: nb.multiple_contact_inverse_dynamics_jacobians(world, st, vt, nodes),
                          "replicated": lambda: replicated(world, st, vt, nodes), "id_jacobians": lambda: nb.inverse_dynamics_jacobians(world, st, vt)}
                times, mem, failed = {r: [] for r in routes}, {}, {}
                for r, f in routes.items():  # warm-up of every shape; a route that does not fit is recorded, not timed
                    try:
                        f()
                    except torch.cuda.OutOfMemoryError:
                        failed[r] = "out of device memory"
                    torch.cuda.empty_cache()
                reps = 1 if B > 10000 else 5
                for _ in range(args.rounds):
                    for r, f in routes.items():
                        if r not in failed:
                            t, mb = timed(f, reps)
                            times[r].append(t)
                            mem[r] = mb
                out = nb.multiple_contact_inverse_dynamics_jacobians(world, st, vt, nodes)
                n = st.shape[1] // 2
                blocks = [out[2], out[3], out[4]] + [x.reshape(B, 6 * k, n) for x in out[6:9]]
                row = {"B": B, "k": k, "rows": n + 6 * k, "dtype": str(dt).replace("torch.", ""),
                       "us_median": {r: float(np.median(v)) for r, v in times.items() if v},
                       "us_min": {r: float(np.min(v)) for r, v in times.items() if v}, "peak_MiB": mem, "failed": failed}
                if dt == torch.float64:
                    out64 = [out[0], out[1].reshape(B, -1)] + blocks
                    if "replicated" not in failed:  # the new blocks against the replicated route's, rows in the same layout
                        ref = replicated(world, st, vt, nodes)
                        new_rows = torch.cat([torch.cat(blocks[:3], 2), torch.cat(blocks[3:], 2)], 1)
                        row["new_vs_replicated_fp64"] = rel_rows(new_rows, ref.double())
                        del ref
                else:
                    got = [out[0], out[1].reshape(B, -1)] + blocks
                    row["fp32_vs_fp64"] = {name: rel_rows(a, b) for name, a, b in zip(["tau", "wrenches"] + BLOCKS, got, out64)}
                res["rows"].append(row)
                print(json.dumps(row), flush=True)
                del out, blocks
                torch.cuda.empty_cache()
    res["card_after"] = card()
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)
    print(json.dumps({"card": res["card"], "card_after": res["card_after"]}))


if __name__ == "__main__":
    main()
