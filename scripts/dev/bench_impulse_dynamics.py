"""Times impulse dynamics (nb2_impulse_dynamics) on Atlas against the composed route (mass_matrix, world_jacobian and torch solves): feet
held 6-D (12 rows) and feet and hands (24 rows), B in {4096, 65536}, fp32 and fp64, forward and forward + backward, restitution 0.5.
CUDA events, the routes alternated over several rounds in one process; peak memory per call; the fp32 outputs against the fp64 kernel; the
card, its power limit and SM clock read in the same run.  Prints one JSON line per configuration and a summary line; --out also writes the
whole result to a JSON file."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import nimblephysics_b200 as nb  # noqa: E402
from scripts.dev.bench_constrained_dynamics import SETS, card, timed  # noqa: E402
from tests.test_forward_dynamics import fd_inputs  # noqa: E402
from tests.util import load_raw  # noqa: E402

E = 0.5


def composed(world, st, nodes):
    n, B, m = st.shape[1] // 2, st.shape[0], 6 * len(nodes)
    q, qd = st[:, :n], st[:, n:]
    M = nb.mass_matrix(world, q)
    J = nb.world_jacobian(world, q, nodes).reshape(B, m, n)
    Y = torch.linalg.solve(M, J.transpose(1, 2))
    lam = -torch.linalg.solve(J @ Y, (1 + E) * (J @ qd[..., None]))
    return qd + (Y @ lam)[..., 0], lam[..., 0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
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
                sg = st.clone().requires_grad_(True)

                def fused_f():
                    with torch.no_grad():
                        return nb.impulse_dynamics(world, st, nodes, restitution=E)

                def fused_fb():
                    v, w = nb.impulse_dynamics(world, sg, nodes, restitution=E)
                    (v.sum() + w.sum()).backward()

                def comp_f():
                    with torch.no_grad():
                        return composed(world, st, nodes)

                def comp_fb():
                    v, lam = composed(world, sg, nodes)
                    (v.sum() + lam.sum()).backward()

                routes = {"fused_fwd": fused_f, "fused_fwd_bwd": fused_fb, "composed_fwd": comp_f, "composed_fwd_bwd": comp_fb}
                for f in routes.values():  # warm-up of every shape
                    f()
                times = {k: [] for k in routes}
                mem = {}
                reps = 3 if B > 10000 else 10
                for _ in range(args.rounds):
                    for k, f in routes.items():
                        t, mb = timed(f, reps)
                        times[k].append(t)
                        mem[k] = mb
                v, w = fused_f()
                row = {"B": B, "rows": m, "dtype": str(dt).replace("torch.", ""), "us_median": {k: float(np.median(x)) for k, x in times.items()},
                       "us_min": {k: float(np.min(x)) for k, x in times.items()}, "peak_MiB": mem}
                if dt == torch.float64:
                    out64 = (v, w)
                else:
                    ev = ((v.double() - out64[0]).norm(dim=1) / out64[0].norm(dim=1).clamp_min(1e-30)).cpu().numpy()
                    ew = ((w.double() - out64[1]).flatten(1).norm(dim=1) / out64[1].flatten(1).norm(dim=1).clamp_min(1e-30)).cpu().numpy()
                    finite = np.isfinite(ev) & np.isfinite(ew)
                    row["fp32_vs_fp64"] = {"vel_worst": float(ev[finite].max()), "vel_median": float(np.median(ev[finite])),
                                           "impulse_worst": float(ew[finite].max()), "impulse_median": float(np.median(ew[finite])),
                                           "nan_worlds": int((~finite).sum())}
                res["rows"].append(row)
                print(json.dumps(row), flush=True)
    res["card_after"] = card()
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)
    print(json.dumps({"card": res["card"], "card_after": res["card_after"]}))


if __name__ == "__main__":
    main()
