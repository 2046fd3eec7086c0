"""Times constrained forward dynamics (nb2_constrained_forward_dynamics) on Atlas against the composed route (inverse_mass_matrix,
world_jacobian, world_jacobian_deriv, forward_dynamics and a torch solve) and forward_dynamics alone: feet held 6-D (12 rows) and feet and
hands (24 rows), B in {4096, 65536}, fp32 and fp64, forward and forward + backward.  CUDA events, the routes alternated over several rounds
in one process; peak memory per call; the fp32 outputs against the fp64 kernel; the card, its power limit and SM clock read in the same run.
Prints one JSON line per configuration and a summary line; --out also writes the whole result to a JSON file."""
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


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()


def composed(world, st, tt, nodes):
    n, B, m = tt.shape[1], tt.shape[0], 6 * len(nodes)
    q = st[:, :n]
    Minv = nb.inverse_mass_matrix(world, q)
    J = nb.world_jacobian(world, q, nodes).reshape(B, m, n)
    Jd = nb.world_jacobian_deriv(world, st, nodes).reshape(B, m, n)
    qf = nb.forward_dynamics(world, st, tt)
    Y = Minv @ J.transpose(1, 2)
    lam = -torch.linalg.solve(J @ Y, (J @ qf[..., None] + Jd @ st[:, n:, None])[..., 0])
    return qf + (Y @ lam[..., None])[..., 0], lam


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
        s, tau = fd_inputs(raw, B, seed=1)
        for m, names in SETS.items():
            nodes = [flat[x] for x in names]
            out64 = None
            for dt in (torch.float64, torch.float32):
                st = torch.tensor(s, dtype=dt, device="cuda")
                tt = torch.tensor(tau, dtype=dt, device="cuda")
                sg, tg = st.clone().requires_grad_(True), tt.clone().requires_grad_(True)

                def fused_f():
                    with torch.no_grad():
                        return nb.constrained_forward_dynamics(world, st, tt, nodes)

                def fused_fb():
                    q, w = nb.constrained_forward_dynamics(world, sg, tg, nodes)
                    (q.sum() + w.sum()).backward()

                def comp_f():
                    with torch.no_grad():
                        return composed(world, st, tt, nodes)

                def comp_fb():
                    q, lam = composed(world, sg, tg, nodes)
                    (q.sum() + lam.sum()).backward()

                def fd_f():
                    with torch.no_grad():
                        return nb.forward_dynamics(world, st, tt)

                routes = {"fused_fwd": fused_f, "fused_fwd_bwd": fused_fb, "composed_fwd": comp_f, "composed_fwd_bwd": comp_fb, "forward_dynamics": fd_f}
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
                q, w = fused_f()
                row = {"B": B, "rows": m, "dtype": str(dt).replace("torch.", ""), "us_median": {k: float(np.median(v)) for k, v in times.items()},
                       "us_min": {k: float(np.min(v)) for k, v in times.items()}, "peak_MiB": mem}
                if dt == torch.float64:
                    out64 = (q, w)
                else:
                    eq = ((q.double() - out64[0]).norm(dim=1) / out64[0].norm(dim=1).clamp_min(1e-30)).cpu().numpy()
                    ew = ((w.double() - out64[1]).flatten(1).norm(dim=1) / out64[1].flatten(1).norm(dim=1).clamp_min(1e-30)).cpu().numpy()
                    finite = np.isfinite(eq) & np.isfinite(ew)
                    row["fp32_vs_fp64"] = {"qdd_worst": float(eq[finite].max()), "qdd_median": float(np.median(eq[finite])),
                                           "wrench_worst": float(ew[finite].max()), "wrench_median": float(np.median(ew[finite])),
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
