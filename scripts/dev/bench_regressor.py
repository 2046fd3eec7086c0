"""Dev: the inverse-dynamics and energy regressors on the flagship model.  Atlas (n = 33, 28 canonical bodies), B worlds (default 4096 and
65536), fp32 and fp64, CUDA events, the median of R rounds in which the legs alternate, in one process:
  reg_call      inverse_dynamics_regressor(world, state, next_vel): the Python call, outputs allocated by it
  reg_kernel    nb2_inverse_dynamics_regressor into preallocated outputs (the kernel alone)
  fill          Y.fill_(0): a write of the same bytes by PyTorch's fill kernel, the write rate this card reaches
  id_saved      nb2_inverse_dynamics with its saved stream: what the ID kernel would cost before a regressor could read V and A from it
  energy        energy_regressor(world, state)
  replicated    the replicated-VJP route: B n worlds through InverseDynamicsLayer with a world_inertia gradient, seeded with e_d
                (fewer steps; skipped where it does not fit in memory)
Per row: the bytes the ID regressor writes (Y and tau_passive) over its kernel time, as a rate and as a share of the data-sheet HBM3
bandwidth of an H100 SXM (3.35 TB/s), and the largest relative difference of the replicated route's Y.  Then the fp32 accuracy against
fp64 on 4096 worlds.  Prints one JSON line per row and one with everything, with the card's name, power limit and maximum SM clock.
    python scripts/dev/bench_regressor.py [--batch B ...] [--steps K] [--rounds R]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", ".."))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import nimblephysics_b200 as nb  # noqa: E402
from nimblephysics_b200.engine import FP32, FP64  # noqa: E402
from nimblephysics_b200.inverse_dynamics import InverseDynamicsLayer  # noqa: E402
from tests.util import load_raw  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12  # H100 SXM data sheet, HBM3


def inputs(raw, B, seed, dtype):
    rng = np.random.default_rng(seed)
    n = raw.ndof
    s = np.concatenate([rng.uniform(-0.4, 0.4, (B, n)), rng.uniform(-1, 1, (B, n))], 1)
    vn = s[:, n:] + raw.dt * rng.uniform(-5, 5, (B, n))
    return torch.tensor(s, dtype=dtype, device="cuda"), torch.tensor(vn, dtype=dtype, device="cuda")


def timed(f, steps):
    for _ in range(2):
        f()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        f()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / steps  # microseconds per call


def replicated(world, st, vt, pi):
    """Y by the replicated-VJP route: world w copied n times, copy d seeded with e_d, the gradient of the per-world inertia table"""
    B, n = vt.shape
    S, V = st.repeat_interleave(n, 0), vt.repeat_interleave(n, 0)
    wi = pi.repeat_interleave(n, 0).requires_grad_(True)
    tau = InverseDynamicsLayer.apply(world, S, V, None, wi)
    tau.backward(torch.eye(n, dtype=tau.dtype, device=tau.device).repeat(B, 1))
    return wi.grad.reshape(B, n, -1, 10)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[4096, 65536])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    world._contacts_disabled = True
    dm = nb.device_model_for(world)
    n, nbod = raw.ndof, dm.cm.nb
    out = {"model": "atlas", "ndof": n, "bodies": nbod, "rows": []}
    stream = lambda: torch.cuda.current_stream().cuda_stream
    for B in args.batch:
        for dtype in (torch.float32, torch.float64):
            prec, word = (FP64, 8) if dtype == torch.float64 else (FP32, 4)
            st, vt = inputs(raw, B, 7, dtype)
            Y = torch.empty((B, n, nbod, 10), dtype=dtype, device="cuda")
            tp = torch.empty((B, n), dtype=dtype, device="cuda")
            tau = torch.empty((B, n), dtype=dtype, device="cuda")
            saved = torch.empty((dm.saved_words, B), dtype=dtype, device="cuda")
            pi = torch.tensor(dm.cm.inertia, device="cuda").expand(B, nbod, 10).contiguous()
            legs = {
                "reg_call": (lambda: nb.inverse_dynamics_regressor(world, st, vt), args.steps),
                "reg_kernel": (lambda: dm.inverse_dynamics_regressor_device(B, st.data_ptr(), vt.data_ptr(), Y.data_ptr(), tp.data_ptr(), stream(), prec),
                               args.steps),
                "fill": (lambda: Y.fill_(0), args.steps),
                "id_saved": (lambda: dm.inverse_dynamics_device(B, st.data_ptr(), vt.data_ptr(), tau.data_ptr(), saved.data_ptr(), stream(), prec),
                             args.steps),
                "energy": (lambda: nb.energy_regressor(world, st), args.steps),
            }
            row = {"B": B, "dtype": str(dtype).split(".")[-1]}
            try:
                with torch.no_grad():
                    ref = nb.inverse_dynamics_regressor(world, st, vt)[0]
                rY = replicated(world, st, vt, pi)
                row["replicated_vs_reg_rel"] = float(((rY - ref).norm() / ref.norm()).item())
                del rY
                legs["replicated"] = (lambda: replicated(world, st, vt, pi), max(1, args.steps // 10))
            except torch.OutOfMemoryError:
                row["replicated"] = "out of memory"
            torch.cuda.empty_cache()
            times = {k: [] for k in legs}
            for _ in range(args.rounds):
                for k, (f, steps) in legs.items():
                    times[k].append(timed(f, steps))
            row.update({k + "_us": round(statistics.median(v), 1) for k, v in times.items()})
            bytes_written = (B * n * nbod * 10 + B * n) * word
            row["reg_bytes"] = bytes_written
            row["reg_GBps"] = round(bytes_written / (row["reg_kernel_us"] * 1e-6) / 1e9, 1)
            row["reg_share_of_3.35TBps"] = round(bytes_written / (row["reg_kernel_us"] * 1e-6) / PEAK_BYTES_PER_S, 3)
            row["fill_share_of_3.35TBps"] = round(B * n * nbod * 10 * word / (row["fill_us"] * 1e-6) / PEAK_BYTES_PER_S, 3)
            out["rows"].append(row)
            print(json.dumps(row), flush=True)
            del Y, tp, tau, saved, pi, legs
            torch.cuda.empty_cache()
    st, vt = inputs(raw, 4096, 11, torch.float64)
    Y64, tp64 = nb.inverse_dynamics_regressor(world, st, vt)
    Y32, tp32 = nb.inverse_dynamics_regressor(world, st.float(), vt.float())
    e64, e32 = nb.energy_regressor(world, st), nb.energy_regressor(world, st.float())
    out["fp32_vs_fp64_rel"] = {k: float((a.double() - b).norm() / b.norm().clamp_min(1e-30)) for k, a, b in
                               zip(("Y", "tau_passive", "Y_T", "Y_U", "U_spring"), (Y32, tp32) + e32, (Y64, tp64) + e64)}
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    out["gpu"] = q.stdout.strip()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
