"""Dev: dense Jacobians of inverse and forward dynamics on the flagship model.  Atlas (n = 33), B worlds (default 4096 and 65536), fp32 and
fp64, CUDA events, the median of R rounds in which the legs alternate, in one process:
  idj / fdj          nb2_inverse_dynamics_jacobians / nb2_forward_dynamics_jacobians: the output and its three n x n blocks, one launch
  id_rep / fd_rep    the replicated VJP route of step_jacobians: every world copied n times, one forward launch (with the saved stream) and
                     one backward launch seeded with the rows of the identity, over B n worlds
  fd_fwd             one nb2_forward_dynamics_batch forward over the B worlds, for scale
with the peak device memory (torch.cuda.max_memory_allocated above what the inputs hold) of one call of each route, and the fp32 accuracy
on 4096 samples: the worst and median norm-wise error of each fp32 block against the fp64 kernel.  Prints one JSON line with the card's
name, power limit and maximum SM clock.
    python scripts/dev/bench_dynamics_jacobians.py [--batch B ...] [--steps K] [--rounds R]"""
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
from tests.util import load_raw  # noqa: E402


def inputs(raw, B, seed, dtype):
    rng = np.random.default_rng(seed)
    n = raw.ndof
    s = np.concatenate([rng.uniform(-0.4, 0.4, (B, n)), rng.uniform(-1, 1, (B, n))], 1)
    vn = s[:, n:] + raw.dt * rng.uniform(-5, 5, (B, n))
    tau = rng.uniform(-20, 20, (B, n))
    return tuple(torch.tensor(a, dtype=dtype, device="cuda") for a in (s, vn, tau))


def timed(f, steps):
    for _ in range(3):
        f()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        f()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / steps  # microseconds per call


def legs_for(dm, raw, B, prec):
    """{name: callable} of one call of every leg, with its buffers allocated inside (so that one call's peak memory is the route's)."""
    dtype = torch.float64 if prec == FP64 else torch.float32
    n, dev = raw.ndof, torch.device("cuda")
    s, vn, tau = inputs(raw, B, 7, dtype)
    stream = torch.cuda.current_stream().cuda_stream
    eye = torch.eye(n, dtype=dtype, device=dev).repeat(B, 1)  # row w * n + i: e_i

    def jac(fd):
        def f():
            out = torch.empty((B, n), dtype=dtype, device=dev)
            J = [torch.empty((B, n, n), dtype=dtype, device=dev) for _ in range(3)]
            run = dm.forward_dynamics_jacobians_device if fd else dm.inverse_dynamics_jacobians_device
            run(B, s.data_ptr(), (tau if fd else vn).data_ptr(), out.data_ptr(), *(j.data_ptr() for j in J), stream, prec)
        return f

    def rep(fd):
        def f():
            Bn = B * n
            sr = s.repeat_interleave(n, 0)
            xr = (tau if fd else vn).repeat_interleave(n, 0)
            out = torch.empty((Bn, n), dtype=dtype, device=dev)
            sv = torch.empty((dm.saved_words, Bn), dtype=dtype, device=dev)
            gs, gx = torch.empty((Bn, 2 * n), dtype=dtype, device=dev), torch.empty((Bn, n), dtype=dtype, device=dev)
            if fd:
                dm.forward_dynamics_device(Bn, sr.data_ptr(), xr.data_ptr(), out.data_ptr(), sv.data_ptr(), stream, prec)
                dm.forward_dynamics_backward_device(Bn, sr.data_ptr(), sv.data_ptr(), eye.data_ptr(), gs.data_ptr(), gx.data_ptr(), stream, prec)
            else:
                dm.inverse_dynamics_device(Bn, sr.data_ptr(), xr.data_ptr(), out.data_ptr(), sv.data_ptr(), stream, prec)
                dm.inverse_dynamics_backward_device(Bn, sr.data_ptr(), sv.data_ptr(), eye.data_ptr(), gs.data_ptr(), gx.data_ptr(), stream, prec)
        return f

    qdd = torch.empty((B, n), dtype=dtype, device=dev)
    legs = {"idj_us": jac(False), "id_rep_us": rep(False), "fdj_us": jac(True), "fd_rep_us": rep(True),
            "fd_fwd_us": lambda: dm.forward_dynamics_device(B, s.data_ptr(), tau.data_ptr(), qdd.data_ptr(), None, stream, prec)}
    return legs


def peak_bytes(f):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    f()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def measure(dm, raw, B, prec, steps, rounds):
    legs = legs_for(dm, raw, B, prec)
    row = {"batch": B, "precision": "fp64" if prec == FP64 else "fp32"}
    row.update({k.replace("_us", "_peak_MB"): round(peak_bytes(f) / 2**20, 1) for k, f in legs.items() if k != "fd_fwd_us"})
    us = {k: [] for k in legs}
    for _ in range(rounds):
        for k, f in legs.items():
            us[k].append(timed(f, steps))
    row.update({k: round(statistics.median(v), 2) for k, v in us.items()})
    return row


def accuracy(world, raw, B=4096):
    """fp32 blocks against the fp64 kernel: (worst, median) over worlds of |J32 - J64|_F / |J64|_F."""
    s, vn, tau = inputs(raw, B, 11, torch.float64)
    out = {}
    for name, fn, x in (("id", nb.inverse_dynamics_jacobians, vn), ("fd", nb.forward_dynamics_jacobians, tau)):
        ref = fn(world, s, x)
        got = fn(world, s.float(), x.float())
        for k, a, b in zip(("out", "d_q", "d_qdot", "d_x"), got, ref):
            e = (a.double() - b).flatten(1).norm(dim=1) / b.flatten(1).norm(dim=1)
            out[f"{name}_{k}"] = {"worst": float(e.max()), "median": float(e.median())}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[4096, 65536])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU (no CPU fallback)"
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    world._contacts_disabled = True
    dm = nb.device_model_for(world)
    rows = [measure(dm, raw, B, prec, args.steps, args.rounds) for B in args.batch for prec in (FP32, FP64)]
    gpu = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"model": "atlas", "steps": args.steps, "rounds": args.rounds, "gpu": gpu, "results": rows,
                      "accuracy_4096": accuracy(world, raw)}))


if __name__ == "__main__":
    main()
