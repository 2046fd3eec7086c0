"""Dev: contact-free forward dynamics on the flagship model.  Atlas (n = 33), B worlds (default 4096 and 65536), fp32 and fp64, CUDA events,
the median of R rounds in which the legs alternate, in one process:
  fd        nb2_forward_dynamics_batch forward, and forward + backward (the state and tau gradients)
  dense     the dense route: inverse_mass_matrix(q), inverse_dynamics(q, qdot, qdot) and a bmm; forward, and forward + autograd backward
  step      the step's forward + backward (nb2_step_forward / _backward, fp32 rows) on the same states: the reference cost of the same passes
  legacy    (fp64, with --parent-lib) nb2_forward_dynamics of this library against the same entry of another build of the library
            (e.g. the parent commit's), alternated
and the fp32 accuracy on 4096 samples: the worst and median norm-wise error of fp32 forward dynamics against the fp64 kernel, next to that
of the step-difference route (v+ - qdot) / dt of the fp32 step.  Prints one JSON line with the card's name, power limit and maximum SM clock.
    python scripts/dev/bench_forward_dynamics.py [--batch B ...] [--steps K] [--rounds R] [--parent-lib PATH]"""
import argparse
import ctypes
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
from nimblephysics_b200 import _cabi  # noqa: E402
from nimblephysics_b200.engine import FP32, FP64, DeviceModel  # noqa: E402
from tests.util import load_raw  # noqa: E402


def inputs(raw, B, seed, dtype):
    rng = np.random.default_rng(seed)
    n = raw.ndof
    s = np.concatenate([rng.uniform(-0.4, 0.4, (B, n)), rng.uniform(-1, 1, (B, n))], 1)
    tau = rng.uniform(-20, 20, (B, n))
    return torch.tensor(s, dtype=dtype, device="cuda"), torch.tensor(tau, dtype=dtype, device="cuda")


def timed(f, steps):
    for _ in range(10):
        f()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        f()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / steps  # microseconds per call


def measure(world, dm, raw, B, prec, steps, rounds, parent):
    dtype = torch.float64 if prec == FP64 else torch.float32
    n, dev = raw.ndof, torch.device("cuda")
    s, tau = inputs(raw, B, 7, dtype)
    qd = s[:, n:].contiguous()
    qdd, gs, gt = torch.empty((B, n), dtype=dtype, device=dev), torch.empty_like(s), torch.empty((B, n), dtype=dtype, device=dev)
    g = torch.randn((B, n), dtype=dtype, device=dev)
    sv = torch.empty((dm.saved_words, B), dtype=dtype, device=dev)
    stream = torch.cuda.current_stream().cuda_stream

    def fd_fwd():
        dm.forward_dynamics_device(B, s.data_ptr(), tau.data_ptr(), qdd.data_ptr(), None, stream, prec)

    def fd_fwd_bwd():
        dm.forward_dynamics_device(B, s.data_ptr(), tau.data_ptr(), qdd.data_ptr(), sv.data_ptr(), stream, prec)
        dm.forward_dynamics_backward_device(B, s.data_ptr(), sv.data_ptr(), g.data_ptr(), gs.data_ptr(), gt.data_ptr(), stream, prec)

    def dense_fwd():
        with torch.no_grad():
            return torch.bmm(nb.inverse_mass_matrix(world, s[:, :n]), (tau - nb.inverse_dynamics(world, s, qd)).unsqueeze(2))

    sg, tg = s.clone().requires_grad_(True), tau.clone().requires_grad_(True)

    def dense_fwd_bwd():
        out = torch.bmm(nb.inverse_mass_matrix(world, sg[:, :n]), (tg - nb.inverse_dynamics(world, sg, sg[:, n:])).unsqueeze(2))
        torch.autograd.grad(out, (sg, tg), g.unsqueeze(2))

    s32, a32 = s.float(), tau.float()[:, :len(raw.action_map)].contiguous()
    nxt, gs32, ga32 = torch.empty_like(s32), torch.empty_like(s32), torch.empty_like(a32)
    g32 = torch.randn_like(s32)
    sv32 = torch.empty((dm.saved_words, B), device=dev)

    def step():
        dm.forward_device(B, s32.data_ptr(), a32.data_ptr(), nxt.data_ptr(), sv32.data_ptr(), stream, FP32)
        dm.backward_device(B, s32.data_ptr(), a32.data_ptr(), sv32.data_ptr(), g32.data_ptr(), gs32.data_ptr(), ga32.data_ptr(), stream, FP32)

    legs = {"fd_fwd_us": fd_fwd, "fd_fwd_bwd_us": fd_fwd_bwd, "dense_fwd_us": dense_fwd, "dense_fwd_bwd_us": dense_fwd_bwd, "step_fwd_bwd_us": step}
    if prec == FP64 and parent is not None:
        pos, vel, acc = s[:, :n].contiguous(), qd, torch.empty((B, n), dtype=dtype, device=dev)
        for key, (L, h) in (("legacy_this_us", (_cabi.lib(), dm.handle)), ("legacy_parent_us", parent)):
            legs[key] = (lambda L=L, h=h: _cabi.check(L.nb2_forward_dynamics(h, B, pos.data_ptr(), vel.data_ptr(), tau.data_ptr(),
                                                                                 acc.data_ptr(), stream)))
    us = {k: [] for k in legs}
    for _ in range(rounds):
        for k, f in legs.items():
            us[k].append(timed(f, steps))
    row = {"batch": B, "precision": "fp64" if prec == FP64 else "fp32"}
    row.update({k: round(statistics.median(v), 2) for k, v in us.items()})
    return row


def accuracy(world, dm, raw, B=4096):
    """fp32 forward dynamics and the fp32 step difference against the fp64 kernel: (worst, median) of |x - ref| / |ref| per world."""
    n = raw.ndof
    s, tau = inputs(raw, B, 11, torch.float64)
    ref = nb.forward_dynamics(world, s, tau)
    fd32 = nb.forward_dynamics(world, s.float(), tau.float()).double()
    nxt = nb.timestep(world, s.float(), tau.float()[:, :len(raw.action_map)])
    sd = ((nxt[:, n:].double() - s.float()[:, n:].double()) / raw.dt)
    err = lambda x: (x - ref).norm(dim=1) / ref.norm(dim=1)
    out = {}
    for k, x in (("fd_fp32", fd32), ("step_difference_fp32", sd)):
        e = err(x)
        out[k] = {"worst": float(e.max()), "median": float(e.median())}
    return out


def parent_model(path, raw):
    """A model of `raw` in another build of libnb2 (its own handle), for the legacy entry's A/B."""
    L = ctypes.CDLL(path)
    L.nb2_model_create.argtypes = [ctypes.POINTER(_cabi.Nb2ModelDesc), ctypes.POINTER(ctypes.c_void_p)]
    L.nb2_forward_dynamics.argtypes = [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 5
    L.nb2_last_error.restype = ctypes.c_char_p
    cm = nb.compile_model(raw, lanes=1)
    cm.shape_body = cm.shape_body[:0]
    desc, keep = _cabi.make_desc(cm, with_contacts=False)
    h = ctypes.c_void_p()
    if L.nb2_model_create(ctypes.byref(desc), ctypes.byref(h)) != 0:
        raise RuntimeError(L.nb2_last_error().decode())
    return L, h, keep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[4096, 65536])
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--parent-lib", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU (no CPU fallback)"
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    world._contacts_disabled = True
    world.setActionSpace(range(raw.ndof))
    dm = nb.device_model_for(world)
    parent = None
    if args.parent_lib:
        L, h, keep = parent_model(args.parent_lib, raw)
        parent = (L, h)
    rows = [measure(world, dm, raw, B, prec, args.steps, args.rounds, parent) for B in args.batch for prec in (FP32, FP64)]
    gpu = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"model": "atlas", "steps": args.steps, "rounds": args.rounds, "gpu": gpu, "results": rows,
                      "accuracy_4096": accuracy(world, dm, raw)}))


if __name__ == "__main__":
    main()
