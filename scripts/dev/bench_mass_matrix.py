"""Mass matrix and its inverse on Atlas: the new kernels (forward and backward) against the batched workaround they replace,
replicated inverse_dynamics (one world per dof, unit accelerations, minus the bias run) plus torch.linalg.inv, forward and autograd
backward, measured in the same process.  CUDA events, warm-up, three alternating rounds; each time is printed next to the store floor
B * n^2 * sizeof(R) / 3.35 TB/s.  Prints the card name and power limit first.  Usage: python scripts/dev/bench_mass_matrix.py [B ...]"""
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import nimblephysics_b200 as nb  # noqa: E402
from tests.util import load_raw  # noqa: E402


def timed(f, reps):
    f()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        f()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def workaround(world, q, inverse):
    """M (or inv(M)) by replicated inverse dynamics: world b*n + j runs next velocity dt * e_j from rest, minus the bias run."""
    B, n = q.shape
    dt = world.getTimeStep()
    qr = q.repeat_interleave(n + 1, 0)
    s = torch.cat([qr, torch.zeros_like(qr)], 1)
    v = torch.zeros_like(qr)
    eye = torch.eye(n, dtype=q.dtype, device=q.device) * dt
    v.view(B, n + 1, n)[:, 1:, :] = eye
    tau = nb.inverse_dynamics(world, s, v).view(B, n + 1, n)
    M = (tau[:, 1:, :] - tau[:, :1, :]).transpose(1, 2)
    return torch.linalg.inv(M) if inverse else M


def main():
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    world._contacts_disabled = True
    n = raw.ndof
    Bs = [int(x) for x in sys.argv[1:]] or [4096, 65536]
    # fp32 accuracy of M^-1 against the fp64 kernels, per world (norm-wise), with the condition numbers of the samples
    q = torch.tensor(np.random.default_rng(0).uniform(-0.3, 0.3, (4096, n)), device="cuda")
    M64, Mi64 = nb.mass_matrix(world, q), nb.inverse_mass_matrix(world, q)
    Mi32 = nb.inverse_mass_matrix(world, q.float()).double()
    err = torch.linalg.matrix_norm(Mi32 - Mi64) / torch.linalg.matrix_norm(Mi64)
    cond = torch.linalg.cond(M64)
    print(f"fp32 M^-1 vs fp64, 4096 Atlas poses: worst {err.max().item():.2e}, median {err.median().item():.2e}; cond(M) min "
          f"{cond.min().item():.3g} median {cond.median().item():.3g} max {cond.max().item():.3g}", flush=True)
    for B in Bs:
        for dt in (torch.float32, torch.float64):
            rng = np.random.default_rng(0)
            q0 = torch.tensor(rng.uniform(-0.3, 0.3, (B, n)), dtype=dt, device="cuda")
            G = torch.randn(B, n, n, dtype=dt, device="cuda")
            floor_us = B * n * n * q0.element_size() / 3.35e12 * 1e6
            for inverse in (False, True):
                f = nb.inverse_mass_matrix if inverse else nb.mass_matrix
                name = "Minv" if inverse else "M"
                q = q0.clone().requires_grad_(True)
                out = f(world, q)

                def new_fwd():
                    with torch.no_grad():
                        f(world, q0)

                def new_bwd():
                    torch.autograd.grad(out, q, G, retain_graph=True)

                def old_fwd():
                    with torch.no_grad():
                        workaround(world, q0, inverse)

                wq = q0.clone().requires_grad_(True)
                wout = workaround(world, wq, inverse) if B * (n + 1) <= 300000 else None

                def old_bwd():
                    torch.autograd.grad(wout, wq, G, retain_graph=True)

                res = {k: [] for k in ("new_fwd", "new_bwd", "old_fwd", "old_bwd")}
                for _ in range(3):
                    res["new_fwd"].append(timed(new_fwd, 10))
                    res["old_fwd"].append(timed(old_fwd, 3))
                    res["new_bwd"].append(timed(new_bwd, 10))
                    if wout is not None:
                        res["old_bwd"].append(timed(old_bwd, 3))
                med = {k: (float(np.median(v)) * 1e3 if v else float("nan")) for k, v in res.items()}
                print(f"atlas n={n} B={B} {str(dt)[6:]} {name}: fwd {med['new_fwd']:.1f} us (workaround {med['old_fwd']:.1f}), "
                      f"bwd {med['new_bwd']:.1f} us (workaround {med['old_bwd']:.1f}), store floor {floor_us:.1f} us", flush=True)


if __name__ == "__main__":
    main()
