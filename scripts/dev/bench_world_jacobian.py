"""World Jacobians on Atlas (nodes l_foot, r_foot, l_hand, r_hand, and the skeleton's COM): the new kernels, forward and backward, in
fp32 and fp64, against the batched workaround in the same process: an IKMapping with the four spatial entries and the COM entry, the
state replicated once per mapped row (6k + 3 rows per world) and one map_to_vel backward of the identity.  The workaround runs in fp32
only and has no position gradient (map_to_vel sends gradients only to qdot), so the backward has nothing to compare against.  CUDA
events, warm-up, three alternating rounds, medians; each forward is printed next to its store floor B * (6k + 3) * n * sizeof(R) / 3.35 TB/s.
Prints the card name and power limit first.  Usage: python scripts/dev/bench_world_jacobian.py [B ...]"""
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import nimblephysics_b200 as nb  # noqa: E402
from tests.util import load_raw  # noqa: E402

NODES = ["l_foot", "r_foot", "l_hand", "r_hand"]


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


def main():
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    world._contacts_disabled = True
    n = raw.ndof
    by = {b.name: b for sk in world.skeletons for b in sk._ordered_bodies()}
    nodes = [by[k] for k in NODES]
    sk = max(world.skeletons, key=lambda s: s.getNumDofs())
    ik = nb.IKMapping(world)
    for b in nodes:
        ik.addSpatialBodyNode(b)
    ik.addSkeletonCOM(sk)
    d = ik.getPosDim()
    Bs = [int(x) for x in sys.argv[1:]] or [4096, 65536]
    for B in Bs:
        rng = np.random.default_rng(0)
        s = np.concatenate([rng.uniform(-0.3, 0.3, (B, n)), rng.uniform(-1, 1, (B, n))], 1)
        for dt in (torch.float32, torch.float64):
            st = torch.tensor(s, dtype=dt, device="cuda")
            q0 = st[:, :n].contiguous()
            G = torch.randn(B, len(nodes), 6, n, dtype=dt, device="cuda")
            Gc = torch.randn(B, 3, n, dtype=dt, device="cuda")
            floor_us = B * (6 * len(nodes) + 3) * n * q0.element_size() / 3.35e12 * 1e6
            q = q0.clone().requires_grad_(True)
            J, Jc = nb.world_jacobian(world, q, nodes), nb.com_jacobian(world, q, sk)

            def new_fwd():
                with torch.no_grad():
                    nb.world_jacobian(world, q0, nodes)
                    nb.com_jacobian(world, q0, sk)

            def new_bwd():
                torch.autograd.grad([J, Jc], q, [G, Gc], retain_graph=True)

            rep = st.float().repeat_interleave(d, 0).requires_grad_(True)
            eye = torch.eye(d, device="cuda").repeat(B, 1)

            def old_fwd():
                rep.grad = None
                nb.map_to_vel(world, ik, rep).backward(eye)

            res = {k: [] for k in ("new_fwd", "new_bwd", "old_fwd")}
            for _ in range(3):
                res["new_fwd"].append(timed(new_fwd, 20))
                res["new_bwd"].append(timed(new_bwd, 20))
                if dt == torch.float32:
                    res["old_fwd"].append(timed(old_fwd, 3))
            med = {k: (float(np.median(v)) * 1e3 if v else float("nan")) for k, v in res.items()}
            print(f"atlas n={n} k={len(nodes)}+COM B={B} {str(dt)[6:]}: fwd {med['new_fwd']:.1f} us (workaround, fp32: {med['old_fwd']:.1f}), "
                  f"bwd {med['new_bwd']:.1f} us (no workaround), store floor {floor_us:.1f} us", flush=True)
        # the two kernels of the forward separately, fp32
        q0 = torch.tensor(s[:, :n], dtype=torch.float32, device="cuda")
        tp = np.median([timed(lambda: nb.world_jacobian(world, q0, nodes), 20) for _ in range(3)]) * 1e3
        tc = np.median([timed(lambda: nb.com_jacobian(world, q0, sk), 20) for _ in range(3)]) * 1e3
        print(f"  B={B} fp32 forward split: body points {tp:.1f} us, COM {tc:.1f} us", flush=True)
        jdot_leg(world, raw, nodes, sk, s)


def jdot_leg(world, raw, nodes, sk, s, h=5e-3):
    """Jdot (world_jacobian_deriv + com_jacobian_deriv) forward and backward, the same-process J forward, and the central-difference
    workaround (J at q (+) h qdot and q (+) -h qdot, positions prepared outside the timed window) with its fp32 error against the fp64
    kernel; the fp32 kernel's own error beside it."""
    from tests.test_world_jacobian_deriv import advance
    from tests.util import rel_err

    B, n = s.shape[0], raw.ndof
    qp = np.stack([advance(raw, s[w, :n], s[w, n:], h) for w in range(B)])
    qm = np.stack([advance(raw, s[w, :n], s[w, n:], -h) for w in range(B)])
    ref = None
    for dt in (torch.float64, torch.float32):
        st = torch.tensor(s, dtype=dt, device="cuda")
        q0, ps, ms = st[:, :n].contiguous(), torch.tensor(qp, dtype=dt, device="cuda"), torch.tensor(qm, dtype=dt, device="cuda")
        G = torch.randn(B, len(nodes), 6, n, dtype=dt, device="cuda")
        Gc = torch.randn(B, 3, n, dtype=dt, device="cuda")
        sg = st.clone().requires_grad_(True)
        dJ, dJc = nb.world_jacobian_deriv(world, sg, nodes), nb.com_jacobian_deriv(world, sg, sk)

        def jd_fwd():
            with torch.no_grad():
                return nb.world_jacobian_deriv(world, st, nodes), nb.com_jacobian_deriv(world, st, sk)

        def jd_bwd():
            torch.autograd.grad([dJ, dJc], sg, [G, Gc], retain_graph=True)

        def j_fwd():
            with torch.no_grad():
                nb.world_jacobian(world, q0, nodes)
                nb.com_jacobian(world, q0, sk)

        def cd_fwd():
            with torch.no_grad():
                return ((nb.world_jacobian(world, ps, nodes) - nb.world_jacobian(world, ms, nodes)) / (2 * h),
                        (nb.com_jacobian(world, ps, sk) - nb.com_jacobian(world, ms, sk)) / (2 * h))

        res = {k: [] for k in ("jd_fwd", "jd_bwd", "j_fwd", "cd_fwd")}
        for _ in range(3):
            for k, f in (("jd_fwd", jd_fwd), ("jd_bwd", jd_bwd), ("j_fwd", j_fwd), ("cd_fwd", cd_fwd)):
                res[k].append(timed(f, 20))
        med = {k: float(np.median(v)) * 1e3 for k, v in res.items()}
        flat = lambda pair: torch.cat([pair[0].reshape(B, -1), pair[1].reshape(B, -1)], 1).double().cpu().numpy()
        if ref is None:
            ref = flat(jd_fwd())
        err = f", fp32 error vs the fp64 kernel: kernel {rel_err(flat(jd_fwd()), ref):.1e}, central differences (h = {h}) " \
              f"{rel_err(flat(cd_fwd()), ref):.1e}" if dt == torch.float32 else ""
        print(f"  B={B} {str(dt)[6:]} Jdot ({len(nodes)} nodes + COM): fwd {med['jd_fwd']:.1f} us, bwd {med['jd_bwd']:.1f} us; "
              f"J fwd {med['j_fwd']:.1f} us; central-difference workaround {med['cd_fwd']:.1f} us{err}", flush=True)


if __name__ == "__main__":
    main()
