"""Dev: kinetic and potential energy and centroidal momentum on the flagship model.  Atlas (n = 33), B worlds (default 4096 and 65536),
fp32 and fp64, CUDA events, the median of R rounds in which the legs alternate, in one process:
  em_fwd / em_fwdbwd        energy_and_momentum: the forward, and the forward plus the backward of a random weighting of (T, U, h)
  comp_fwd / comp_fwdbwd    the composed route: T = 1/2 qdot^T M qdot (mass_matrix), p = m_tot J_com qdot (com_jacobian), the angular
                            momentum from world_jacobian of every body (k <= 32 per call) with the inertias rotated into world axes in
                            torch, U from the COM; the same outputs and the same backward
and the fp32 accuracy on 4096 samples: the norm-wise relative error of each fp32 output over the batch against the fp64 kernel.  Prints one JSON line with
the card's name, power limit and maximum SM clock.
    python scripts/dev/bench_energy.py [--batch B ...] [--steps K] [--rounds R]"""
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
from tests.util import load_raw  # noqa: E402


def inputs(raw, B, seed, dtype):
    rng = np.random.default_rng(seed)
    n = raw.ndof
    s = np.concatenate([rng.uniform(-0.4, 0.4, (B, n)), rng.uniform(-1, 1, (B, n))], 1)
    return torch.tensor(s, dtype=dtype, device="cuda")


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


def composed(world, sk, st, bodies, G6, Mt):
    """(T, U, h) from mass_matrix, com_jacobian and world_jacobian: G6 [k, 6, 6] the bodies' spatial inertias in their frames"""
    n = world.getNumDofs()
    q, qd = st[:, :n], st[:, n:]
    T = 0.5 * torch.einsum("bi,bij,bj->b", qd, nb.mass_matrix(world, q), qd)
    Jc = nb.com_jacobian(world, q, sk)
    vc = torch.einsum("brn,bn->br", Jc, qd)
    p = Mt * vc
    # body twists in world axes at the body origins, then their momenta about the world origin
    A = torch.zeros_like(p)
    for k0 in range(0, len(bodies), 32):
        bs = bodies[k0:k0 + 32]
        J = nb.world_jacobian(world, q, bs)
        V = torch.einsum("bkrn,bn->bkr", J, qd)
        W = world_poses(world, bs, st)
        R, o = W[..., :3, :3], W[..., :3, 3]
        Vb = torch.cat([torch.einsum("bkji,bkj->bki", R, V[..., :3]), torch.einsum("bkji,bkj->bki", R, V[..., 3:])], -1)
        Pb = torch.einsum("kij,bkj->bki", G6[k0:k0 + 32].to(st.dtype), Vb)
        l = torch.einsum("bkij,bkj->bki", R, Pb[..., 3:])
        A = A + (torch.einsum("bkij,bkj->bki", R, Pb[..., :3]) + torch.cross(o, l, dim=-1)).sum(1)
    ik_com = _com(world, sk, st)
    g = torch.tensor(world.getGravity(), dtype=st.dtype, device=st.device)
    U = -Mt * ik_com @ g
    h = torch.cat([A - torch.cross(ik_com, p, dim=-1), p], 1)
    return T, U, h


_IK = {}


def _com(world, sk, st):
    if id(world) not in _IK:
        ik = nb.IKMapping(world)
        ik.addSkeletonCOM(sk)
        _IK[id(world)] = ik
    return nb.map_to_pos(world, _IK[id(world)], st).to(st.dtype)


_POSE = {}


def world_poses(world, bodies, st):
    """[B, k, 4, 4] world poses of the bodies (IKMapping spatial entries: rotation vector and origin)"""
    key = (id(world), tuple(id(b) for b in bodies))
    if key not in _POSE:
        ik = nb.IKMapping(world)
        for b in bodies:
            ik.addSpatialBodyNode(b)
        _POSE[key] = ik
    x = nb.map_to_pos(world, _POSE[key], st).to(st.dtype).reshape(st.shape[0], len(bodies), 6)
    th = x[..., :3]
    a = th.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    K = torch.zeros(x.shape[:-1] + (3, 3), dtype=st.dtype, device=st.device)
    k = th / a
    K[..., 0, 1], K[..., 0, 2], K[..., 1, 2] = -k[..., 2], k[..., 1], -k[..., 0]
    K = K - K.transpose(-1, -2)
    s, c = torch.sin(a)[..., None], torch.cos(a)[..., None]
    R = torch.eye(3, dtype=st.dtype, device=st.device) + s * K + (1 - c) * K @ K
    W = torch.zeros(x.shape[:-1] + (4, 4), dtype=st.dtype, device=st.device)
    W[..., :3, :3], W[..., :3, 3], W[..., 3, 3] = R, x[..., 3:], 1
    return W


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[4096, 65536])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    sk = max(world.skeletons, key=lambda s: s.getNumDofs())
    bodies = sk._ordered_bodies()
    G6 = []
    for b in bodies:
        m, c, I = b.mass, np.asarray(b.com), np.asarray(b.moment)
        C = np.array([[0, -c[2], c[1]], [c[2], 0, -c[0]], [-c[1], c[0], 0]])
        G = np.zeros((6, 6))
        G[:3, :3], G[:3, 3:], G[3:, :3], G[3:, 3:] = I + m * C @ C.T, m * C, m * C.T, m * np.eye(3)
        G6.append(G)
    G6 = torch.tensor(np.stack(G6), device="cuda")
    Mt = float(sum(b.mass for b in bodies))
    out = {"model": "atlas", "ndof": raw.ndof, "rows": []}
    for B in args.batch:
        for dtype in (torch.float32, torch.float64):
            st = inputs(raw, B, 7, dtype)
            w8 = torch.randn(B, 8, dtype=dtype, device="cuda")

            def loss(T, U, h):
                return (torch.cat([T[:, None], U[:, None], h], 1) * w8).sum()

            def leg(route, bwd):
                def f():
                    x = st.clone().requires_grad_(bwd)
                    r = nb.energy_and_momentum(world, x, sk) if route == "em" else composed(world, sk, x, bodies, G6, Mt)
                    if bwd:
                        loss(*r).backward()
                return f
            legs = {f"{r}_{'fwdbwd' if b else 'fwd'}": leg(r, b) for r in ("em", "comp") for b in (False, True)}
            times = {k: [] for k in legs}
            for _ in range(args.rounds):
                for k, f in legs.items():
                    times[k].append(timed(f, args.steps))
            row = {"B": B, "dtype": str(dtype).split(".")[-1]}
            row.update({k + "_us": round(statistics.median(v), 1) for k, v in times.items()})
            with torch.no_grad():
                a, b = nb.energy_and_momentum(world, st, sk), composed(world, sk, st, bodies, G6, Mt)
            row["composed_vs_em_rel"] = max(float((x - y).norm() / y.norm()) for x, y in zip(b, a))
            out["rows"].append(row)
            print(json.dumps(row), flush=True)
    s64 = inputs(raw, 4096, 11, torch.float64)
    r64 = nb.energy_and_momentum(world, s64, sk)
    r32 = nb.energy_and_momentum(world, s64.float(), sk)
    out["fp32_vs_fp64_rel"] = {k: float((a.double() - b).norm() / b.norm()) for k, a, b in zip(("T", "U", "h"), r32, r64)}
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    out["gpu"] = q.stdout.strip()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
