"""Dev: per-stage cycles of the contact-free step kernels (k_step_fwd / k_step_bwd), Atlas fp32, from a -DNB2_STEP_CLOCKS build.

    nvcc <the flags of __graft_entry__.NVCC_FLAGS> -DNB2_STEP_CLOCKS -o build/clk/libnb2.so nimblephysics_b200/csrc/nb2_kernels.cu nimblephysics_b200/csrc/nb2_fd.cu
    NB2_LIB=build/clk/libnb2.so python scripts/dev/stage_clocks.py [--batch 4096] [--lanes 4 1] [--reps 20]

Thread 0 of a few groups spread over the grid records clock64() at kernel entry, after the wait for the previous kernel
(griddepcontrol.wait), after the input staging and after every stage with its barrier (nb2_kernels.cu, NB2_CLK).
The backward of a rep is launched right behind its forward, so its wait covers the forward's tail.  Thread 0 of a group is in
its warp 0, lane 0 of the schedule: the lane that sweeps the trunk.  For every stage the table gives the median over the sampled groups and
launches, and for the body sweeps the number of bodies lane 0 walks in it and the cycles per body.  Cycles are SM clocks; the
instrumented build adds a few instructions per stage, so compare stages with each other, not with the default build's kernel
times.
"""
import argparse
import ctypes
import os
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", ".."))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import nimblephysics_b200 as nb
from nimblephysics_b200 import _cabi
from nimblephysics_b200.engine import FP32
from bench import make_inputs

GROUPS, SLOTS = 8, 16
# stage names and which body set lane 0 sweeps in it ("trunk", "limb" or None): world_forward_stage / world_backward_stage
FWD = [("load q, v, tau", None), ("kinematics trunk", "trunk"), ("kinematics limbs", "limb"), ("inertias limbs", "limb"),
       ("inertias trunk", "trunk"), ("accelerations trunk", "trunk"), ("accelerations limbs", "limb"), ("store q+, v+", None)]
BWD = [("load g, q, v, tau", None), ("B1 limbs", "limb"), ("B1 trunk", "trunk"), ("B2 trunk", "trunk"), ("B2 limbs", "limb"),
       ("B3 limbs", "limb"), ("assemble limbs", "limb"), ("B3 trunk", "trunk"), ("assemble trunk", "trunk"), ("clip + store", None)]


def bodies(ranges):
    return sum(hi - lo for lo, hi in ranges)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--lanes", type=int, nargs="+", default=[4, 1])
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "stage_clocks.py needs a GPU"
    L = _cabi.lib()
    buf = (ctypes.c_longlong * (2 * GROUPS * SLOTS))()
    if not hasattr(L, "nb2_step_clocks_read") or not L.nb2_step_clocks_read(buf, 1):
        sys.exit("stage_clocks.py needs a library built with -DNB2_STEP_CLOCKS (set NB2_LIB to it)")
    raw = nb.RawModel.load(os.path.join(ROOT, "tests", "golden", "models", "atlas.json"))
    dm = nb.DeviceModel.from_raw(raw)
    B, n, na = args.batch, raw.ndof, len(raw.action_map)
    s, a, g = (torch.tensor(x, device="cuda") for x in make_inputs(raw, B, 1234))
    nxt, gs, ga = torch.empty((B, 2 * n), device="cuda"), torch.empty((B, 2 * n), device="cuda"), torch.empty((B, na), device="cuda")
    saved = torch.empty((dm.saved_words, B), device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    print(f"{torch.cuda.get_device_name()}  Atlas fp32, B = {B}; cycles = median over {args.reps} launches x up to {GROUPS} sampled groups")
    for K in args.lanes:
        dm.set_lanes(K)
        assert dm.lanes_for(B, False, FP32) == K and dm.lanes_for(B, True, FP32) == K, f"no {K}-lane schedule"
        cm = next(c for c in dm.schedules if c.lanes == K)
        nbody = {"trunk": bodies(cm.trunk_ranges), "limb": bodies(cm.limb_ranges[0]) if cm.limb_ranges else 0}
        runs = [[], []]
        for rep in range(args.reps + 3):
            L.nb2_step_clocks_read(None, 1)
            dm.forward_device(B, s.data_ptr(), a.data_ptr(), nxt.data_ptr(), saved.data_ptr(), stream, FP32)
            dm.backward_device(B, s.data_ptr(), a.data_ptr(), saved.data_ptr(), g.data_ptr(), gs.data_ptr(), ga.data_ptr(), stream, FP32)
            torch.cuda.synchronize()
            L.nb2_step_clocks_read(buf, 0)
            if rep < 3:  # warm-up launches
                continue
            c = np.frombuffer(buf, dtype=np.int64).reshape(2, GROUPS, SLOTS)
            for d, stages in ((0, FWD), (1, BWD)):
                for w in range(GROUPS):
                    t = c[d, w, :len(stages) + 3]
                    if t[0] and np.all(t[1:] >= t[:-1]):
                        runs[d].append(np.diff(t))
        print(f"\n--- K = {K} lanes per world: lane 0 sweeps {nbody['trunk']} trunk bodies and {nbody['limb']} limb bodies ---")
        for d, (kname, stages) in enumerate((("k_step_fwd", FWD), ("k_step_bwd", BWD))):
            if not runs[d]:
                print(f"{kname}: no samples")
                continue
            med = np.median(np.stack(runs[d]), axis=0)
            print(f"{kname} ({len(runs[d])} samples)   {'stage':<22}{'cycles':>9}{'bodies':>8}{'per body':>10}")
            print(f"{'':<24}{'entry: wait for previous kernel':<33}{med[0]:>9.0f}")
            print(f"{'':<24}{'entry: input staging':<33}{med[1]:>9.0f}")
            groups = {"fixed": med[1], "trunk": 0.0, "limb": 0.0}
            for k, (name, part) in enumerate(stages):
                cyc = med[2 + k]
                nbk = nbody[part] if part else 0
                per = f"{cyc / nbk:>10.0f}" if nbk else ""
                print(f"{'':<24}{k:>2} {name:<30}{cyc:>9.0f}{(nbk or ''):>8}{per}")
                groups[part or "fixed"] += cyc
            tot = sum(groups.values())  # without the wait: the chain of the kernel itself
            print(f"{'':<24}total {tot:.0f} cycles: fixed {groups['fixed'] / tot:.0%}, trunk stages {groups['trunk'] / tot:.0%}, "
                  f"limb stages {groups['limb'] / tot:.0%}")
    dm.set_lanes(0)


if __name__ == "__main__":
    main()
