"""The contact-free step kernels are launched as programmatic dependents of the kernel before them in the stream (griddepcontrol):
a launch is processed while its predecessor completes, and waits for it before its first global memory access.  Every chain below
is queued with no host synchronise and must give, bit for bit, what the same launches give with torch.cuda.synchronize() between
them: read-after-write across forwards, forward -> backward and the backward's accumulating rollout mode, a torch kernel writing
the backward's input, and write-after-read (a forward overwriting the state and saved stream a backward is still reading).
Racecheck does not see hazards between kernels; these tests and the SASS order check are the guard."""
import os
import re
import shutil
import subprocess

import pytest

from nimblephysics_b200._cabi import LIB_PATH
from tests.util import load_raw, sample_inputs

T = 16
# SASS opcodes that touch global memory (loads, stores, async and bulk copies, atomics and reductions, generic accesses)
GLOBAL_ACCESS = {"LDG", "STG", "LDGSTS", "UBLKCP", "UTMALDG", "UTMASTG", "ATOM", "ATOMG", "RED", "REDG", "LD", "ST"}


def _cuobjdump():
    exe = shutil.which("cuobjdump") or os.path.join(os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")), "cuobjdump")
    return exe if os.path.exists(exe) else None


def test_wait_precedes_every_global_access_in_sass():
    """In every k_step_fwd / k_step_bwd instantiation the first ACQBULK (griddepcontrol.wait) comes before any global access:
    nothing that reads or writes global memory may run while the previous kernel is still running."""
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found")
    assert os.path.exists(LIB_PATH), f"{LIB_PATH} is not built"
    sass = subprocess.run([exe, "-sass", LIB_PATH], check=True, capture_output=True, text=True).stdout
    checked = []
    for fn in re.split(r"\n\s*Function : ", sass)[1:]:
        name = fn.split("\n", 1)[0].strip()
        if "k_step_fwd" not in name and "k_step_bwd" not in name:
            continue
        waited = False
        for m in re.finditer(r"/\*([0-9a-f]{4,})\*/\s+(?:@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9_]*)", fn):
            op = m.group(2)
            if op == "ACQBULK":
                waited = True
                break
            assert op not in GLOBAL_ACCESS, f"{name}: {op} at /*{m.group(1)}*/ before griddepcontrol.wait"
        assert waited, f"{name}: no griddepcontrol.wait"
        checked.append(name)
    # float / double x every lane count x shared / per-world inertia, forward and backward
    assert len(checked) >= 8 and any("k_step_fwd" in n for n in checked) and any("k_step_bwd" in n for n in checked), checked


@pytest.fixture(scope="module")
def atlas():
    import nimblephysics_b200 as nb

    raw = load_raw("atlas")
    world = nb.World.from_raw(raw)
    world._contacts_disabled = True
    dm = nb.device_model_for(world)
    yield raw, dm
    dm.set_lanes(0)


def _lane_counts(dm):
    lanes = sorted(int(c.lanes) for c in dm.schedules)
    assert lanes[0] == 1 and len(lanes) > 1
    return lanes


def _chain(ops, sync):
    import torch

    for op in ops:
        op()
        if sync:
            torch.cuda.synchronize()
    torch.cuda.synchronize()


def _same(a, b, what):
    import torch

    for k in a:
        assert torch.equal(a[k], b[k]), f"{what}: {k} differs between the chained and the synchronised launches"


def _each_schedule(dm, B, precision, run):
    """run(sync) -> dict of tensors, compared between sync=False and sync=True under every lane count the model offers"""
    for K in _lane_counts(dm):
        dm.set_lanes(K)
        assert dm.lanes_for(B, False, precision) == K and dm.lanes_for(B, True, precision) == K
        _same(run(False), run(True), f"{K} lanes")
    dm.set_lanes(0)


CASES = [(B, p) for B in (4096, 4093) for p in (0, 1)]  # B = 4093: a partial last group; precision 0 = fp32, 1 = fp64
IDS = [f"B{B}-{'fp64' if p else 'fp32'}" for B, p in CASES]


@pytest.mark.gpu
@pytest.mark.parametrize("B,precision", CASES, ids=IDS)
def test_rollout_forward_then_accumulating_backward(atlas, B, precision):
    """nb2_rollout_forward then nb2_rollout_backward, T = 16, queued back to back: each forward reads the previous forward's
    state, the first backward reads the last forward's saved stream, and each backward reads grad_states[t+1] from the previous
    backward and adds into grad_states[t].  The synchronised chain launches the same kernels one step per call."""
    import torch

    raw, dm = atlas
    n2, na, sw = 2 * raw.ndof, len(raw.action_map), dm.saved_words
    rtype = torch.float64 if precision else torch.float32
    gen = torch.Generator().manual_seed(7)
    s, _, _ = sample_inputs(raw, B, seed=41)
    acts = (torch.rand((T, B, na), generator=gen) * 40 - 20).cuda()
    acts[:, :, :6] = 0
    gin = torch.randn((T + 1, B, n2), generator=gen).cuda()
    stream = torch.cuda.current_stream().cuda_stream

    def run(sync):
        states = torch.zeros((T + 1, B, n2), device="cuda")
        states[0] = torch.from_numpy(s).cuda()
        saved = torch.zeros((T, sw, B), device="cuda", dtype=rtype)
        gs, ga = gin.clone(), torch.zeros((T, B, na), device="cuda")
        torch.cuda.synchronize()
        sp, ap, vp, gp, gap = states.data_ptr(), acts.data_ptr(), saved.data_ptr(), gs.data_ptr(), ga.data_ptr()
        if not sync:
            ops = [lambda: dm.rollout_forward_device(B, T, sp, ap, vp, stream, precision),
                   lambda: dm.rollout_backward_device(B, T, sp, ap, vp, gp, gap, stream, precision)]
        else:
            f4, e = 4, saved.element_size()
            ops = [lambda t=t: dm.rollout_forward_device(B, 1, sp + f4 * t * B * n2, ap + f4 * t * B * na, vp + e * t * sw * B, stream, precision)
                   for t in range(T)]
            ops += [lambda t=t: dm.rollout_backward_device(B, 1, sp + f4 * t * B * n2, ap + f4 * t * B * na, vp + e * t * sw * B,
                                                           gp + f4 * t * B * n2, gap + f4 * t * B * na, stream, precision)
                    for t in reversed(range(T))]
        _chain(ops, sync)
        return {"states": states, "saved": saved, "grad_states": gs, "grad_actions": ga}

    _each_schedule(dm, B, precision, run)


@pytest.mark.gpu
@pytest.mark.parametrize("B,precision", CASES, ids=IDS)
def test_torch_kernel_writes_the_backward_input(atlas, B, precision):
    """A torch elementwise kernel writes dL/dx' right before the backward; and a backward launched right after its forward
    reads a dL/dx' that a torch kernel wrote two launches earlier."""
    import torch

    raw, dm = atlas
    rtype = torch.float64 if precision else torch.float32
    s, a, g = (torch.from_numpy(x).cuda() for x in sample_inputs(raw, B, seed=42))
    stream = torch.cuda.current_stream().cuda_stream

    def run(sync):
        nxt, nxt2 = torch.zeros_like(s), torch.zeros_like(s)
        sv, sv2 = (torch.zeros((dm.saved_words, B), device="cuda", dtype=rtype) for _ in range(2))
        g1, g2 = torch.zeros_like(g), torch.zeros_like(g)
        gs, gs2 = torch.zeros_like(s), torch.zeros_like(s)
        ga, ga2 = torch.zeros_like(a), torch.zeros_like(a)
        torch.cuda.synchronize()
        ops = [lambda: dm.forward_device(B, s.data_ptr(), a.data_ptr(), nxt.data_ptr(), sv.data_ptr(), stream, precision),
               lambda: torch.mul(g, 1.5, out=g1),
               lambda: dm.backward_device(B, s.data_ptr(), a.data_ptr(), sv.data_ptr(), g1.data_ptr(), gs.data_ptr(), ga.data_ptr(), stream, precision),
               lambda: torch.mul(g, -0.5, out=g2),
               lambda: dm.forward_device(B, nxt.data_ptr(), a.data_ptr(), nxt2.data_ptr(), sv2.data_ptr(), stream, precision),
               lambda: dm.backward_device(B, nxt.data_ptr(), a.data_ptr(), sv2.data_ptr(), g2.data_ptr(), gs2.data_ptr(), ga2.data_ptr(), stream,
                                          precision)]
        _chain(ops, sync)
        return {"next": nxt, "next2": nxt2, "grad_state": gs, "grad_action": ga, "grad_state2": gs2, "grad_action2": ga2}

    _each_schedule(dm, B, precision, run)


@pytest.mark.gpu
@pytest.mark.parametrize("B,precision", CASES, ids=IDS)
def test_forward_overwrites_what_the_backward_reads(atlas, B, precision):
    """Write-after-read with ping-pong state buffers: fwd(A -> N), bwd(A, g), then fwd(N -> A) writes A and the saved stream
    while the backward before it may still be reading both."""
    import torch

    raw, dm = atlas
    rtype = torch.float64 if precision else torch.float32
    s, a, g = (torch.from_numpy(x).cuda() for x in sample_inputs(raw, B, seed=43))
    stream = torch.cuda.current_stream().cuda_stream

    def run(sync):
        A, N = s.clone(), torch.zeros_like(s)
        sv = torch.zeros((dm.saved_words, B), device="cuda", dtype=rtype)
        gs, ga = torch.zeros_like(s), torch.zeros_like(a)
        torch.cuda.synchronize()
        ops = [lambda: dm.forward_device(B, A.data_ptr(), a.data_ptr(), N.data_ptr(), sv.data_ptr(), stream, precision),
               lambda: dm.backward_device(B, A.data_ptr(), a.data_ptr(), sv.data_ptr(), g.data_ptr(), gs.data_ptr(), ga.data_ptr(), stream, precision),
               lambda: dm.forward_device(B, N.data_ptr(), a.data_ptr(), A.data_ptr(), sv.data_ptr(), stream, precision)]
        _chain(ops, sync)
        return {"grad_state": gs, "grad_action": ga, "A": A, "N": N, "saved": sv}

    _each_schedule(dm, B, precision, run)
