"""``timestep(world, state, action, mass=None)`` — the reference's autograd boundary, batched.

reference: python/nimblephysics/timestep.py:13-69 (TimestepLayer).  Same call, same gradient outputs
(None, d/dstate, d/daction, d/dmass); what changes:
  * ``state`` / ``action`` may be 2-D ``[B, 2n]`` / ``[B, a]`` tensors: B independent worlds advance in one launch;
  * tensors stay on the GPU (fp32); nothing goes through numpy;
  * 1-D tensors keep the legacy single-world meaning, including the side effect that ``world`` is left at the
    post-step state (NeuralUtils.cpp:46 idempotent=False) and the fp64 return dtype (timestep.py:40);
  * ``mass`` may be 2-D ``[B, getMassDims()]``: every world steps with its own masses and the World is left alone.
The work is done by libnb2.so through the C ABI (include/nb2.h).  There is no CPU implementation.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from ._cabi import MAX_CONTACTS, MAX_ROWS
from .engine import FP32, FP64, device_model_for


def _ptr(t: torch.Tensor) -> int:
    return t.data_ptr()


def _word_major_inertia(dm, world_inertia, B, dev):
    """[B, nb, 10] per-world inertia -> the kernels' word-major [10*nb, B] fp64 layout on `dev`, so that the worlds of a warp read
    adjacent words (None stays None)."""
    if world_inertia is None:
        return None
    return world_inertia.detach().to(device=dev, dtype=torch.float64).reshape(B, 10 * dm.cm.nb).t().contiguous()


def _inertia_grad(gi, like):
    """The kernels' [10*nb, B] inertia gradient -> world w's own dL/d(inertia) in the [B, nb, 10] layout (dtype, device) of the
    per-world inertia input (None stays None)."""
    if gi is None:
        return None
    return gi.t().to(torch.float64).reshape(like.shape).to(device=like.device, dtype=like.dtype)


class TimestepLayer(torch.autograd.Function):
    """world_inertia (optional): per-world canonical inertia [B, nb, 10] (modelspec.mass_to_inertia); it replaces the model's table for
    world w only, and its gradient is the kernels' per-world dL/d(inertia).  Exclusive with the 1-D `mass` argument."""

    @staticmethod
    def forward(ctx, world, state, action, mass, world_inertia=None):
        dm = device_model_for(world)
        if mass is not None and world_inertia is not None:
            raise ValueError("TimestepLayer: give either a mass vector or a per-world inertia table, not both")
        if mass is not None:
            # reference: world.setMasses(mass) before the step (timestep.py:33-35); the masses stay set afterwards.
            # One mass vector per call: every world of the batch shares the model (the gradient sums over the batch).
            if mass.dim() != 1 or mass.numel() != world.getMassDims():
                raise ValueError(f"timestep(): mass has shape {tuple(mass.shape)}, expected [{world.getMassDims()}] (= getMassDims(); "
                                 "register parameters with world.tuneMass)")
            # (a device -> host copy, i.e. a sync: skipped when this very tensor, unchanged since the last call, is already what the world holds)
            from .world import edit_epoch

            mkey = (mass.data_ptr(), mass._version, tuple(mass.shape), str(mass.device), edit_epoch())
            if getattr(world, "_mass_key", None) != mkey:
                world.setMasses(mass.detach().cpu().numpy().astype(np.float64))
                dm = device_model_for(world)   # setMasses edited the model: the device model follows (inertia refresh)
                world._mass_key = mkey
                world._mass_P = None
        n2, na = 2 * dm.ndof, dm.na
        legacy = state.dim() == 1
        if legacy and (state.numel() != n2 or action.numel() != na):
            # reference: message on stderr and the call is ignored (World.cpp:2027-2033, :2063-2070); we raise
            raise ValueError(f"timestep(): got state of size {state.numel()} / action of size {action.numel()}, expected "
                             f"getStateSize()={n2} / getActionSize()={na}")
        s2 = state.detach().reshape(-1, n2) if legacy else state.detach()
        a2 = action.detach().reshape(-1, na) if legacy else action.detach()
        if s2.dim() != 2 or s2.shape[1] != n2:
            raise ValueError(f"timestep(): state has shape {tuple(state.shape)}, expected [..., {n2}] (= getStateSize())")
        if a2.dim() != 2 or a2.shape[1] != na or a2.shape[0] != s2.shape[0]:
            raise ValueError(f"timestep(): action has shape {tuple(action.shape)}, expected [{s2.shape[0]}, {na}] (= getActionSize())")
        if not torch.cuda.is_available():
            raise RuntimeError("nimblephysics_b200.timestep needs a CUDA device; there is no CPU fallback")
        dev = s2.device if s2.is_cuda else torch.device("cuda", torch.cuda.current_device())
        sd = s2.to(device=dev, dtype=torch.float32, non_blocking=True).contiguous()
        ad = a2.to(device=dev, dtype=torch.float32, non_blocking=True).contiguous()
        B = sd.shape[0]
        if world_inertia is not None and (legacy or tuple(world_inertia.shape) != (B, dm.cm.nb, 10)):
            raise ValueError(f"timestep(): per-world inertia has shape {tuple(world_inertia.shape)}, expected [{B}, {dm.cm.nb}, 10] "
                             "with a 2-D state")
        wi = _word_major_inertia(dm, world_inertia, B, dev)
        wi_ptr = _ptr(wi) if wi is not None else None
        ctx.wi_grad = world_inertia is not None and ctx.needs_input_grad[4]
        ctx.wi_like = world_inertia
        ctx.mass_grad = mass is not None and ctx.needs_input_grad[3]
        if ctx.mass_grad:
            if getattr(world, "_mass_P", None) is None or world._mass_P.device != dev:
                world._mass_P = torch.from_numpy(dm.inertia_param_jacobian(world)).to(dev)  # [mass_dims, 10*nb], fp64; cached with the mass key
            ctx.mass_P = world._mass_P
            ctx.mass_like = mass
        need_grad = any(ctx.needs_input_grad[1:5])
        ctx.contact = dm.has_contacts
        with torch.cuda.device(dev):
            nxt = torch.empty_like(sd)
            stream = torch.cuda.current_stream().cuda_stream
            if dm.has_contacts:
                # contact / boxed-LCP stage: fp64 kernels; the LCP cache (BoxedLcpConstraintSolver::mX in the reference)
                # lives on the world and flows from step to step like the reference's solver state
                cache = contact_cache(world, B, dev)
                # saved stream (world-major): the apply kernel of the three-kernel forward reads the tree data back from it, the
                # backward too; the ~1 KB/world record only when a backward will follow
                saved = torch.empty((B, dm.saved_words), dtype=torch.float64, device=dev)
                crec = torch.empty((B, dm.contact_record_bytes(B) // (8 * B)), dtype=torch.float64, device=dev) if need_grad else None
                dm.forward_contact_device(B, _ptr(sd), _ptr(ad), _ptr(nxt), _ptr(saved) if saved is not None else None, _ptr(cache["ws"]),
                                          _ptr(cache["x"]), _ptr(cache["m"]), _ptr(cache["labels"]), _ptr(cache["status"]), _ptr(cache["nc"]),
                                          _ptr(cache["cinfo"]), _ptr(crec) if crec is not None else None, _ptr(cache["sticky"]), stream,
                                          wi_ptr=wi_ptr)
                ctx.crec = crec
                ctx.ws = cache["ws"]
                ctx.sticky = cache["sticky"]
                if getattr(world, "_strict_contact_checks", False) or legacy:
                    check_contact_status(world)  # host sync: off by default for batches (call it once per rollout instead)
            else:
                saved = torch.empty((dm.saved_words, B), dtype=torch.float32, device=dev) if need_grad else None
                dm.forward_device(B, _ptr(sd), _ptr(ad), _ptr(nxt), _ptr(saved) if saved is not None else None, stream, FP32, wi_ptr=wi_ptr)
        ctx.dm = dm
        ctx.legacy = legacy
        ctx.in_device = state.device
        ctx.in_dtype = state.dtype
        ctx.act_device = action.device
        ctx.act_dtype = action.dtype
        ctx.B = B
        if need_grad:
            ctx.save_for_backward(sd, ad, saved, wi)
        if legacy:
            out = nxt[0].to(dtype=torch.float64).cpu() if not state.is_cuda else nxt[0].to(torch.float64)
            world._state = out.detach().cpu().numpy().astype(np.float64)
            return out
        return nxt.to(device=state.device, dtype=state.dtype)

    @staticmethod
    def backward(ctx, grad_state):
        dm = ctx.dm
        sd, ad, saved, wi = ctx.saved_tensors
        wi_ptr = _ptr(wi) if wi is not None else None
        want_gi = ctx.mass_grad or ctx.wi_grad
        dev = sd.device
        g = grad_state.detach().reshape(ctx.B, 2 * dm.ndof).to(device=dev, dtype=torch.float32).contiguous()
        with torch.cuda.device(dev):
            gs = torch.empty_like(sd)
            ga = torch.empty_like(ad)
            stream = torch.cuda.current_stream().cuda_stream
            if ctx.contact:
                # adjoint of the contact stage with the classification frozen at the forward solution (csrc/nb2_cw.cuh contact_backward)
                gi = torch.empty((10 * dm.cm.nb, ctx.B), dtype=torch.float32, device=dev) if want_gi else None
                # worlds that cannot be back-propagated get NaN gradients and bit 2048 in the world's sticky status word: no host
                # sync here — check_contact_status(world) reports them (rollout() / sharded_trajectory_loss() call it once)
                dm.backward_contact_device(ctx.B, _ptr(sd), _ptr(ad), _ptr(saved), _ptr(ctx.crec), _ptr(ctx.ws), _ptr(g), _ptr(gs),
                                           _ptr(ga), stream, _ptr(gi) if gi is not None else None, _ptr(ctx.sticky), wi_ptr=wi_ptr)
                if ctx.legacy:
                    _raise_on_status(int(ctx.sticky[0].item()), [0], backward=True)
            else:
                gi = torch.empty((10 * dm.cm.nb, ctx.B), dtype=torch.float32, device=dev) if want_gi else None
                dm.backward_device(ctx.B, _ptr(sd), _ptr(ad), _ptr(saved), _ptr(g), _ptr(gs), _ptr(ga), stream, FP32,
                                   _ptr(gi) if gi is not None else None, wi_ptr=wi_ptr)
        gm = None
        if ctx.mass_grad:
            # lossWrtMass = massVel^T g_v' (BackpropSnapshot.cpp:177-178), summed over the worlds that share the model
            gm = (ctx.mass_P @ gi.to(torch.float64).sum(dim=1)).to(device=ctx.mass_like.device, dtype=ctx.mass_like.dtype)
        gw = _inertia_grad(gi, ctx.wi_like) if ctx.wi_grad else None
        if ctx.legacy:
            # reference returns fp64 grads (timestep.py:55-60)
            gs = gs[0].to(device=ctx.in_device, dtype=torch.float64 if ctx.in_dtype == torch.float64 else ctx.in_dtype)
            ga = ga[0].to(device=ctx.act_device, dtype=ctx.act_dtype)
            return None, gs, ga, gm, gw
        return None, gs.to(device=ctx.in_device, dtype=ctx.in_dtype), ga.to(device=ctx.act_device, dtype=ctx.act_dtype), gm, gw


def contact_cache(world, B: int, device) -> dict:
    """Per-world, per-batch-size device buffers of the contact stage: the cached LCP solution x/m (the reference's
    BoxedLcpConstraintSolver::mX, warm start of the next step), and this step's labels / status / contact list."""
    device = torch.device(device)
    if device.type == "cuda" and device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())  # "cuda" and "cuda:0" are the same cache
    key = (B, str(device), world._version)
    c = getattr(world, "_lcp_cache", None)
    if c is None or c.get("key") != key:
        dm = device_model_for(world)
        c = dict(key=key,
                 x=torch.zeros((B, MAX_ROWS), dtype=torch.float64, device=device),
                 m=torch.full((B,), -1, dtype=torch.int32, device=device),
                 labels=torch.zeros((B, MAX_ROWS), dtype=torch.int32, device=device),
                 status=torch.zeros((B,), dtype=torch.int32, device=device),
                 sticky=torch.zeros((B,), dtype=torch.int32, device=device),  # OR of every step's problem bits since the last check
                 nc=torch.zeros((B,), dtype=torch.int32, device=device),
                 cinfo=torch.zeros((B, MAX_CONTACTS, 10), dtype=torch.float32, device=device),
                 ws=torch.empty((dm.contact_workspace_bytes(B) // 8,), dtype=torch.float64, device=device))
        world._lcp_cache = c
    return c


ST_NAN, ST_UNSUPPORTED, ST_OVERFLOW, ST_BOUNCE, ST_BWD_ERROR = 32, 128, 256, 1024, 2048


def _raise_on_status(bits: int, worlds, backward=False):
    if bits & ST_BWD_ERROR:
        raise RuntimeError(
            f"backward through the contact stage failed for worlds {list(worlds)[:16]} (their gradients are NaN): the contact rows "
            "regenerated in the backward pass did not match the forward's")
    if bits & ST_OVERFLOW:
        raise RuntimeError(f"contact stage: worlds {list(worlds)[:16]} generated more than {MAX_CONTACTS} contacts / {MAX_ROWS} LCP rows "
                           "(or the overflow pool was exhausted): the extra contacts were DROPPED — the step differs from the reference")
    if bits & ST_UNSUPPORTED:
        raise RuntimeError(f"contact stage: worlds {list(worlds)[:16]} hit a contact configuration without a generator (a capsule lying flat "
                           "on a box: the reference asks libccd's MPR): those contacts were NOT generated")


def check_contact_status(world, reset: bool = True) -> int:
    """Read the world's sticky contact-stage status (ONE host sync) and raise if any world dropped contacts, met an unsupported
    geometry or could not be back-propagated since the last check; otherwise return the OR of all status words.
    timestep() itself never synchronises on batches: call this once per rollout / optimiser step."""
    c = getattr(world, "_lcp_cache", None)
    if c is None:
        return 0
    st = c["sticky"].cpu().numpy()
    if reset:
        c["sticky"].zero_()
    bits = int(np.bitwise_or.reduce(st)) if st.size else 0
    bad = np.nonzero(st & (ST_BWD_ERROR | ST_OVERFLOW | ST_UNSUPPORTED))[0]
    if bad.size:
        _raise_on_status(int(np.bitwise_or.reduce(st[bad])), bad.tolist())
    return bits


def reset_contact_cache(world):
    """Forget the cached LCP solutions (the next step starts from LCPUtils::guessSolution like a fresh solver)."""
    world._lcp_cache = None


def per_world_inertia(world, state: torch.Tensor, mass: torch.Tensor) -> torch.Tensor:
    """Checks a 2-D mass argument against a batch of states and maps it to the per-world inertia table the kernels read."""
    from .modelspec import mass_to_inertia

    if state.dim() != 2:
        raise ValueError(f"timestep(): a per-world mass [B, getMassDims()] needs a batched state [B, 2n], got state of shape {tuple(state.shape)}")
    if mass.shape[0] != state.shape[0]:
        raise ValueError(f"timestep(): mass has {mass.shape[0]} rows for a batch of {state.shape[0]} worlds")
    return mass_to_inertia(world, mass)


def timestep(world, state: torch.Tensor, action: torch.Tensor, mass: Optional[torch.Tensor] = None) -> torch.Tensor:
    """One differentiable step of every world in the batch (forward stores what backward needs).

    mass: None, a 1-D vector [getMassDims()] (the reference's meaning: world.setMasses(mass) first, shared by every world, the masses stay
    set, the gradient sums over the batch), or a 2-D tensor [B, getMassDims()]: world w steps with mass[w], mass.grad[w] is world w's
    lossWrtMass, and the World is NOT modified (no setMasses, no host sync).  Per-world masses are not checked on the device: a world
    with a non-positive mass gets non-finite outputs, and no other world is affected."""
    if mass is not None and mass.dim() == 2:
        return TimestepLayer.apply(world, state, action, None, per_world_inertia(world, state, mass))
    return TimestepLayer.apply(world, state, action, mass)
