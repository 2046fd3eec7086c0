"""T-step rollouts with backprop through the horizon, and batch sharding across the GPUs of one box.

reference: dart/trajectory/SingleShot.cpp:635-686 (getSnapshots: unroll T forward passes) and :539-631
(backpropGradientWrt: reverse sweep carrying dL/dq, dL/dqdot and adding per-step loss gradients);
MultiShot runs shots on std::async threads with one cloned World each (MultiShot.cpp:57-72, 1245-1275).
Here a "shot" is simply a slice of the batch: worlds are independent, so the batch shards across ranks with NO
data-path collective; the only collective is the all-reduce of the scalar loss / of gradients of parameters shared by
all worlds (torch.distributed, NCCL over NVLink), outside the timestep.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence, Tuple

import torch

from .timestep import TimestepLayer, per_world_inertia, timestep


def rollout(world, state0: torch.Tensor, actions: Sequence[torch.Tensor], keep_states: bool = False, mass: Optional[torch.Tensor] = None):
    """Unroll len(actions) differentiable steps.  state0: [B, 2n]; actions[t]: [B, a]; mass: as for timestep() (a 2-D [B, m] mass is
    mapped to the per-world inertia once and held constant over the horizon).
    Returns the final state (and the list of intermediate states when keep_states)."""
    x = state0
    states: List[torch.Tensor] = []
    wi = per_world_inertia(world, state0, mass) if mass is not None and mass.dim() == 2 else None
    for a in actions:
        x = TimestepLayer.apply(world, x, a, None, wi) if wi is not None else timestep(world, x, a, mass)
        if keep_states:
            states.append(x)
    return (x, states) if keep_states else x


class _FusedRollout(torch.autograd.Function):
    """Whole-horizon rollout behind ONE C-ABI call per direction (include/nb2.h nb2_rollout_forward / _backward): the 2T
    kernels are queued back to back on the stream, the trajectory and the saved streams never leave the device, and
    autograd sees a single node instead of T."""

    @staticmethod
    def forward(ctx, world, state0, actions, world_inertia=None):
        from .engine import FP32, device_model_for

        dm = device_model_for(world)
        T, B = actions.shape[0], actions.shape[1]
        n2, na = 2 * dm.ndof, dm.na
        if state0.shape != (B, n2) or actions.shape[2] != na:
            raise ValueError(f"rollout(): state0 {tuple(state0.shape)} / actions {tuple(actions.shape)} do not match [B,{n2}] / [T,B,{na}]")
        dev = state0.device
        states = torch.empty((T + 1, B, n2), dtype=torch.float32, device=dev)
        states[0].copy_(state0.detach())
        acts = actions.detach().to(dtype=torch.float32).contiguous()
        wi = _word_major_inertia(dm, world_inertia, B, dev)
        need = any(ctx.needs_input_grad[1:4])
        saved = torch.empty((T, dm.saved_words, B), dtype=torch.float32, device=dev) if need else None
        with torch.cuda.device(dev):
            dm.rollout_forward_device(B, T, states.data_ptr(), acts.data_ptr(), saved.data_ptr() if need else None,
                                      torch.cuda.current_stream().cuda_stream, FP32, wi_ptr=wi.data_ptr() if wi is not None else None)
        ctx.dm, ctx.T, ctx.B = dm, T, B
        ctx.dtypes = (state0.dtype, actions.dtype)
        ctx.wi_like = world_inertia
        if need:
            ctx.save_for_backward(states, acts, saved, wi)
        return states.to(state0.dtype)

    @staticmethod
    def backward(ctx, grad_states):
        from .engine import FP32

        states, acts, saved, wi = ctx.saved_tensors
        dm, T, B = ctx.dm, ctx.T, ctx.B
        gs = grad_states.detach().to(dtype=torch.float32).contiguous().clone()  # in: loss gradient per state; out: total dL/dx_t
        ga = torch.empty_like(acts)
        gi = torch.zeros((10 * dm.cm.nb, B), dtype=torch.float64, device=states.device) if ctx.needs_input_grad[3] else None
        with torch.cuda.device(states.device):
            dm.rollout_backward_device(B, T, states.data_ptr(), acts.data_ptr(), saved.data_ptr(), gs.data_ptr(), ga.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream, FP32, wi_ptr=wi.data_ptr() if wi is not None else None,
                                       ginertia_ptr=gi.data_ptr() if gi is not None else None)
        return None, gs[0].to(ctx.dtypes[0]), ga.to(ctx.dtypes[1]), _inertia_grad(gi, ctx.wi_like)


class _ContactRollout(torch.autograd.Function):
    """Whole-horizon rollout of a world with collision pairs behind ONE C-ABI call per direction (nb2_rollout_forward_contact /
    nb2_rollout_backward_contact): every kernel of the horizon is queued from C, the solver's LCP cache flows on the device, the tape
    (saved streams + contact records) is one device buffer, optionally checkpointed every k steps."""

    @staticmethod
    def forward(ctx, world, state0, actions, checkpoint_every, world_inertia=None):
        from .engine import device_model_for
        from .timestep import contact_cache

        dm = device_model_for(world)
        T, B = actions.shape[0], actions.shape[1]
        n2, na = 2 * dm.ndof, dm.na
        if state0.shape != (B, n2) or actions.shape[2] != na:
            raise ValueError(f"rollout(): state0 {tuple(state0.shape)} / actions {tuple(actions.shape)} do not match [B,{n2}] / [T,B,{na}]")
        if not state0.is_cuda:
            raise RuntimeError("rollout_fused needs CUDA tensors; there is no CPU fallback")
        dev = state0.device
        states = torch.empty((T + 1, B, n2), dtype=torch.float32, device=dev)
        states[0].copy_(state0.detach())
        acts = actions.detach().to(dtype=torch.float32).contiguous()
        k = int(checkpoint_every or 0)
        cache = contact_cache(world, B, dev)
        tape = torch.empty((dm.rollout_contact_tape_bytes(B, T, k) // 8,), dtype=torch.float64, device=dev)
        wi = _word_major_inertia(dm, world_inertia, B, dev)
        with torch.cuda.device(dev):
            dm.rollout_forward_contact_device(B, T, states.data_ptr(), acts.data_ptr(), cache["x"].data_ptr(), cache["m"].data_ptr(), tape.data_ptr(), k,
                                              cache["ws"].data_ptr(), cache["sticky"].data_ptr(), torch.cuda.current_stream().cuda_stream,
                                              wi_ptr=wi.data_ptr() if wi is not None else None)
        ctx.dm, ctx.T, ctx.B, ctx.k, ctx.cache = dm, T, B, k, cache
        ctx.dtypes = (state0.dtype, actions.dtype)
        ctx.peak_tape_bytes = tape.numel() * 8
        ctx.wi_like = world_inertia
        if any(ctx.needs_input_grad[1:3]) or ctx.needs_input_grad[4]:
            ctx.save_for_backward(states, acts, tape, wi)
        return states.to(state0.dtype)

    @staticmethod
    def backward(ctx, grad_states):
        states, acts, tape, wi = ctx.saved_tensors
        dm, T, B, cache = ctx.dm, ctx.T, ctx.B, ctx.cache
        gs = grad_states.detach().to(dtype=torch.float32).contiguous().clone()  # in: loss gradient per state; out: total dL/dx_t
        ga = torch.empty_like(acts)
        gi = torch.zeros((10 * dm.cm.nb, B), dtype=torch.float64, device=states.device) if ctx.needs_input_grad[4] else None
        with torch.cuda.device(states.device):
            dm.rollout_backward_contact_device(B, T, states.data_ptr(), acts.data_ptr(), cache["x"].data_ptr(), cache["m"].data_ptr(), tape.data_ptr(),
                                               ctx.k, gs.data_ptr(), ga.data_ptr(), cache["ws"].data_ptr(), cache["sticky"].data_ptr(),
                                               torch.cuda.current_stream().cuda_stream, wi_ptr=wi.data_ptr() if wi is not None else None,
                                               ginertia_ptr=gi.data_ptr() if gi is not None else None)
        return None, gs[0].to(ctx.dtypes[0]), ga.to(ctx.dtypes[1]), None, _inertia_grad(gi, ctx.wi_like)


def _word_major_inertia(dm, world_inertia, B, dev):
    """[B, nb, 10] per-world inertia -> the kernels' word-major [10*nb, B] fp64 layout on `dev` (None stays None)."""
    if world_inertia is None:
        return None
    return world_inertia.detach().to(device=dev, dtype=torch.float64).reshape(B, 10 * dm.cm.nb).t().contiguous()


def _inertia_grad(gi, like):
    """[10*nb, B] gradient summed over the horizon -> the [B, nb, 10] layout (dtype, device) of the per-world inertia input."""
    if gi is None:
        return None
    return gi.t().reshape(like.shape).to(device=like.device, dtype=like.dtype)


def rollout_fused(world, state0: torch.Tensor, actions: torch.Tensor, checkpoint_every: int = 0, mass: Optional[torch.Tensor] = None) -> torch.Tensor:
    """states[T+1, B, 2n] of the T-step rollout x_{t+1} = timestep(x_t, actions[t])
    (SingleShot::getSnapshots, dart/trajectory/SingleShot.cpp:635-686), differentiable with respect to state0 and every
    action (SingleShot::backpropGradientWrt, :539-631); losses may look at any state of the trajectory.  One C call per direction.
    Worlds with collision pairs run the contact / boxed-LCP stage every step with the world's LCP cache flowing exactly as when
    chaining timestep() (bit-identical states and gradients); `checkpoint_every=k` keeps the backward tape of k steps instead of T and
    re-runs each segment's forward in the reverse sweep.  Problems (dropped contacts, worlds that cannot be back-propagated) are
    reported by check_contact_status(world), one host sync per rollout.
    mass (optional) [B, getMassDims()]: world w rolls out with masses mass[w], constant over the horizon; mass.grad sums over the steps
    (bit-identical to rollout(..., mass=)); the World is not modified."""
    from .engine import device_model_for

    wi = None
    if mass is not None:
        if mass.dim() != 2:
            raise ValueError(f"rollout_fused(): mass must be [B, getMassDims()], got shape {tuple(mass.shape)}")
        wi = per_world_inertia(world, state0, mass)
    if device_model_for(world).has_contacts:
        return _ContactRollout.apply(world, state0, actions, checkpoint_every, wi)
    return _FusedRollout.apply(world, state0, actions, wi)


def rollout_tape_bytes(world, B: int, T: int, checkpoint_every: int = 0) -> int:
    """Device bytes the backward tape of rollout_fused(world, ...) takes for a world with collision pairs."""
    from .engine import device_model_for

    return device_model_for(world).rollout_contact_tape_bytes(B, T, int(checkpoint_every or 0))


def multishot_rollout(world, start_states: torch.Tensor, actions: torch.Tensor, shot_length: int, rollout_fn: Optional[Callable] = None):
    """MultiShot as a batch: the S = ceil(T / shot_length) shots of a T-step problem run as S*B independent worlds of ONE rollout
    (the reference gives each shot a cloned World and a std::async thread, dart/trajectory/MultiShot.cpp:24-72, 1228-1334).
      start_states [S, B, 2n]: the start state of every shot (knot points; start_states[0] is the trajectory's x_0);
      actions      [T, B, a].
    Returns (states [T, B, 2n], defects [S-1, B, 2n]):
      states[t]  = the state after step t (MultiShot::getStates concatenates the shots' snapshots, MultiShot.cpp:902-975);
      defects[i] = final state of shot i - start state of shot i+1, the knot-point constraints of MultiShot::computeConstraints
                   (MultiShot.cpp:164-213).
    Differentiable with respect to start_states and actions; a last shot shorter than shot_length is padded with zero actions whose
    steps are discarded (they receive no gradient)."""
    S, B, n2 = start_states.shape
    T, na = actions.shape[0], actions.shape[2]
    L = int(shot_length)
    if L <= 0 or S != (T + L - 1) // L or actions.shape[1] != B:
        raise ValueError(f"multishot_rollout(): {T} steps in shots of {L} need start_states [{(T + L - 1) // max(L, 1)}, {actions.shape[1]}, 2n], got {tuple(start_states.shape)}")
    pad = S * L - T
    acts = torch.cat([actions, actions.new_zeros((pad, B, na))], 0) if pad else actions
    acts = acts.reshape(S, L, B, na).permute(1, 0, 2, 3).reshape(L, S * B, na)
    traj = (rollout_fn or rollout_fused)(world, start_states.reshape(S * B, n2), acts)  # [L+1, S*B, 2n]
    traj = traj.reshape(L + 1, S, B, n2)
    states = traj[1:].permute(1, 0, 2, 3).reshape(S * L, B, n2)[:T]
    defects = traj[L, : S - 1] - start_states[1:]
    return states, defects


def shard_range(total: int, rank: int, world_size: int) -> Tuple[int, int]:
    """Contiguous slice [lo, hi) of a batch of `total` worlds owned by `rank` (sizes differ by at most one)."""
    if world_size <= 0 or not (0 <= rank < world_size):
        raise ValueError("bad rank / world_size")
    base, rem = divmod(total, world_size)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_batch(t: torch.Tensor, rank: int, world_size: int) -> torch.Tensor:
    lo, hi = shard_range(t.shape[0], rank, world_size)
    return t[lo:hi]


def allreduce_sum_(t: torch.Tensor, group=None) -> torch.Tensor:
    """In-place SUM all-reduce when torch.distributed is initialised (no-op otherwise)."""
    import torch.distributed as dist

    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
    return t


def sharded_trajectory_loss(world, state0: torch.Tensor, actions: Sequence[torch.Tensor],
                            loss_fn: Callable[[torch.Tensor], torch.Tensor], rank: int, world_size: int,
                            step_fn: Optional[Callable] = None, checkpoint_every: int = 0):
    """Each rank rolls out its slice of the batch, backpropagates its part of the loss, and the scalar loss is
    all-reduced (config 5 of BASELINE.json).  Returns (global_loss, local_state0_grad, local_action_grads).
    Without `step_fn` the horizon runs through rollout_fused (one C call per direction); with one, step by step."""
    lo, hi = shard_range(state0.shape[0], rank, world_size)
    x0 = state0[lo:hi].detach().clone().requires_grad_(True)
    if step_fn is None:
        acts = torch.stack([a[lo:hi].detach() for a in actions], 0).requires_grad_(True)
        states = rollout_fused(world, x0, acts, checkpoint_every)
        loss = loss_fn(states[-1])
        loss.backward()
        grads = list(acts.grad.unbind(0))
    else:
        alist = [a[lo:hi].detach().clone().requires_grad_(True) for a in actions]
        x = x0
        for a in alist:
            x = step_fn(world, x, a)
        loss = loss_fn(x)
        loss.backward()
        grads = [a.grad for a in alist]
    total = allreduce_sum_(loss.detach().clone())
    if step_fn is None or step_fn is timestep:
        from .timestep import check_contact_status

        check_contact_status(world)  # ONE host sync per rollout: worlds that dropped contacts / could not be back-propagated raise here
    return total, x0.grad, grads
