"""Jacobian blocks of one step, state_{t+1} with respect to (state_t, action_t).

reference: BackpropSnapshot::getStateJacobian / getActionJacobian (dart/neural/BackpropSnapshot.cpp:1230-1260), the [2n, 2n] and
[2n, a] matrices the reference assembles from its pos-pos / pos-vel / vel-pos / vel-vel / force-vel blocks; World::getStateJacobian /
getActionJacobian (dart/simulation/World.cpp) return the same thing for the world's current state.

Here no block is ever formed inside the step: the backward kernels are vector-Jacobian products.  The getters seed that VJP with the rows
of an identity: world w of the batch is replicated 2n times, replica i back-propagates e_i, and its gradient IS row i of the Jacobian.  One
forward launch and one backward launch for the whole batch, on the GPU; the result is exactly what backprop through timestep() applies
(including the frozen contact classification and the bound clipping of BackpropSnapshot.cpp:425-479 at states sitting ON a limit).
"""
from __future__ import annotations

from typing import Tuple

import torch

from .engine import device_model_for
from .timestep import contact_cache, timestep


def step_jacobians(world, state: torch.Tensor, action: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """state [B, 2n], action [B, a] (CUDA) -> (next_state [B, 2n], d next/d state [B, 2n, 2n], d next/d action [B, 2n, a]).
    Does not disturb the world's LCP cache (contact worlds warm-start from a copy of it when the batch sizes agree)."""
    dm = device_model_for(world)
    n2, na = 2 * dm.ndof, dm.na
    if state.dim() != 2 or state.shape[1] != n2 or action.shape != (state.shape[0], na):
        raise ValueError(f"step_jacobians(): state {tuple(state.shape)} / action {tuple(action.shape)} do not match [B,{n2}] / [B,{na}]")
    if not state.is_cuda:
        raise RuntimeError("step_jacobians needs CUDA tensors; there is no CPU fallback")
    B = state.shape[0]
    s = state.detach().to(torch.float32).repeat_interleave(n2, dim=0).requires_grad_(True)
    a = action.detach().to(device=state.device, dtype=torch.float32).repeat_interleave(n2, dim=0).requires_grad_(True)
    seed = torch.eye(n2, device=state.device, dtype=torch.float32).repeat(B, 1)
    keep = getattr(world, "_lcp_cache", None)
    try:
        if dm.has_contacts:
            world._lcp_cache = None
            tmp = contact_cache(world, B * n2, state.device)
            if keep is not None and keep["x"].shape[0] == B and keep["x"].device == state.device:
                tmp["x"].copy_(keep["x"].repeat_interleave(n2, dim=0))
                tmp["m"].copy_(keep["m"].repeat_interleave(n2, dim=0))
        nxt = timestep(world, s, a)
        nxt.backward(seed)
    finally:
        world._lcp_cache = keep
    Js = s.grad.reshape(B, n2, n2)
    Ja = a.grad.reshape(B, n2, na)
    return nxt.detach().reshape(B, n2, n2)[:, 0, :], Js, Ja


def state_jacobian(world, state: torch.Tensor, action: torch.Tensor) -> torch.Tensor:
    return step_jacobians(world, state, action)[1]


def action_jacobian(world, state: torch.Tensor, action: torch.Tensor) -> torch.Tensor:
    return step_jacobians(world, state, action)[2]
