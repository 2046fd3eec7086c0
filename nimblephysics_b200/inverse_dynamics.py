"""``inverse_dynamics(world, state, next_vel, mass=None)`` — contact-free inverse dynamics, batched and differentiable.

It answers the reverse question of ``timestep``: which generalised force takes each world from ``state = [q; qdot]`` to the
velocity ``next_vel`` in one contact-free step?

    a = (next_vel - qdot) / dt ,   tau = M(q) a + C(q, qdot) + g(q) + K (q - q0 + qdot dt) + D qdot

tau is per dof (not gathered through the action map); free joints use the step's conventions.  Contacts, joint-limit rows and
force limits are ignored, and a world's LCP cache is never touched.  With an action space covering every dof,
``timestep(world, state, tau)`` returns ``next_vel`` up to rounding.  The nearest call of the reference is the contact-free
``Skeleton::getInverseDynamics(nextVel)`` for one skeleton.  Whether its spring term carries ``qdot * dt`` is unverified here;
this one uses the step's semi-implicit spring so that the round trip holds.

Precision follows the state's dtype: float64 tensors run the fp64 kernels with fp64 rows, anything else the fp32 ones.
Gradients flow to ``state``, ``next_vel`` and ``mass`` (1-D: ``setMasses``, shared by the batch, gradient summed; 2-D ``[B, m]``:
per world, the World is left untouched).  The work is done by libnb2.so (include/nb2.h ``nb2_inverse_dynamics``).
"""
from __future__ import annotations

from typing import Optional

import torch

from .engine import FP32, FP64, device_model_for
from .timestep import _inertia_grad, _word_major_inertia, per_world_inertia, set_shared_masses, shared_mass_jacobian

_WHO = "inverse_dynamics()"


class InverseDynamicsLayer(torch.autograd.Function):
    """world_inertia (optional): per-world canonical inertia [B, nb, 10] (modelspec.mass_to_inertia), exclusive with the 1-D `mass`."""

    @staticmethod
    def forward(ctx, world, state, next_vel, mass, world_inertia=None):
        if mass is not None and world_inertia is not None:
            raise ValueError(f"{_WHO}: give either a mass vector or a per-world inertia table, not both")
        dm = set_shared_masses(world, mass, _WHO) if mass is not None else device_model_for(world)
        n = dm.ndof
        single = state.dim() == 1
        s2 = state.detach().reshape(1, -1) if single else state.detach()
        v2 = next_vel.detach().reshape(1, -1) if single else next_vel.detach()
        if s2.dim() != 2 or s2.shape[1] != 2 * n:
            raise ValueError(f"{_WHO}: state has shape {tuple(state.shape)}, expected [..., {2 * n}] (= getStateSize())")
        if v2.dim() != 2 or tuple(v2.shape) != (s2.shape[0], n) or next_vel.dim() != state.dim():
            raise ValueError(f"{_WHO}: next_vel has shape {tuple(next_vel.shape)}, expected the state's batch shape with {n} (= getNumDofs()) entries")
        if not torch.cuda.is_available():
            raise RuntimeError("nimblephysics_b200.inverse_dynamics needs a CUDA device; there is no CPU fallback")
        dev = s2.device if s2.is_cuda else torch.device("cuda", torch.cuda.current_device())
        rdt = torch.float64 if state.dtype == torch.float64 else torch.float32
        prec = FP64 if rdt == torch.float64 else FP32
        sd = s2.to(device=dev, dtype=rdt).contiguous()
        vd = v2.to(device=dev, dtype=rdt).contiguous()
        B = sd.shape[0]
        if world_inertia is not None and (single or tuple(world_inertia.shape) != (B, dm.cm.nb, 10)):
            raise ValueError(f"{_WHO}: per-world inertia has shape {tuple(world_inertia.shape)}, expected [{B}, {dm.cm.nb}, 10] with a 2-D state")
        wi = _word_major_inertia(dm, world_inertia, B, dev)
        wi_ptr = wi.data_ptr() if wi is not None else None
        ctx.wi_grad = world_inertia is not None and ctx.needs_input_grad[4]
        ctx.wi_like = world_inertia
        ctx.mass_grad = mass is not None and ctx.needs_input_grad[3]
        if ctx.mass_grad:
            ctx.mass_P = shared_mass_jacobian(world, dm, dev)
            ctx.mass_like = mass
        need_grad = any(ctx.needs_input_grad[1:5])
        with torch.cuda.device(dev):
            tau = torch.empty((B, n), dtype=rdt, device=dev)
            saved = torch.empty((dm.saved_words, B), dtype=rdt, device=dev) if need_grad else None
            dm.inverse_dynamics_device(B, sd.data_ptr(), vd.data_ptr(), tau.data_ptr(), saved.data_ptr() if saved is not None else None,
                                       torch.cuda.current_stream().cuda_stream, prec, wi_ptr=wi_ptr)
        ctx.dm, ctx.B, ctx.prec, ctx.single = dm, B, prec, single
        ctx.in_meta = (state.device, state.dtype, next_vel.device, next_vel.dtype)
        if need_grad:
            ctx.save_for_backward(sd, saved, wi)
        out = tau[0] if single else tau
        return out.to(device=state.device, dtype=state.dtype)

    @staticmethod
    def backward(ctx, grad_tau):
        dm, B = ctx.dm, ctx.B
        sd, saved, wi = ctx.saved_tensors
        dev, n = sd.device, dm.ndof
        want_gi = ctx.mass_grad or ctx.wi_grad
        g = grad_tau.detach().reshape(B, n).to(device=dev, dtype=sd.dtype).contiguous()
        with torch.cuda.device(dev):
            gs = torch.empty_like(sd)
            gn = torch.empty((B, n), dtype=sd.dtype, device=dev)
            gi = torch.empty((10 * dm.cm.nb, B), dtype=torch.float64, device=dev) if want_gi else None
            dm.inverse_dynamics_backward_device(B, sd.data_ptr(), saved.data_ptr(), g.data_ptr(), gs.data_ptr(), gn.data_ptr(),
                                                torch.cuda.current_stream().cuda_stream, ctx.prec,
                                                ginertia_ptr=gi.data_ptr() if gi is not None else None,
                                                wi_ptr=wi.data_ptr() if wi is not None else None)
        gm = None
        if ctx.mass_grad:  # one mass vector shared by the batch: the worlds' gradients add up
            gm = (ctx.mass_P @ gi.sum(dim=1)).to(device=ctx.mass_like.device, dtype=ctx.mass_like.dtype)
        gw = _inertia_grad(gi, ctx.wi_like) if ctx.wi_grad else None
        sdev, sdt, vdev, vdt = ctx.in_meta
        if ctx.single:
            gs, gn = gs[0], gn[0]
        return None, gs.to(device=sdev, dtype=sdt), gn.to(device=vdev, dtype=vdt), gm, gw


def inverse_dynamics(world, state: torch.Tensor, next_vel: torch.Tensor, mass: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Generalised force [B, n] (or [n] for a 1-D state) that takes every world from `state` [B, 2n] to `next_vel` [B, n] in one
    contact-free step (see the module docstring).  mass: None, a 1-D vector [getMassDims()] (world.setMasses(mass) first, shared by the
    batch, the masses stay set, the gradient sums over the batch), or a 2-D tensor [B, getMassDims()]: world w uses mass[w],
    mass.grad[w] is its own, and the World is not modified."""
    if mass is not None and mass.dim() == 2:
        return InverseDynamicsLayer.apply(world, state, next_vel, None, per_world_inertia(world, state, mass, _WHO))
    return InverseDynamicsLayer.apply(world, state, next_vel, mass)
