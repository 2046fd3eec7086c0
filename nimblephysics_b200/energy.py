"""``energy_and_momentum(world, state, skeleton, mass=None)``: the kinetic and potential energy and the centroidal momentum of a skeleton,
batched and differentiable (DESIGN.md §6m).

At states [q ; qdot] in the step's velocity coordinates (free joints: body twist), over the skeleton's bodies i and dofs d:

- kinetic energy T = 1/2 sum_i V_i . G_i V_i (V_i the body's spatial velocity, G_i its spatial inertia) = 1/2 qdot^T M qdot;
- potential energy U = -g . sum_i (m_i p_i + R_i h_i) + 1/2 sum_d k_d (q_d - q0_d)^2: gravity at each body's centre of mass and the
  joint springs (``spring``, ``rest``);
- momentum h [6] = [angular momentum about the skeleton's COM ; linear momentum], in world axes.  h is linear in qdot, so dh/dqdot is
  the centroidal momentum matrix; its linear rows are m_tot J_com.

The skeleton's root must move (as for ``com_jacobian``).  Contacts, limits and the contact cache play no part; the dofs of other
skeletons get exactly zero gradient.  Precision follows the state's dtype; gradients of all three outputs reach both halves of the state
and ``mass`` (1-D: ``setMasses``, shared by the batch, gradient summed; 2-D ``[B, m]``: per world, the World is left untouched).  The work
is done by libnb2.so (include/nb2.h ``nb2_energy_momentum`` and its backward).
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from .engine import FP32, FP64, device_model_for
from .mass_matrix import _ptr
from .timestep import _inertia_grad, _word_major_inertia, per_world_inertia, set_shared_masses, shared_mass_jacobian
from .world_jacobian import _check_skeleton, _check_state, _device, com_root

_WHO = "energy_and_momentum()"


class EnergyMomentumLayer(torch.autograd.Function):
    """(T, U, h) of the tree rooted at canonical body `root` at states [q ; qdot]; mass as ComJacobianLayer, world_inertia an optional
    per-world inertia table [B, nb, 10] (the model's is used where it is None)."""

    @staticmethod
    def forward(ctx, world, state, root, mass, world_inertia=None):
        dm = set_shared_masses(world, mass, _WHO) if mass is not None else device_model_for(world)
        single = state.dim() == 1
        s2 = state.detach().reshape(1, -1) if single else state.detach()
        dev = _device(s2, _WHO)
        rdt = torch.float64 if state.dtype == torch.float64 else torch.float32
        sd = s2.to(device=dev, dtype=rdt).contiguous()
        B = sd.shape[0]
        if world_inertia is not None and tuple(world_inertia.shape) != (B, dm.cm.nb, 10):
            raise ValueError(f"{_WHO}: world_inertia has shape {tuple(world_inertia.shape)}, expected [{B}, {dm.cm.nb}, 10]")
        wi = _word_major_inertia(dm, world_inertia, B, dev)
        prec = FP64 if rdt == torch.float64 else FP32
        with torch.cuda.device(dev):
            T = torch.empty(B, dtype=rdt, device=dev)
            U = torch.empty(B, dtype=rdt, device=dev)
            h = torch.empty((B, 6), dtype=rdt, device=dev)
            dm.energy_momentum_device(B, sd.data_ptr(), root, T.data_ptr(), U.data_ptr(), h.data_ptr(), torch.cuda.current_stream().cuda_stream,
                                      prec, wi_ptr=_ptr(wi))
        ctx.save_for_backward(sd, wi)
        ctx.dm, ctx.root, ctx.prec, ctx.single = dm, root, prec, single
        ctx.wi_grad = world_inertia is not None and ctx.needs_input_grad[4]
        ctx.wi_like = world_inertia
        ctx.mass_grad = mass is not None and ctx.needs_input_grad[3]
        if ctx.mass_grad:
            ctx.mass_P = shared_mass_jacobian(world, dm, dev)
            ctx.mass_like = mass
        ctx.in_meta = (state.device, state.dtype)
        if single:
            T, U, h = T[0], U[0], h[0]
        return tuple(x.to(device=state.device, dtype=state.dtype) for x in (T, U, h))

    @staticmethod
    def backward(ctx, gT, gU, gh):
        sd, wi = ctx.saved_tensors
        dm, dev = ctx.dm, sd.device
        B, n = sd.shape[0], dm.ndof
        g = lambda x, shape: (torch.zeros(shape, dtype=sd.dtype, device=dev) if x is None
                              else x.detach().reshape(shape).to(device=dev, dtype=sd.dtype).contiguous())
        gT, gU, gh = g(gT, (B,)), g(gU, (B,)), g(gh, (B, 6))
        with torch.cuda.device(dev):
            gs = torch.empty((B, 2 * n), dtype=sd.dtype, device=dev)
            gi = torch.empty((10 * dm.cm.nb, B), dtype=torch.float64, device=dev) if (ctx.mass_grad or ctx.wi_grad) else None
            dm.energy_momentum_backward_device(B, sd.data_ptr(), ctx.root, gT.data_ptr(), gU.data_ptr(), gh.data_ptr(), gs.data_ptr(),
                                               torch.cuda.current_stream().cuda_stream, ctx.prec, ginertia_ptr=_ptr(gi), wi_ptr=_ptr(wi))
        gm = None
        if ctx.mass_grad:  # one mass vector shared by the batch: the worlds' gradients add up
            gm = (ctx.mass_P @ gi.sum(dim=1)).to(device=ctx.mass_like.device, dtype=ctx.mass_like.dtype)
        gw = _inertia_grad(gi, ctx.wi_like) if ctx.wi_grad else None
        dev0, dt0 = ctx.in_meta
        gs = (gs[0] if ctx.single else gs).to(device=dev0, dtype=dt0)
        return None, gs, None, gm, gw


def energy_and_momentum(world, state: torch.Tensor, skeleton, mass: Optional[torch.Tensor] = None):
    """(kinetic [B], potential [B], momentum [B, 6]) of `skeleton` at states [B, 2n] = [q ; qdot] ([], [] and [6] for [2n]); see the module
    docstring.  mass as for com_jacobian.  ValueError before any device work for a wrong shape, a skeleton of another world, a skeleton
    whose root is fixed to the world, a world without dofs or a mass of the wrong size."""
    _check_state(world, state, _WHO)
    _check_skeleton(world, skeleton, _WHO)
    m = world.getMassDims()
    if mass is not None:
        if mass.dim() == 2 and state.dim() != 2:
            raise ValueError(f"{_WHO}: a [B, getMassDims()] mass needs [B, 2n] states")
        want = (m,) if mass.dim() == 1 else (state.shape[0], m)
        if mass.dim() not in (1, 2) or tuple(mass.shape) != want:
            raise ValueError(f"{_WHO}: mass has shape {tuple(mass.shape)}, expected [{m}] or [B, {m}] (= getMassDims())")
    root = com_root(world, skeleton, _WHO)
    if mass is not None and mass.dim() == 2:
        return EnergyMomentumLayer.apply(world, state, root, None, per_world_inertia(world, state, mass, _WHO))
    return EnergyMomentumLayer.apply(world, state, root, mass)


def _single_world_energy(world, skeleton, who):
    """(T, U) as Python floats at the world's current state (fp64 kernels, B = 1)."""
    s = torch.tensor(np.concatenate([world.getPositions(), world.getVelocities()]).astype(np.float64), dtype=torch.float64)
    _check_state(world, s, who)
    _check_skeleton(world, skeleton, who)
    if not torch.cuda.is_available():
        raise RuntimeError(f"nimblephysics_b200.{who} needs a CUDA device; there is no CPU fallback")
    with torch.no_grad():
        T, U, _ = energy_and_momentum(world, s.to("cuda"), skeleton)
    return float(T), float(U)
