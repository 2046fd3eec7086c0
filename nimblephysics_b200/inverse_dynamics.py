"""``inverse_dynamics(world, state, next_vel, mass=None)`` — contact-free inverse dynamics, batched and differentiable — and
``contact_inverse_dynamics(world, state, next_vel, contact_body, mass=None)``, the same force split into a contact wrench and joint torques.

It answers the reverse question of ``timestep``: which generalised force takes each world from ``state = [q; qdot]`` to the
velocity ``next_vel`` in one contact-free step?

    a = (next_vel - qdot) / dt ,   tau = M(q) a + C(q, qdot) + g(q) + K (q - q0 + qdot dt) + D qdot

tau is per dof (not gathered through the action map); free joints use the step's conventions.  Contacts, joint-limit rows and
force limits are ignored, and a world's LCP cache is never touched.  With an action space covering every dof,
``timestep(world, state, tau)`` returns ``next_vel`` up to rounding.  The nearest call of the reference is the contact-free
``Skeleton::getInverseDynamics(nextVel)`` for one skeleton.  Whether its spring term carries ``qdot * dt`` is unverified here;
this one uses the step's semi-implicit spring so that the round trip holds.

Contact inverse dynamics (the reference's ``Skeleton::getContactInverseDynamics(nextVel, contactBody)``): with tau_ID the force above
and J_c(q) the Jacobian from qdot to the spatial velocity [omega; v_origin] of ``contact_body`` in world axes about the world origin,

    tau + J_c(q)^T wrench = tau_ID   on every dof ,     tau = 0 on the six dofs of the free root of the contact body's skeleton.

wrench [6] is [torque; force] in world axes about the world origin (the convention of the world wrenches of ``ik_fk_vjp``).  It is the
total external wrench the motion needs, the ground reaction of a robot standing on that body, and is the same whichever body of the
skeleton is named.  tau differs from tau_ID only on the joints between the contact body and the root; every other dof, other skeletons
included, is tau_ID bit for bit.  The frame in which the reference reports its ``contactWrench`` is not checked here.

Precision follows the state's dtype: float64 tensors run the fp64 kernels with fp64 rows, anything else the fp32 ones.
Gradients flow to ``state``, ``next_vel`` and ``mass`` (1-D: ``setMasses``, shared by the batch, gradient summed; 2-D ``[B, m]``:
per world, the World is left untouched).  The work is done by libnb2.so (include/nb2.h ``nb2_inverse_dynamics``,
``nb2_contact_inverse_dynamics``).
"""
from __future__ import annotations

from typing import Optional

import torch

from .engine import FP32, FP64, device_model_for
from .timestep import _inertia_grad, _word_major_inertia, per_world_inertia, set_shared_masses, shared_mass_jacobian
from .world import FREE

_WHO = "inverse_dynamics()"
_WHO_CONTACT = "contact_inverse_dynamics()"


def _check_rows(world, state, next_vel, who):
    """ValueError unless state is [2n] / [B, 2n] and next_vel [n] / [B, n] (n = getNumDofs()); nothing touches the device."""
    n = world.getNumDofs()
    if state.dim() not in (1, 2) or state.shape[-1] != 2 * n:
        raise ValueError(f"{who}: state has shape {tuple(state.shape)}, expected [..., {2 * n}] (= getStateSize())")
    if next_vel.dim() != state.dim() or tuple(next_vel.shape) != tuple(state.shape[:-1]) + (n,):
        raise ValueError(f"{who}: next_vel has shape {tuple(next_vel.shape)}, expected the state's batch shape with {n} (= getNumDofs()) entries")


def _prepare(ctx, world, state, next_vel, mass, world_inertia, who):
    """The shared front of both layers: mass handling, device rows in the arithmetic type and what backward needs of it on ctx.
    Returns (dm, sd, vd, wi, need_grad)."""
    if mass is not None and world_inertia is not None:
        raise ValueError(f"{who}: give either a mass vector or a per-world inertia table, not both")
    _check_rows(world, state, next_vel, who)
    dm = set_shared_masses(world, mass, who) if mass is not None else device_model_for(world)
    single = state.dim() == 1
    s2 = state.detach().reshape(1, -1) if single else state.detach()
    v2 = next_vel.detach().reshape(1, -1) if single else next_vel.detach()
    if not torch.cuda.is_available():
        raise RuntimeError(f"nimblephysics_b200.{who[:-2]} needs a CUDA device; there is no CPU fallback")
    dev = s2.device if s2.is_cuda else torch.device("cuda", torch.cuda.current_device())
    rdt = torch.float64 if state.dtype == torch.float64 else torch.float32
    sd = s2.to(device=dev, dtype=rdt).contiguous()
    vd = v2.to(device=dev, dtype=rdt).contiguous()
    B = sd.shape[0]
    if world_inertia is not None and (single or tuple(world_inertia.shape) != (B, dm.cm.nb, 10)):
        raise ValueError(f"{who}: per-world inertia has shape {tuple(world_inertia.shape)}, expected [{B}, {dm.cm.nb}, 10] with a 2-D state")
    wi = _word_major_inertia(dm, world_inertia, B, dev)
    ctx.wi_grad = world_inertia is not None and ctx.needs_input_grad[4]
    ctx.wi_like = world_inertia
    ctx.mass_grad = mass is not None and ctx.needs_input_grad[3]
    if ctx.mass_grad:
        ctx.mass_P = shared_mass_jacobian(world, dm, dev)
        ctx.mass_like = mass
    ctx.dm, ctx.B, ctx.prec, ctx.single = dm, B, FP64 if rdt == torch.float64 else FP32, single
    ctx.in_meta = (state.device, state.dtype, next_vel.device, next_vel.dtype)
    return dm, sd, vd, wi, any(ctx.needs_input_grad[1:5])


def _backward_buffers(ctx, dev, dtype):
    """g_state, g_next_vel and (when a mass or inertia gradient is wanted) the [10*nb, B] fp64 inertia gradient."""
    dm, B = ctx.dm, ctx.B
    gs = torch.empty((B, 2 * dm.ndof), dtype=dtype, device=dev)
    gn = torch.empty((B, dm.ndof), dtype=dtype, device=dev)
    gi = torch.empty((10 * dm.cm.nb, B), dtype=torch.float64, device=dev) if (ctx.mass_grad or ctx.wi_grad) else None
    return gs, gn, gi


def _input_grads(ctx, gs, gn, gi):
    """(g_state, g_next_vel, g_mass, g_world_inertia) in the inputs' shapes, dtypes and devices."""
    gm = None
    if ctx.mass_grad:  # one mass vector shared by the batch: the worlds' gradients add up
        gm = (ctx.mass_P @ gi.sum(dim=1)).to(device=ctx.mass_like.device, dtype=ctx.mass_like.dtype)
    gw = _inertia_grad(gi, ctx.wi_like) if ctx.wi_grad else None
    sdev, sdt, vdev, vdt = ctx.in_meta
    if ctx.single:
        gs, gn = gs[0], gn[0]
    return gs.to(device=sdev, dtype=sdt), gn.to(device=vdev, dtype=vdt), gm, gw


def _ptr(t):
    return t.data_ptr() if t is not None else None


class InverseDynamicsLayer(torch.autograd.Function):
    """world_inertia (optional): per-world canonical inertia [B, nb, 10] (modelspec.mass_to_inertia), exclusive with the 1-D `mass`."""

    @staticmethod
    def forward(ctx, world, state, next_vel, mass, world_inertia=None):
        dm, sd, vd, wi, need_grad = _prepare(ctx, world, state, next_vel, mass, world_inertia, _WHO)
        B, dev = ctx.B, sd.device
        with torch.cuda.device(dev):
            tau = torch.empty((B, dm.ndof), dtype=sd.dtype, device=dev)
            saved = torch.empty((dm.saved_words, B), dtype=sd.dtype, device=dev) if need_grad else None
            dm.inverse_dynamics_device(B, sd.data_ptr(), vd.data_ptr(), tau.data_ptr(), _ptr(saved), torch.cuda.current_stream().cuda_stream,
                                       ctx.prec, wi_ptr=_ptr(wi))
        if need_grad:
            ctx.save_for_backward(sd, saved, wi)
        out = tau[0] if ctx.single else tau
        return out.to(device=state.device, dtype=state.dtype)

    @staticmethod
    def backward(ctx, grad_tau):
        dm, B = ctx.dm, ctx.B
        sd, saved, wi = ctx.saved_tensors
        dev = sd.device
        g = grad_tau.detach().reshape(B, dm.ndof).to(device=dev, dtype=sd.dtype).contiguous()
        with torch.cuda.device(dev):
            gs, gn, gi = _backward_buffers(ctx, dev, sd.dtype)
            dm.inverse_dynamics_backward_device(B, sd.data_ptr(), saved.data_ptr(), g.data_ptr(), gs.data_ptr(), gn.data_ptr(),
                                                torch.cuda.current_stream().cuda_stream, ctx.prec, ginertia_ptr=_ptr(gi), wi_ptr=_ptr(wi))
        return (None,) + _input_grads(ctx, gs, gn, gi)


def contact_body_index(world, body, who: str = _WHO_CONTACT) -> int:
    """The canonical index (of the device model) of `body`, a BodyNode of `world` under a FreeJoint root; a welded body maps to the body it
    is welded to.  ValueError, before any device work, for a body of another world, of an immobile skeleton, or under another root joint."""
    bodies = [b for sk in world.skeletons for b in sk._ordered_bodies()]
    raw = next((k for k, b in enumerate(bodies) if b is body), None)
    if raw is None:
        raise ValueError(f"{who}: the contact body {getattr(body, 'name', body)!r} is not a body of this world")
    sk = body.skeleton
    if sk is None or not sk.mobile or sk.getNumDofs() == 0:
        raise ValueError(f"{who}: the contact body {body.name!r} belongs to an immobile skeleton")
    root = body
    while root.parent_body is not None:
        root = root.parent_body
    if root.parent_joint is None or root.parent_joint.jtype != FREE:
        raise ValueError(f"{who}: the root joint of the contact body's skeleton is not a FreeJoint: its root dofs are not an external wrench")
    return raw


class ContactInverseDynamicsLayer(torch.autograd.Function):
    """Contact inverse dynamics of one contact body (raw body index `raw_body`, see contact_body_index); world_inertia as for
    InverseDynamicsLayer.  Returns (tau, wrench)."""

    @staticmethod
    def forward(ctx, world, state, next_vel, mass, world_inertia, raw_body):
        dm, sd, vd, wi, need_grad = _prepare(ctx, world, state, next_vel, mass, world_inertia, _WHO_CONTACT)
        body = int(dm.cm.body_owner[raw_body])
        B, dev = ctx.B, sd.device
        with torch.cuda.device(dev):
            tau = torch.empty((B, dm.ndof), dtype=sd.dtype, device=dev)
            wrench = torch.empty((B, 6), dtype=sd.dtype, device=dev)
            saved = torch.empty((dm.saved_words, B), dtype=sd.dtype, device=dev) if need_grad else None
            dm.contact_inverse_dynamics_device(B, body, sd.data_ptr(), vd.data_ptr(), tau.data_ptr(), wrench.data_ptr(), _ptr(saved),
                                               torch.cuda.current_stream().cuda_stream, ctx.prec, wi_ptr=_ptr(wi))
        ctx.body = body
        if need_grad:
            ctx.save_for_backward(sd, saved, wi, wrench)
        if ctx.single:
            tau, wrench = tau[0], wrench[0]
        return tau.to(device=state.device, dtype=state.dtype), wrench.to(device=state.device, dtype=state.dtype)

    @staticmethod
    def backward(ctx, grad_tau, grad_wrench):
        dm, B = ctx.dm, ctx.B
        sd, saved, wi, wrench = ctx.saved_tensors
        dev = sd.device
        g = grad_tau.detach().reshape(B, dm.ndof).to(device=dev, dtype=sd.dtype).contiguous()
        gw = grad_wrench.detach().reshape(B, 6).to(device=dev, dtype=sd.dtype).contiguous()
        with torch.cuda.device(dev):
            gs, gn, gi = _backward_buffers(ctx, dev, sd.dtype)
            seed = torch.empty((B, dm.ndof), dtype=sd.dtype, device=dev)
            dm.contact_inverse_dynamics_backward_device(B, ctx.body, sd.data_ptr(), saved.data_ptr(), wrench.data_ptr(), g.data_ptr(), gw.data_ptr(),
                                                        seed.data_ptr(), gs.data_ptr(), gn.data_ptr(), torch.cuda.current_stream().cuda_stream,
                                                        ctx.prec, ginertia_ptr=_ptr(gi), wi_ptr=_ptr(wi))
        return (None,) + _input_grads(ctx, gs, gn, gi) + (None,)


def inverse_dynamics(world, state: torch.Tensor, next_vel: torch.Tensor, mass: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Generalised force [B, n] (or [n] for a 1-D state) that takes every world from `state` [B, 2n] to `next_vel` [B, n] in one
    contact-free step (see the module docstring).  mass: None, a 1-D vector [getMassDims()] (world.setMasses(mass) first, shared by the
    batch, the masses stay set, the gradient sums over the batch), or a 2-D tensor [B, getMassDims()]: world w uses mass[w],
    mass.grad[w] is its own, and the World is not modified."""
    if mass is not None and mass.dim() == 2:
        return InverseDynamicsLayer.apply(world, state, next_vel, None, per_world_inertia(world, state, mass, _WHO))
    return InverseDynamicsLayer.apply(world, state, next_vel, mass)


def contact_inverse_dynamics(world, state: torch.Tensor, next_vel: torch.Tensor, contact_body, mass: Optional[torch.Tensor] = None):
    """(tau, wrench): tau [B, n] (or [n]) and wrench [B, 6] (or [6]) with tau + J_c^T wrench = inverse_dynamics(world, state, next_vel, mass)
    and tau = 0 on the free root of `contact_body`'s skeleton (see the module docstring).  contact_body: a BodyNode of `world` whose
    skeleton is mobile and has a FreeJoint root (ValueError otherwise, before any device work).  state, next_vel and mass as for
    inverse_dynamics; gradients of both outputs reach state, next_vel and mass."""
    raw_body = contact_body_index(world, contact_body)
    _check_rows(world, state, next_vel, _WHO_CONTACT)
    if mass is not None and mass.dim() == 2:
        return ContactInverseDynamicsLayer.apply(world, state, next_vel, None, per_world_inertia(world, state, mass, _WHO_CONTACT), raw_body)
    return ContactInverseDynamicsLayer.apply(world, state, next_vel, mass, None, raw_body)
