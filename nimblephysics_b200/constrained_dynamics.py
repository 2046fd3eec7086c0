"""``constrained_forward_dynamics(world, state, tau, contact_nodes, offsets=None, point_contacts=False, damping=0.0, mass=None)``:
joint accelerations and contact wrenches of worlds whose contact points are held by bilateral constraints, batched and differentiable.

For whole-body control, trajectory optimisation over a fixed stance schedule, MPC and policy learning through stance phases: the contact
set is known, and qdd and the contact wrenches are wanted as smooth functions of the state, the force and the masses.  With k contact
points p_i (1 <= k <= 4; each on a BodyNode, at an offset o_i in the node's frame, as in ``world_jacobian``), J the stack of their
world-Jacobian rows ([omega ; pdot], or only the three linear rows with ``point_contacts=True``), Jdot its time derivative
(``world_jacobian_deriv``) and rho = ``damping`` >= 0,

    M qdd + C + g + K (q - q0 + qdot dt) + D qdot = tau + J^T lam ,     J qdd + Jdot qdot = -rho lam ,

the dynamics of ``forward_dynamics`` with the contact forces added, so that

    lam = -(J M^-1 J^T + rho I)^-1 (J qdd_free + Jdot qdot) ,   qdd = forward_dynamics(state, tau + J^T lam) ,   qdd_free = forward_dynamics(state, tau).

lam_i is [torque about p_i ; force] in world axes.  The returned wrench of a 6-D contact is the wrench about the world origin,
[lam_a + p_i x lam_l ; lam_l], the convention of ``multiple_contact_inverse_dynamics``; a point contact returns its force lam_l.  The
constraints are equalities: no unilateral limits, friction cones or Baumgarte terms, and the world's own contacts, joint-limit rows and LCP
cache play no part.  tau is per dof and free joints use the step's velocity coordinates, as in ``forward_dynamics``.

A contact set that does not fix independent directions (J M^-1 J^T singular: e.g. a leg at a straight knee, or two 6-D contacts on one
chain) has no unique wrench.  A world whose J M^-1 J^T + rho I has a Cholesky pivot at or below 64 eps max(diagonal) (eps of the
arithmetic type) returns NaN in its qdd and wrench rows, and in its gradients; other worlds are unaffected.  A small rho > 0 makes the
problem regular: it picks the solution with the least wrench norm in the limit.

``constrained_forward_dynamics_jacobians`` returns qdd, the wrenches and their dense Jacobians in state and tau in one launch, for iLQR /
DDP, linearised MPC and contact-force constraints that need the matrices rather than products with one gradient.

``impulse_dynamics`` is the impact map at a phase switch of the same contact description: when the points strike, the pre-impact velocity
qdot- jumps to a qdot+ that satisfies the new constraints, with restitution e in [0, 1]:

    M (qdot+ - qdot-) = J^T Lam ,     J qdot+ = -e J qdot- - rho Lam .

``impulse_dynamics_jacobians`` returns qdot+, the impulses and their dense Jacobians in q and qdot- in one launch: the linearisation of the
reset map at a touchdown, for hybrid iLQR / DDP and trajectory optimisers.

The reference simulator has no counterpart: it resolves contact and impacts only through its LCP step.  The work is done by libnb2.so
(include/nb2.h ``nb2_constrained_forward_dynamics``, its backward, ``nb2_constrained_forward_dynamics_jacobians`` and
``nb2_impulse_dynamics`` with its backward and ``nb2_impulse_dynamics_jacobians``), one warp per world.
"""
from __future__ import annotations

import math
from typing import Optional, Sequence

import torch

from .engine import FP32, FP64, device_model_for
from .inverse_dynamics import MAX_CONTACT_BODIES, _backward_buffers, _check_fd, _input_grads, _prepare, _ptr
from .timestep import _inertia_grad, _word_major_inertia, per_world_inertia, set_shared_masses, shared_mass_jacobian
from .world_jacobian import _body_index, resolve_nodes

_WHO = "constrained_forward_dynamics()"
_WHO_J = "constrained_forward_dynamics_jacobians()"
_WHO_I = "impulse_dynamics()"
_WHO_IJ = "impulse_dynamics_jacobians()"


def _check_contacts(world, state, tau, nodes, offsets, damping, who=_WHO):
    """ValueError before any device work for a bad contact set, offsets, damping or dtype; returns the nodes as a list.  tau None: the
    checks of impulse_dynamics, which takes no force."""
    if tau is None:  # impulse dynamics: the state alone
        if world.getNumDofs() == 0:
            raise ValueError(f"{who}: the world has no degrees of freedom")
        n = world.getNumDofs()
        if state.dim() not in (1, 2) or state.shape[-1] != 2 * n:
            raise ValueError(f"{who}: state has shape {tuple(state.shape)}, expected [..., {2 * n}] (= getStateSize())")
    else:
        _check_fd(world, state, tau, who, "tau")
    for name, t in (("state", state), ("tau", tau)):
        if t is not None and not t.dtype.is_floating_point:
            raise ValueError(f"{who}: {name} has dtype {t.dtype}, expected a floating-point tensor")
    nodes = list(nodes)
    if not 1 <= len(nodes) <= MAX_CONTACT_BODIES:
        raise ValueError(f"{who}: {len(nodes)} contact nodes, expected 1 to {MAX_CONTACT_BODIES}")
    if len({id(b) for b in nodes}) != len(nodes):
        raise ValueError(f"{who}: a contact node appears twice")
    index = _body_index(world)
    for node in nodes:
        if id(node) not in index:
            raise ValueError(f"{who}: body node {getattr(node, 'name', node)!r} does not belong to this world")
        sk = node.skeleton
        if sk is None or not sk.mobile or sk.getNumDofs() == 0:
            raise ValueError(f"{who}: body node {node.name!r} belongs to an immobile skeleton")
    k = len(nodes)
    if offsets is not None:
        ok = offsets.dtype.is_floating_point and ((offsets.dim() == 2 and tuple(offsets.shape) == (k, 3)) or (
            offsets.dim() == 3 and state.dim() == 2 and tuple(offsets.shape) == (state.shape[0], k, 3)))
        if not ok:
            want = f"[{k}, 3]" + (f" or [{state.shape[0]}, {k}, 3]" if state.dim() == 2 else "")
            raise ValueError(f"{who}: offsets has shape {tuple(offsets.shape)} and dtype {offsets.dtype}, expected a floating-point {want}")
    if isinstance(damping, torch.Tensor) or not isinstance(damping, (int, float)) or not math.isfinite(damping) or damping < 0:
        raise ValueError(f"{who}: damping must be a finite float >= 0, got {damping!r}")
    return nodes


def _check_restitution(restitution, who):
    if isinstance(restitution, (torch.Tensor, bool)) or not isinstance(restitution, (int, float)) or not math.isfinite(restitution) \
            or not 0.0 <= restitution <= 1.0:
        raise ValueError(f"{who}: restitution must be a finite float in [0, 1], got {restitution!r}")


def _resolve(world, nodes, who=_WHO):
    """(canonical bodies, T12) of checked contact nodes; ValueError when two of them move with the same body."""
    bodies, T12 = resolve_nodes(world, nodes, who)
    if len(set(bodies.tolist())) != len(nodes) or (bodies < 0).any():
        raise ValueError(f"{who}: two contact nodes move with the same body (several points on one body are not supported)")
    return bodies, T12


class ConstrainedForwardDynamicsLayer(torch.autograd.Function):
    """(qdd, wrenches) of the canonical contact bodies `bodies` with placements T12 (world_jacobian.resolve_nodes); world_inertia as for
    InverseDynamicsLayer (exclusive with the 1-D `mass`); offsets None, [k, 3] or [B, k, 3]; point and damping as
    constrained_forward_dynamics."""

    @staticmethod
    def forward(ctx, world, state, tau, mass, world_inertia, offsets, bodies, T12, point, damping):
        dm, sd, td, wi, need_grad = _prepare(ctx, world, state, tau, mass, world_inertia, _WHO, "tau")
        need_grad = need_grad or ctx.needs_input_grad[5]
        B, dev, k = ctx.B, sd.device, len(bodies)
        od = None if offsets is None else offsets.detach().to(device=dev, dtype=sd.dtype).contiguous()
        ctx.bodies, ctx.T12, ctx.point, ctx.damping, ctx.off_like = bodies, T12, bool(point), float(damping), offsets
        with torch.cuda.device(dev):
            qdd = torch.empty((B, dm.ndof), dtype=sd.dtype, device=dev)
            wr = torch.empty((B, k, 3 if point else 6), dtype=sd.dtype, device=dev)
            dm.constrained_forward_dynamics_device(B, sd.data_ptr(), td.data_ptr(), bodies, T12, _ptr(od), od is not None and od.dim() == 3,
                                                   ctx.point, ctx.damping, qdd.data_ptr(), wr.data_ptr(), torch.cuda.current_stream().cuda_stream,
                                                   ctx.prec, wi_ptr=_ptr(wi))
        if need_grad:
            ctx.save_for_backward(sd, td, od, wi)
        if ctx.single:
            qdd, wr = qdd[0], wr[0]
        return qdd.to(device=state.device, dtype=state.dtype), wr.to(device=state.device, dtype=state.dtype)

    @staticmethod
    def backward(ctx, grad_qdd, grad_wrenches):
        dm, B = ctx.dm, ctx.B
        sd, td, od, wi = ctx.saved_tensors
        dev, k = sd.device, len(ctx.bodies)
        g = grad_qdd.detach().reshape(B, dm.ndof).to(device=dev, dtype=sd.dtype).contiguous()
        gw = grad_wrenches.detach().reshape(B, k, 3 if ctx.point else 6).to(device=dev, dtype=sd.dtype).contiguous()
        want_off = ctx.off_like is not None and ctx.needs_input_grad[5]
        with torch.cuda.device(dev):
            gs, gt, gi = _backward_buffers(ctx, dev, sd.dtype)
            go = torch.empty((B, k, 3), dtype=sd.dtype, device=dev) if want_off else None
            dm.constrained_forward_dynamics_backward_device(B, sd.data_ptr(), td.data_ptr(), ctx.bodies, ctx.T12, _ptr(od),
                                                            od is not None and od.dim() == 3, ctx.point, ctx.damping, g.data_ptr(), gw.data_ptr(),
                                                            gs.data_ptr(), gt.data_ptr(), _ptr(go), torch.cuda.current_stream().cuda_stream,
                                                            ctx.prec, ginertia_ptr=_ptr(gi), wi_ptr=_ptr(wi))
        if want_off:
            if ctx.off_like.dim() == 2:  # offsets shared by the batch: the worlds' gradients add up
                go = go.sum(dim=0)
            go = go.to(device=ctx.off_like.device, dtype=ctx.off_like.dtype)
        return (None,) + _input_grads(ctx, gs, gt, gi) + (go, None, None, None, None)


def constrained_forward_dynamics(world, state: torch.Tensor, tau: torch.Tensor, contact_nodes: Sequence, offsets: Optional[torch.Tensor] = None,
                                 point_contacts: bool = False, damping: float = 0.0, mass: Optional[torch.Tensor] = None):
    """(qdd, wrenches): qdd [B, n] and wrenches [B, k, 6] ([B, k, 3] with point_contacts; [n] and [k, 6] / [k, 3] for a 1-D state) of every
    world at `state` [B, 2n] under the per-dof force `tau` [B, n] with the k `contact_nodes` held (see the module docstring).
    contact_nodes: 1 to 4 distinct BodyNodes of mobile skeletons of `world` (different skeletons allowed; a welded node counts through the
    body it is welded to, and no two may move with the same body).  offsets: None (the nodes' origins), [k, 3] (shared by the batch) or
    [B, k, 3], in each node's frame.  damping: rho >= 0, a float.  mass as for forward_dynamics: None, 1-D (setMasses, shared) or
    [B, getMassDims()] (per world).  Precision follows state.dtype.  Gradients of both outputs reach state, tau, offsets and mass.
    ValueError before any device work for a bad contact set, shape, dtype or damping."""
    nodes = _check_contacts(world, state, tau, contact_nodes, offsets, damping)
    if mass is not None and mass.dim() == 2:
        wi = per_world_inertia(world, state, mass, _WHO)
        return ConstrainedForwardDynamicsLayer.apply(world, state, tau, None, wi, offsets, *_resolve(world, nodes), point_contacts, damping)
    bodies, T12 = _resolve(world, nodes)
    return ConstrainedForwardDynamicsLayer.apply(world, state, tau, mass, None, offsets, bodies, T12, point_contacts, damping)


def constrained_forward_dynamics_jacobians(world, state: torch.Tensor, tau: torch.Tensor, contact_nodes: Sequence,
                                           offsets: Optional[torch.Tensor] = None, point_contacts: bool = False, damping: float = 0.0,
                                           mass: Optional[torch.Tensor] = None):
    """(qdd, wrenches, dqdd_dq, dqdd_dqdot, dqdd_dtau, dwrench_dq, dwrench_dqdot, dwrench_dtau): the outputs of
    constrained_forward_dynamics for the same arguments and their dense Jacobians in the layout of torch.autograd.functional.jacobian,
    dqdd_dx [B, n, n] and dwrench_dx [B, k, r, n] (r = 6, or 3 with point_contacts), entry [w, ..., j] = d out / d x_j, x = the positions,
    the velocities and tau.  Row i of each block is constrained_forward_dynamics's vector-Jacobian product with the seed e_i on that output,
    so the blocks equal autograd's Jacobian up to rounding; free joints follow its conventions (position columns for the six stored
    coordinates, body-twist velocity columns) and the wrenches are about the world origin.  From the definition, with A = J M^-1 J^T + rho I:

        dqdd_dtau = M^-1 - M^-1 J^T A^-1 J M^-1 ,   dlam_dtau = -A^-1 J M^-1 ,   J dqdd_dtau = -rho dlam_dtau .

    Arguments, shapes, masses and precision as constrained_forward_dynamics; a 1-D state gives the same blocks without B.  The outputs carry
    no autograd history: there are no second derivatives and no offset or mass Jacobian.  A singular world gets NaN in every output and
    block.  ValueError before any device work for the argument errors of constrained_forward_dynamics."""
    nodes = _check_contacts(world, state, tau, contact_nodes, offsets, damping, _WHO_J)
    wi = per_world_inertia(world, state, mass, _WHO_J) if mass is not None and mass.dim() == 2 else None
    bodies, T12 = _resolve(world, nodes, _WHO_J)
    dm = set_shared_masses(world, mass, _WHO_J) if mass is not None and wi is None else device_model_for(world)
    if not torch.cuda.is_available():
        raise RuntimeError(f"nimblephysics_b200.{_WHO_J[:-2]} needs a CUDA device; there is no CPU fallback")
    single = state.dim() == 1
    s2 = state.detach().reshape(1, -1) if single else state.detach()
    t2 = tau.detach().reshape(1, -1) if single else tau.detach()
    dev = s2.device if s2.is_cuda else torch.device("cuda", torch.cuda.current_device())
    rdt = torch.float64 if state.dtype == torch.float64 else torch.float32
    sd = s2.to(device=dev, dtype=rdt).contiguous()
    td = t2.to(device=dev, dtype=rdt).contiguous()
    od = None if offsets is None else offsets.detach().to(device=dev, dtype=rdt).contiguous()
    B, n, k, r = sd.shape[0], dm.ndof, len(nodes), 3 if point_contacts else 6
    with torch.cuda.device(dev):
        qdd = torch.empty((B, n), dtype=rdt, device=dev)
        wr = torch.empty((B, k, r), dtype=rdt, device=dev)
        J = [torch.empty((B, n, n), dtype=rdt, device=dev) for _ in range(3)] + [torch.empty((B, k, r, n), dtype=rdt, device=dev) for _ in range(3)]
        if B > 0:  # an empty batch has no rows to hand over (its data pointers may be NULL)
            dm.constrained_forward_dynamics_jacobians_device(B, sd.data_ptr(), td.data_ptr(), bodies, T12, _ptr(od), od is not None and od.dim() == 3,
                                                             bool(point_contacts), float(damping), qdd.data_ptr(), wr.data_ptr(),
                                                             [x.data_ptr() for x in J], torch.cuda.current_stream().cuda_stream,
                                                             FP64 if rdt == torch.float64 else FP32,
                                                             wi_ptr=_ptr(_word_major_inertia(dm, wi, B, dev)))
    res = [qdd, wr] + J
    if single:
        res = [x[0] for x in res]
    return tuple(x.to(device=state.device, dtype=state.dtype) for x in res)


class ImpulseDynamicsLayer(torch.autograd.Function):
    """(qdot_after, impulses) of the canonical contact bodies `bodies` with placements T12 (world_jacobian.resolve_nodes); world_inertia
    as for InverseDynamicsLayer (exclusive with the 1-D `mass`); offsets None, [k, 3] or [B, k, 3]; point, restitution and damping as
    impulse_dynamics.  No gradient reaches restitution or damping."""

    @staticmethod
    def forward(ctx, world, state, mass, world_inertia, offsets, bodies, T12, point, restitution, damping):
        if mass is not None and world_inertia is not None:
            raise ValueError(f"{_WHO_I}: give either a mass vector or a per-world inertia table, not both")
        dm = set_shared_masses(world, mass, _WHO_I) if mass is not None else device_model_for(world)
        if not torch.cuda.is_available():
            raise RuntimeError(f"nimblephysics_b200.{_WHO_I[:-2]} needs a CUDA device; there is no CPU fallback")
        ctx.single = state.dim() == 1
        s2 = state.detach().reshape(1, -1) if ctx.single else state.detach()
        dev = s2.device if s2.is_cuda else torch.device("cuda", torch.cuda.current_device())
        rdt = torch.float64 if state.dtype == torch.float64 else torch.float32
        sd = s2.to(device=dev, dtype=rdt).contiguous()
        B, k = sd.shape[0], len(bodies)
        if world_inertia is not None and (ctx.single or tuple(world_inertia.shape) != (B, dm.cm.nb, 10)):
            raise ValueError(f"{_WHO_I}: per-world inertia has shape {tuple(world_inertia.shape)}, expected [{B}, {dm.cm.nb}, 10] with a 2-D state")
        wi = _word_major_inertia(dm, world_inertia, B, dev)
        od = None if offsets is None else offsets.detach().to(device=dev, dtype=rdt).contiguous()
        ctx.dm, ctx.B, ctx.prec = dm, B, FP64 if rdt == torch.float64 else FP32
        ctx.bodies, ctx.T12, ctx.point, ctx.e, ctx.damping, ctx.off_like = bodies, T12, bool(point), float(restitution), float(damping), offsets
        ctx.state_meta = (state.device, state.dtype)
        ctx.mass_grad = mass is not None and ctx.needs_input_grad[2]
        if ctx.mass_grad:
            ctx.mass_P, ctx.mass_like = shared_mass_jacobian(world, dm, dev), mass
        ctx.wi_grad, ctx.wi_like = world_inertia is not None and ctx.needs_input_grad[3], world_inertia
        with torch.cuda.device(dev):
            vel = torch.empty((B, dm.ndof), dtype=rdt, device=dev)
            imp = torch.empty((B, k, 3 if point else 6), dtype=rdt, device=dev)
            if B > 0:  # an empty batch has no rows to hand over (its data pointers may be NULL)
                dm.impulse_dynamics_device(B, sd.data_ptr(), bodies, T12, _ptr(od), od is not None and od.dim() == 3, ctx.point, ctx.e, ctx.damping,
                                           vel.data_ptr(), imp.data_ptr(), torch.cuda.current_stream().cuda_stream, ctx.prec, wi_ptr=_ptr(wi))
        if any(ctx.needs_input_grad[1:5]):
            ctx.save_for_backward(sd, od, wi)
        if ctx.single:
            vel, imp = vel[0], imp[0]
        return vel.to(device=state.device, dtype=state.dtype), imp.to(device=state.device, dtype=state.dtype)

    @staticmethod
    def backward(ctx, grad_vel, grad_impulses):
        dm, B = ctx.dm, ctx.B
        sd, od, wi = ctx.saved_tensors
        dev, k = sd.device, len(ctx.bodies)
        g = grad_vel.detach().reshape(B, dm.ndof).to(device=dev, dtype=sd.dtype).contiguous()
        gw = grad_impulses.detach().reshape(B, k, 3 if ctx.point else 6).to(device=dev, dtype=sd.dtype).contiguous()
        want_off = ctx.off_like is not None and ctx.needs_input_grad[4]
        with torch.cuda.device(dev):
            gs = torch.empty((B, 2 * dm.ndof), dtype=sd.dtype, device=dev)
            gi = torch.empty((10 * dm.cm.nb, B), dtype=torch.float64, device=dev) if (ctx.mass_grad or ctx.wi_grad) else None
            go = torch.empty((B, k, 3), dtype=sd.dtype, device=dev) if want_off else None
            if B > 0:
                dm.impulse_dynamics_backward_device(B, sd.data_ptr(), ctx.bodies, ctx.T12, _ptr(od), od is not None and od.dim() == 3, ctx.point,
                                                    ctx.e, ctx.damping, g.data_ptr(), gw.data_ptr(), gs.data_ptr(), _ptr(go),
                                                    torch.cuda.current_stream().cuda_stream, ctx.prec, ginertia_ptr=_ptr(gi), wi_ptr=_ptr(wi))
            elif gi is not None:
                gi.zero_()
        gm = (ctx.mass_P @ gi.sum(dim=1)).to(device=ctx.mass_like.device, dtype=ctx.mass_like.dtype) if ctx.mass_grad else None
        gwi = _inertia_grad(gi, ctx.wi_like) if ctx.wi_grad else None
        if want_off:
            if ctx.off_like.dim() == 2:  # offsets shared by the batch: the worlds' gradients add up
                go = go.sum(dim=0)
            go = go.to(device=ctx.off_like.device, dtype=ctx.off_like.dtype)
        gs = gs[0] if ctx.single else gs
        return None, gs.to(device=ctx.state_meta[0], dtype=ctx.state_meta[1]), gm, gwi, go, None, None, None, None, None


def impulse_dynamics(world, state: torch.Tensor, contact_nodes: Sequence, offsets: Optional[torch.Tensor] = None, point_contacts: bool = False,
                     restitution: float = 0.0, damping: float = 0.0, mass: Optional[torch.Tensor] = None):
    """(qdot_after, impulses): the post-impact velocities [B, n] and contact impulses [B, k, 6] ([B, k, 3] with point_contacts; [n] and
    [k, 6] / [k, 3] for a 1-D state) of every world at `state` [B, 2n] = [q ; qdot-] when the k `contact_nodes` strike and are held, with
    restitution e = `restitution` and damping rho = `damping`:

        Lam = -(J M^-1 J^T + rho I)^-1 (1 + e) J qdot- ,   qdot_after = qdot- + M^-1 J^T Lam .

    Lam_i is [angular impulse about p_i ; linear impulse] in world axes, in N s; a 6-D contact returns it about the world origin,
    [Lam_a + p_i x Lam_l ; Lam_l], a point contact Lam_l (the wrench convention of constrained_forward_dynamics).  The impact is
    instantaneous: gravity, joint springs and damping, limits, the world's own contacts and the LCP cache play no part.  With rho = 0,
    e = 1 keeps the kinetic energy and e < 1 loses (1 - e^2) / 2 (J qdot-)^T (J M^-1 J^T)^-1 (J qdot-); at e = 0 a second impact changes
    nothing.  Velocities are in the step's coordinates (free joints use the body twist).

    contact_nodes, offsets, point_contacts, damping and mass as constrained_forward_dynamics; restitution: a Python number in [0, 1].
    Precision follows state.dtype.  Gradients of both outputs reach state (both halves), offsets and mass; none reach restitution or
    damping.  A singular contact set gives NaN rows in that world only, as in constrained_forward_dynamics.  ValueError before any device
    work for a bad contact set, shape, dtype, damping or restitution."""
    nodes = _check_contacts(world, state, None, contact_nodes, offsets, damping, _WHO_I)
    _check_restitution(restitution, _WHO_I)
    wi = per_world_inertia(world, state, mass, _WHO_I) if mass is not None and mass.dim() == 2 else None
    bodies, T12 = _resolve(world, nodes, _WHO_I)
    return ImpulseDynamicsLayer.apply(world, state, None if wi is not None else mass, wi, offsets, bodies, T12, point_contacts,
                                      float(restitution), float(damping))


def impulse_dynamics_jacobians(world, state: torch.Tensor, contact_nodes: Sequence, offsets: Optional[torch.Tensor] = None,
                               point_contacts: bool = False, restitution: float = 0.0, damping: float = 0.0, mass: Optional[torch.Tensor] = None):
    """(qdot_after, impulses, dv_dq, dv_dqdot, dimp_dq, dimp_dqdot): the outputs of impulse_dynamics for the same arguments (equal to them
    bit for bit) and their dense Jacobians in the layout of torch.autograd.functional.jacobian, dv_dx [B, n, n] and dimp_dx [B, k, r, n]
    (r = 6, or 3 with point_contacts), entry [w, ..., j] = d out / d x_j, x = the positions q or the pre-impact velocities qdot-.  Row i of
    each block is impulse_dynamics's vector-Jacobian product with the seed e_i on that output, so the blocks equal autograd's Jacobian up
    to rounding; free joints follow its conventions (position columns for the six stored coordinates, body-twist velocity columns) and
    the impulses of 6-D contacts are about the world origin.  With A = J M^-1 J^T + rho I, e the restitution and Lam in point form (the
    returned 6-D impulse is [Lam_a + p x Lam_l ; Lam_l]):

        dv_dqdot = I - (1 + e) M^-1 J^T A^-1 J ,   dLam_dqdot = -(1 + e) A^-1 J ,

    and qdot_after and Lam are linear in qdot- at fixed q (qdot_after = dv_dqdot qdot-, Lam = dLam_dqdot qdot-).  With rho = 0,
    J dv_dqdot = -e J, and at e = 0 dv_dqdot is a projector whose product with M is symmetric.  Differentiating the constraint in q:
    J dv_dq + d(J(q) v)/dq |_(v = qdot_after + e qdot-) = -rho dLam_dq.  For the hybrid state x = [q ; qdot], the reset map at the
    touchdown has the Jacobian

        dDelta/dx = [[I, 0], [dv_dq, dv_dqdot]] .

    Arguments, shapes, masses and precision as impulse_dynamics; a 1-D state gives the same blocks without B.  The outputs carry no
    autograd history: there are no second derivatives and no offset, mass, restitution or damping Jacobian.  A singular world gets NaN in
    every output and block; the other worlds are unaffected.  ValueError before any device work for the argument errors of
    impulse_dynamics."""
    nodes = _check_contacts(world, state, None, contact_nodes, offsets, damping, _WHO_IJ)
    _check_restitution(restitution, _WHO_IJ)
    wi = per_world_inertia(world, state, mass, _WHO_IJ) if mass is not None and mass.dim() == 2 else None
    bodies, T12 = _resolve(world, nodes, _WHO_IJ)
    dm = set_shared_masses(world, mass, _WHO_IJ) if mass is not None and wi is None else device_model_for(world)
    if not torch.cuda.is_available():
        raise RuntimeError(f"nimblephysics_b200.{_WHO_IJ[:-2]} needs a CUDA device; there is no CPU fallback")
    single = state.dim() == 1
    s2 = state.detach().reshape(1, -1) if single else state.detach()
    dev = s2.device if s2.is_cuda else torch.device("cuda", torch.cuda.current_device())
    rdt = torch.float64 if state.dtype == torch.float64 else torch.float32
    sd = s2.to(device=dev, dtype=rdt).contiguous()
    od = None if offsets is None else offsets.detach().to(device=dev, dtype=rdt).contiguous()
    B, n, k, r = sd.shape[0], dm.ndof, len(nodes), 3 if point_contacts else 6
    with torch.cuda.device(dev):
        vel = torch.empty((B, n), dtype=rdt, device=dev)
        imp = torch.empty((B, k, r), dtype=rdt, device=dev)
        J = [torch.empty((B, n, n), dtype=rdt, device=dev) for _ in range(2)] + [torch.empty((B, k, r, n), dtype=rdt, device=dev) for _ in range(2)]
        if B > 0:  # an empty batch has no rows to hand over (its data pointers may be NULL)
            dm.impulse_dynamics_jacobians_device(B, sd.data_ptr(), bodies, T12, _ptr(od), od is not None and od.dim() == 3, bool(point_contacts),
                                                 float(restitution), float(damping), vel.data_ptr(), imp.data_ptr(), [x.data_ptr() for x in J],
                                                 torch.cuda.current_stream().cuda_stream, FP64 if rdt == torch.float64 else FP32,
                                                 wi_ptr=_ptr(_word_major_inertia(dm, wi, B, dev)))
    res = [vel, imp] + J
    if single:
        res = [x[0] for x in res]
    return tuple(x.to(device=state.device, dtype=state.dtype) for x in res)
