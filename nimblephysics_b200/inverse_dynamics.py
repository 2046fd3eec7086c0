"""``inverse_dynamics(world, state, next_vel, mass=None)`` — contact-free inverse dynamics, batched and differentiable —,
``contact_inverse_dynamics(world, state, next_vel, contact_body, mass=None)``, the same force split into a contact wrench and joint torques,
and ``multiple_contact_inverse_dynamics(world, state, next_vel, contact_bodies, mass=None, wrench_guesses=None)``, split over several bodies.

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

Multiple-contact inverse dynamics (the reference's ``Skeleton::getMultipleContactInverseDynamics(nextVel, bodies, bodyWrenchGuesses)``):
with k contact bodies c_1..c_k of one skeleton, J_i their Jacobians as above, p_i the world position of c_i's own origin and g_i guesses,

    tau + sum_i J_i(q)^T w_i = tau_ID   on every dof ,     tau = 0 on the free root ,
    minimise  sum_i | Gamma(p_i)^-1 (w_i - g_i) |^2 ,      Gamma(p) = [[I, [p]x], [0, I]] ,

so the deviation from each guess is measured as [torque about p_i; force], independently of where the world origin is.  The w_i sum to the
one-body wrench; the objective and the wrench frame are this package's, the reference's could not be checked.

Forward dynamics, ``forward_dynamics(world, state, tau, mass=None)`` (the reference's ``Skeleton::computeForwardDynamics()`` followed by
``getAccelerations()``, and ``SimpleFeatherstone::forwardDynamics``), is the exact inverse of ``inverse_dynamics``: the acceleration the
contact-free step applies under the per-dof force tau,

    qdd = M(q)^-1 ( tau - C(q, qdot) - g(q) - K (q - q0 + qdot dt) - D qdot ) ,    so that  v+ = qdot + dt qdd  and
    inverse_dynamics(world, state, qdot + dt qdd) = tau  up to rounding.

tau is per dof like the output of ``inverse_dynamics`` (any action space works); contacts, joint-limit rows, velocity and force limits are
ignored, no gradient clipping is applied and the LCP cache is never touched.  Gradients flow to ``state``, ``tau`` and ``mass``.

Precision follows the state's dtype: float64 tensors run the fp64 kernels with fp64 rows, anything else the fp32 ones.
Gradients flow to ``state``, ``next_vel`` and ``mass`` (1-D: ``setMasses``, shared by the batch, gradient summed; 2-D ``[B, m]``:
per world, the World is left untouched).  The work is done by libnb2.so (include/nb2.h ``nb2_inverse_dynamics``,
``nb2_contact_inverse_dynamics``, ``nb2_multiple_contact_inverse_dynamics``, ``nb2_forward_dynamics_batch``).

``inverse_dynamics_jacobians`` and ``forward_dynamics_jacobians`` return the dense Jacobians of ``inverse_dynamics`` and
``forward_dynamics`` (with their outputs) in one launch (``nb2_inverse_dynamics_jacobians`` / ``nb2_forward_dynamics_jacobians``), for
iLQR / DDP, Gauss-Newton or linearised-MPC users who need the matrices rather than products with one gradient.
``contact_inverse_dynamics_jacobians`` and ``multiple_contact_inverse_dynamics_jacobians`` do the same for the two contact splits
(``nb2_multiple_contact_inverse_dynamics_jacobians``).
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch

from .engine import FP32, FP64, device_model_for
from .timestep import _inertia_grad, _word_major_inertia, per_world_inertia, set_shared_masses, shared_mass_jacobian
from .world import FREE

_WHO = "inverse_dynamics()"
_WHO_CONTACT = "contact_inverse_dynamics()"
_WHO_MULTI = "multiple_contact_inverse_dynamics()"
_WHO_FD = "forward_dynamics()"
_WHO_IDJ = "inverse_dynamics_jacobians()"
_WHO_FDJ = "forward_dynamics_jacobians()"
_WHO_CIDJ = "contact_inverse_dynamics_jacobians()"
_WHO_MCIDJ = "multiple_contact_inverse_dynamics_jacobians()"
MAX_CONTACT_BODIES = 4  # include/nb2.h NB2_MAX_CONTACT_BODIES


def _check_rows(world, state, next_vel, who, second="next_vel"):
    """ValueError unless state is [2n] / [B, 2n] and the second row argument (`second`: its name in the message) [n] / [B, n]
    (n = getNumDofs()); nothing touches the device."""
    n = world.getNumDofs()
    if state.dim() not in (1, 2) or state.shape[-1] != 2 * n:
        raise ValueError(f"{who}: state has shape {tuple(state.shape)}, expected [..., {2 * n}] (= getStateSize())")
    if next_vel.dim() != state.dim() or tuple(next_vel.shape) != tuple(state.shape[:-1]) + (n,):
        raise ValueError(f"{who}: {second} has shape {tuple(next_vel.shape)}, expected the state's batch shape with {n} (= getNumDofs()) entries")


def _prepare(ctx, world, state, next_vel, mass, world_inertia, who, second="next_vel"):
    """The shared front of the layers: mass handling, device rows in the arithmetic type and what backward needs of it on ctx.
    Returns (dm, sd, vd, wi, need_grad)."""
    if mass is not None and world_inertia is not None:
        raise ValueError(f"{who}: give either a mass vector or a per-world inertia table, not both")
    _check_rows(world, state, next_vel, who, second)
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
    """g_state, the gradient of the second row argument and (when a mass or inertia gradient is wanted) the [10*nb, B] fp64 inertia gradient."""
    dm, B = ctx.dm, ctx.B
    gs = torch.empty((B, 2 * dm.ndof), dtype=dtype, device=dev)
    gn = torch.empty((B, dm.ndof), dtype=dtype, device=dev)
    gi = torch.empty((10 * dm.cm.nb, B), dtype=torch.float64, device=dev) if (ctx.mass_grad or ctx.wi_grad) else None
    return gs, gn, gi


def _input_grads(ctx, gs, gn, gi):
    """(g_state, g of the second row argument, g_mass, g_world_inertia) in the inputs' shapes, dtypes and devices."""
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


def _check_fd(world, state, tau, who=_WHO_FD, second="tau"):
    """ValueError unless the world has dofs and state / tau are rows as inverse_dynamics takes them; nothing touches the device."""
    if world.getNumDofs() == 0:
        raise ValueError(f"{who}: the world has no degrees of freedom")
    _check_rows(world, state, tau, who, second)


class ForwardDynamicsLayer(torch.autograd.Function):
    """Forward dynamics qdd = FD(state, tau); world_inertia as for InverseDynamicsLayer (exclusive with the 1-D `mass`)."""

    @staticmethod
    def forward(ctx, world, state, tau, mass, world_inertia=None):
        _check_fd(world, state, tau)
        dm, sd, td, wi, need_grad = _prepare(ctx, world, state, tau, mass, world_inertia, _WHO_FD, "tau")
        B, dev = ctx.B, sd.device
        with torch.cuda.device(dev):
            qdd = torch.empty((B, dm.ndof), dtype=sd.dtype, device=dev)
            saved = torch.empty((dm.saved_words, B), dtype=sd.dtype, device=dev) if need_grad else None
            if B > 0:  # an empty batch has no rows to hand over (its data pointers may be NULL)
                dm.forward_dynamics_device(B, sd.data_ptr(), td.data_ptr(), qdd.data_ptr(), _ptr(saved), torch.cuda.current_stream().cuda_stream,
                                           ctx.prec, wi_ptr=_ptr(wi))
        if need_grad:
            ctx.save_for_backward(sd, saved, wi)
        out = qdd[0] if ctx.single else qdd
        return out.to(device=state.device, dtype=state.dtype)

    @staticmethod
    def backward(ctx, grad_qdd):
        dm, B = ctx.dm, ctx.B
        sd, saved, wi = ctx.saved_tensors
        dev = sd.device
        g = grad_qdd.detach().reshape(B, dm.ndof).to(device=dev, dtype=sd.dtype).contiguous()
        with torch.cuda.device(dev):
            gs, gt, gi = _backward_buffers(ctx, dev, sd.dtype)
            if B > 0:
                dm.forward_dynamics_backward_device(B, sd.data_ptr(), saved.data_ptr(), g.data_ptr(), gs.data_ptr(), gt.data_ptr(),
                                                    torch.cuda.current_stream().cuda_stream, ctx.prec, ginertia_ptr=_ptr(gi), wi_ptr=_ptr(wi))
        return (None,) + _input_grads(ctx, gs, gt, gi)


def forward_dynamics(world, state: torch.Tensor, tau: torch.Tensor, mass: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Joint accelerations qdd [B, n] (or [n] for a 1-D state) of every world at `state` [B, 2n] under the per-dof generalised force `tau`
    [B, n]: the acceleration the contact-free step applies, the exact inverse of inverse_dynamics (see the module docstring).  mass as for
    inverse_dynamics.  ValueError before any device work for a wrong shape, a world without dofs or a mass of the wrong size."""
    _check_fd(world, state, tau)
    if mass is not None and mass.dim() == 2:
        return ForwardDynamicsLayer.apply(world, state, tau, None, per_world_inertia(world, state, mass, _WHO_FD))
    return ForwardDynamicsLayer.apply(world, state, tau, mass)


def _dynamics_jacobians(world, state, x, mass, who, second, fd):
    """The shared body of inverse_dynamics_jacobians / forward_dynamics_jacobians: (out, J_q, J_qdot, J_x) in the state's dtype and device."""
    _check_fd(world, state, x, who, second)
    wi = per_world_inertia(world, state, mass, who) if mass is not None and mass.dim() == 2 else None
    dm = set_shared_masses(world, mass, who) if mass is not None and wi is None else device_model_for(world)
    if not torch.cuda.is_available():
        raise RuntimeError(f"nimblephysics_b200.{who[:-2]} needs a CUDA device; there is no CPU fallback")
    single = state.dim() == 1
    s2 = state.detach().reshape(1, -1) if single else state.detach()
    x2 = x.detach().reshape(1, -1) if single else x.detach()
    dev = s2.device if s2.is_cuda else torch.device("cuda", torch.cuda.current_device())
    rdt = torch.float64 if state.dtype == torch.float64 else torch.float32
    sd = s2.to(device=dev, dtype=rdt).contiguous()
    xd = x2.to(device=dev, dtype=rdt).contiguous()
    B, n = sd.shape[0], dm.ndof
    with torch.cuda.device(dev):
        out = torch.empty((B, n), dtype=rdt, device=dev)
        J = [torch.empty((B, n, n), dtype=rdt, device=dev) for _ in range(3)]
        if B > 0:  # an empty batch has no rows to hand over (its data pointers may be NULL)
            run = dm.forward_dynamics_jacobians_device if fd else dm.inverse_dynamics_jacobians_device
            run(B, sd.data_ptr(), xd.data_ptr(), out.data_ptr(), J[0].data_ptr(), J[1].data_ptr(), J[2].data_ptr(), torch.cuda.current_stream().cuda_stream,
                FP64 if rdt == torch.float64 else FP32, wi_ptr=_ptr(_word_major_inertia(dm, wi, B, dev)))
    res = [out] + J
    if single:
        res = [r[0] for r in res]
    return tuple(r.to(device=state.device, dtype=state.dtype) for r in res)


def inverse_dynamics_jacobians(world, state: torch.Tensor, next_vel: torch.Tensor, mass: Optional[torch.Tensor] = None):
    """(tau, dtau_dq, dtau_dqdot, dtau_dnext_vel): tau = inverse_dynamics(world, state, next_vel, mass) [B, n] and its dense Jacobians
    [B, n, n], J[w, i, j] = d tau_i / d x_j (the layout of torch.autograd.functional.jacobian), next_vel held fixed in the first two:

        dtau_dnext_vel = M / dt ,   dtau_dqdot = dID_a/dqdot + D + dt K - M / dt ,   dtau_dq = dID_a/dq + K ,

    with ID_a(q, qdot, a) = M a + C + g at a = (next_vel - qdot) / dt.  Row i is inverse_dynamics's vector-Jacobian product with the seed
    e_i, so the blocks equal autograd's Jacobian of inverse_dynamics up to rounding; free joints follow its conventions (body-twist velocity
    columns, position columns for the six stored coordinates).  state [B, 2n] or [2n] (then [n] and [n, n] outputs), mass as for
    inverse_dynamics; precision follows state.dtype.  Contacts, limits and clipping are ignored and the LCP cache is not touched.
    The outputs carry no autograd history: there are no second derivatives and no mass Jacobian.  ValueError before any device work for a
    wrong shape, a world without dofs or a mass of the wrong size."""
    return _dynamics_jacobians(world, state, next_vel, mass, _WHO_IDJ, "next_vel", False)


def forward_dynamics_jacobians(world, state: torch.Tensor, tau: torch.Tensor, mass: Optional[torch.Tensor] = None):
    """(qdd, dqdd_dq, dqdd_dqdot, dqdd_dtau): qdd = forward_dynamics(world, state, tau, mass) [B, n] and its dense Jacobians [B, n, n],
    J[w, i, j] = d qdd_i / d x_j:

        dqdd_dtau = M^-1 ,   dqdd_dq = -M^-1 (dID_a/dq + K) ,   dqdd_dqdot = -M^-1 (dID_a/dqdot + D + dt K)    at a = qdd.

    Row i is forward_dynamics's vector-Jacobian product with the seed e_i, so the blocks equal autograd's Jacobian of forward_dynamics up to
    rounding.  Arguments, shapes, precision and what is ignored as for inverse_dynamics_jacobians; unlike forward_dynamics this runs on
    every model inverse_mass_matrix runs on, in both precisions.  The outputs carry no autograd history: there are no second derivatives
    and no mass Jacobian.  ValueError before any device work for a wrong shape, a world without dofs or a mass of the wrong size."""
    return _dynamics_jacobians(world, state, tau, mass, _WHO_FDJ, "tau", True)


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


def contact_body_indices(world, bodies, who: str = _WHO_MULTI) -> list:
    """The raw indices of `bodies`, 1..MAX_CONTACT_BODIES distinct BodyNodes of one skeleton of `world`, each as contact_body_index
    requires.  ValueError before any device work otherwise."""
    bodies = list(bodies)
    if not 1 <= len(bodies) <= MAX_CONTACT_BODIES:
        raise ValueError(f"{who}: {len(bodies)} contact bodies, expected 1 to {MAX_CONTACT_BODIES}")
    if len({id(b) for b in bodies}) != len(bodies):
        raise ValueError(f"{who}: a contact body appears twice")
    raw = [contact_body_index(world, b, who) for b in bodies]
    if any(b.skeleton is not bodies[0].skeleton for b in bodies):
        raise ValueError(f"{who}: the contact bodies belong to different skeletons")
    return raw


def _check_guesses(state, k, guesses, who):
    """ValueError unless guesses is None or [B, k, 6] ([k, 6] for a 1-D state); nothing touches the device."""
    if guesses is not None:
        want = tuple(state.shape[:-1]) + (k, 6)
        if tuple(guesses.shape) != want:
            raise ValueError(f"{who}: wrench_guesses has shape {tuple(guesses.shape)}, expected {list(want)}")


class MultipleContactInverseDynamicsLayer(torch.autograd.Function):
    """Multiple-contact inverse dynamics of the raw bodies `raw_bodies` (see contact_body_indices); guesses: [B, k, 6] / [k, 6] or None;
    world_inertia as for InverseDynamicsLayer.  Returns (tau, wrenches)."""

    @staticmethod
    def forward(ctx, world, state, next_vel, mass, world_inertia, guesses, raw_bodies):
        dm, sd, vd, wi, need_grad = _prepare(ctx, world, state, next_vel, mass, world_inertia, _WHO_MULTI)
        need_grad = need_grad or ctx.needs_input_grad[5]
        k, cm = len(raw_bodies), dm.cm
        ctx.bodies = [int(cm.body_owner[r]) for r in raw_bodies]
        ctx.points = [cm.body_T[r][:3, 3].astype(float) for r in raw_bodies]  # each body's own origin in its owner's canonical frame
        B, dev = ctx.B, sd.device
        gd = guesses.detach().reshape(B, k, 6).to(device=dev, dtype=sd.dtype).contiguous() if guesses is not None else None
        with torch.cuda.device(dev):
            tau = torch.empty((B, dm.ndof), dtype=sd.dtype, device=dev)
            wrenches = torch.empty((B, k, 6), dtype=sd.dtype, device=dev)
            saved = torch.empty((dm.saved_words, B), dtype=sd.dtype, device=dev) if need_grad else None
            dm.multiple_contact_inverse_dynamics_device(B, ctx.bodies, ctx.points, sd.data_ptr(), vd.data_ptr(), _ptr(gd), tau.data_ptr(),
                                                        wrenches.data_ptr(), _ptr(saved), torch.cuda.current_stream().cuda_stream, ctx.prec,
                                                        wi_ptr=_ptr(wi))
        ctx.guess_grad = ctx.needs_input_grad[5]
        ctx.guess_like = guesses
        if need_grad:
            ctx.save_for_backward(sd, saved, wi, wrenches, gd)
        if ctx.single:
            tau, wrenches = tau[0], wrenches[0]
        return tau.to(device=state.device, dtype=state.dtype), wrenches.to(device=state.device, dtype=state.dtype)

    @staticmethod
    def backward(ctx, grad_tau, grad_wrenches):
        dm, B = ctx.dm, ctx.B
        sd, saved, wi, wrenches, gd = ctx.saved_tensors
        dev, k = sd.device, wrenches.shape[1]
        g = grad_tau.detach().reshape(B, dm.ndof).to(device=dev, dtype=sd.dtype).contiguous()
        gw = grad_wrenches.detach().reshape(B, k, 6).to(device=dev, dtype=sd.dtype).contiguous()
        with torch.cuda.device(dev):
            gs, gn, gi = _backward_buffers(ctx, dev, sd.dtype)
            seed = torch.empty((B, dm.ndof), dtype=sd.dtype, device=dev)
            gg = torch.empty((B, k, 6), dtype=sd.dtype, device=dev) if ctx.guess_grad else None
            dm.multiple_contact_inverse_dynamics_backward_device(B, ctx.bodies, ctx.points, sd.data_ptr(), saved.data_ptr(), wrenches.data_ptr(),
                                                                 _ptr(gd), g.data_ptr(), gw.data_ptr(), seed.data_ptr(), gs.data_ptr(),
                                                                 gn.data_ptr(), torch.cuda.current_stream().cuda_stream, ctx.prec,
                                                                 ginertia_ptr=_ptr(gi), gguess_ptr=_ptr(gg), wi_ptr=_ptr(wi))
        if gg is not None:
            gg = gg.reshape(ctx.guess_like.shape).to(device=ctx.guess_like.device, dtype=ctx.guess_like.dtype)
        return (None,) + _input_grads(ctx, gs, gn, gi) + (gg, None)


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


def multiple_contact_inverse_dynamics(world, state: torch.Tensor, next_vel: torch.Tensor, contact_bodies: Sequence, mass: Optional[torch.Tensor] = None,
                                      wrench_guesses: Optional[torch.Tensor] = None):
    """(tau, wrenches): tau [B, n] (or [n]) and wrenches [B, k, 6] (or [k, 6]) with tau + sum_i J_i^T w_i =
    inverse_dynamics(world, state, next_vel, mass), tau = 0 on the free root, and the w_i as close as possible to `wrench_guesses` (see
    the module docstring).  contact_bodies: 1 to 4 distinct BodyNodes of one mobile skeleton of `world` with a FreeJoint root; each wrench
    is [torque; force] in world axes about the world origin, on that body's own origin.  wrench_guesses: [B, k, 6] ([k, 6] for a 1-D
    state) in the same convention, or None (0).  ValueError for any of these, before any device work.

    The motion fixes only the total wrench.  Without guesses the split is the minimum-norm one, not a prediction of how the load is
    actually shared; with measured per-body wrenches (force plates) as guesses it is the dynamically consistent set closest to them, with
    the matching joint torques.  With one body the result is contact_inverse_dynamics's.  Gradients of both outputs reach state, next_vel,
    mass and the guesses."""
    raw_bodies = contact_body_indices(world, contact_bodies)
    _check_rows(world, state, next_vel, _WHO_MULTI)
    _check_guesses(state, len(raw_bodies), wrench_guesses, _WHO_MULTI)
    if mass is not None and mass.dim() == 2:
        return MultipleContactInverseDynamicsLayer.apply(world, state, next_vel, None, per_world_inertia(world, state, mass, _WHO_MULTI),
                                                         wrench_guesses, raw_bodies)
    return MultipleContactInverseDynamicsLayer.apply(world, state, next_vel, mass, None, wrench_guesses, raw_bodies)


def _contact_jacobians(world, state, next_vel, raw_bodies, mass, guesses, who, guess_blocks):
    """The body of the two contact Jacobian calls: (tau [B, n], wrenches [B, k, 6], T_q, T_qdot, T_next_vel [B, n, n], T_guess [B, n, k, 6],
    W_q, W_qdot, W_next_vel [B, k, 6, n], W_guess [B, k, 6, k, 6]) in the state's dtype and device, the guess blocks None unless
    guess_blocks.  Every argument is checked before any device work."""
    _check_rows(world, state, next_vel, who)
    _check_guesses(state, len(raw_bodies), guesses, who)
    wi = per_world_inertia(world, state, mass, who) if mass is not None and mass.dim() == 2 else None
    dm = set_shared_masses(world, mass, who) if mass is not None and wi is None else device_model_for(world)
    if not torch.cuda.is_available():
        raise RuntimeError(f"nimblephysics_b200.{who[:-2]} needs a CUDA device; there is no CPU fallback")
    single = state.dim() == 1
    s2 = state.detach().reshape(1, -1) if single else state.detach()
    v2 = next_vel.detach().reshape(1, -1) if single else next_vel.detach()
    dev = s2.device if s2.is_cuda else torch.device("cuda", torch.cuda.current_device())
    rdt = torch.float64 if state.dtype == torch.float64 else torch.float32
    sd = s2.to(device=dev, dtype=rdt).contiguous()
    vd = v2.to(device=dev, dtype=rdt).contiguous()
    B, n, k, cm = sd.shape[0], dm.ndof, len(raw_bodies), dm.cm
    gd = guesses.detach().reshape(B, k, 6).to(device=dev, dtype=rdt).contiguous() if guesses is not None else None
    bodies = [int(cm.body_owner[r]) for r in raw_bodies]
    points = [cm.body_T[r][:3, 3].astype(float) for r in raw_bodies]  # each body's own origin in its owner's canonical frame
    with torch.cuda.device(dev):
        tau = torch.empty((B, n), dtype=rdt, device=dev)
        w = torch.empty((B, k, 6), dtype=rdt, device=dev)
        T = [torch.empty((B, n, n), dtype=rdt, device=dev) for _ in range(3)]
        W = [torch.empty((B, k, 6, n), dtype=rdt, device=dev) for _ in range(3)]
        Tg = torch.empty((B, n, k, 6), dtype=rdt, device=dev) if guess_blocks else None
        Wg = torch.empty((B, k, 6, k, 6), dtype=rdt, device=dev) if guess_blocks else None
        if B > 0:  # an empty batch has no rows to hand over (its data pointers may be NULL)
            dm.multiple_contact_inverse_dynamics_jacobians_device(B, bodies, points, sd.data_ptr(), vd.data_ptr(), _ptr(gd), tau.data_ptr(),
                                                                  w.data_ptr(), [_ptr(x) for x in T + [Tg] + W + [Wg]],
                                                                  torch.cuda.current_stream().cuda_stream, FP64 if rdt == torch.float64 else FP32,
                                                                  wi_ptr=_ptr(_word_major_inertia(dm, wi, B, dev)))
    res = [tau, w] + T + [Tg] + W + [Wg]
    if single:
        res = [r[0] if r is not None else None for r in res]
    return tuple(r.to(device=state.device, dtype=state.dtype) if r is not None else None for r in res)


def contact_inverse_dynamics_jacobians(world, state: torch.Tensor, next_vel: torch.Tensor, contact_body, mass: Optional[torch.Tensor] = None):
    """(tau, wrench, dtau_dq, dtau_dqdot, dtau_dnext_vel, dw_dq, dw_dqdot, dw_dnext_vel): (tau [B, n], wrench [B, 6]) =
    contact_inverse_dynamics(world, state, next_vel, contact_body, mass), bit for bit, and their dense Jacobians, dtau_* [B, n, n] and
    dw_* [B, 6, n], J[w, i, j] = d out_i / d x_j (the layout of torch.autograd.functional.jacobian), next_vel held fixed in the q and qdot
    blocks.  From tau + J_c^T wrench = tau_ID and wrench = X*(root -> world) F_r (F_r: tau_ID's six free-root entries):

        dtau_dx + J_c^T dw_dx = dtau_ID/dx   for x = qdot, next_vel  (J_c does not depend on them),   dtau_dnext_vel + J_c^T dw_dnext_vel = M / dt,

    the root's six rows of every dtau block are 0, and the rows of dofs off the chain from the root to contact_body are
    inverse_dynamics_jacobians's.  Row i is contact_inverse_dynamics's vector-Jacobian product with the seed e_i, so the blocks equal
    autograd's Jacobian of that layer up to rounding; free joints follow its conventions (position columns for the six stored coordinates,
    body-twist velocity columns).  Arguments, precision and masses as contact_inverse_dynamics (a 1-D state gives unbatched shapes); the
    outputs carry no autograd history and there is no mass Jacobian.  ValueError before any device work as contact_inverse_dynamics."""
    raw_body = contact_body_index(world, contact_body, _WHO_CIDJ)
    out = _contact_jacobians(world, state, next_vel, [raw_body], mass, None, _WHO_CIDJ, False)
    tau, w, Tq, Tqd, Tn, _, Wq, Wqd, Wn, _ = out
    return (tau, w[..., 0, :], Tq, Tqd, Tn, Wq[..., 0, :, :], Wqd[..., 0, :, :], Wn[..., 0, :, :])


def multiple_contact_inverse_dynamics_jacobians(world, state: torch.Tensor, next_vel: torch.Tensor, contact_bodies: Sequence,
                                                mass: Optional[torch.Tensor] = None, wrench_guesses: Optional[torch.Tensor] = None):
    """(tau, wrenches, dtau_dq, dtau_dqdot, dtau_dnext_vel, dtau_dguess, dw_dq, dw_dqdot, dw_dnext_vel, dw_dguess): (tau [B, n],
    wrenches [B, k, 6]) = multiple_contact_inverse_dynamics(world, state, next_vel, contact_bodies, mass, wrench_guesses), bit for bit,
    and their dense Jacobians in the layout of torch.autograd.functional.jacobian: dtau_dq, dtau_dqdot, dtau_dnext_vel [B, n, n],
    dtau_dguess [B, n, k, 6], dw_dq, dw_dqdot, dw_dnext_vel [B, k, 6, n], dw_dguess [B, k, 6, k, 6]; next_vel held fixed in the q and qdot
    blocks.  With J_i the contact Jacobians:

        dtau_dx + sum_i J_i^T dw_i_dx = dtau_ID/dx   for x = qdot, next_vel ,     sum_i dw_i_dx = the one-body wrench block (x = q, qdot, next_vel),
        sum_i dw_i_dg = 0 ,   dtau_dg = -sum_i J_i^T dw_i_dg ,

    the root's six rows of every dtau block are 0, and rows of dofs off the union of the chains are inverse_dynamics_jacobians's.  With
    one body the guess is not read and both guess blocks are 0.  Row i is the layer's vector-Jacobian product with the seed e_i, so the
    blocks equal autograd's Jacobian of multiple_contact_inverse_dynamics up to rounding; free joints follow its conventions.  Arguments,
    precision and masses as multiple_contact_inverse_dynamics (a 1-D state gives unbatched shapes); the outputs carry no autograd history
    and there is no mass Jacobian.  ValueError before any device work as multiple_contact_inverse_dynamics."""
    raw_bodies = contact_body_indices(world, contact_bodies, _WHO_MCIDJ)
    return _contact_jacobians(world, state, next_vel, raw_bodies, mass, wrench_guesses, _WHO_MCIDJ, True)
