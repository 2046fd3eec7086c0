"""``world_jacobian(world, positions, nodes, offsets=None)`` and ``com_jacobian(world, positions, skeleton, mass=None)``: the kinematic
Jacobians of body points and of a skeleton's centre of mass, batched and differentiable.

Columns are in the step's velocity coordinates, in the world's dof order: revolute and prismatic dofs as usual, free joints in their
body twist (S = I6), the convention of ``mass_matrix``, so that e.g. J M^-1 J^T needs no conversion.

- Body point: for a BodyNode e and an offset o_e in the node's own frame, p_e = W_b T_e o_e (b the body the node moves with: welded
  nodes count through the body they are welded to, T_e the node's placement on it).  J_e [6, n] maps qdot to [omega_b ; d/dt p_e], both in
  world axes.  With o_e = 0 this is the velocity of an IKMapping spatial entry (``map_to_vel``).  Columns of dofs that do not move b are
  exactly 0; a static node gets an all-zero block.
- Centre of mass: J_com [3, n] maps qdot to the skeleton's COM velocity (``Skeleton::getCOMLinearVelocity``, the IKMapping COM entry).  It
  depends on the masses.
- Time derivatives: ``world_jacobian_deriv(world, state, nodes, offsets=None)`` and ``com_jacobian_deriv(world, state, skeleton,
  mass=None)`` return Jdot = d/dt J(q(t)) at states [q ; qdot], so that J qddot + Jdot qdot is the acceleration of the point (with the
  body's angular acceleration) or of the COM.  Their gradients reach both halves of the state.

Precision follows the positions' dtype: float64 tensors run the fp64 kernels with fp64 rows, anything else the fp32 ones.  Gradients flow
to ``positions``, ``offsets`` and ``mass`` (1-D: ``setMasses``, shared by the batch, gradient summed; 2-D ``[B, m]``: per world, the
World is left untouched).  The work is done by libnb2.so (include/nb2.h ``nb2_world_jacobian``, ``nb2_com_jacobian``, their
``_deriv`` counterparts and their backwards).
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np
import torch

from .engine import FP32, FP64, device_model_for
from .mass_matrix import _check_positions, _ptr
from .world import WELD
from .timestep import _inertia_grad, _word_major_inertia, per_world_inertia, set_shared_masses, shared_mass_jacobian

_WHO = "world_jacobian()"
_WHO_COM = "com_jacobian()"
MAX_NODES = 32  # NB2_MAX_JACOBIAN_NODES (include/nb2.h)


def _body_index(world):
    index, k = {}, 0
    for sk in world.skeletons:
        for b in sk._ordered_bodies():
            index[id(b)] = k
            k += 1
    return index


def resolve_nodes(world, nodes, who=_WHO):
    """BodyNodes of this world -> (canonical bodies [k] int32, body <- node transforms [k, 12] fp64: R row-major, p), as
    IKMapping.device_handle maps its entries."""
    index = _body_index(world)
    cm = device_model_for(world).cm
    bodies, Ts = [], []
    for node in nodes:
        ri = index[id(node)]
        T = np.asarray(cm.body_T[ri], np.float64)
        bodies.append(int(cm.body_owner[ri]))
        Ts.append(np.concatenate([T[:3, :3].reshape(-1), T[:3, 3]]))
    return np.asarray(bodies, np.int32), np.ascontiguousarray(np.stack(Ts), np.float64)


def _check_skeleton(world, skeleton, who):
    """ValueError for another world's skeleton or one whose root is fixed to the world (as for IKMapping's COM entry: its COM would count
    bodies that no dof moves); nothing touches the device."""
    if not any(s is skeleton for s in world.skeletons):
        raise ValueError(f"{who}: the skeleton does not belong to this world")
    roots = [b for b in skeleton._ordered_bodies() if b.parent_body is None]
    if not roots or roots[0].parent_joint is None or roots[0].parent_joint.jtype == WELD:
        raise ValueError(f"{who}: the skeleton's root is fixed to the world (no moving tree to take the COM of)")
    return roots[0]


def com_root(world, skeleton, who=_WHO_COM):
    """The canonical root body of a skeleton of this world (checked as _check_skeleton)."""
    root = _check_skeleton(world, skeleton, who)
    cm = device_model_for(world).cm
    owner = int(cm.body_owner[_body_index(world)[id(root)]])
    while cm.parent[owner] >= 0:
        owner = int(cm.parent[owner])
    return owner


def _device(p2, who):
    if not torch.cuda.is_available():
        raise RuntimeError(f"nimblephysics_b200.{who[:-2]} needs a CUDA device; there is no CPU fallback")
    return p2.device if p2.is_cuda else torch.device("cuda", torch.cuda.current_device())


class WorldJacobianLayer(torch.autograd.Function):
    """J_e of the given nodes.  Arguments as world_jacobian, the nodes already resolved (resolve_nodes)."""

    @staticmethod
    def forward(ctx, world, positions, bodies, T12, offsets):
        dm = device_model_for(world)
        single = positions.dim() == 1
        p2 = positions.detach().reshape(1, -1) if single else positions.detach()
        dev = _device(p2, _WHO)
        rdt = torch.float64 if positions.dtype == torch.float64 else torch.float32
        pd = p2.to(device=dev, dtype=rdt).contiguous()
        B, n, k = pd.shape[0], dm.ndof, len(bodies)
        od = None if offsets is None else offsets.detach().to(device=dev, dtype=rdt).contiguous()
        prec = FP64 if rdt == torch.float64 else FP32
        with torch.cuda.device(dev):
            out = torch.empty((B, k, 6, n), dtype=rdt, device=dev)
            dm.world_jacobian_device(B, pd.data_ptr(), bodies, T12, _ptr(od), od is not None and od.dim() == 3, out.data_ptr(),
                                     torch.cuda.current_stream().cuda_stream, prec)
        ctx.save_for_backward(pd, od)
        ctx.dm, ctx.bodies, ctx.T12, ctx.prec, ctx.single = dm, bodies, T12, prec, single
        ctx.in_meta = (positions.device, positions.dtype)
        ctx.off_like = offsets
        out = out[0] if single else out
        return out.to(device=positions.device, dtype=positions.dtype)

    @staticmethod
    def backward(ctx, grad):
        pd, od = ctx.saved_tensors
        dm, dev = ctx.dm, pd.device
        B, n, k = pd.shape[0], dm.ndof, len(ctx.bodies)
        g = grad.detach().reshape(B, k, 6, n).to(device=dev, dtype=pd.dtype).contiguous()
        want_off = ctx.off_like is not None and ctx.needs_input_grad[4]
        with torch.cuda.device(dev):
            gp = torch.empty((B, n), dtype=pd.dtype, device=dev)
            go = torch.empty((B, k, 3), dtype=pd.dtype, device=dev) if want_off else None
            dm.world_jacobian_backward_device(B, pd.data_ptr(), ctx.bodies, ctx.T12, _ptr(od), od is not None and od.dim() == 3, g.data_ptr(),
                                              gp.data_ptr(), _ptr(go), torch.cuda.current_stream().cuda_stream, ctx.prec)
        dev0, dt0 = ctx.in_meta
        gp = (gp[0] if ctx.single else gp).to(device=dev0, dtype=dt0)
        if want_off:
            if ctx.off_like.dim() == 2:  # offsets shared by the batch: the worlds' gradients add up
                go = go.sum(dim=0)
            go = go.to(device=ctx.off_like.device, dtype=ctx.off_like.dtype)
        return None, gp, None, None, go


class ComJacobianLayer(torch.autograd.Function):
    """J_com of the tree rooted at canonical body `root`; mass / world_inertia as MassMatrixLayer."""

    @staticmethod
    def forward(ctx, world, positions, root, mass, world_inertia=None):
        dm = set_shared_masses(world, mass, _WHO_COM) if mass is not None else device_model_for(world)
        single = positions.dim() == 1
        p2 = positions.detach().reshape(1, -1) if single else positions.detach()
        dev = _device(p2, _WHO_COM)
        rdt = torch.float64 if positions.dtype == torch.float64 else torch.float32
        pd = p2.to(device=dev, dtype=rdt).contiguous()
        B, n = pd.shape[0], dm.ndof
        wi = _word_major_inertia(dm, world_inertia, B, dev)
        prec = FP64 if rdt == torch.float64 else FP32
        with torch.cuda.device(dev):
            out = torch.empty((B, 3, n), dtype=rdt, device=dev)
            dm.com_jacobian_device(B, pd.data_ptr(), root, out.data_ptr(), torch.cuda.current_stream().cuda_stream, prec, wi_ptr=_ptr(wi))
        ctx.save_for_backward(pd, wi)
        ctx.dm, ctx.root, ctx.prec, ctx.single = dm, root, prec, single
        ctx.wi_grad = world_inertia is not None and ctx.needs_input_grad[4]
        ctx.wi_like = world_inertia
        ctx.mass_grad = mass is not None and ctx.needs_input_grad[3]
        if ctx.mass_grad:
            ctx.mass_P = shared_mass_jacobian(world, dm, dev)
            ctx.mass_like = mass
        ctx.in_meta = (positions.device, positions.dtype)
        out = out[0] if single else out
        return out.to(device=positions.device, dtype=positions.dtype)

    @staticmethod
    def backward(ctx, grad):
        pd, wi = ctx.saved_tensors
        dm, dev = ctx.dm, pd.device
        B, n = pd.shape[0], dm.ndof
        g = grad.detach().reshape(B, 3, n).to(device=dev, dtype=pd.dtype).contiguous()
        with torch.cuda.device(dev):
            gp = torch.empty((B, n), dtype=pd.dtype, device=dev)
            gi = torch.empty((10 * dm.cm.nb, B), dtype=torch.float64, device=dev) if (ctx.mass_grad or ctx.wi_grad) else None
            dm.com_jacobian_backward_device(B, pd.data_ptr(), ctx.root, g.data_ptr(), gp.data_ptr(), torch.cuda.current_stream().cuda_stream,
                                            ctx.prec, ginertia_ptr=_ptr(gi), wi_ptr=_ptr(wi))
        gm = None
        if ctx.mass_grad:  # one mass vector shared by the batch: the worlds' gradients add up
            gm = (ctx.mass_P @ gi.sum(dim=1)).to(device=ctx.mass_like.device, dtype=ctx.mass_like.dtype)
        gw = _inertia_grad(gi, ctx.wi_like) if ctx.wi_grad else None
        dev0, dt0 = ctx.in_meta
        gp = (gp[0] if ctx.single else gp).to(device=dev0, dtype=dt0)
        return None, gp, None, gm, gw


def world_jacobian(world, positions: torch.Tensor, nodes: Sequence, offsets: Optional[torch.Tensor] = None) -> torch.Tensor:
    """J_e [B, k, 6, n] of the k BodyNodes `nodes` at positions [B, n] ([k, 6, n] for [n]); see the module docstring.  offsets: None (the
    nodes' origins), [k, 3] (shared by the batch, the gradient sums over it) or [B, k, 3] (one set per world), in each node's own frame.
    ValueError before any device work for a wrong shape, an empty node list, more than MAX_NODES nodes, a node of another world or a
    world without dofs."""
    _check_positions(world, positions, _WHO)
    nodes = list(nodes)
    if not nodes or len(nodes) > MAX_NODES:
        raise ValueError(f"{_WHO}: {len(nodes)} nodes given, expected 1 to {MAX_NODES}")
    index = _body_index(world)
    for node in nodes:
        if id(node) not in index:
            raise ValueError(f"{_WHO}: body node {getattr(node, 'name', node)!r} does not belong to this world")
    k = len(nodes)
    if offsets is not None:
        ok = (offsets.dim() == 2 and tuple(offsets.shape) == (k, 3)) or (
            offsets.dim() == 3 and positions.dim() == 2 and tuple(offsets.shape) == (positions.shape[0], k, 3))
        if not ok:
            want = f"[{k}, 3]" + (f" or [{positions.shape[0]}, {k}, 3]" if positions.dim() == 2 else "")
            raise ValueError(f"{_WHO}: offsets has shape {tuple(offsets.shape)}, expected {want}")
    bodies, T12 = resolve_nodes(world, nodes, _WHO)
    return WorldJacobianLayer.apply(world, positions, bodies, T12, offsets)


def com_jacobian(world, positions: torch.Tensor, skeleton, mass: Optional[torch.Tensor] = None) -> torch.Tensor:
    """J_com [B, 3, n] of `skeleton` at positions [B, n] ([3, n] for [n]); see the module docstring.  mass as for mass_matrix: None, a 1-D
    vector [getMassDims()] (world.setMasses(mass) first, shared by the batch) or [B, getMassDims()] (per world, the World is not
    modified).  ValueError before any device work for a wrong shape, a skeleton of another world, a skeleton whose root is fixed to the
    world, a mass of the wrong size or a world without dofs."""
    _check_positions(world, positions, _WHO_COM)
    _check_skeleton(world, skeleton, _WHO_COM)
    m = world.getMassDims()
    if mass is not None:
        if mass.dim() == 2 and positions.dim() != 2:
            raise ValueError(f"{_WHO_COM}: a [B, getMassDims()] mass needs [B, n] positions")
        want = (m,) if mass.dim() == 1 else (positions.shape[0], m)
        if mass.dim() not in (1, 2) or tuple(mass.shape) != want:
            raise ValueError(f"{_WHO_COM}: mass has shape {tuple(mass.shape)}, expected [{m}] or [B, {m}] (= getMassDims())")
    root = com_root(world, skeleton, _WHO_COM)
    if mass is not None and mass.dim() == 2:
        return ComJacobianLayer.apply(world, positions, root, None, per_world_inertia(world, positions, mass, _WHO_COM))
    return ComJacobianLayer.apply(world, positions, root, mass)


_WHO_D = "world_jacobian_deriv()"
_WHO_COM_D = "com_jacobian_deriv()"


def _check_state(world, state, who):
    """ValueError unless the world has dofs and state is [2n] / [B, 2n] = [q ; qdot]; nothing touches the device."""
    n = world.getNumDofs()
    if n == 0:
        raise ValueError(f"{who}: the world has no degrees of freedom")
    if state.dim() not in (1, 2) or state.shape[-1] != 2 * n or (state.dim() == 2 and state.shape[0] == 0):
        raise ValueError(f"{who}: state has shape {tuple(state.shape)}, expected [{2 * n}] or [B, {2 * n}] (= getStateSize())")


class WorldJacobianDerivLayer(torch.autograd.Function):
    """Jdot_e of the given nodes at states [q ; qdot].  Arguments as world_jacobian_deriv, the nodes already resolved (resolve_nodes)."""

    @staticmethod
    def forward(ctx, world, state, bodies, T12, offsets):
        dm = device_model_for(world)
        single = state.dim() == 1
        s2 = state.detach().reshape(1, -1) if single else state.detach()
        dev = _device(s2, _WHO_D)
        rdt = torch.float64 if state.dtype == torch.float64 else torch.float32
        sd = s2.to(device=dev, dtype=rdt).contiguous()
        B, n, k = sd.shape[0], dm.ndof, len(bodies)
        od = None if offsets is None else offsets.detach().to(device=dev, dtype=rdt).contiguous()
        prec = FP64 if rdt == torch.float64 else FP32
        with torch.cuda.device(dev):
            out = torch.empty((B, k, 6, n), dtype=rdt, device=dev)
            dm.world_jacobian_deriv_device(B, sd.data_ptr(), bodies, T12, _ptr(od), od is not None and od.dim() == 3, out.data_ptr(),
                                           torch.cuda.current_stream().cuda_stream, prec)
        ctx.save_for_backward(sd, od)
        ctx.dm, ctx.bodies, ctx.T12, ctx.prec, ctx.single = dm, bodies, T12, prec, single
        ctx.in_meta = (state.device, state.dtype)
        ctx.off_like = offsets
        out = out[0] if single else out
        return out.to(device=state.device, dtype=state.dtype)

    @staticmethod
    def backward(ctx, grad):
        sd, od = ctx.saved_tensors
        dm, dev = ctx.dm, sd.device
        B, n, k = sd.shape[0], dm.ndof, len(ctx.bodies)
        g = grad.detach().reshape(B, k, 6, n).to(device=dev, dtype=sd.dtype).contiguous()
        want_off = ctx.off_like is not None and ctx.needs_input_grad[4]
        with torch.cuda.device(dev):
            gs = torch.empty((B, 2 * n), dtype=sd.dtype, device=dev)
            go = torch.empty((B, k, 3), dtype=sd.dtype, device=dev) if want_off else None
            dm.world_jacobian_deriv_backward_device(B, sd.data_ptr(), ctx.bodies, ctx.T12, _ptr(od), od is not None and od.dim() == 3, g.data_ptr(),
                                                    gs.data_ptr(), _ptr(go), torch.cuda.current_stream().cuda_stream, ctx.prec)
        dev0, dt0 = ctx.in_meta
        gs = (gs[0] if ctx.single else gs).to(device=dev0, dtype=dt0)
        if want_off:
            if ctx.off_like.dim() == 2:  # offsets shared by the batch: the worlds' gradients add up
                go = go.sum(dim=0)
            go = go.to(device=ctx.off_like.device, dtype=ctx.off_like.dtype)
        return None, gs, None, None, go


class ComJacobianDerivLayer(torch.autograd.Function):
    """Jdot_com of the tree rooted at canonical body `root` at states [q ; qdot]; mass / world_inertia as ComJacobianLayer."""

    @staticmethod
    def forward(ctx, world, state, root, mass, world_inertia=None):
        dm = set_shared_masses(world, mass, _WHO_COM_D) if mass is not None else device_model_for(world)
        single = state.dim() == 1
        s2 = state.detach().reshape(1, -1) if single else state.detach()
        dev = _device(s2, _WHO_COM_D)
        rdt = torch.float64 if state.dtype == torch.float64 else torch.float32
        sd = s2.to(device=dev, dtype=rdt).contiguous()
        B, n = sd.shape[0], dm.ndof
        wi = _word_major_inertia(dm, world_inertia, B, dev)
        prec = FP64 if rdt == torch.float64 else FP32
        with torch.cuda.device(dev):
            out = torch.empty((B, 3, n), dtype=rdt, device=dev)
            dm.com_jacobian_deriv_device(B, sd.data_ptr(), root, out.data_ptr(), torch.cuda.current_stream().cuda_stream, prec, wi_ptr=_ptr(wi))
        ctx.save_for_backward(sd, wi)
        ctx.dm, ctx.root, ctx.prec, ctx.single = dm, root, prec, single
        ctx.wi_grad = world_inertia is not None and ctx.needs_input_grad[4]
        ctx.wi_like = world_inertia
        ctx.mass_grad = mass is not None and ctx.needs_input_grad[3]
        if ctx.mass_grad:
            ctx.mass_P = shared_mass_jacobian(world, dm, dev)
            ctx.mass_like = mass
        ctx.in_meta = (state.device, state.dtype)
        out = out[0] if single else out
        return out.to(device=state.device, dtype=state.dtype)

    @staticmethod
    def backward(ctx, grad):
        sd, wi = ctx.saved_tensors
        dm, dev = ctx.dm, sd.device
        B, n = sd.shape[0], dm.ndof
        g = grad.detach().reshape(B, 3, n).to(device=dev, dtype=sd.dtype).contiguous()
        with torch.cuda.device(dev):
            gs = torch.empty((B, 2 * n), dtype=sd.dtype, device=dev)
            gi = torch.empty((10 * dm.cm.nb, B), dtype=torch.float64, device=dev) if (ctx.mass_grad or ctx.wi_grad) else None
            dm.com_jacobian_deriv_backward_device(B, sd.data_ptr(), ctx.root, g.data_ptr(), gs.data_ptr(), torch.cuda.current_stream().cuda_stream,
                                                  ctx.prec, ginertia_ptr=_ptr(gi), wi_ptr=_ptr(wi))
        gm = None
        if ctx.mass_grad:  # one mass vector shared by the batch: the worlds' gradients add up
            gm = (ctx.mass_P @ gi.sum(dim=1)).to(device=ctx.mass_like.device, dtype=ctx.mass_like.dtype)
        gw = _inertia_grad(gi, ctx.wi_like) if ctx.wi_grad else None
        dev0, dt0 = ctx.in_meta
        gs = (gs[0] if ctx.single else gs).to(device=dev0, dtype=dt0)
        return None, gs, None, gm, gw


def world_jacobian_deriv(world, state: torch.Tensor, nodes: Sequence, offsets: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Jdot_e [B, k, 6, n] of the k BodyNodes `nodes` at states [B, 2n] = [q ; qdot] ([k, 6, n] for [2n]): d/dt J_e(q(t)) along a motion
    through q with velocity qdot (free joints: Rdot = R [omega]x, pdot = R v, the step's position update), so that the acceleration
    [alpha_b ; d2/dt2 p_e] is J_e qddot + Jdot_e qdot.  Linear in qdot; columns, nodes and offsets as world_jacobian.  Gradients flow to
    the state (both halves) and the offsets.  ValueError before any device work as world_jacobian, for a state that is not [2n] / [B, 2n]."""
    _check_state(world, state, _WHO_D)
    nodes = list(nodes)
    if not nodes or len(nodes) > MAX_NODES:
        raise ValueError(f"{_WHO_D}: {len(nodes)} nodes given, expected 1 to {MAX_NODES}")
    index = _body_index(world)
    for node in nodes:
        if id(node) not in index:
            raise ValueError(f"{_WHO_D}: body node {getattr(node, 'name', node)!r} does not belong to this world")
    k = len(nodes)
    if offsets is not None:
        ok = (offsets.dim() == 2 and tuple(offsets.shape) == (k, 3)) or (
            offsets.dim() == 3 and state.dim() == 2 and tuple(offsets.shape) == (state.shape[0], k, 3))
        if not ok:
            want = f"[{k}, 3]" + (f" or [{state.shape[0]}, {k}, 3]" if state.dim() == 2 else "")
            raise ValueError(f"{_WHO_D}: offsets has shape {tuple(offsets.shape)}, expected {want}")
    bodies, T12 = resolve_nodes(world, nodes, _WHO_D)
    return WorldJacobianDerivLayer.apply(world, state, bodies, T12, offsets)


def com_jacobian_deriv(world, state: torch.Tensor, skeleton, mass: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Jdot_com [B, 3, n] of `skeleton` at states [B, 2n] = [q ; qdot] ([3, n] for [2n]), so that the COM's acceleration is
    J_com qddot + Jdot_com qdot; mass and the ValueErrors as com_jacobian, for a state that is not [2n] / [B, 2n]."""
    _check_state(world, state, _WHO_COM_D)
    _check_skeleton(world, skeleton, _WHO_COM_D)
    m = world.getMassDims()
    if mass is not None:
        if mass.dim() == 2 and state.dim() != 2:
            raise ValueError(f"{_WHO_COM_D}: a [B, getMassDims()] mass needs [B, 2n] states")
        want = (m,) if mass.dim() == 1 else (state.shape[0], m)
        if mass.dim() not in (1, 2) or tuple(mass.shape) != want:
            raise ValueError(f"{_WHO_COM_D}: mass has shape {tuple(mass.shape)}, expected [{m}] or [B, {m}] (= getMassDims())")
    root = com_root(world, skeleton, _WHO_COM_D)
    if mass is not None and mass.dim() == 2:
        return ComJacobianDerivLayer.apply(world, state, root, None, per_world_inertia(world, state, mass, _WHO_COM_D))
    return ComJacobianDerivLayer.apply(world, state, root, mass)


def _current(world, who):
    q = torch.tensor(np.asarray(world.getPositions(), dtype=np.float64), dtype=torch.float64)
    if not torch.cuda.is_available():
        raise RuntimeError(f"nimblephysics_b200.{who} needs a CUDA device; there is no CPU fallback")
    return q.to("cuda")


def _single_world_point(world, node, offset, who):
    """[6, n] numpy fp64 of one node at the world's current positions (fp64 kernels, B = 1)."""
    q = _current(world, who)
    off = None if offset is None else torch.as_tensor(np.asarray(offset, np.float64).reshape(1, 3), dtype=torch.float64, device=q.device)
    with torch.no_grad():
        return world_jacobian(world, q, [node], off)[0].cpu().numpy()


def _single_world_com(world, skeleton, who):
    q = _current(world, who)
    with torch.no_grad():
        return com_jacobian(world, q, skeleton).cpu().numpy()


def _current_state(world, who):
    s = torch.tensor(np.concatenate([world.getPositions(), world.getVelocities()]).astype(np.float64), dtype=torch.float64)
    if not torch.cuda.is_available():
        raise RuntimeError(f"nimblephysics_b200.{who} needs a CUDA device; there is no CPU fallback")
    return s.to("cuda")


def _single_world_point_deriv(world, node, offset, who):
    """[6, n] numpy fp64 Jdot of one node at the world's current state (fp64 kernels, B = 1)."""
    s = _current_state(world, who)
    off = None if offset is None else torch.as_tensor(np.asarray(offset, np.float64).reshape(1, 3), dtype=torch.float64, device=s.device)
    with torch.no_grad():
        return world_jacobian_deriv(world, s, [node], off)[0].cpu().numpy()


def _single_world_com_deriv(world, skeleton, who):
    s = _current_state(world, who)
    with torch.no_grad():
        return com_jacobian_deriv(world, s, skeleton).cpu().numpy()
