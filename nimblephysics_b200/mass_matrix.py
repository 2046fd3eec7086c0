"""``mass_matrix(world, positions, mass=None)`` and ``inverse_mass_matrix(world, positions, mass=None)``: the joint-space mass matrix M(q)
and its inverse, batched and differentiable.

M is the matrix the step inverts, in the step's velocity coordinates: revolute and prismatic dofs as usual, free joints in their body
twist (S = I6).  In exact arithmetic

    inverse_dynamics(q, qdot, v') - inverse_dynamics(q, qdot, qdot) = M(q) (v' - qdot) / dt ,
    qddot of the contact-free step = M(q)^-1 (tau - inverse_dynamics(q, qdot, qdot)) .

A world's M is block-diagonal over its skeletons, in the world's dof order; welded bodies count through the body they are welded to.
M does not depend on a free root's pose (that root's position entries get a gradient of exactly 0).  Contacts, joint limits, springs
and damping are not part of M, and a world's LCP cache is never touched.  Both outputs are exactly symmetric.  The reference's
``getCoriolisAndGravityForces`` is ``inverse_dynamics(q, qdot, qdot)`` minus the spring and damping forces.

Precision follows the positions' dtype: float64 tensors run the fp64 kernels with fp64 rows, anything else the fp32 ones.  Gradients
flow to ``positions`` and ``mass`` (1-D: ``setMasses``, shared by the batch, gradient summed; 2-D ``[B, m]``: per world, the World is left
untouched).  The work is done by libnb2.so (include/nb2.h ``nb2_mass_matrix``, ``nb2_inverse_mass_matrix`` and their backwards): M by the
composite-rigid-body algorithm, M^-1 by the step's articulated inertias with one unit-force sweep pair per column.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from .engine import FP32, FP64, device_model_for
from .timestep import _inertia_grad, _word_major_inertia, per_world_inertia, set_shared_masses, shared_mass_jacobian

_WHO = "mass_matrix()"
_WHO_INV = "inverse_mass_matrix()"


def _check_positions(world, positions, who):
    """ValueError unless the world has dofs and positions is [n] / [B, n] (n = getNumDofs()); nothing touches the device."""
    n = world.getNumDofs()
    if n == 0:
        raise ValueError(f"{who}: the world has no degrees of freedom")
    if positions.dim() not in (1, 2) or positions.shape[-1] != n or (positions.dim() == 2 and positions.shape[0] == 0):
        raise ValueError(f"{who}: positions has shape {tuple(positions.shape)}, expected [{n}] or [B, {n}] (n = getNumDofs())")


def _ptr(t):
    return t.data_ptr() if t is not None else None


class _MassMatrixBase(torch.autograd.Function):
    WHO = _WHO

    @staticmethod
    def _prepare(ctx, world, positions, mass, world_inertia, who):
        if mass is not None and world_inertia is not None:
            raise ValueError(f"{who}: give either a mass vector or a per-world inertia table, not both")
        _check_positions(world, positions, who)
        dm = set_shared_masses(world, mass, who) if mass is not None else device_model_for(world)
        single = positions.dim() == 1
        p2 = positions.detach().reshape(1, -1) if single else positions.detach()
        if not torch.cuda.is_available():
            raise RuntimeError(f"nimblephysics_b200.{who[:-2]} needs a CUDA device; there is no CPU fallback")
        dev = p2.device if p2.is_cuda else torch.device("cuda", torch.cuda.current_device())
        rdt = torch.float64 if positions.dtype == torch.float64 else torch.float32
        pd = p2.to(device=dev, dtype=rdt).contiguous()
        B = pd.shape[0]
        if world_inertia is not None and (single or tuple(world_inertia.shape) != (B, dm.cm.nb, 10)):
            raise ValueError(f"{who}: per-world inertia has shape {tuple(world_inertia.shape)}, expected [{B}, {dm.cm.nb}, 10] with 2-D positions")
        wi = _word_major_inertia(dm, world_inertia, B, dev)
        ctx.wi_grad = world_inertia is not None and ctx.needs_input_grad[3]
        ctx.wi_like = world_inertia
        ctx.mass_grad = mass is not None and ctx.needs_input_grad[2]
        if ctx.mass_grad:
            ctx.mass_P = shared_mass_jacobian(world, dm, dev)
            ctx.mass_like = mass
        ctx.dm, ctx.B, ctx.prec, ctx.single = dm, B, FP64 if rdt == torch.float64 else FP32, single
        ctx.in_meta = (positions.device, positions.dtype)
        return dm, pd, wi

    @staticmethod
    def _grads(ctx, gp, gi):
        gm = None
        if ctx.mass_grad:  # one mass vector shared by the batch: the worlds' gradients add up
            gm = (ctx.mass_P @ gi.sum(dim=1)).to(device=ctx.mass_like.device, dtype=ctx.mass_like.dtype)
        gw = _inertia_grad(gi, ctx.wi_like) if ctx.wi_grad else None
        dev, dt = ctx.in_meta
        if ctx.single:
            gp = gp[0]
        return None, gp.to(device=dev, dtype=dt), gm, gw


class MassMatrixLayer(_MassMatrixBase):
    """M(q).  world_inertia (optional): per-world canonical inertia [B, nb, 10] (modelspec.mass_to_inertia), exclusive with the 1-D `mass`."""

    @staticmethod
    def forward(ctx, world, positions, mass, world_inertia=None):
        dm, pd, wi = _MassMatrixBase._prepare(ctx, world, positions, mass, world_inertia, _WHO)
        n, dev = dm.ndof, pd.device
        with torch.cuda.device(dev):
            out = torch.empty((ctx.B, n, n), dtype=pd.dtype, device=dev)
            dm.mass_matrix_device(ctx.B, pd.data_ptr(), out.data_ptr(), torch.cuda.current_stream().cuda_stream, ctx.prec, wi_ptr=_ptr(wi))
        ctx.save_for_backward(pd, wi)
        out = out[0] if ctx.single else out
        return out.to(device=positions.device, dtype=positions.dtype)

    @staticmethod
    def backward(ctx, grad):
        dm, B = ctx.dm, ctx.B
        pd, wi = ctx.saved_tensors
        dev, n = pd.device, dm.ndof
        g = grad.detach().reshape(B, n, n).to(device=dev, dtype=pd.dtype).contiguous()
        with torch.cuda.device(dev):
            gp = torch.empty((B, n), dtype=pd.dtype, device=dev)
            gi = torch.empty((10 * dm.cm.nb, B), dtype=torch.float64, device=dev) if (ctx.mass_grad or ctx.wi_grad) else None
            dm.mass_matrix_backward_device(B, pd.data_ptr(), g.data_ptr(), gp.data_ptr(), torch.cuda.current_stream().cuda_stream, ctx.prec,
                                           ginertia_ptr=_ptr(gi), wi_ptr=_ptr(wi))
        return _MassMatrixBase._grads(ctx, gp, gi)


class InverseMassMatrixLayer(_MassMatrixBase):
    """M(q)^-1; world_inertia as for MassMatrixLayer.  The backward uses the forward's output, dL/dM = -M^-1 Gs M^-1 (Gs the symmetrised
    incoming gradient), and then the M backward, all in one kernel."""

    @staticmethod
    def forward(ctx, world, positions, mass, world_inertia=None):
        dm, pd, wi = _MassMatrixBase._prepare(ctx, world, positions, mass, world_inertia, _WHO_INV)
        n, dev = dm.ndof, pd.device
        with torch.cuda.device(dev):
            out = torch.empty((ctx.B, n, n), dtype=pd.dtype, device=dev)
            dm.inverse_mass_matrix_device(ctx.B, pd.data_ptr(), out.data_ptr(), torch.cuda.current_stream().cuda_stream, ctx.prec,
                                          wi_ptr=_ptr(wi))
        ctx.save_for_backward(pd, wi, out)
        res = out[0] if ctx.single else out
        return res.to(device=positions.device, dtype=positions.dtype)

    @staticmethod
    def backward(ctx, grad):
        dm, B = ctx.dm, ctx.B
        pd, wi, minv = ctx.saved_tensors
        dev, n = pd.device, dm.ndof
        g = grad.detach().reshape(B, n, n).to(device=dev, dtype=pd.dtype).contiguous()
        with torch.cuda.device(dev):
            gp = torch.empty((B, n), dtype=pd.dtype, device=dev)
            ws = torch.empty((B, n, n), dtype=pd.dtype, device=dev)
            gi = torch.empty((10 * dm.cm.nb, B), dtype=torch.float64, device=dev) if (ctx.mass_grad or ctx.wi_grad) else None
            dm.inverse_mass_matrix_backward_device(B, pd.data_ptr(), minv.data_ptr(), g.data_ptr(), ws.data_ptr(), gp.data_ptr(),
                                                   torch.cuda.current_stream().cuda_stream, ctx.prec, ginertia_ptr=_ptr(gi), wi_ptr=_ptr(wi))
        return _MassMatrixBase._grads(ctx, gp, gi)


def _apply(layer, who, world, positions, mass):
    _check_positions(world, positions, who)
    if mass is not None and mass.dim() == 2:
        if positions.dim() != 2:
            raise ValueError(f"{who}: a [B, getMassDims()] mass needs [B, n] positions")
        # per_world_inertia checks the mass against a batch of rows; it reads only the batch size
        return layer.apply(world, positions, None, per_world_inertia(world, positions, mass, who))
    return layer.apply(world, positions, mass)


def mass_matrix(world, positions: torch.Tensor, mass: Optional[torch.Tensor] = None) -> torch.Tensor:
    """M(q) [B, n, n] for positions [B, n] ([n, n] for [n]); see the module docstring.  mass: None, a 1-D vector [getMassDims()]
    (world.setMasses(mass) first, shared by the batch, the gradient sums over the batch) or [B, getMassDims()] (world w uses mass[w], the
    World is not modified).  ValueError before any device work for a wrong shape, a world without dofs or a mass of the wrong size."""
    return _apply(MassMatrixLayer, _WHO, world, positions, mass)


def inverse_mass_matrix(world, positions: torch.Tensor, mass: Optional[torch.Tensor] = None) -> torch.Tensor:
    """M(q)^-1, with the shapes and arguments of mass_matrix."""
    return _apply(InverseMassMatrixLayer, _WHO_INV, world, positions, mass)


def _single_world(world, who, inverse):
    """The fp64 matrix of the world at its current positions (B = 1, fp64 kernels), as a numpy array."""
    q = torch.tensor(np.asarray(world.getPositions(), dtype=np.float64), dtype=torch.float64)
    if not torch.cuda.is_available():
        raise RuntimeError(f"nimblephysics_b200.{who} needs a CUDA device; there is no CPU fallback")
    q = q.to("cuda")
    with torch.no_grad():
        out = (inverse_mass_matrix if inverse else mass_matrix)(world, q)
    return out.cpu().numpy()
