"""``inverse_dynamics_regressor(world, state, next_vel)`` and ``energy_regressor(world, state)``: the joint forces of inverse dynamics and the
kinetic and potential energy as linear maps of every body's inertial parameters, batched (DESIGN.md §6n).

The inertial parameters are the canonical inertia table pi [nb, 10] of ``mass_to_inertia`` / ``InverseDynamicsLayer``'s ``world_inertia``:
one row per canonical body (welded bodies folded into the body they are welded to), (m, h = m c, Ibar) about the canonical body's origin
in the order of ``modelspec.body_inertia_contribution``.  The model's own table is
``mass_to_inertia(world, torch.zeros(1, world.getMassDims()))[0]`` when no body is registered with ``tuneMass`` (the mass vector is then
empty), and ``mass_to_inertia(world, torch.tensor([world.getMasses()]))[0]`` in general.

- Inverse dynamics is affine in pi:  inverse_dynamics(world, state, next_vel, world_inertia = pi) = einsum("bdjk,bjk->bd", Y, pi) + tau_passive,
  tau_passive = K (q - q0 + qdot dt) + D qdot.  Y[b, d, j] is zero unless dof d's joint is at or above body j.
- Kinetic energy: einsum("bjk,bjk->b", Y_T, pi) = 1/2 qdot^T M(pi) qdot, Y_T[j] = 1/2 t(V_j, V_j).
- Potential energy: einsum("bjk,bjk->b", Y_U, pi) + U_spring, Y_U[j] = (-g . p_j, -R_j^T g, 0, ..., 0) (gravity at each body's centre
  of mass), U_spring = 1/2 sum_d k_d (q_d - q0_d)^2 over all dofs.  Summing one skeleton's columns gives energy_and_momentum's T, and its U
  less the springs of other skeletons' dofs.

This is the regressor Y(q, qdot, qdd) of robot identification: least squares over a trajectory, identifiability (the SVD of the stacked
rows) and constrained fits become batched linear algebra.  A mass vector of ``tuneMass`` entries enters through the d(table)/d(mass) map
``modelspec.inertia_param_jacobian``: for INERTIA_MASS entries the table is affine in the mass vector, so Y P^T is its exact regressor.
Momentum about the centre of mass is not linear in pi (the centre of mass depends on the masses) and has no regressor here.

Contacts, joint limits and clipping are ignored and the LCP cache is never touched.  Precision follows the state's dtype.  The outputs
carry no autograd history.  The work is done by libnb2.so (include/nb2.h ``nb2_inverse_dynamics_regressor``, ``nb2_energy_regressor``).
"""
from __future__ import annotations

import torch

from .engine import FP32, FP64, device_model_for
from .inverse_dynamics import _check_fd

_WHO_ID = "inverse_dynamics_regressor()"
_WHO_E = "energy_regressor()"


def _rows(world, state, x, who):
    """(dm, device rows of state and x (or None), precision, single) after the checks, nothing on the device before them"""
    dm = device_model_for(world)
    if not torch.cuda.is_available():
        raise RuntimeError(f"nimblephysics_b200.{who[:-2]} needs a CUDA device; there is no CPU fallback")
    single = state.dim() == 1
    dev = state.device if state.is_cuda else torch.device("cuda", torch.cuda.current_device())
    rdt = torch.float64 if state.dtype == torch.float64 else torch.float32
    rows = [None if t is None else t.detach().reshape(-1, t.shape[-1]).to(device=dev, dtype=rdt).contiguous() for t in (state, x)]
    return dm, rows[0], rows[1], FP64 if rdt == torch.float64 else FP32, single


def _out(res, state, single):
    return tuple((r[0] if single else r).to(device=state.device, dtype=state.dtype) for r in res)


@torch.no_grad()
def inverse_dynamics_regressor(world, state: torch.Tensor, next_vel: torch.Tensor):
    """(Y, tau_passive): Y [B, n, nb, 10] and tau_passive [B, n] ([n, nb, 10] and [n] for a 1-D state) with
    inverse_dynamics(world, state, next_vel, world_inertia = pi) = einsum("bdjk,bjk->bd", Y, pi) + tau_passive for any canonical inertia
    table pi [B, nb, 10] (see the module docstring).  state [B, 2n] / [2n], next_vel [B, n] / [n] as for inverse_dynamics; precision follows
    state.dtype.  Y does not depend on pi.  The outputs carry no autograd history.  ValueError before any device work for a wrong shape
    or a world without dofs."""
    _check_fd(world, state, next_vel, _WHO_ID, "next_vel")
    dm, sd, vd, prec, single = _rows(world, state, next_vel, _WHO_ID)
    B, n, nb = sd.shape[0], dm.ndof, dm.cm.nb
    with torch.cuda.device(sd.device):
        Y = torch.empty((B, n, nb, 10), dtype=sd.dtype, device=sd.device)
        tp = torch.empty((B, n), dtype=sd.dtype, device=sd.device)
        if B > 0:  # an empty batch has no rows to hand over (its data pointers may be NULL)
            dm.inverse_dynamics_regressor_device(B, sd.data_ptr(), vd.data_ptr(), Y.data_ptr(), tp.data_ptr(), torch.cuda.current_stream().cuda_stream,
                                                 prec)
    return _out((Y, tp), state, single)


@torch.no_grad()
def energy_regressor(world, state: torch.Tensor):
    """(Y_T, Y_U, U_spring): Y_T and Y_U [B, nb, 10] and U_spring [B] ([nb, 10], [nb, 10] and [] for a 1-D state) with
    T = einsum("bjk,bjk->b", Y_T, pi) and U = einsum("bjk,bjk->b", Y_U, pi) + U_spring (see the module docstring).  state [B, 2n] / [2n];
    precision follows state.dtype.  The outputs carry no autograd history.  ValueError before any device work for a wrong shape or a world
    without dofs."""
    n = world.getNumDofs()
    if n == 0:
        raise ValueError(f"{_WHO_E}: the world has no degrees of freedom")
    if state.dim() not in (1, 2) or state.shape[-1] != 2 * n:
        raise ValueError(f"{_WHO_E}: state has shape {tuple(state.shape)}, expected [..., {2 * n}] (= getStateSize())")
    dm, sd, _, prec, single = _rows(world, state, None, _WHO_E)
    B, nb = sd.shape[0], dm.cm.nb
    with torch.cuda.device(sd.device):
        YT = torch.empty((B, nb, 10), dtype=sd.dtype, device=sd.device)
        YU = torch.empty((B, nb, 10), dtype=sd.dtype, device=sd.device)
        Us = torch.empty(B, dtype=sd.dtype, device=sd.device)
        if B > 0:
            dm.energy_regressor_device(B, sd.data_ptr(), YT.data_ptr(), YU.data_ptr(), Us.data_ptr(), torch.cuda.current_stream().cuda_stream, prec)
    return _out((YT, YU, Us), state, single)
