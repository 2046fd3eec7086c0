"""nimblephysics_b200 — H100-native batched differentiable timestep behind the
Nimble ``timestep(world, state, action)`` surface.  See DESIGN.md."""
from . import world as _world
from .world import (World, Skeleton, BodyNode, Joint, Isometry3, BoxShape, SphereShape, CapsuleShape)
from .loader import loadWorld, load_skeleton
from .modelspec import RawModel, CanonModel, flatten_world, compile_model, mass_to_inertia
from .timestep import timestep, TimestepLayer, contact_cache, reset_contact_cache, check_contact_status
from .inverse_dynamics import (inverse_dynamics, InverseDynamicsLayer, contact_inverse_dynamics, ContactInverseDynamicsLayer,
                               multiple_contact_inverse_dynamics, MultipleContactInverseDynamicsLayer, forward_dynamics,
                               ForwardDynamicsLayer, inverse_dynamics_jacobians, forward_dynamics_jacobians,
                               contact_inverse_dynamics_jacobians, multiple_contact_inverse_dynamics_jacobians)
from .mass_matrix import mass_matrix, inverse_mass_matrix, MassMatrixLayer, InverseMassMatrixLayer
from .world_jacobian import world_jacobian, com_jacobian, WorldJacobianLayer, ComJacobianLayer
from .world_jacobian import world_jacobian_deriv, com_jacobian_deriv, WorldJacobianDerivLayer, ComJacobianDerivLayer
from .energy import energy_and_momentum, EnergyMomentumLayer
from .regressor import inverse_dynamics_regressor, energy_regressor
from .constrained_dynamics import constrained_forward_dynamics, constrained_forward_dynamics_jacobians, ConstrainedForwardDynamicsLayer
from .constrained_dynamics import impulse_dynamics, impulse_dynamics_jacobians, ImpulseDynamicsLayer
from .engine import DeviceModel, device_model_for
from .rollout import rollout, rollout_fused, rollout_tape_bytes, multishot_rollout, shard_range, shard_batch, allreduce_sum_, sharded_trajectory_loss

__all__ = ["World", "Skeleton", "BodyNode", "Joint", "Isometry3", "BoxShape", "SphereShape", "CapsuleShape",
           "loadWorld", "load_skeleton", "timestep", "TimestepLayer", "inverse_dynamics", "InverseDynamicsLayer", "contact_inverse_dynamics", "ContactInverseDynamicsLayer",
           "multiple_contact_inverse_dynamics", "MultipleContactInverseDynamicsLayer", "forward_dynamics", "ForwardDynamicsLayer",
           "inverse_dynamics_jacobians", "forward_dynamics_jacobians", "contact_inverse_dynamics_jacobians",
           "multiple_contact_inverse_dynamics_jacobians", "mass_matrix", "inverse_mass_matrix", "MassMatrixLayer", "InverseMassMatrixLayer",
           "world_jacobian", "com_jacobian", "WorldJacobianLayer", "ComJacobianLayer",
           "world_jacobian_deriv", "com_jacobian_deriv", "WorldJacobianDerivLayer", "ComJacobianDerivLayer", "energy_and_momentum", "EnergyMomentumLayer", "inverse_dynamics_regressor", "energy_regressor", "constrained_forward_dynamics", "constrained_forward_dynamics_jacobians", "ConstrainedForwardDynamicsLayer", "impulse_dynamics", "impulse_dynamics_jacobians", "ImpulseDynamicsLayer", "rollout", "rollout_fused", "DeviceModel", "device_model_for", "RawModel", "CanonModel", "flatten_world", "compile_model", "mass_to_inertia"]
from .lcp import solve_boxed_lcp_batch
from .jacobians import step_jacobians, state_jacobian, action_jacobian
from .mapping import IKMapping, map_to_pos, map_to_vel
