"""nimblephysics_b200 — H100-native batched differentiable timestep behind the
Nimble ``timestep(world, state, action)`` surface.  See DESIGN.md."""
from . import world as _world
from .world import (World, Skeleton, BodyNode, Joint, Isometry3, BoxShape, SphereShape, CapsuleShape)
from .loader import loadWorld, load_skeleton
from .modelspec import RawModel, CanonModel, flatten_world, compile_model
from .timestep import timestep, TimestepLayer, contact_cache, reset_contact_cache, check_contact_status
from .engine import DeviceModel, device_model_for
from .rollout import rollout, rollout_fused, rollout_tape_bytes, multishot_rollout, shard_range, shard_batch, allreduce_sum_, sharded_trajectory_loss

__all__ = ["World", "Skeleton", "BodyNode", "Joint", "Isometry3", "BoxShape", "SphereShape", "CapsuleShape",
           "loadWorld", "load_skeleton", "timestep", "TimestepLayer", "rollout", "rollout_fused", "DeviceModel", "device_model_for", "RawModel", "CanonModel", "flatten_world", "compile_model"]
from .lcp import solve_boxed_lcp_batch
from .jacobians import step_jacobians, state_jacobian, action_jacobian
from .mapping import IKMapping, map_to_pos, map_to_vel
