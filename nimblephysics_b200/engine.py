"""Device-side handle of a World: builds the canonical model and owns the nb2_model created through the C ABI."""
from __future__ import annotations

import ctypes

import numpy as np

from . import _cabi
from .modelspec import CanonModel, RawModel, compile_model, flatten_world

FP32, FP64 = 0, 1


class DeviceModel:
    """nb2_model wrapper (include/nb2.h).  One per (World version)."""

    def __init__(self, cm: CanonModel, schedules=()):
        """cm: the canonical model (its own schedule, normally lanes=1, is what the contact kernels sweep with);
        schedules: further compilations of the SAME RawModel with other lane counts (modelspec.compile_model(raw, lanes=K));
        the library picks one per launch from the batch size (include/nb2.h nb2_model_add_schedule)."""
        self.cm = cm
        self.ndof = cm.ndof
        self.na = len(cm.action_map)
        L = _cabi.lib()
        self._desc, self._keep = _cabi.make_desc(cm, with_contacts=len(cm.shape_body) > 0 or len(getattr(cm, "limit_bodies", [])) > 0)
        h = ctypes.c_void_p()
        _cabi.check(L.nb2_model_create(ctypes.byref(self._desc), ctypes.byref(h)))
        self.handle = h
        self.saved_words = L.nb2_saved_words_per_world(h)
        self.has_contacts = bool(L.nb2_model_has_contacts(h))
        self.schedules = [cm]
        for c in schedules:
            d, keep = _cabi.make_desc(c, with_contacts=False)
            _cabi.check(L.nb2_model_add_schedule(h, ctypes.byref(d)))
            self.schedules.append(c)

    @classmethod
    def from_raw(cls, raw: RawModel, lanes=(1, 2, 4, 8), contacts=True):
        """Compile `raw` once per lane count that shortens the sequential depth of a sweep (trunk + longest limb set)."""
        cms, best = [], None
        for K in sorted(lanes):
            try:
                c = compile_model(raw, lanes=K)
            except ValueError:
                if K == 1:
                    raise
                continue
            depth = sum(hi - lo for lo, hi in c.trunk_ranges) + max(sum(hi - lo for lo, hi in rs) for rs in c.limb_ranges)
            if best is None or depth < best:
                cms.append(c)
                best = depth
        if not contacts:
            for c in cms:
                c.shape_body = c.shape_body[:0]
        return cls(cms[0], cms[1:])

    def refresh_inertia(self, world):
        """The World's masses / COMs / moments changed (World.setMasses): recompute the canonical inertias (welded bodies
        summed into their owner) and push them to the device model; the tree, schedules and slots are unchanged."""
        from .modelspec import body_inertia_contribution

        raw = world._raw_model
        k = 0
        for sk in world.skeletons:
            for b in sk._ordered_bodies():
                raw.mass[k], raw.com[k] = b.mass, b.com
                I = b.moment
                raw.moment[k] = [I[0, 0], I[1, 1], I[2, 2], I[0, 1], I[0, 2], I[1, 2]]
                k += 1
        cm = self.cm
        inertia = np.zeros((cm.nb, 10))
        for i in range(raw.nb):
            o = int(cm.body_owner[i])
            if o >= 0:
                inertia[o] += body_inertia_contribution(cm.body_T[i], raw.mass[i], raw.com[i], raw.moment[i])
        for c in self.schedules:
            c.inertia = inertia.copy()
        buf = np.ascontiguousarray(inertia, dtype=np.float64)
        _cabi.check(_cabi.lib().nb2_model_set_inertia(self.handle, buf.ctypes.data))

    def inertia_param_jacobian(self, world) -> np.ndarray:
        """[getMassDims(), 10*nb] : d(canonical inertia parameters)/d(mass vector) at the world's current values."""
        from .modelspec import inertia_param_jacobian

        return inertia_param_jacobian(world._raw_model, self.cm, world._mass_entries())

    def set_lanes(self, lanes: int):
        """Pin the lane count (0 = automatic choice per launch)."""
        _cabi.check(_cabi.lib().nb2_model_set_lanes(self.handle, int(lanes)))

    def lanes_for(self, B: int, backward: bool = False, precision: int = FP32) -> int:
        return int(_cabi.lib().nb2_model_lanes_for(self.handle, int(B), int(backward), int(precision)))

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                _cabi.lib().nb2_model_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    # ---- device pointers (torch tensors on the current CUDA device) ----
    # wi_ptr (optional, every step / rollout call): per-world canonical inertia, fp64 [10*nb, B] (include/nb2.h nb2_step_forward_pw);
    # None = the model's table.  A backward takes the same wi_ptr as its forward.
    def forward_device(self, B, state_ptr, action_ptr, next_ptr, saved_ptr, stream, precision=FP32, wi_ptr=None):
        _cabi.check(_cabi.lib().nb2_step_forward_pw(self.handle, B, state_ptr, action_ptr, wi_ptr, next_ptr, saved_ptr, precision, stream))

    def backward_device(self, B, state_ptr, action_ptr, saved_ptr, gnext_ptr, gstate_ptr, gaction_ptr, stream,
                        precision=FP32, ginertia_ptr=None, wi_ptr=None):
        """ginertia_ptr: optional [10*nb, B] float32 buffer receiving dL/d(inertia parameters) per body and world."""
        _cabi.check(_cabi.lib().nb2_step_backward_pw(self.handle, B, state_ptr, action_ptr, wi_ptr, saved_ptr, gnext_ptr,
                                                     gstate_ptr, gaction_ptr, ginertia_ptr, precision, stream))

    def rollout_forward_device(self, B, T, states_ptr, actions_ptr, saved_ptr, stream, precision=FP32, wi_ptr=None):
        _cabi.check(_cabi.lib().nb2_rollout_forward_pw(self.handle, B, T, states_ptr, actions_ptr, wi_ptr, saved_ptr, precision, stream))

    def rollout_backward_device(self, B, T, states_ptr, actions_ptr, saved_ptr, gstates_ptr, gactions_ptr, stream, precision=FP32,
                                wi_ptr=None, ginertia_ptr=None):
        """ginertia_ptr: optional [10*nb, B] float64 buffer to which every step ADDS its dL/d(inertia parameters)."""
        _cabi.check(_cabi.lib().nb2_rollout_backward_pw(self.handle, B, T, states_ptr, actions_ptr, wi_ptr, saved_ptr, gstates_ptr,
                                                        gactions_ptr, ginertia_ptr, precision, stream))

    def rollout_contact_tape_bytes(self, B, T, checkpoint_every):
        return int(_cabi.lib().nb2_rollout_contact_tape_bytes(self.handle, B, T, checkpoint_every))

    def rollout_forward_contact_device(self, B, T, states_ptr, actions_ptr, x_ptr, m_ptr, tape_ptr, checkpoint_every, ws_ptr, sticky_ptr, stream,
                                       wi_ptr=None):
        _cabi.check(_cabi.lib().nb2_rollout_forward_contact_pw(self.handle, B, T, states_ptr, actions_ptr, wi_ptr, x_ptr, m_ptr, tape_ptr,
                                                               checkpoint_every, ws_ptr, sticky_ptr, stream))

    def rollout_backward_contact_device(self, B, T, states_ptr, actions_ptr, x_ptr, m_ptr, tape_ptr, checkpoint_every, gstates_ptr, gactions_ptr,
                                        ws_ptr, sticky_ptr, stream, wi_ptr=None, ginertia_ptr=None):
        _cabi.check(_cabi.lib().nb2_rollout_backward_contact_pw(self.handle, B, T, states_ptr, actions_ptr, wi_ptr, x_ptr, m_ptr, tape_ptr,
                                                                checkpoint_every, gstates_ptr, gactions_ptr, ginertia_ptr, ws_ptr, sticky_ptr, stream))

    def forward_dynamics(self, pos, vel, force):
        """q-ddot [B, n] (float64 CUDA tensors in and out): pointer-style ABA, no integration, no contact stage
        (SimpleFeatherstone::forwardDynamics / Skeleton::computeForwardDynamics + getAccelerations); the fp64 kernel of
        forward_dynamics_device.  Needs an action space covering every dof."""
        import torch

        dev = pos.device
        f = lambda t: t.to(device=dev, dtype=torch.float64).contiguous()
        pos, vel, force = f(pos), f(vel), f(force)
        acc = torch.empty_like(pos)
        with torch.cuda.device(dev):
            _cabi.check(_cabi.lib().nb2_forward_dynamics(self.handle, pos.shape[0], pos.data_ptr(), vel.data_ptr(), force.data_ptr(), acc.data_ptr(),
                                                         torch.cuda.current_stream().cuda_stream))
        return acc

    def inverse_dynamics_device(self, B, state_ptr, next_vel_ptr, tau_ptr, saved_ptr, stream, precision=FP32, wi_ptr=None):
        """Contact-free inverse dynamics (include/nb2.h nb2_inverse_dynamics): rows in the arithmetic type of `precision`."""
        _cabi.check(_cabi.lib().nb2_inverse_dynamics(self.handle, B, state_ptr, next_vel_ptr, wi_ptr, tau_ptr, saved_ptr, precision, stream))

    def inverse_dynamics_backward_device(self, B, state_ptr, saved_ptr, gtau_ptr, gstate_ptr, gnext_ptr, stream, precision=FP32,
                                         ginertia_ptr=None, wi_ptr=None):
        """VJP of inverse_dynamics_device; ginertia_ptr: optional [10*nb, B] float64 buffer receiving dL/d(inertia parameters)."""
        _cabi.check(_cabi.lib().nb2_inverse_dynamics_backward(self.handle, B, state_ptr, None, wi_ptr, saved_ptr, gtau_ptr, gstate_ptr,
                                                              gnext_ptr, ginertia_ptr, precision, stream))

    def forward_dynamics_device(self, B, state_ptr, tau_ptr, qdd_ptr, saved_ptr, stream, precision=FP32, wi_ptr=None):
        """Contact-free forward dynamics (include/nb2.h nb2_forward_dynamics_batch): rows in the arithmetic type of `precision`, tau per dof."""
        _cabi.check(_cabi.lib().nb2_forward_dynamics_batch(self.handle, B, state_ptr, tau_ptr, wi_ptr, qdd_ptr, saved_ptr, precision, stream))

    def forward_dynamics_backward_device(self, B, state_ptr, saved_ptr, gqdd_ptr, gstate_ptr, gtau_ptr, stream, precision=FP32,
                                         ginertia_ptr=None, wi_ptr=None):
        """VJP of forward_dynamics_device; ginertia_ptr: optional [10*nb, B] float64 buffer receiving dL/d(inertia parameters)."""
        _cabi.check(_cabi.lib().nb2_forward_dynamics_backward(self.handle, B, state_ptr, wi_ptr, saved_ptr, gqdd_ptr, gstate_ptr, gtau_ptr,
                                                              ginertia_ptr, precision, stream))

    def inverse_dynamics_jacobians_device(self, B, state_ptr, next_vel_ptr, tau_ptr, jq_ptr, jqdot_ptr, jnext_ptr, stream, precision=FP32, wi_ptr=None):
        """tau and its dense Jacobians [B, n, n] d/dq, d/dqdot, d/dnext_vel (include/nb2.h nb2_inverse_dynamics_jacobians)."""
        _cabi.check(_cabi.lib().nb2_inverse_dynamics_jacobians(self.handle, B, state_ptr, next_vel_ptr, wi_ptr, tau_ptr, jq_ptr, jqdot_ptr, jnext_ptr,
                                                               precision, stream))

    def forward_dynamics_jacobians_device(self, B, state_ptr, tau_ptr, qdd_ptr, jq_ptr, jqdot_ptr, jtau_ptr, stream, precision=FP32, wi_ptr=None):
        """qdd and its dense Jacobians [B, n, n] d/dq, d/dqdot, d/dtau (include/nb2.h nb2_forward_dynamics_jacobians)."""
        _cabi.check(_cabi.lib().nb2_forward_dynamics_jacobians(self.handle, B, state_ptr, tau_ptr, wi_ptr, qdd_ptr, jq_ptr, jqdot_ptr, jtau_ptr,
                                                               precision, stream))

    def contact_inverse_dynamics_device(self, B, body, state_ptr, next_vel_ptr, tau_ptr, wrench_ptr, saved_ptr, stream, precision=FP32,
                                        wi_ptr=None):
        """Contact inverse dynamics (include/nb2.h nb2_contact_inverse_dynamics); body: canonical index of the contact body."""
        _cabi.check(_cabi.lib().nb2_contact_inverse_dynamics(self.handle, B, body, state_ptr, next_vel_ptr, wi_ptr, tau_ptr, wrench_ptr,
                                                             saved_ptr, precision, stream))

    def contact_inverse_dynamics_backward_device(self, B, body, state_ptr, saved_ptr, wrench_ptr, gtau_ptr, gwrench_ptr, seed_ptr, gstate_ptr,
                                                 gnext_ptr, stream, precision=FP32, ginertia_ptr=None, wi_ptr=None):
        """VJP of contact_inverse_dynamics_device; seed_ptr: caller-owned [B, ndof] workspace in the arithmetic type."""
        _cabi.check(_cabi.lib().nb2_contact_inverse_dynamics_backward(self.handle, B, body, state_ptr, None, wi_ptr, saved_ptr, wrench_ptr,
                                                                      gtau_ptr, gwrench_ptr, seed_ptr, gstate_ptr, gnext_ptr, ginertia_ptr,
                                                                      precision, stream))

    @staticmethod
    def _contact_set(bodies, points):
        b = np.ascontiguousarray(bodies, np.int32).reshape(-1)
        p = np.ascontiguousarray(points, np.float64).reshape(len(b), 3)
        return len(b), b, p

    def multiple_contact_inverse_dynamics_device(self, B, bodies, points, state_ptr, next_vel_ptr, guess_ptr, tau_ptr, wrench_ptr, saved_ptr,
                                                 stream, precision=FP32, wi_ptr=None):
        """Multiple-contact inverse dynamics (include/nb2.h nb2_multiple_contact_inverse_dynamics); bodies [k]: canonical indices, points
        [k, 3]: each body's own origin in its canonical frame; guess_ptr: [B, k, 6] or None; wrench_ptr: [B, k, 6]."""
        k, b, p = self._contact_set(bodies, points)
        _cabi.check(_cabi.lib().nb2_multiple_contact_inverse_dynamics(self.handle, B, k, b.ctypes.data, p.ctypes.data, state_ptr, next_vel_ptr,
                                                                      wi_ptr, guess_ptr, tau_ptr, wrench_ptr, saved_ptr, precision, stream))

    def multiple_contact_inverse_dynamics_backward_device(self, B, bodies, points, state_ptr, saved_ptr, wrench_ptr, guess_ptr, gtau_ptr,
                                                          gwrench_ptr, seed_ptr, gstate_ptr, gnext_ptr, stream, precision=FP32, ginertia_ptr=None,
                                                          gguess_ptr=None, wi_ptr=None):
        """VJP of multiple_contact_inverse_dynamics_device; seed_ptr: caller-owned [B, ndof] workspace in the arithmetic type; gguess_ptr:
        optional [B, k, 6] buffer receiving dL/d(guess)."""
        k, b, p = self._contact_set(bodies, points)
        _cabi.check(_cabi.lib().nb2_multiple_contact_inverse_dynamics_backward(self.handle, B, k, b.ctypes.data, p.ctypes.data, state_ptr, None,
                                                                               wi_ptr, saved_ptr, wrench_ptr, guess_ptr, gtau_ptr, gwrench_ptr,
                                                                               seed_ptr, gstate_ptr, gnext_ptr, ginertia_ptr, gguess_ptr,
                                                                               precision, stream))

    def multiple_contact_inverse_dynamics_jacobians_device(self, B, bodies, points, state_ptr, next_vel_ptr, guess_ptr, tau_ptr, wrench_ptr,
                                                           jac_ptrs, stream, precision=FP32, wi_ptr=None):
        """tau, the wrenches and the dense Jacobians of multiple_contact_inverse_dynamics_device (include/nb2.h
        nb2_multiple_contact_inverse_dynamics_jacobians); jac_ptrs: (T_q, T_qdot, T_next_vel [B, n, n], T_guess [B, n, 6k] or None,
        W_q, W_qdot, W_next_vel [B, 6k, n], W_guess [B, 6k, 6k] or None)."""
        k, b, p = self._contact_set(bodies, points)
        _cabi.check(_cabi.lib().nb2_multiple_contact_inverse_dynamics_jacobians(self.handle, B, k, b.ctypes.data, p.ctypes.data, state_ptr,
                                                                                next_vel_ptr, wi_ptr, guess_ptr, tau_ptr, wrench_ptr, *jac_ptrs,
                                                                                precision, stream))

    def mass_matrix_device(self, B, pos_ptr, out_ptr, stream, precision=FP32, wi_ptr=None):
        """M(q) [B, n, n] (include/nb2.h nb2_mass_matrix): rows in the arithmetic type of `precision`."""
        _cabi.check(_cabi.lib().nb2_mass_matrix(self.handle, B, pos_ptr, wi_ptr, out_ptr, precision, stream))

    def inverse_mass_matrix_device(self, B, pos_ptr, out_ptr, stream, precision=FP32, wi_ptr=None):
        """M(q)^-1 [B, n, n] (include/nb2.h nb2_inverse_mass_matrix)."""
        _cabi.check(_cabi.lib().nb2_inverse_mass_matrix(self.handle, B, pos_ptr, wi_ptr, out_ptr, precision, stream))

    def mass_matrix_backward_device(self, B, pos_ptr, gM_ptr, gpos_ptr, stream, precision=FP32, ginertia_ptr=None, wi_ptr=None):
        """VJP of mass_matrix_device; ginertia_ptr: optional [10*nb, B] float64 buffer receiving dL/d(inertia parameters)."""
        _cabi.check(_cabi.lib().nb2_mass_matrix_backward(self.handle, B, pos_ptr, wi_ptr, gM_ptr, gpos_ptr, ginertia_ptr, precision, stream))

    def inverse_mass_matrix_backward_device(self, B, pos_ptr, minv_ptr, gMinv_ptr, ws_ptr, gpos_ptr, stream, precision=FP32, ginertia_ptr=None,
                                            wi_ptr=None):
        """VJP of inverse_mass_matrix_device from its output minv_ptr; ws_ptr: caller-owned [B, n, n] workspace in the arithmetic type."""
        _cabi.check(_cabi.lib().nb2_inverse_mass_matrix_backward(self.handle, B, pos_ptr, wi_ptr, minv_ptr, gMinv_ptr, ws_ptr, gpos_ptr,
                                                                 ginertia_ptr, precision, stream))

    def world_jacobian_device(self, B, pos_ptr, bodies, T12, off_ptr, off_per_world, out_ptr, stream, precision=FP32):
        """J [B, k, 6, n] of body points (include/nb2.h nb2_world_jacobian); bodies [k] int32 and T12 [k, 12] fp64 are host arrays."""
        b = np.ascontiguousarray(bodies, np.int32)
        T = np.ascontiguousarray(T12, np.float64)
        _cabi.check(_cabi.lib().nb2_world_jacobian(self.handle, B, pos_ptr, len(b), b.ctypes.data, T.ctypes.data, off_ptr, int(off_per_world),
                                                   out_ptr, precision, stream))

    def world_jacobian_backward_device(self, B, pos_ptr, bodies, T12, off_ptr, off_per_world, gJ_ptr, gpos_ptr, goff_ptr, stream, precision=FP32):
        """VJP of world_jacobian_device; goff_ptr: optional [B, k, 3] buffer (one row per world, also for shared offsets)."""
        b = np.ascontiguousarray(bodies, np.int32)
        T = np.ascontiguousarray(T12, np.float64)
        _cabi.check(_cabi.lib().nb2_world_jacobian_backward(self.handle, B, pos_ptr, len(b), b.ctypes.data, T.ctypes.data, off_ptr,
                                                            int(off_per_world), gJ_ptr, gpos_ptr, goff_ptr, precision, stream))

    def com_jacobian_device(self, B, pos_ptr, root, out_ptr, stream, precision=FP32, wi_ptr=None):
        """J_com [B, 3, n] of the tree rooted at canonical body `root` (include/nb2.h nb2_com_jacobian)."""
        _cabi.check(_cabi.lib().nb2_com_jacobian(self.handle, B, pos_ptr, int(root), wi_ptr, out_ptr, precision, stream))

    def com_jacobian_backward_device(self, B, pos_ptr, root, gJ_ptr, gpos_ptr, stream, precision=FP32, ginertia_ptr=None, wi_ptr=None):
        """VJP of com_jacobian_device; ginertia_ptr: optional [10*nb, B] float64 buffer receiving dL/d(inertia parameters)."""
        _cabi.check(_cabi.lib().nb2_com_jacobian_backward(self.handle, B, pos_ptr, int(root), wi_ptr, gJ_ptr, gpos_ptr, ginertia_ptr, precision,
                                                          stream))

    def world_jacobian_deriv_device(self, B, state_ptr, bodies, T12, off_ptr, off_per_world, out_ptr, stream, precision=FP32):
        """Jdot [B, k, 6, n] of body points at states [B, 2n] (include/nb2.h nb2_world_jacobian_deriv); nodes as world_jacobian_device."""
        b = np.ascontiguousarray(bodies, np.int32)
        T = np.ascontiguousarray(T12, np.float64)
        _cabi.check(_cabi.lib().nb2_world_jacobian_deriv(self.handle, B, state_ptr, len(b), b.ctypes.data, T.ctypes.data, off_ptr,
                                                         int(off_per_world), out_ptr, precision, stream))

    def world_jacobian_deriv_backward_device(self, B, state_ptr, bodies, T12, off_ptr, off_per_world, gJ_ptr, gstate_ptr, goff_ptr, stream,
                                             precision=FP32):
        """VJP of world_jacobian_deriv_device into gstate [B, 2n]; goff_ptr: optional [B, k, 3] buffer (one row per world)."""
        b = np.ascontiguousarray(bodies, np.int32)
        T = np.ascontiguousarray(T12, np.float64)
        _cabi.check(_cabi.lib().nb2_world_jacobian_deriv_backward(self.handle, B, state_ptr, len(b), b.ctypes.data, T.ctypes.data, off_ptr,
                                                                  int(off_per_world), gJ_ptr, gstate_ptr, goff_ptr, precision, stream))

    def com_jacobian_deriv_device(self, B, state_ptr, root, out_ptr, stream, precision=FP32, wi_ptr=None):
        """Jdot_com [B, 3, n] of the tree rooted at canonical body `root` at states [B, 2n] (include/nb2.h nb2_com_jacobian_deriv)."""
        _cabi.check(_cabi.lib().nb2_com_jacobian_deriv(self.handle, B, state_ptr, int(root), wi_ptr, out_ptr, precision, stream))

    def com_jacobian_deriv_backward_device(self, B, state_ptr, root, gJ_ptr, gstate_ptr, stream, precision=FP32, ginertia_ptr=None, wi_ptr=None):
        """VJP of com_jacobian_deriv_device into gstate [B, 2n]; ginertia_ptr: optional [10*nb, B] float64 buffer."""
        _cabi.check(_cabi.lib().nb2_com_jacobian_deriv_backward(self.handle, B, state_ptr, int(root), wi_ptr, gJ_ptr, gstate_ptr, ginertia_ptr,
                                                                precision, stream))

    def energy_momentum_device(self, B, state_ptr, root, kin_ptr, pot_ptr, mom_ptr, stream, precision=FP32, wi_ptr=None):
        """kinetic [B], potential [B] and momentum [B, 6] of the tree rooted at canonical body `root` at states [B, 2n] (include/nb2.h
        nb2_energy_momentum)."""
        _cabi.check(_cabi.lib().nb2_energy_momentum(self.handle, B, state_ptr, int(root), wi_ptr, kin_ptr, pot_ptr, mom_ptr, precision, stream))

    def energy_momentum_backward_device(self, B, state_ptr, root, gkin_ptr, gpot_ptr, gmom_ptr, gstate_ptr, stream, precision=FP32,
                                        ginertia_ptr=None, wi_ptr=None):
        """VJP of energy_momentum_device into gstate [B, 2n]; ginertia_ptr: optional [10*nb, B] float64 buffer."""
        _cabi.check(_cabi.lib().nb2_energy_momentum_backward(self.handle, B, state_ptr, int(root), wi_ptr, gkin_ptr, gpot_ptr, gmom_ptr, gstate_ptr,
                                                             ginertia_ptr, precision, stream))

    def inverse_dynamics_regressor_device(self, B, state_ptr, next_vel_ptr, Y_ptr, tau_passive_ptr, stream, precision=FP32):
        """Y [B, n, nb, 10] and tau_passive [B, n] of inverse dynamics at states [B, 2n] and next velocities [B, n] (include/nb2.h
        nb2_inverse_dynamics_regressor)."""
        _cabi.check(_cabi.lib().nb2_inverse_dynamics_regressor(self.handle, B, state_ptr, next_vel_ptr, Y_ptr, tau_passive_ptr, precision, stream))

    def energy_regressor_device(self, B, state_ptr, YT_ptr, YU_ptr, spring_ptr, stream, precision=FP32):
        """Y_kinetic, Y_potential [B, nb, 10] and the spring energy [B] at states [B, 2n] (include/nb2.h nb2_energy_regressor)."""
        _cabi.check(_cabi.lib().nb2_energy_regressor(self.handle, B, state_ptr, YT_ptr, YU_ptr, spring_ptr, precision, stream))

    def constrained_forward_dynamics_device(self, B, state_ptr, tau_ptr, bodies, T12, off_ptr, off_per_world, point, damping, qdd_ptr, wrench_ptr,
                                            stream, precision=FP32, wi_ptr=None):
        """qdd [B, n] and contact wrenches [B, k, 6 or 3] with the bodies held (include/nb2.h nb2_constrained_forward_dynamics); bodies [k]
        int32 and T12 [k, 12] fp64 are host arrays."""
        b = np.ascontiguousarray(bodies, np.int32)
        T = np.ascontiguousarray(T12, np.float64)
        _cabi.check(_cabi.lib().nb2_constrained_forward_dynamics(self.handle, B, state_ptr, tau_ptr, len(b), b.ctypes.data, T.ctypes.data, off_ptr,
                                                                 int(off_per_world), int(point), float(damping), wi_ptr, qdd_ptr, wrench_ptr,
                                                                 precision, stream))

    def constrained_forward_dynamics_backward_device(self, B, state_ptr, tau_ptr, bodies, T12, off_ptr, off_per_world, point, damping, gqdd_ptr,
                                                     gwrench_ptr, gstate_ptr, gtau_ptr, goff_ptr, stream, precision=FP32, ginertia_ptr=None,
                                                     wi_ptr=None):
        """VJP of constrained_forward_dynamics_device; goff_ptr: optional [B, k, 3], ginertia_ptr: optional [10*nb, B] float64."""
        b = np.ascontiguousarray(bodies, np.int32)
        T = np.ascontiguousarray(T12, np.float64)
        _cabi.check(_cabi.lib().nb2_constrained_forward_dynamics_backward(self.handle, B, state_ptr, tau_ptr, len(b), b.ctypes.data, T.ctypes.data,
                                                                          off_ptr, int(off_per_world), int(point), float(damping), wi_ptr, gqdd_ptr,
                                                                          gwrench_ptr, gstate_ptr, gtau_ptr, goff_ptr, ginertia_ptr, precision,
                                                                          stream))

    def constrained_forward_dynamics_jacobians_device(self, B, state_ptr, tau_ptr, bodies, T12, off_ptr, off_per_world, point, damping, qdd_ptr,
                                                      wrench_ptr, jac_ptrs, stream, precision=FP32, wi_ptr=None):
        """qdd, wrenches and the dense Jacobians of constrained_forward_dynamics_device (include/nb2.h
        nb2_constrained_forward_dynamics_jacobians); jac_ptrs: (J_q, J_qdot, J_tau [B, n, n], W_q, W_qdot, W_tau [B, m, n])."""
        b = np.ascontiguousarray(bodies, np.int32)
        T = np.ascontiguousarray(T12, np.float64)
        _cabi.check(_cabi.lib().nb2_constrained_forward_dynamics_jacobians(self.handle, B, state_ptr, tau_ptr, len(b), b.ctypes.data, T.ctypes.data,
                                                                           off_ptr, int(off_per_world), int(point), float(damping), wi_ptr, qdd_ptr,
                                                                           wrench_ptr, *jac_ptrs, precision, stream))

    def impulse_dynamics_device(self, B, state_ptr, bodies, T12, off_ptr, off_per_world, point, restitution, damping, vel_ptr, imp_ptr, stream,
                                precision=FP32, wi_ptr=None):
        """Post-impact velocities [B, n] and contact impulses [B, k, 6 or 3] with the bodies held (include/nb2.h nb2_impulse_dynamics);
        bodies [k] int32 and T12 [k, 12] fp64 are host arrays."""
        b = np.ascontiguousarray(bodies, np.int32)
        T = np.ascontiguousarray(T12, np.float64)
        _cabi.check(_cabi.lib().nb2_impulse_dynamics(self.handle, B, state_ptr, len(b), b.ctypes.data, T.ctypes.data, off_ptr, int(off_per_world),
                                                     int(point), float(restitution), float(damping), wi_ptr, vel_ptr, imp_ptr, precision, stream))

    def impulse_dynamics_backward_device(self, B, state_ptr, bodies, T12, off_ptr, off_per_world, point, restitution, damping, gvel_ptr,
                                         gimp_ptr, gstate_ptr, goff_ptr, stream, precision=FP32, ginertia_ptr=None, wi_ptr=None):
        """VJP of impulse_dynamics_device; goff_ptr: optional [B, k, 3], ginertia_ptr: optional [10*nb, B] float64."""
        b = np.ascontiguousarray(bodies, np.int32)
        T = np.ascontiguousarray(T12, np.float64)
        _cabi.check(_cabi.lib().nb2_impulse_dynamics_backward(self.handle, B, state_ptr, len(b), b.ctypes.data, T.ctypes.data, off_ptr,
                                                              int(off_per_world), int(point), float(restitution), float(damping), wi_ptr,
                                                              gvel_ptr, gimp_ptr, gstate_ptr, goff_ptr, ginertia_ptr, precision, stream))

    def impulse_dynamics_jacobians_device(self, B, state_ptr, bodies, T12, off_ptr, off_per_world, point, restitution, damping, vel_ptr, imp_ptr,
                                          jac_ptrs, stream, precision=FP32, wi_ptr=None):
        """qdot_after, impulses and the dense Jacobians of impulse_dynamics_device (include/nb2.h nb2_impulse_dynamics_jacobians); jac_ptrs:
        (V_q, V_qdot [B, n, n], I_q, I_qdot [B, m, n])."""
        b = np.ascontiguousarray(bodies, np.int32)
        T = np.ascontiguousarray(T12, np.float64)
        _cabi.check(_cabi.lib().nb2_impulse_dynamics_jacobians(self.handle, B, state_ptr, len(b), b.ctypes.data, T.ctypes.data, off_ptr,
                                                               int(off_per_world), int(point), float(restitution), float(damping), wi_ptr,
                                                               vel_ptr, imp_ptr, *jac_ptrs, precision, stream))

    def contact_workspace_bytes(self, B):
        return int(_cabi.lib().nb2_contact_workspace_bytes(self.handle, B))

    def contact_record_bytes(self, B):
        return int(_cabi.lib().nb2_contact_record_bytes(self.handle, B))

    def forward_contact_device(self, B, state_ptr, action_ptr, next_ptr, saved_ptr, ws_ptr, x_ptr, m_ptr, labels_ptr,
                               status_ptr, nc_ptr, cinfo_ptr, crec_ptr, status_accum_ptr, stream, wi_ptr=None):
        """fused fp64 step with the contact / boxed-LCP stage, one warp per world (include/nb2.h nb2_step_forward_contact)."""
        _cabi.check(_cabi.lib().nb2_step_forward_contact_pw(self.handle, B, state_ptr, action_ptr, wi_ptr, next_ptr, saved_ptr, ws_ptr, x_ptr,
                                                            m_ptr, labels_ptr, status_ptr, nc_ptr, cinfo_ptr, crec_ptr, status_accum_ptr, stream))

    def backward_contact_device(self, B, state_ptr, action_ptr, saved_ptr, crec_ptr, ws_ptr, gnext_ptr, gstate_ptr, gaction_ptr,
                                stream, ginertia_ptr=None, status_ptr=None, wi_ptr=None):
        """status_ptr: the forward's status array; worlds that cannot be back-propagated get bit 2048 (and NaN gradients)."""
        _cabi.check(_cabi.lib().nb2_step_backward_contact_pw(self.handle, B, state_ptr, action_ptr, wi_ptr, saved_ptr, crec_ptr, ws_ptr,
                                                             gnext_ptr, gstate_ptr, gaction_ptr, ginertia_ptr, status_ptr, stream))

    def set_contact_capacity(self, max_contacts: int):
        _cabi.check(_cabi.lib().nb2_model_set_contact_capacity(self.handle, int(max_contacts)))

    def contact_capacity(self) -> int:
        return int(_cabi.lib().nb2_model_contact_capacity(self.handle))

    # ---- host pointers (numpy / CPU tensors): copies included ----
    def forward_host(self, state: np.ndarray, action: np.ndarray, keep_for_backward=True, precision=FP32,
                     out: np.ndarray = None) -> np.ndarray:
        B = state.shape[0]
        if out is None:
            out = np.empty_like(state)
        _cabi.check(_cabi.lib().nb2_step_forward_host(self.handle, B, state.ctypes.data, action.ctypes.data,
                                                      out.ctypes.data, int(keep_for_backward), precision))
        return out

    def backward_host(self, grad_next: np.ndarray, precision=FP32, out_state=None, out_action=None):
        B = grad_next.shape[0]
        gs = np.empty_like(grad_next) if out_state is None else out_state
        ga = np.empty((B, self.na), np.float32) if out_action is None else out_action
        _cabi.check(_cabi.lib().nb2_step_backward_host(self.handle, B, grad_next.ctypes.data, gs.ctypes.data,
                                                       ga.ctypes.data, precision))
        return gs, ga

    def forward_contact_host(self, state: np.ndarray, action: np.ndarray, keep_for_backward=True, reset_cache=False, out=None, status_out=None):
        """Contact step on HOST arrays (float32 [B, 2n] / [B, a]); the solver cache lives in the model between calls."""
        B = state.shape[0]
        if out is None:
            out = np.empty_like(state)
        _cabi.check(_cabi.lib().nb2_step_forward_contact_host(self.handle, B, state.ctypes.data, action.ctypes.data, out.ctypes.data,
                                                              int(keep_for_backward), int(reset_cache),
                                                              status_out.ctypes.data if status_out is not None else None))
        return out

    def backward_contact_host(self, grad_next: np.ndarray, out_state=None, out_action=None, sticky_out=None):
        B = grad_next.shape[0]
        gs = np.empty_like(grad_next) if out_state is None else out_state
        ga = np.empty((B, self.na), np.float32) if out_action is None else out_action
        _cabi.check(_cabi.lib().nb2_step_backward_contact_host(self.handle, B, grad_next.ctypes.data, gs.ctypes.data, ga.ctypes.data,
                                                               sticky_out.ctypes.data if sticky_out is not None else None))
        return gs, ga


def device_model_for(world) -> DeviceModel:
    """Lazily (re)build the device model of a World.  The cache is validated against the object graph: any setter of a BodyNode / Joint /
    Skeleton / ShapeNode bumps a global edit epoch (world.py); a World whose model was built at an older epoch is re-flattened and,
    when its description really changed, rebuilt (with its LCP cache dropped)."""
    import hashlib

    from .world import edit_epoch

    dm = getattr(world, "_device_model", None)
    if dm is not None and getattr(world, "_dm_epoch", -1) == edit_epoch():
        return dm
    raw = flatten_world(world)
    h = hashlib.sha1(raw.to_json().encode()).hexdigest() + ("|nc" if getattr(world, "_contacts_disabled", False) else "")
    if dm is not None and getattr(world, "_dm_hash", None) == h:
        world._dm_epoch = edit_epoch()
        return dm
    world._raw_model = raw
    # contact-free step requested explicitly -> contacts=False
    dm = DeviceModel.from_raw(raw, contacts=not getattr(world, "_contacts_disabled", False))
    world._device_model = dm
    world._dm_hash, world._dm_epoch = h, edit_epoch()
    world._lcp_cache = None
    return dm
