"""ctypes binding of the C ABI declared in include/nb2.h (libnb2.so, built in-tree by __graft_entry__.build()).

There is no CPU fallback: if the CUDA library is missing or fails to load, importing the compute path raises.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import numpy as np

from .modelspec import CanonModel

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("NB2_LIB") or os.path.join(_HERE, "csrc", "libnb2.so")  # NB2_LIB: a dev build (e.g. with -DNB2_CW_PROFILE)

_I32P = ctypes.POINTER(ctypes.c_int32)
_F64P = ctypes.POINTER(ctypes.c_double)
_F32P = ctypes.POINTER(ctypes.c_float)


class Nb2ModelDesc(ctypes.Structure):
    _fields_ = [
        ("nb", ctypes.c_int32), ("ndof", ctypes.c_int32), ("na", ctypes.c_int32), ("nslots", ctypes.c_int32),
        ("parent", _I32P), ("jtype", _I32P), ("dof_off", _I32P), ("flags", _I32P), ("slot_self", _I32P),
        ("slot_parent", _I32P), ("slot_count", _I32P),
        ("Xtree", _F64P), ("inertia", _F64P),
        ("damping", _F64P), ("spring", _F64P), ("rest", _F64P),
        ("pos_lo", _F64P), ("pos_hi", _F64P), ("vel_lo", _F64P), ("vel_hi", _F64P), ("force_lo", _F64P),
        ("force_hi", _F64P),
        ("action_map", _I32P),
        ("gravity", ctypes.c_double * 3), ("dt", ctypes.c_double),
        ("nshapes", ctypes.c_int32), ("npairs", ctypes.c_int32),
        ("shape_body", _I32P), ("shape_type", _I32P), ("shape_orig_body", _I32P),
        ("shape_dims", _F64P), ("shape_T", _F64P), ("shape_mu", _F64P), ("shape_rest", _F64P),
        ("pair_a", _I32P), ("pair_b", _I32P),
        ("penetration_correction", ctypes.c_int32),
        ("contact_clipping_depth", ctypes.c_double), ("fallback_cfm", ctypes.c_double),
        ("lanes", ctypes.c_int32), ("nsched", ctypes.c_int32), ("sched", _I32P),
        ("nlimits", ctypes.c_int32), ("limit_body", _I32P),
    ]

MAX_CONTACTS, MAX_ROWS = 16, 48  # include/nb2.h


def make_desc(cm: CanonModel, with_contacts: bool = True):
    """-> (Nb2ModelDesc, keepalive list).  The arrays must outlive the descriptor."""
    keep = []

    def i32(a):
        a = np.ascontiguousarray(a, dtype=np.int32)
        keep.append(a)
        return a.ctypes.data_as(_I32P)

    def f64(a):
        a = np.ascontiguousarray(a, dtype=np.float64)
        keep.append(a)
        return a.ctypes.data_as(_F64P)

    d = Nb2ModelDesc()
    d.nb, d.ndof, d.na, d.nslots = cm.nb, cm.ndof, len(cm.action_map), cm.nslots
    d.parent, d.jtype, d.dof_off = i32(cm.parent), i32(cm.jtype), i32(cm.dof_off)
    d.flags, d.slot_self, d.slot_parent = i32(cm.flags), i32(cm.slot_self), i32(cm.slot_parent)
    d.slot_count = i32(cm.slot_count)
    sched = [len(cm.trunk_ranges)] + [x for r in cm.trunk_ranges for x in r]
    for lr in cm.limb_ranges:
        sched += [len(lr)] + [x for r in lr for x in r]
    d.lanes, d.nsched, d.sched = int(cm.lanes), len(sched), i32(sched)
    d.Xtree, d.inertia = f64(cm.Xtree), f64(cm.inertia)
    d.damping, d.spring, d.rest = f64(cm.damping), f64(cm.spring), f64(cm.rest)
    d.pos_lo, d.pos_hi = f64(cm.pos_lo), f64(cm.pos_hi)
    d.vel_lo, d.vel_hi = f64(cm.vel_lo), f64(cm.vel_hi)
    d.force_lo, d.force_hi = f64(cm.force_lo), f64(cm.force_hi)
    d.action_map = i32(cm.action_map)
    for k in range(3):
        d.gravity[k] = float(cm.gravity[k])
    d.dt = float(cm.dt)
    # contact stage: shapes + the collision pairs in the reference's enumeration order (objects i < j in insertion
    # order, DARTCollisionDetector.cpp:150-175) after the static part of BodyNodeCollisionFilter (CollisionFilter.cpp:105-152)
    pa, pb = collision_pairs(cm) if with_contacts else ([], [])
    ns = len(cm.shape_body) if (with_contacts and pa) else 0
    d.nshapes, d.npairs = ns, len(pa) if ns else 0
    d.shape_body, d.shape_type, d.shape_orig_body = i32(cm.shape_body[:ns]), i32(cm.shape_type[:ns]), i32(cm.shape_orig_body[:ns])
    d.shape_dims, d.shape_T = f64(cm.shape_dims[:ns]), f64(cm.shape_T[:ns])
    d.shape_mu, d.shape_rest = f64(cm.shape_friction[:ns]), f64(cm.shape_restitution[:ns])
    d.pair_a, d.pair_b = i32(pa), i32(pb)
    lb = list(getattr(cm, "limit_bodies", [])) if with_contacts else []
    d.nlimits, d.limit_body = len(lb), i32(lb)
    d.penetration_correction = int(cm.penetration_correction)
    d.contact_clipping_depth = float(cm.contact_clipping_depth)
    d.fallback_cfm = float(cm.fallback_cfm)
    return d, keep


def collision_pairs(cm: CanonModel):
    """Shape pairs the narrow phase visits, in the reference's enumeration order (object i < object j), after the static part of
    BodyNodeCollisionFilter::ignoresCollision (dart/collision/CollisionFilter.cpp:105-152): same BodyNode, two immobile skeletons, the same
    skeleton unless it enabled self-collision checking — and then adjacent BodyNodes only when it also enabled the adjacent-body check.
    One addition: two BodyNodes welded into the same moving body cannot move against each other; their pair is dropped."""
    pa, pb = [], []
    ns = len(cm.shape_body)
    selfcol = getattr(cm, "shape_selfcol", None)
    for i in range(ns - 1):
        for j in range(i + 1, ns):
            bi, bj = int(cm.shape_orig_body[i]), int(cm.shape_orig_body[j])
            if bi == bj:
                continue  # same BodyNode
            if cm.shape_body[i] < 0 and cm.shape_body[j] < 0:
                continue  # neither can move
            if cm.shape_skel[i] == cm.shape_skel[j]:
                if selfcol is None or not selfcol[i]:
                    continue  # self-collision checking is off by default in the reference
                if not cm.shape_adjcheck[i] and (cm.orig_parent[bi] == bj or cm.orig_parent[bj] == bi):
                    continue  # adjacent bodies (areAdjacentBodies, CollisionFilter.cpp:155-170)
                if cm.shape_body[i] == cm.shape_body[j]:
                    continue  # welded together
            pa.append(i)
            pb.append(j)
    return pa, pb


_lib: Optional[ctypes.CDLL] = None


class Nb2Error(RuntimeError):
    pass


def lib() -> ctypes.CDLL:
    """Load libnb2.so; fail loudly when it is absent (no fallback path exists)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise Nb2Error(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(nvcc, sm_90a). nimblephysics_b200 has no CPU fallback.")
        L = ctypes.CDLL(LIB_PATH)
        L.nb2_last_error.restype = ctypes.c_char_p
        L.nb2_version.restype = ctypes.c_char_p
        L.nb2_launch_count.restype = ctypes.c_longlong
        L.nb2_model_create.argtypes = [ctypes.POINTER(Nb2ModelDesc), ctypes.POINTER(ctypes.c_void_p)]
        L.nb2_model_destroy.argtypes = [ctypes.c_void_p]
        L.nb2_model_add_schedule.argtypes = [ctypes.c_void_p, ctypes.POINTER(Nb2ModelDesc)]
        L.nb2_model_set_inertia.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.nb2_model_set_lanes.argtypes = [ctypes.c_void_p, ctypes.c_int]
        L.nb2_model_lanes_for.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.nb2_model_ndof.argtypes = [ctypes.c_void_p]
        L.nb2_model_na.argtypes = [ctypes.c_void_p]
        L.nb2_saved_words_per_world.argtypes = [ctypes.c_void_p]
        vp = ctypes.c_void_p
        L.nb2_step_forward.argtypes = [vp, ctypes.c_int, vp, vp, vp, vp, ctypes.c_int, vp]
        L.nb2_step_backward.argtypes = [vp, ctypes.c_int, vp, vp, vp, vp, vp, vp, vp, ctypes.c_int, vp]
        L.nb2_rollout_forward.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp, vp, vp, ctypes.c_int, vp]
        L.nb2_rollout_backward.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp, vp, vp, vp, vp, ctypes.c_int, vp]
        # per-world inertia variants: the same arguments with `world_inertia` after the action(s) (rollout backward: + grad_inertia)
        L.nb2_step_forward_pw.argtypes = [vp, ctypes.c_int, vp, vp, vp, vp, vp, ctypes.c_int, vp]
        L.nb2_step_backward_pw.argtypes = [vp, ctypes.c_int, vp, vp, vp, vp, vp, vp, vp, vp, ctypes.c_int, vp]
        L.nb2_rollout_forward_pw.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp, vp, vp, vp, ctypes.c_int, vp]
        L.nb2_rollout_backward_pw.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp, vp, vp, vp, vp, vp, vp, ctypes.c_int, vp]
        L.nb2_step_forward_contact_pw.argtypes = [vp, ctypes.c_int] + [vp] * 15
        L.nb2_step_backward_contact_pw.argtypes = [vp, ctypes.c_int] + [vp] * 12
        L.nb2_rollout_forward_contact_pw.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp, vp, vp, vp, vp, vp, ctypes.c_int, vp, vp, vp]
        L.nb2_rollout_backward_contact_pw.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp, vp, vp, vp, vp, vp, ctypes.c_int, vp, vp, vp, vp, vp, vp]
        L.nb2_ik_create.argtypes = [vp, ctypes.c_int, vp, vp, vp, ctypes.POINTER(ctypes.c_void_p)]
        L.nb2_ik_destroy.argtypes = [vp]
        L.nb2_ik_destroy.restype = None
        L.nb2_ik_pos_dim.argtypes = [vp]
        L.nb2_ik_vel_dim.argtypes = [vp]
        L.nb2_ik_forward.argtypes = [vp, ctypes.c_int, vp, vp, vp, vp]
        L.nb2_ik_backward.argtypes = [vp, ctypes.c_int, vp, vp, vp, vp, vp]
        L.nb2_rollout_contact_tape_bytes.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.nb2_rollout_contact_tape_bytes.restype = ctypes.c_size_t
        L.nb2_rollout_forward_contact.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp, vp, vp, vp, vp, ctypes.c_int, vp, vp, vp]
        L.nb2_rollout_backward_contact.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp, vp, vp, vp, vp, ctypes.c_int, vp, vp, vp, vp, vp]
        L.nb2_model_has_contacts.argtypes = [vp]
        L.nb2_contact_workspace_bytes.argtypes = [vp, ctypes.c_int]
        L.nb2_contact_workspace_bytes.restype = ctypes.c_size_t
        L.nb2_step_forward_contact.argtypes = [vp, ctypes.c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
        L.nb2_contact_record_bytes.argtypes = [vp, ctypes.c_int]
        L.nb2_contact_record_bytes.restype = ctypes.c_size_t
        L.nb2_step_backward_contact.argtypes = [vp, ctypes.c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
        L.nb2_step_forward_contact_host.argtypes = [vp, ctypes.c_int, vp, vp, vp, ctypes.c_int, ctypes.c_int, vp]
        L.nb2_step_backward_contact_host.argtypes = [vp, ctypes.c_int, vp, vp, vp, vp]
        L.nb2_forward_dynamics.argtypes = [vp, ctypes.c_int, vp, vp, vp, vp, vp]
        L.nb2_forward_dynamics_batch.argtypes = [vp, ctypes.c_int, vp, vp, vp, vp, vp, ctypes.c_int, vp]
        L.nb2_forward_dynamics_backward.argtypes = [vp, ctypes.c_int, vp, vp, vp, vp, vp, vp, vp, ctypes.c_int, vp]
        L.nb2_inverse_dynamics_jacobians.argtypes = [vp, ctypes.c_int] + [vp] * 7 + [ctypes.c_int, vp]
        L.nb2_forward_dynamics_jacobians.argtypes = [vp, ctypes.c_int] + [vp] * 7 + [ctypes.c_int, vp]
        L.nb2_inverse_dynamics.argtypes = [vp, ctypes.c_int, vp, vp, vp, vp, vp, ctypes.c_int, vp]
        L.nb2_inverse_dynamics_backward.argtypes = [vp, ctypes.c_int, vp, vp, vp, vp, vp, vp, vp, vp, ctypes.c_int, vp]
        L.nb2_contact_inverse_dynamics.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp, vp, vp, vp, vp, vp, ctypes.c_int, vp]
        L.nb2_contact_inverse_dynamics_backward.argtypes = [vp, ctypes.c_int, ctypes.c_int] + [vp] * 11 + [ctypes.c_int, vp]
        L.nb2_multiple_contact_inverse_dynamics.argtypes = [vp, ctypes.c_int, ctypes.c_int] + [vp] * 9 + [ctypes.c_int, vp]
        L.nb2_multiple_contact_inverse_dynamics_backward.argtypes = [vp, ctypes.c_int, ctypes.c_int] + [vp] * 15 + [ctypes.c_int, vp]
        L.nb2_multiple_contact_inverse_dynamics_jacobians.argtypes = [vp, ctypes.c_int, ctypes.c_int] + [vp] * 16 + [ctypes.c_int, vp]
        L.nb2_mass_matrix.argtypes = [vp, ctypes.c_int, vp, vp, vp, ctypes.c_int, vp]
        L.nb2_inverse_mass_matrix.argtypes = [vp, ctypes.c_int, vp, vp, vp, ctypes.c_int, vp]
        L.nb2_mass_matrix_backward.argtypes = [vp, ctypes.c_int] + [vp] * 5 + [ctypes.c_int, vp]
        L.nb2_inverse_mass_matrix_backward.argtypes = [vp, ctypes.c_int] + [vp] * 7 + [ctypes.c_int, vp]
        L.nb2_world_jacobian.argtypes = [vp, ctypes.c_int, vp, ctypes.c_int, vp, vp, vp, ctypes.c_int, vp, ctypes.c_int, vp]
        L.nb2_world_jacobian_backward.argtypes = [vp, ctypes.c_int, vp, ctypes.c_int, vp, vp, vp, ctypes.c_int, vp, vp, vp, ctypes.c_int, vp]
        L.nb2_com_jacobian.argtypes = [vp, ctypes.c_int, vp, ctypes.c_int, vp, vp, ctypes.c_int, vp]
        L.nb2_com_jacobian_backward.argtypes = [vp, ctypes.c_int, vp, ctypes.c_int] + [vp] * 4 + [ctypes.c_int, vp]
        L.nb2_world_jacobian_deriv.argtypes = [vp, ctypes.c_int, vp, ctypes.c_int, vp, vp, vp, ctypes.c_int, vp, ctypes.c_int, vp]
        L.nb2_world_jacobian_deriv_backward.argtypes = [vp, ctypes.c_int, vp, ctypes.c_int, vp, vp, vp, ctypes.c_int, vp, vp, vp, ctypes.c_int, vp]
        L.nb2_com_jacobian_deriv.argtypes = [vp, ctypes.c_int, vp, ctypes.c_int, vp, vp, ctypes.c_int, vp]
        L.nb2_com_jacobian_deriv_backward.argtypes = [vp, ctypes.c_int, vp, ctypes.c_int] + [vp] * 4 + [ctypes.c_int, vp]
        L.nb2_energy_momentum.argtypes = [vp, ctypes.c_int, vp, ctypes.c_int] + [vp] * 4 + [ctypes.c_int, vp]
        L.nb2_energy_momentum_backward.argtypes = [vp, ctypes.c_int, vp, ctypes.c_int] + [vp] * 6 + [ctypes.c_int, vp]
        L.nb2_inverse_dynamics_regressor.argtypes = [vp, ctypes.c_int] + [vp] * 4 + [ctypes.c_int, vp]
        L.nb2_energy_regressor.argtypes = [vp, ctypes.c_int] + [vp] * 4 + [ctypes.c_int, vp]
        L.nb2_constrained_forward_dynamics.argtypes = ([vp, ctypes.c_int, vp, vp, ctypes.c_int, vp, vp, vp, ctypes.c_int, ctypes.c_int, ctypes.c_double]
                                                       + [vp] * 3 + [ctypes.c_int, vp])
        L.nb2_constrained_forward_dynamics_backward.argtypes = ([vp, ctypes.c_int, vp, vp, ctypes.c_int, vp, vp, vp, ctypes.c_int, ctypes.c_int,
                                                                 ctypes.c_double] + [vp] * 7 + [ctypes.c_int, vp])
        L.nb2_constrained_forward_dynamics_jacobians.argtypes = ([vp, ctypes.c_int, vp, vp, ctypes.c_int, vp, vp, vp, ctypes.c_int, ctypes.c_int,
                                                                  ctypes.c_double] + [vp] * 9 + [ctypes.c_int, vp])
        L.nb2_impulse_dynamics.argtypes = ([vp, ctypes.c_int, vp, ctypes.c_int, vp, vp, vp, ctypes.c_int, ctypes.c_int, ctypes.c_double,
                                            ctypes.c_double] + [vp] * 3 + [ctypes.c_int, vp])
        L.nb2_impulse_dynamics_backward.argtypes = ([vp, ctypes.c_int, vp, ctypes.c_int, vp, vp, vp, ctypes.c_int, ctypes.c_int,
                                                     ctypes.c_double, ctypes.c_double] + [vp] * 6 + [ctypes.c_int, vp])
        L.nb2_impulse_dynamics_jacobians.argtypes = ([vp, ctypes.c_int, vp, ctypes.c_int, vp, vp, vp, ctypes.c_int, ctypes.c_int,
                                                      ctypes.c_double, ctypes.c_double] + [vp] * 7 + [ctypes.c_int, vp])
        L.nb2_lcp_solve_batch.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double] + [vp] * 11
        L.nb2_model_set_contact_capacity.argtypes = [vp, ctypes.c_int]
        L.nb2_model_contact_capacity.argtypes = [vp]
        L.nb2_step_forward_host.argtypes = [vp, ctypes.c_int, vp, vp, vp, ctypes.c_int, ctypes.c_int]
        L.nb2_step_backward_host.argtypes = [vp, ctypes.c_int, vp, vp, vp, ctypes.c_int]
        _lib = L
    return _lib


def check(rc: int):
    if rc != 0:
        raise Nb2Error(f"nb2 error {rc}: {lib().nb2_last_error().decode()}")
