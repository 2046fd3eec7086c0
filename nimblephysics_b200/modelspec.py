"""ModelSpec: World description -> flat arrays.

Two formats:

* ``RawModel``  — one entry per reference BodyNode, in the reference's own
  parametrisation (parent->joint and child->joint transforms, joint axis,
  mass / COM / moment, weld joints as bodies).  This is what the fp64 oracle
  consumes (oracle/nb_oracle.cpp) and what is stored as JSON fixtures.
  reference: the quantities are those of dart/dynamics/detail/JointAspect.hpp,
  BodyNodeAspect.hpp, Inertia.cpp:1368-1383.

* ``CanonModel`` — what the CUDA kernels consume (include/nb2.h `nb2_model_desc`).
  ``compile_model`` (a) folds weld-jointed bodies into their parents (rigidly
  attached: identical dynamics), (b) moves every body frame onto its joint
  frame with the joint axis along +z, so the motion subspace is a unit vector
  (revolute [0,0,1,0,0,0], prismatic [0,0,0,0,0,1], free = identity), (c)
  renumbers bodies in DFS pre-order so that leaf->root sweeps can hand results
  to the parent in registers, and assigns accumulator slots for branch nodes.
  None of this changes the generalized coordinates: q, qdot, tau keep the
  reference's DoF order.
"""
from __future__ import annotations

import json
from dataclasses import dataclass, field
from typing import Dict, List

import numpy as np

from .world import FREE, JOINT_NDOF, PRISMATIC, REVOLUTE, WELD, World

_ARRAY_FIELDS_F = ["axis", "Tpj", "Tcj", "mass", "com", "moment", "friction", "restitution", "damping", "spring",
                   "rest", "pos_lo", "pos_hi", "vel_lo", "vel_hi", "force_lo", "force_hi", "init_pos", "gravity",
                   "shape_dims", "shape_T"]
_ARRAY_FIELDS_I = ["parent", "jtype", "dof_off", "mobile", "gravity_mode", "skel_id", "shape_body", "shape_type",
                   "action_map", "self_collision", "adjacent_check", "limit_enforced"]


def T_to_12(T: np.ndarray) -> np.ndarray:
    """4x4 -> [R row-major (9), p (3)]"""
    return np.concatenate([T[:3, :3].reshape(9), T[:3, 3]])


def T_from_12(v) -> np.ndarray:
    T = np.eye(4)
    T[:3, :3] = np.asarray(v[:9]).reshape(3, 3)
    T[:3, 3] = v[9:12]
    return T


@dataclass
class RawModel:
    nb: int = 0
    ndof: int = 0
    parent: np.ndarray = None
    jtype: np.ndarray = None
    dof_off: np.ndarray = None
    axis: np.ndarray = None
    Tpj: np.ndarray = None
    Tcj: np.ndarray = None
    mass: np.ndarray = None
    com: np.ndarray = None
    moment: np.ndarray = None  # [nb,6] xx,yy,zz,xy,xz,yz about the COM
    mobile: np.ndarray = None
    gravity_mode: np.ndarray = None
    skel_id: np.ndarray = None
    self_collision: np.ndarray = None   # [nb] 1 when the body's skeleton has self-collision checking enabled (Skeleton::enableSelfCollisionCheck)
    adjacent_check: np.ndarray = None   # [nb] 1 when that skeleton also checks ADJACENT bodies (Skeleton::enableAdjacentBodyCheck)
    limit_enforced: np.ndarray = None   # [nb] 1 when the body's parent joint enforces its position limits (Joint::setPositionLimitEnforced)
    friction: np.ndarray = None
    restitution: np.ndarray = None
    damping: np.ndarray = None
    spring: np.ndarray = None
    rest: np.ndarray = None
    pos_lo: np.ndarray = None
    pos_hi: np.ndarray = None
    vel_lo: np.ndarray = None
    vel_hi: np.ndarray = None
    force_lo: np.ndarray = None
    force_hi: np.ndarray = None
    init_pos: np.ndarray = None
    gravity: np.ndarray = None
    dt: float = 1e-3
    shape_body: np.ndarray = None
    shape_type: np.ndarray = None
    shape_dims: np.ndarray = None
    shape_T: np.ndarray = None
    action_map: np.ndarray = None
    penetration_correction: bool = False
    contact_clipping_depth: float = 0.03
    fallback_cfm: float = 1e-4
    body_names: List[str] = field(default_factory=list)
    dof_names: List[str] = field(default_factory=list)

    @property
    def ns(self):
        return int(self.shape_body.shape[0])

    def to_json(self) -> str:
        d = {}
        for k, v in self.__dict__.items():
            d[k] = v.tolist() if isinstance(v, np.ndarray) else v
        return json.dumps(d)

    @staticmethod
    def from_json(s: str) -> "RawModel":
        d = json.loads(s)
        m = RawModel()
        for k, v in d.items():
            if k in _ARRAY_FIELDS_F:
                v = np.array(v, dtype=np.float64)
            elif k in _ARRAY_FIELDS_I:
                v = np.array(v, dtype=np.int32)
            setattr(m, k, v)
        m._fix_shapes()
        return m

    def _fix_shapes(self):
        nb, n = self.nb, self.ndof
        if self.self_collision is None:  # fixtures written before these fields existed: the reference's defaults (both off)
            self.self_collision = np.zeros(nb, np.int32)
        if self.adjacent_check is None:
            self.adjacent_check = np.zeros(nb, np.int32)
        if self.limit_enforced is None:
            self.limit_enforced = np.zeros(nb, np.int32)
        self.axis = self.axis.reshape(nb, 3)
        self.Tpj = self.Tpj.reshape(nb, 12)
        self.Tcj = self.Tcj.reshape(nb, 12)
        self.com = self.com.reshape(nb, 3)
        self.moment = self.moment.reshape(nb, 6)
        ns = self.shape_body.shape[0]
        self.shape_dims = self.shape_dims.reshape(ns, 3)
        self.shape_T = self.shape_T.reshape(ns, 12)

    def save(self, path: str):
        with open(path, "w") as f:
            f.write(self.to_json())

    @staticmethod
    def load(path: str) -> "RawModel":
        with open(path) as f:
            return RawModel.from_json(f.read())


def flatten_world(world: World) -> RawModel:
    m = RawModel()
    bodies = []
    for si, skel in enumerate(world.skeletons):
        for b in skel._ordered_bodies():
            bodies.append((si, skel, b))
    index = {id(b): i for i, (_, _, b) in enumerate(bodies)}
    nb = len(bodies)
    m.nb = nb
    m.parent = np.full(nb, -1, np.int32)
    m.jtype = np.zeros(nb, np.int32)
    m.dof_off = np.zeros(nb, np.int32)
    m.axis = np.zeros((nb, 3))
    m.Tpj = np.zeros((nb, 12))
    m.Tcj = np.zeros((nb, 12))
    m.mass = np.zeros(nb)
    m.com = np.zeros((nb, 3))
    m.moment = np.zeros((nb, 6))
    m.mobile = np.zeros(nb, np.int32)
    m.gravity_mode = np.zeros(nb, np.int32)
    m.skel_id = np.zeros(nb, np.int32)
    m.self_collision = np.zeros(nb, np.int32)
    m.adjacent_check = np.zeros(nb, np.int32)
    m.limit_enforced = np.zeros(nb, np.int32)
    m.friction = np.zeros(nb)
    m.restitution = np.zeros(nb)
    per_dof = {k: [] for k in ("damping", "spring", "rest", "pos_lo", "pos_hi", "vel_lo", "vel_hi", "force_lo",
                               "force_hi", "init_pos")}
    sb, st, sd, sT = [], [], [], []
    off = 0
    for i, (si, skel, b) in enumerate(bodies):
        j = b.parent_joint
        m.parent[i] = index[id(b.parent_body)] if b.parent_body is not None else -1
        m.jtype[i] = j.jtype
        m.dof_off[i] = off
        off += j.ndof
        m.axis[i] = j.axis
        m.Tpj[i] = T_to_12(j.T_pj)
        m.Tcj[i] = T_to_12(j.T_cj)
        m.mass[i] = b.mass
        m.com[i] = b.com
        I = b.moment
        m.moment[i] = [I[0, 0], I[1, 1], I[2, 2], I[0, 1], I[0, 2], I[1, 2]]
        m.mobile[i] = 1 if skel.mobile else 0
        m.gravity_mode[i] = 1 if b.gravity_mode else 0
        m.skel_id[i] = si
        m.self_collision[i] = 1 if getattr(skel, "self_collision", False) else 0
        m.adjacent_check[i] = 1 if getattr(skel, "adjacent_check", False) else 0
        m.limit_enforced[i] = 1 if getattr(j, "limit_enforced", False) else 0
        m.friction[i] = b.friction
        m.restitution[i] = b.restitution
        for k in per_dof:
            per_dof[k].append(getattr(j, k))
        m.body_names.append(b.name)
        for d in range(j.ndof):
            m.dof_names.append(f"{j.name}[{d}]" if j.ndof > 1 else j.name)
        for sn in b.shapes:
            if not (sn.has_collision and sn.collidable):
                continue
            sb.append(i)
            st.append(sn.shape.kind)
            sd.append(sn.shape.dims)
            sT.append(T_to_12(sn.T_local))
    m.ndof = off
    for k, v in per_dof.items():
        setattr(m, k, np.concatenate(v) if v else np.zeros(0))
    m.gravity = world.gravity.copy()
    m.dt = world.dt
    m.shape_body = np.array(sb, np.int32)
    m.shape_type = np.array(st, np.int32)
    m.shape_dims = np.array(sd, np.float64).reshape(len(sb), 3)
    m.shape_T = np.array(sT, np.float64).reshape(len(sb), 12)
    m.action_map = np.array(world.action_space, np.int32)
    m.penetration_correction = world.penetration_correction
    m.contact_clipping_depth = world.contact_clipping_depth
    m.fallback_cfm = world.fallback_cfm
    return m


# --------------------------------------------------------------------------
# kernel format
# --------------------------------------------------------------------------
CANON_REV, CANON_PRIS, CANON_FREE = 1, 2, 3


@dataclass
class CanonModel:
    nb: int = 0
    ndof: int = 0
    parent: np.ndarray = None  # [nb] canonical parent index, -1 world
    jtype: np.ndarray = None  # CANON_*
    dof_off: np.ndarray = None
    Xtree: np.ndarray = None  # [nb,12] parent frame <- child frame at q=0 (R row-major, p)
    inertia: np.ndarray = None  # [nb,10] m, h(3)=m*c, Ibar(6: xx,yy,zz,xy,xz,yz) about body origin
    flags: np.ndarray = None  # bit0: hand result to parent in registers (parent == i-1, same lane range)
    #                            bit2: body owns accumulator slots (has non-handoff children)
    slot_self: np.ndarray = None  # first incoming accumulator slot of this body (or -1); it owns slot_count consecutive slots
    slot_count: np.ndarray = None  # number of incoming slots (= children that cannot hand off in registers)
    slot_parent: np.ndarray = None  # slot this body deposits its contribution to the parent into, or -1 (register handoff / root)
    nslots: int = 0
    # cooperative-lane schedule: `lanes` threads work on one world.  Phase "trunk" is run by lane 0 over trunk_ranges,
    # phase "limbs" by every lane over its own limb_ranges; ranges are [lo, hi) in canonical (DFS pre-order) numbering.
    lanes: int = 1
    trunk_ranges: List = field(default_factory=list)
    limb_ranges: List = field(default_factory=list)  # per lane: list of (lo, hi)
    orig_body: np.ndarray = None  # [nb] raw body index this canonical body stems from
    body_owner: np.ndarray = None  # [raw nb] canonical body a raw body is (rigidly) part of, -1 = static
    body_T: np.ndarray = None  # [raw nb,4,4] canonical owner frame <- raw body frame
    # per dof
    damping: np.ndarray = None
    spring: np.ndarray = None
    rest: np.ndarray = None
    pos_lo: np.ndarray = None
    pos_hi: np.ndarray = None
    vel_lo: np.ndarray = None
    vel_hi: np.ndarray = None
    force_lo: np.ndarray = None
    force_hi: np.ndarray = None
    gravity: np.ndarray = None
    dt: float = 1e-3
    action_map: np.ndarray = None
    # collision shapes: body == -1 -> static (world-fixed)
    shape_body: np.ndarray = None  # canonical body index or -1
    shape_orig_body: np.ndarray = None
    shape_type: np.ndarray = None
    shape_dims: np.ndarray = None
    shape_T: np.ndarray = None  # [ns,12] in canonical body frame (or world for static)
    shape_friction: np.ndarray = None
    shape_restitution: np.ndarray = None
    shape_skel: np.ndarray = None
    shape_selfcol: np.ndarray = None   # per shape: its skeleton checks self-collisions / adjacent bodies too
    shape_adjcheck: np.ndarray = None
    orig_parent: np.ndarray = None     # [raw nb] parent BodyNode (adjacency test of the collision filter)
    limit_bodies: List[int] = field(default_factory=list)  # canonical bodies whose parent joint enforces its position limits
    penetration_correction: bool = False
    contact_clipping_depth: float = 0.03
    fallback_cfm: float = 1e-4
    max_depth: int = 0


def _rot_z_to(axis: np.ndarray) -> np.ndarray:
    """A rotation R with R @ ez == axis (deterministic choice of the other two columns)."""
    a = axis / np.linalg.norm(axis)
    # exact shortcuts keep common models free of rounding noise
    for k, (x, y) in enumerate((((0, 1, 0), (0, 0, 1)), ((0, 0, 1), (1, 0, 0)), ((1, 0, 0), (0, 1, 0)))):
        e = np.zeros(3)
        e[k] = 1.0
        if np.allclose(a, e, atol=0, rtol=0):
            return np.stack([np.array(x, float), np.array(y, float), e], axis=1)
        if np.allclose(a, -e, atol=0, rtol=0):
            return np.stack([np.array(y, float), np.array(x, float), -e], axis=1)
    ref = np.array([1.0, 0.0, 0.0]) if abs(a[0]) < 0.9 else np.array([0.0, 1.0, 0.0])
    x = np.cross(ref, a)
    x /= np.linalg.norm(x)
    y = np.cross(a, x)
    return np.stack([x, y, a], axis=1)


def _spatial_inertia_about_origin(mass, com, Ic):
    """-> (m, h=m c, Ibar = Ic + m (|c|^2 I - c c^T)); reference Inertia.cpp:1368-1383."""
    c = np.asarray(com)
    Ibar = Ic + mass * (np.dot(c, c) * np.eye(3) - np.outer(c, c))
    return mass, mass * c, Ibar


def body_inertia_contribution(T, mass, com, mom6):
    """(m, h, Ibar about the origin) of one rigid body expressed in frame `T <- body`; polynomial in (mass, com, mom6),
    written so that complex arguments pass through unchanged (complex-step differentiation in inertia_param_jacobian)."""
    R, p = T[:3, :3], T[:3, 3]
    mom = mom6
    Ic = np.array([[mom[0], mom[3], mom[4]], [mom[3], mom[1], mom[5]], [mom[4], mom[5], mom[2]]])
    c = R @ np.asarray(com) + p
    RIR = R @ Ic @ R.T
    Ibar = RIR + mass * (np.sum(c * c) * np.eye(3) - np.outer(c, c))
    h = mass * c
    return np.array([mass, h[0], h[1], h[2], Ibar[0, 0], Ibar[1, 1], Ibar[2, 2], Ibar[0, 1], Ibar[0, 2], Ibar[1, 2]])


# WrtMassBodyNodeEntryType (dart/neural/WithRespectToMass.hpp:19-27)
INERTIA_MASS, INERTIA_COM, INERTIA_COM_MU, INERTIA_DIAGONAL, INERTIA_OFF_DIAGONAL, INERTIA_FULL = range(6)
WRT_MASS_DIMS = {INERTIA_MASS: 1, INERTIA_COM: 3, INERTIA_COM_MU: 1, INERTIA_DIAGONAL: 3, INERTIA_OFF_DIAGONAL: 3, INERTIA_FULL: 10}


def _apply_mass_entry(kind, value, mass, com, mom6):
    """(mass, com, mom6) of a body after WrtMassBodyNodyEntry::set (WithRespectToMass.cpp:44-134).  INERTIA_MASS goes
    through Inertia::setMass, which keeps the body's dimensions: the moment scales with the mass (Inertia.cpp:157-177)."""
    if kind == INERTIA_MASS:
        scale = (value[0] / mass) if (mass > 0 and np.any(np.asarray(mom6) != 0)) else 1.0
        return value[0], com, np.asarray(mom6) * scale
    if kind == INERTIA_COM:
        return mass, value[0:3], mom6
    if kind == INERTIA_DIAGONAL:
        return mass, com, np.array([value[0], value[1], value[2], mom6[3], mom6[4], mom6[5]])
    if kind == INERTIA_OFF_DIAGONAL:
        return mass, com, np.array([mom6[0], mom6[1], mom6[2], value[0], value[1], value[2]])
    if kind == INERTIA_FULL:
        return value[0], value[1:4], value[4:10]
    raise NotImplementedError("INERTIA_COM_MU needs BodyNode::getBeta(), which this builder surface does not carry")


def _mass_entry_value(kind, mass, com, mom6):
    """WrtMassBodyNodyEntry::get (WithRespectToMass.cpp:136-185)."""
    if kind == INERTIA_MASS:
        return np.array([mass])
    if kind == INERTIA_COM:
        return np.array(com, dtype=np.float64)
    if kind == INERTIA_DIAGONAL:
        return np.array(mom6[0:3], dtype=np.float64)
    if kind == INERTIA_OFF_DIAGONAL:
        return np.array(mom6[3:6], dtype=np.float64)
    if kind == INERTIA_FULL:
        return np.concatenate([[mass], com, mom6])
    raise NotImplementedError("INERTIA_COM_MU needs BodyNode::getBeta(), which this builder surface does not carry")


def inertia_param_jacobian(raw: RawModel, cm: "CanonModel", entries) -> np.ndarray:
    """d(canonical inertia [nb*10]) / d(mass vector), shape [mass_dims, nb*10], at the current values.
    entries: [(raw body index, WrtMassBodyNodeEntryType)] in registration order (WithRespectToMass::get order).
    The map raw (mass, com, moment) -> canonical (m, h, Ibar) is polynomial, so a complex step gives its exact derivative."""
    rows = []
    eps = 1e-30
    for (bi, kind) in entries:
        k = int(cm.body_owner[bi])
        x0 = _mass_entry_value(kind, raw.mass[bi], raw.com[bi], raw.moment[bi]).astype(np.complex128)
        for j in range(len(x0)):
            row = np.zeros(cm.nb * 10)
            if k >= 0:
                x = x0.copy()
                x[j] += 1j * eps
                m_, c_, mom_ = _apply_mass_entry(kind, x, raw.mass[bi], raw.com[bi], raw.moment[bi])
                row[10 * k:10 * k + 10] = np.imag(body_inertia_contribution(cm.body_T[bi].astype(np.complex128), m_, np.asarray(c_, np.complex128),
                                                                            np.asarray(mom_, np.complex128))) / eps
            rows.append(row)
    return np.array(rows).reshape(len(rows), cm.nb * 10)


def _mass_map_constants(world, raw: RawModel, cm: "CanonModel", device):
    """What mass_to_inertia needs besides the mass vectors, as tensors on `device`: the canonical table of every body that is NOT
    registered with tuneMass (fixed), and per registered body its current (mass, com, moment), its frame in the owner and the
    mass-vector columns that overwrite those values."""
    import torch

    entries = world._mass_entries()
    reg = {bi for bi, _ in entries}
    cur = {i: (raw.mass[i], raw.com[i], raw.moment[i]) for i in range(raw.nb)}
    base = np.zeros((cm.nb, 10))
    for i in range(raw.nb):
        o = int(cm.body_owner[i])
        if o >= 0 and i not in reg:
            base[o] += body_inertia_contribution(cm.body_T[i], *cur[i])
    E = len(entries)
    p0 = np.zeros((E, 10))       # (mass, com(3), moment(6)) before the mass vector is applied
    Rs, ps = np.zeros((E, 3, 3)), np.zeros((E, 3))
    owner = np.zeros((cm.nb, E))  # one-hot: canonical body <- registered raw body (0 for static bodies)
    dst, src, scaled = [], [], []  # columns of the mass vector -> (entry, parameter) slots; INERTIA_MASS entries whose moment scales
    col = 0
    for e, (bi, kind) in enumerate(entries):
        m0, c0, mom0 = cur[bi]
        p0[e] = np.concatenate([[m0], c0, mom0])
        T = cm.body_T[bi]
        Rs[e], ps[e] = T[:3, :3], T[:3, 3]
        if cm.body_owner[bi] >= 0:
            owner[int(cm.body_owner[bi]), e] = 1.0
        slots = {INERTIA_MASS: [0], INERTIA_COM: [1, 2, 3], INERTIA_DIAGONAL: [4, 5, 6], INERTIA_OFF_DIAGONAL: [7, 8, 9],
                 INERTIA_FULL: list(range(10))}.get(kind)
        if slots is None:
            raise NotImplementedError("INERTIA_COM_MU needs BodyNode::getBeta(), which this builder surface does not carry")
        dst += [10 * e + s for s in slots]
        src += list(range(col, col + len(slots)))
        if kind == INERTIA_MASS and m0 > 0 and np.any(mom0 != 0):  # Inertia::setMass keeps the body's dimensions (_apply_mass_entry)
            scaled.append((e, col))
        col += len(slots)
    t = lambda a, dt=torch.float64: torch.as_tensor(np.asarray(a), dtype=dt, device=device)
    return dict(base=t(base), p0=t(p0), R=t(Rs), p=t(ps), owner=t(owner), dst=t(dst, torch.long), src=t(src, torch.long),
                sc_e=t([e for e, _ in scaled], torch.long), sc_col=t([c for _, c in scaled], torch.long))


def mass_to_inertia(world, mass):
    """Per-world canonical inertia of B mass vectors: mass [B, getMassDims()] -> [B, nb, 10] float64 on mass's device, row w = the
    (m, h, Ibar) table that world.setMasses(mass[w]) followed by DeviceModel.refresh_inertia would produce from the World's current
    body parameters (INERTIA_MASS scales the moment by mass[w] / current mass).  The World is not modified.  Written in torch, so autograd
    carries a gradient with respect to the table (the kernels' per-world grad_inertia) back to `mass`.  The bodies that are not registered
    are folded into a constant table that is rebuilt only when the model or the body parameters change."""
    import torch

    from .world import edit_epoch

    if mass.dim() != 2 or mass.shape[1] != world.getMassDims():
        raise ValueError(f"mass_to_inertia(): mass has shape {tuple(mass.shape)}, expected [B, {world.getMassDims()}] (= getMassDims())")
    regs = [(id(b), t, b.mass, np.asarray(b.com).tobytes(), np.asarray(b.moment).tobytes()) for b, t, _, _ in getattr(world, "_wrt_mass", [])]
    key = (edit_epoch(), tuple(regs), str(mass.device))
    c = getattr(world, "_mass_map", None)
    if c is None or c[0] != key:
        raw = flatten_world(world)  # the current body parameters; the canonical numbering is the device model's (any lane count)
        c = (key, _mass_map_constants(world, raw, compile_model(raw), mass.device))
        world._mass_map = c
    K = c[1]
    B, E = mass.shape[0], K["p0"].shape[0]
    x = mass.to(torch.float64)
    prm = K["p0"].reshape(1, E * 10).expand(B, E * 10).clone()
    prm[:, K["dst"]] = x[:, K["src"]]
    prm = prm.reshape(B, E, 10)
    if K["sc_e"].numel():
        mom = prm[:, :, 4:].clone()
        mom[:, K["sc_e"]] = K["p0"][K["sc_e"], 4:] * (x[:, K["sc_col"]] / K["p0"][K["sc_e"], 0]).unsqueeze(-1)
        prm = torch.cat([prm[:, :, :4], mom], -1)
    m, com, m6 = prm[..., 0], prm[..., 1:4], prm[..., 4:]
    # body_inertia_contribution, batched: c = R com + p ; Ibar = R Ic R^T + m (|c|^2 1 - c c^T) ; h = m c
    Ic = torch.stack([m6[..., 0], m6[..., 3], m6[..., 4], m6[..., 3], m6[..., 1], m6[..., 5], m6[..., 4], m6[..., 5], m6[..., 2]], -1).reshape(B, E, 3, 3)
    cw = torch.einsum("eij,bej->bei", K["R"], com) + K["p"]
    RIR = K["R"] @ Ic @ K["R"].transpose(-1, -2)
    cc = (cw * cw).sum(-1)
    I3 = torch.eye(3, dtype=torch.float64, device=mass.device)
    Ibar = RIR + m[..., None, None] * (cc[..., None, None] * I3 - cw[..., :, None] * cw[..., None, :])
    h = m[..., None] * cw
    contrib = torch.stack([m, h[..., 0], h[..., 1], h[..., 2], Ibar[..., 0, 0], Ibar[..., 1, 1], Ibar[..., 2, 2],
                           Ibar[..., 0, 1], Ibar[..., 0, 2], Ibar[..., 1, 2]], -1)      # [B, E, 10]
    return K["base"] + torch.einsum("ke,bej->bkj", K["owner"], contrib)


def _ranges(idx):
    """sorted indices -> list of contiguous [lo, hi) ranges"""
    out = []
    for i in idx:
        if out and out[-1][1] == i:
            out[-1][1] = i + 1
        else:
            out.append([i, i + 1])
    return [(a, b) for a, b in out]


def _partition_tree(parent, lanes):
    """Split a forest (DFS pre-order numbering) into an ancestor-closed TRUNK and disjoint LIMB subtrees so that
    |trunk| + max(load per lane) — the sequential depth of one sweep with `lanes` cooperating threads — is small."""
    nb = len(parent)
    if lanes <= 1 or nb == 0:
        return list(range(nb)), []
    kids = {i: [] for i in range(-1, nb)}
    for i in range(nb):
        kids[int(parent[i])].append(i)
    size = [1] * nb
    for i in range(nb - 1, -1, -1):
        if parent[i] >= 0:
            size[int(parent[i])] += size[i]

    def subtree(r):
        return list(range(r, r + size[r]))  # contiguous in pre-order

    def cost(trunk_n, limb_roots):
        loads = [0] * lanes
        for sz in sorted((size[r] for r in limb_roots), reverse=True):
            loads[loads.index(min(loads))] += sz
        return trunk_n + max(loads) if limb_roots else trunk_n

    trunk = set()
    limb_roots = list(kids[-1])
    best = (cost(0, limb_roots), set(trunk), list(limb_roots))
    for _ in range(nb):
        if not limb_roots:
            break
        r = max(limb_roots, key=lambda x: size[x])
        limb_roots.remove(r)
        trunk.add(r)
        limb_roots.extend(kids[r])
        c = cost(len(trunk), limb_roots)
        if c < best[0]:
            best = (c, set(trunk), list(limb_roots))
    _, trunk, limb_roots = best
    return sorted(trunk), [subtree(r) for r in limb_roots]


def compile_model(raw: RawModel, lanes: int = 1) -> CanonModel:
    nb = raw.nb
    # world pose bookkeeping is done with 4x4s: for every raw body keep
    #   rel[i]  : constant transform parent-body-frame <- joint frame (T_pj)
    #   Tcj[i]  : child-body-frame <- joint frame
    Tpj = [T_from_12(raw.Tpj[i]) for i in range(nb)]
    Tcj = [T_from_12(raw.Tcj[i]) for i in range(nb)]

    # ---- (a) resolve welds: attach[i] = (canonical owner raw index or -1 for world, T_owner_body<-this_body)
    attach: Dict[int, tuple] = {}

    def owner(i):
        if i in attach:
            return attach[i]
        if raw.jtype[i] != WELD:
            attach[i] = (i, np.eye(4))
            return attach[i]
        T_rel = Tpj[i] @ np.linalg.inv(Tcj[i])  # parent body <- this body
        p = raw.parent[i]
        if p < 0:
            attach[i] = (-1, T_rel)
        else:
            po, pT = owner(p)
            attach[i] = (po, pT @ T_rel)
        return attach[i]

    for i in range(nb):
        owner(i)
        if not raw.mobile[i] and JOINT_NDOF[int(raw.jtype[i])] > 0:
            raise NotImplementedError(
                "immobile skeletons with degrees of freedom are not supported by the batched engine; "
                "weld them to the world instead")
        if not raw.gravity_mode[i]:
            raise NotImplementedError("per-body gravity mode off is not supported")

    movers = [i for i in range(nb) if raw.jtype[i] != WELD]
    # ---- (b) canonical frames: C[i] = body_i frame <- canonical frame of i
    C = {}
    for i in movers:
        Ci = Tcj[i].copy()
        if raw.jtype[i] in (REVOLUTE, PRISMATIC):
            Ra = np.eye(4)
            Ra[:3, :3] = _rot_z_to(raw.axis[i])
            Ci = Ci @ Ra
        C[i] = Ci

    def canon_parent(i):
        p = raw.parent[i]
        if p < 0:
            return -1, np.eye(4)
        po, pT = attach[p]  # owner body frame <- body p frame
        return po, pT

    # children lists (in raw order) over movers
    kids: Dict[int, List[int]] = {-1: []}
    for i in movers:
        kids[i] = []
    Xtree_raw = {}
    for i in movers:
        po, pT = canon_parent(i)
        kids[po].append(i)
        # owner-body frame <- joint frame of i :  pT @ Tpj[i];   then into the owner's canonical frame
        X = pT @ Tpj[i]
        if raw.jtype[i] in (REVOLUTE, PRISMATIC):
            Ra = np.eye(4)
            Ra[:3, :3] = _rot_z_to(raw.axis[i])
            X = X @ Ra
        if po >= 0:
            X = np.linalg.inv(C[po]) @ X
        Xtree_raw[i] = X

    # ---- (c) DFS pre-order
    order: List[int] = []
    depth = {}

    def dfs(i, d):
        order.append(i)
        depth[i] = d
        for c in kids[i]:
            dfs(c, d + 1)

    import sys
    sys.setrecursionlimit(max(10000, sys.getrecursionlimit()))
    for r in kids[-1]:
        dfs(r, 0)
    new_index = {ri: k for k, ri in enumerate(order)}
    cm = CanonModel()
    cm.nb = len(order)
    cm.ndof = raw.ndof
    cm.parent = np.array([(-1 if canon_parent(ri)[0] < 0 else new_index[canon_parent(ri)[0]]) for ri in order], np.int32)
    cm.jtype = np.array([{REVOLUTE: CANON_REV, PRISMATIC: CANON_PRIS, FREE: CANON_FREE}[int(raw.jtype[ri])] for ri in order], np.int32)
    cm.dof_off = np.array([raw.dof_off[ri] for ri in order], np.int32)
    cm.Xtree = np.array([T_to_12(Xtree_raw[ri]) for ri in order]).reshape(cm.nb, 12)
    cm.orig_body = np.array(order, np.int32)
    cm.max_depth = (max(depth.values()) + 1) if depth else 0

    # inertia: sum over every raw body attached to the owner, expressed in the owner's canonical frame
    inertia = np.zeros((cm.nb, 10))
    cm.body_owner = np.full(nb, -1, np.int32)
    cm.body_T = np.tile(np.eye(4), (nb, 1, 1))
    for i in range(nb):
        o, T_ob = attach[i]
        if o < 0:
            continue  # static body, no dynamics
        T = np.linalg.inv(C[o]) @ T_ob  # canonical(o) <- body i
        k = new_index[o]
        cm.body_owner[i], cm.body_T[i] = k, T
        inertia[k] += body_inertia_contribution(T, raw.mass[i], raw.com[i], raw.moment[i])
    cm.inertia = inertia

    # ---- cooperative-lane schedule + accumulator slots for the leaf->root sweeps
    trunk, limbs = _partition_tree(cm.parent, lanes)
    cm.lanes = lanes
    cm.trunk_ranges = _ranges(sorted(trunk))
    lane_bodies = [[] for _ in range(lanes)]
    for li, limb in enumerate(sorted(limbs, key=lambda l: -len(l))):
        k = min(range(lanes), key=lambda kk: len(lane_bodies[kk]))  # greedy balance
        lane_bodies[k].extend(limb)
    cm.limb_ranges = [_ranges(sorted(bs)) for bs in lane_bodies]
    if len(cm.trunk_ranges) > 8 or any(len(rs) > 8 for rs in cm.limb_ranges):  # NB2_MAX_RANGES (csrc/nb2_model.h)
        raise ValueError(f"the {lanes}-lane schedule of this tree needs more than 8 body ranges per lane")
    # which range does a body belong to?  register handoff (child -> parent = child-1) only inside one range
    range_id = {}
    rid = 0
    for (lo, hi) in cm.trunk_ranges:
        for i in range(lo, hi):
            range_id[i] = rid
        rid += 1
    for rs in cm.limb_ranges:
        for (lo, hi) in rs:
            for i in range(lo, hi):
                range_id[i] = rid
            rid += 1
    flags = np.zeros(cm.nb, np.int32)
    slot_self = np.full(cm.nb, -1, np.int32)
    slot_count = np.zeros(cm.nb, np.int32)
    slot_parent = np.full(cm.nb, -1, np.int32)
    nslots = 0
    for p_ in range(cm.nb):
        kids_ = [c for c in range(cm.nb) if cm.parent[c] == p_]
        cross = [c for c in kids_ if not (c == p_ + 1 and range_id[c] == range_id[p_])]
        for c in kids_:
            if c not in cross:
                flags[c] |= 1  # NB2_F_HANDOFF
        if cross:
            slot_self[p_] = nslots
            slot_count[p_] = len(cross)
            flags[p_] |= 4  # NB2_F_HAS_SLOT
            for c in cross:
                slot_parent[c] = nslots
                nslots += 1
    cm.flags, cm.slot_self, cm.slot_count, cm.slot_parent, cm.nslots = flags, slot_self, slot_count, slot_parent, nslots

    for k in ("damping", "spring", "rest", "pos_lo", "pos_hi", "vel_lo", "vel_hi", "force_lo", "force_hi"):
        setattr(cm, k, getattr(raw, k).copy())
    cm.gravity = raw.gravity.copy()
    cm.dt = raw.dt
    cm.action_map = raw.action_map.copy()

    # shapes
    sb, so, st, sd, sT, sf, sr, ss = [], [], [], [], [], [], [], []
    for s in range(raw.ns):
        i = int(raw.shape_body[s])
        o, T_ob = attach[i]
        Ts = T_from_12(raw.shape_T[s])
        if o < 0:
            T = T_ob @ Ts
            sb.append(-1)
        else:
            T = np.linalg.inv(C[o]) @ T_ob @ Ts
            sb.append(new_index[o])
        so.append(i)
        st.append(int(raw.shape_type[s]))
        sd.append(raw.shape_dims[s])
        sT.append(T_to_12(T))
        sf.append(raw.friction[i])
        sr.append(raw.restitution[i])
        ss.append(int(raw.skel_id[i]))
    ns = len(sb)
    cm.shape_body = np.array(sb, np.int32)
    cm.shape_orig_body = np.array(so, np.int32)
    cm.shape_type = np.array(st, np.int32)
    cm.shape_dims = np.array(sd, np.float64).reshape(ns, 3)
    cm.shape_T = np.array(sT, np.float64).reshape(ns, 12)
    cm.shape_friction = np.array(sf, np.float64)
    cm.shape_restitution = np.array(sr, np.float64)
    cm.shape_skel = np.array(ss, np.int32)
    cm.shape_selfcol = np.array([int(raw.self_collision[i]) for i in so], np.int32)
    cm.shape_adjcheck = np.array([int(raw.adjacent_check[i]) for i in so], np.int32)
    cm.orig_parent = np.array(raw.parent, np.int32)
    # joints with enforced position limits (1-dof joints of mobile skeletons), in raw joint order: canonical body of each
    canon_of_raw = {int(r): k for k, r in enumerate(cm.orig_body)}
    cm.limit_bodies = [canon_of_raw[i] for i in range(raw.nb)
                       if raw.limit_enforced[i] and raw.mobile[i] and raw.jtype[i] in (REVOLUTE, PRISMATIC) and i in canon_of_raw]
    cm.penetration_correction = raw.penetration_correction
    cm.contact_clipping_depth = raw.contact_clipping_depth
    cm.fallback_cfm = raw.fallback_cfm
    return cm
