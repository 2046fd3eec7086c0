"""Host-side World / Skeleton / Joint / BodyNode builder surface.

This mirrors the small part of the reference's object model that training
scripts touch before calling ``timestep`` (reference: pybind `World`
python/_nimblephysics/simulation_and_neural/World.cpp, `Skeleton` builder
calls used in python/new_examples/cartpole.py:12-46).  It holds *description*
only; all arithmetic happens on the GPU through the C-ABI (csrc/) after
``modelspec.flatten_world`` / ``modelspec.compile_model`` turn it into flat
arrays.

Conventions follow the reference: spatial quantities are [angular; linear],
transforms are 4x4 homogeneous (``T_parent_child``), default gravity is
(0, 0, -9.81) and default dt 1e-3 (dart/simulation/World.cpp:75-76).
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import numpy as np

# joint type ids shared with oracle/ and csrc/ (include/nb2.h)
WELD, REVOLUTE, PRISMATIC, FREE = 0, 1, 2, 3
JOINT_NDOF = {WELD: 0, REVOLUTE: 1, PRISMATIC: 1, FREE: 6}

# shape type ids (include/nb2.h)
SHAPE_BOX, SHAPE_SPHERE, SHAPE_CAPSULE = 0, 1, 2

INF = float("inf")


def _eye4():
    return np.eye(4, dtype=np.float64)


class Isometry3:
    """Tiny stand-in for nimble.math.Isometry3 (set_translation / set_rotation)."""

    def __init__(self, m: Optional[np.ndarray] = None):
        self._m = _eye4() if m is None else np.array(m, dtype=np.float64).reshape(4, 4)

    def set_translation(self, t):
        self._m[:3, 3] = np.asarray(t, dtype=np.float64)

    def set_rotation(self, r):
        self._m[:3, :3] = np.asarray(r, dtype=np.float64).reshape(3, 3)

    def translation(self):
        return self._m[:3, 3].copy()

    def rotation(self):
        return self._m[:3, :3].copy()

    def matrix(self):
        return self._m.copy()


def _as_T(T) -> np.ndarray:
    if isinstance(T, Isometry3):
        return T.matrix()
    return np.array(T, dtype=np.float64).reshape(4, 4)


class Shape:
    def __init__(self, kind: int, dims: Sequence[float]):
        self.kind = kind
        self.dims = np.zeros(3)
        self.dims[: len(dims)] = dims

    def compute_inertia(self, mass: float) -> np.ndarray:
        """Moment about the shape's own centre, shape-frame axes.
        reference: dart/dynamics/BoxShape.cpp:74-83, CapsuleShape.cpp:107-131,
        SphereShape (2/5 m r^2)."""
        if self.kind == SHAPE_BOX:
            sx, sy, sz = self.dims
            return np.diag([
                mass / 12.0 * (sy * sy + sz * sz),
                mass / 12.0 * (sx * sx + sz * sz),
                mass / 12.0 * (sx * sx + sy * sy),
            ])
        if self.kind == SHAPE_SPHERE:
            r = self.dims[0]
            return np.eye(3) * (0.4 * mass * r * r)
        if self.kind == SHAPE_CAPSULE:
            r, h = self.dims[0], self.dims[1]
            r2, h2 = r * r, h * h
            vc = math.pi * r2 * h
            vs = 4.0 / 3.0 * math.pi * r2 * r
            dens = mass / (vc + vs)
            mc, ms = dens * vc, dens * vs
            ixx = mc * (h2 / 12.0 + r2 / 4.0) + ms * (h2 + 0.375 * h * r + 0.4 * r2)
            izz = mc * (r2 / 2.0) + ms * (0.4 * r2)
            return np.diag([ixx, ixx, izz])
        raise ValueError("unknown shape kind")


def BoxShape(size):
    return Shape(SHAPE_BOX, list(size))


def SphereShape(radius):
    return Shape(SHAPE_SPHERE, [radius])


def CapsuleShape(radius, height):
    return Shape(SHAPE_CAPSULE, [radius, height])


# Every setter of the object graph bumps this counter.  device_model_for() re-flattens a World whose cached device model was built at
# an older epoch and rebuilds it when the flattened description really changed (domain randomisation / system identification edit
# masses, damping, friction between rollouts: the GPU model must follow).
_EDIT_EPOCH = [0]


def _edited():
    _EDIT_EPOCH[0] += 1


def edit_epoch() -> int:
    return _EDIT_EPOCH[0]


class ShapeNode:
    def __init__(self, shape: Shape, T_local: Optional[np.ndarray] = None, collidable=True):
        self.shape = shape
        self.T_local = _eye4() if T_local is None else _as_T(T_local)
        self.collidable = collidable
        self.has_collision = False

    # the reference's visual calls are accepted and ignored (no renderer here)
    def createVisualAspect(self):
        return self

    def createCollisionAspect(self):
        _edited()
        self.has_collision = True
        return self

    def setColor(self, *_):
        return None

    def setRelativeTransform(self, T):
        _edited()
        self.T_local = _as_T(T)


class BodyNode:
    """reference defaults: mass 1, com 0, moment I (dart/dynamics/Inertia.hpp
    default ctor); friction 1.0, restitution 0 (detail/BodyNodeAspect.hpp:47-48)."""

    def __init__(self, name: str):
        self.name = name
        self.mass = 1.0
        self.com = np.zeros(3)
        self.moment = np.eye(3)  # about the COM, body-frame axes
        self.shapes: List[ShapeNode] = []
        self.friction = 1.0
        self.restitution = 0.0
        self.gravity_mode = True
        self.parent_joint: Optional["Joint"] = None
        self.parent_body: Optional["BodyNode"] = None
        self.skeleton: Optional["Skeleton"] = None

    def setMass(self, m):
        """Inertia::setMass with preserveDimsAndEuler=true (dart/dynamics/Inertia.cpp:157-177): the body keeps its
        dimensions, so a non-zero moment scales with the mass."""
        _edited()
        m = float(m)
        if m == self.mass:
            return
        if self.mass > 0 and np.any(self.moment != 0):
            self.moment = self.moment * (m / self.mass)
        self.mass = m

    def getMass(self):
        return self.mass

    def setLocalCOM(self, c):
        _edited()
        self.com = np.asarray(c, dtype=np.float64).copy()

    def setMomentOfInertia(self, ixx, iyy, izz, ixy=0.0, ixz=0.0, iyz=0.0):
        _edited()
        self.moment = np.array([[ixx, ixy, ixz], [ixy, iyy, iyz], [ixz, iyz, izz]], dtype=np.float64)

    def setFrictionCoeff(self, mu):
        _edited()
        self.friction = float(mu)

    def setRestitutionCoeff(self, e):
        _edited()
        self.restitution = float(e)

    def createShapeNode(self, shape: Shape) -> ShapeNode:
        _edited()
        sn = ShapeNode(shape)
        self.shapes.append(sn)
        return sn

    def getName(self):
        return self.name


class Joint:
    def __init__(self, jtype: int, name: str):
        self.jtype = jtype
        self.name = name
        self.axis = np.array([0.0, 0.0, 1.0]) if jtype == REVOLUTE else np.array([1.0, 0.0, 0.0])
        self.T_pj = _eye4()  # parent body -> joint
        self.T_cj = _eye4()  # child body -> joint
        nd = JOINT_NDOF[jtype]
        self.ndof = nd
        self.damping = np.zeros(nd)
        self.spring = np.zeros(nd)
        self.rest = np.zeros(nd)
        self.pos_lo = np.full(nd, -INF)
        self.pos_hi = np.full(nd, INF)
        self.vel_lo = np.full(nd, -INF)
        self.vel_hi = np.full(nd, INF)
        self.force_lo = np.full(nd, -INF)
        self.force_hi = np.full(nd, INF)
        self.init_pos = np.zeros(nd)

    # --- subset of the reference Joint API used by example scripts ---
    def setAxis(self, a):
        _edited()
        a = np.asarray(a, dtype=np.float64)
        self.axis = a / np.linalg.norm(a)  # reference normalises (RevoluteJoint.cpp setAxis)

    def setTransformFromParentBodyNode(self, T):
        _edited()
        self.T_pj = _as_T(T)

    def setTransformFromChildBodyNode(self, T):
        _edited()
        self.T_cj = _as_T(T)

    def setPositionUpperLimit(self, i, v):
        _edited()
        self.pos_hi[i] = v

    def setPositionLowerLimit(self, i, v):
        _edited()
        self.pos_lo[i] = v

    def setVelocityUpperLimit(self, i, v):
        _edited()
        self.vel_hi[i] = v

    def setVelocityLowerLimit(self, i, v):
        _edited()
        self.vel_lo[i] = v

    def setControlForceUpperLimit(self, i, v):
        _edited()
        self.force_hi[i] = v

    def setControlForceLowerLimit(self, i, v):
        _edited()
        self.force_lo[i] = v

    def setPositionLimitEnforced(self, enforced: bool = True):
        """Joint::setPositionLimitEnforced (dart/dynamics/Joint.cpp:1366): the constraint solver adds a JointLimitConstraint row while the
        position sits on or beyond a limit (off by default, like the reference's loaders leave it)."""
        self.limit_enforced = bool(enforced)
        _edited()

    def setLimitEnforcement(self, enforced: bool = True):
        self.setPositionLimitEnforced(enforced)

    def isPositionLimitEnforced(self) -> bool:
        return bool(getattr(self, "limit_enforced", False))

    def setDampingCoefficient(self, i, v):
        _edited()
        self.damping[i] = v

    def setSpringStiffness(self, i, v):
        _edited()
        self.spring[i] = v

    def setRestPosition(self, i, v):
        _edited()
        self.rest[i] = v

    def getNumDofs(self):
        return self.ndof


class Skeleton:
    def __init__(self, name: str = "skeleton"):
        self.name = name
        self.bodies: List[BodyNode] = []
        self.mobile = True

    # ----- self-collision (Skeleton::enableSelfCollisionCheck / enableAdjacentBodyCheck, dart/dynamics/Skeleton.cpp; both off by default)
    def setSelfCollisionCheck(self, enable: bool):
        self.self_collision = bool(enable)
        self._touch_world()

    def enableSelfCollisionCheck(self):
        self.setSelfCollisionCheck(True)

    def disableSelfCollisionCheck(self):
        self.setSelfCollisionCheck(False)

    def isEnabledSelfCollisionCheck(self) -> bool:
        return bool(getattr(self, "self_collision", False))

    def getSelfCollisionCheck(self) -> bool:
        return self.isEnabledSelfCollisionCheck()

    def setAdjacentBodyCheck(self, enable: bool):
        self.adjacent_check = bool(enable)
        self._touch_world()

    def enableAdjacentBodyCheck(self):
        self.setAdjacentBodyCheck(True)

    def disableAdjacentBodyCheck(self):
        self.setAdjacentBodyCheck(False)

    def isEnabledAdjacentBodyCheck(self) -> bool:
        return bool(getattr(self, "adjacent_check", False))

    def setMobile(self, m: bool):
        _edited()
        self.mobile = bool(m)

    def isMobile(self):
        return self.mobile

    def _create(self, jtype: int, parent: Optional[BodyNode], jname=None, bname=None):
        _edited()
        j = Joint(jtype, jname or f"joint_{len(self.bodies)}")
        b = BodyNode(bname or f"body_{len(self.bodies)}")
        b.parent_joint, b.parent_body, b.skeleton = j, parent, self
        if parent is not None and parent.skeleton is not self:
            raise ValueError("parent body belongs to a different skeleton")
        self.bodies.append(b)
        return j, b

    def createRevoluteJointAndBodyNodePair(self, parent=None):
        return self._create(REVOLUTE, parent)

    def createPrismaticJointAndBodyNodePair(self, parent=None):
        return self._create(PRISMATIC, parent)

    def createFreeJointAndBodyNodePair(self, parent=None):
        return self._create(FREE, parent)

    def createWeldJointAndBodyNodePair(self, parent=None):
        return self._create(WELD, parent)

    def getNumDofs(self):
        return sum(b.parent_joint.ndof for b in self.bodies)

    def getNumBodyNodes(self):
        return len(self.bodies)

    def getBodyNode(self, key):
        if isinstance(key, int):
            return self.bodies[key]
        for b in self.bodies:
            if b.name == key:
                return b
        return None

    def getJoint(self, key):
        if isinstance(key, int):
            return self.bodies[key].parent_joint
        for b in self.bodies:
            if b.parent_joint.name == key:
                return b.parent_joint
        return None

    # ----- per-dof access in the skeleton's own dof order (dart/dynamics/MetaSkeleton.hpp) -----
    def _dof_slots(self):
        """[(joint, local index)] in dof order."""
        out = []
        for b in self._ordered_bodies():
            out.extend((b.parent_joint, k) for k in range(b.parent_joint.ndof))
        return out

    def _dof_offset_in_world(self):
        w = getattr(self, "_world", None)
        if w is None:
            return None, 0
        off = 0
        for sk in w.skeletons:
            if sk is self:
                return w, off
            off += sk.getNumDofs()
        return None, 0

    def setPosition(self, i, v):
        """Skeleton::setPosition: the pose the world starts from (and its current legacy state, if it has one)."""
        j, k = self._dof_slots()[i]
        j.init_pos[k] = float(v)
        w, off = self._dof_offset_in_world()
        if w is not None and w._state is not None:
            w._state[off + i] = float(v)

    def setPositions(self, q):
        for i, v in enumerate(np.asarray(q, dtype=np.float64).reshape(-1)):
            self.setPosition(i, v)

    def getPositions(self):
        w, off = self._dof_offset_in_world()
        if w is not None and w._state is not None:
            return w._state[off:off + self.getNumDofs()].copy()
        return np.array([j.init_pos[k] for j, k in self._dof_slots()])

    def _mass_matrix_block(self, inverse):
        w, off = self._dof_offset_in_world()
        if w is None:
            raise ValueError("Skeleton.getMassMatrix(): the skeleton is not part of a World")
        n = self.getNumDofs()
        return w._mass_matrix(inverse)[off:off + n, off:off + n].copy()

    def getMassMatrix(self):
        """Skeleton::getMassMatrix: this skeleton's block of its World's mass matrix at the current positions (numpy fp64; fp64 kernels,
        nimblephysics_b200.mass_matrix)."""
        return self._mass_matrix_block(False)

    def getInvMassMatrix(self):
        """Skeleton::getInvMassMatrix: this skeleton's block of M^-1 (M is block-diagonal over skeletons)."""
        return self._mass_matrix_block(True)

    def _jacobian_columns(self, who, node=None, offset=None):
        from .world_jacobian import _single_world_com, _single_world_point

        w, off = self._dof_offset_in_world()
        if w is None:
            raise ValueError(f"Skeleton.{who}: the skeleton is not part of a World")
        J = _single_world_com(w, self, who) if node is None else _single_world_point(w, node, offset, who)
        return J[:, off:off + self.getNumDofs()].copy()

    def getWorldJacobian(self, node, offset=None):
        """Skeleton::getWorldJacobian(node[, offset]) [6, n_skel]: [omega; velocity of the point] in world axes at the current positions,
        the columns of this skeleton's dofs (numpy fp64; fp64 kernels, nimblephysics_b200.world_jacobian)."""
        return self._jacobian_columns("getWorldJacobian()", node, offset)

    def getLinearJacobian(self, node, offset=None):
        """Skeleton::getLinearJacobian(node[, offset]) [3, n_skel]: the point's velocity rows of getWorldJacobian."""
        return self._jacobian_columns("getLinearJacobian()", node, offset)[3:]

    def getAngularJacobian(self, node):
        """Skeleton::getAngularJacobian(node) [3, n_skel]: the angular-velocity rows of getWorldJacobian."""
        return self._jacobian_columns("getAngularJacobian()", node)[:3]

    def getCOMLinearJacobian(self):
        """Skeleton::getCOMLinearJacobian() [3, n_skel] (numpy fp64; fp64 kernels, nimblephysics_b200.com_jacobian)."""
        return self._jacobian_columns("getCOMLinearJacobian()")

    def _jacobian_deriv_columns(self, who, node=None, offset=None):
        from .world_jacobian import _single_world_com_deriv, _single_world_point_deriv

        w, off = self._dof_offset_in_world()
        if w is None:
            raise ValueError(f"Skeleton.{who}: the skeleton is not part of a World")
        dJ = _single_world_com_deriv(w, self, who) if node is None else _single_world_point_deriv(w, node, offset, who)
        return dJ[:, off:off + self.getNumDofs()].copy()

    def getJacobianClassicDeriv(self, node, offset=None):
        """Skeleton::getJacobianClassicDeriv(node[, offset]) [6, n_skel]: d/dt getWorldJacobian at the current positions and velocities,
        the columns of this skeleton's dofs (numpy fp64; fp64 kernels, nimblephysics_b200.world_jacobian_deriv)."""
        return self._jacobian_deriv_columns("getJacobianClassicDeriv()", node, offset)

    def getLinearJacobianDeriv(self, node, offset=None):
        """Skeleton::getLinearJacobianDeriv(node[, offset]) [3, n_skel]: the point's rows of getJacobianClassicDeriv."""
        return self._jacobian_deriv_columns("getLinearJacobianDeriv()", node, offset)[3:]

    def getAngularJacobianDeriv(self, node):
        """Skeleton::getAngularJacobianDeriv(node) [3, n_skel]: the angular rows of getJacobianClassicDeriv."""
        return self._jacobian_deriv_columns("getAngularJacobianDeriv()", node)[:3]

    def getCOMLinearJacobianDeriv(self):
        """Skeleton::getCOMLinearJacobianDeriv() [3, n_skel] (numpy fp64; fp64 kernels, nimblephysics_b200.com_jacobian_deriv)."""
        return self._jacobian_deriv_columns("getCOMLinearJacobianDeriv()")

    def _energies(self, who):
        from .energy import _single_world_energy

        w, _ = self._dof_offset_in_world()
        if w is None:
            raise ValueError(f"Skeleton.{who}: the skeleton is not part of a World")
        return _single_world_energy(w, self, who)

    def computeKineticEnergy(self):
        """Skeleton::computeKineticEnergy() at the current positions and velocities (float, fp64 kernels,
        nimblephysics_b200.energy_and_momentum)."""
        return self._energies("computeKineticEnergy()")[0]

    def computePotentialEnergy(self):
        """Skeleton::computePotentialEnergy(): gravity at each body's centre of mass plus the joint springs (float; DESIGN.md §6m)."""
        return self._energies("computePotentialEnergy()")[1]

    def computeLagrangian(self):
        """Skeleton::computeLagrangian() = computeKineticEnergy() - computePotentialEnergy() (float)."""
        T, U = self._energies("computeLagrangian()")
        return T - U

    def setVelocity(self, i, v):
        w, off = self._dof_offset_in_world()
        if w is None:
            raise ValueError("setVelocity(): add the skeleton to a World first (velocities live in the world state)")
        st = w.getState()
        st[w.getNumDofs() + off + i] = float(v)
        w.setState(st)

    def setVelocities(self, v):
        for i, x in enumerate(np.asarray(v, dtype=np.float64).reshape(-1)):
            self.setVelocity(i, x)

    def setControlForceUpperLimits(self, limits):
        for (j, k), v in zip(self._dof_slots(), np.asarray(limits, dtype=np.float64).reshape(-1)):
            j.force_hi[k] = v
        self._touch_world()

    def setControlForceLowerLimits(self, limits):
        for (j, k), v in zip(self._dof_slots(), np.asarray(limits, dtype=np.float64).reshape(-1)):
            j.force_lo[k] = v
        self._touch_world()

    def _touch_world(self):
        w = getattr(self, "_world", None)
        if w is not None:
            w._touch()

    def _ordered_bodies(self) -> List[BodyNode]:
        """Bodies in an order where every parent precedes its children and that
        is otherwise creation order (the reference's tree/DoF order for
        single-tree skeletons, dart/dynamics/Skeleton.cpp registerBodyNode)."""
        done, out = set(), []
        pending = list(self.bodies)
        while pending:
            progressed = False
            rest = []
            for b in pending:
                if b.parent_body is None or id(b.parent_body) in done:
                    out.append(b)
                    done.add(id(b))
                    progressed = True
                else:
                    rest.append(b)
            if not progressed:
                raise ValueError("skeleton has a body whose parent is missing")
            pending = rest
        return out

    def getPositionLowerLimits(self):
        return np.concatenate([b.parent_joint.pos_lo for b in self._ordered_bodies()] or [np.zeros(0)])

    def getPositionUpperLimits(self):
        return np.concatenate([b.parent_joint.pos_hi for b in self._ordered_bodies()] or [np.zeros(0)])


class Contact:
    """collision::Contact (dart/collision/Contact.hpp:82-230), the fields the Python binding exposes: point and normal in the world frame
    (normal from object 2 towards object 1), penetrationDepth, type (collision::ContactType), names of the two BodyNodes."""

    def __init__(self, point, normal, penetrationDepth, type, bodyNodeA, bodyNodeB):
        self.point, self.normal, self.penetrationDepth, self.type = point, normal, penetrationDepth, type
        self.bodyNodeA, self.bodyNodeB = bodyNodeA, bodyNodeB

    def __repr__(self):
        return f"Contact({self.bodyNodeA} / {self.bodyNodeB}, depth={self.penetrationDepth:.4g}, type={self.type})"


class CollisionResult:
    """collision::CollisionResult (pybind collision/CollisionResult.cpp:49-65)."""

    def __init__(self, contacts):
        self._contacts = list(contacts)

    def getNumContacts(self) -> int:
        return len(self._contacts)

    def getContacts(self):
        return list(self._contacts)

    def getContact(self, i):
        return self._contacts[i]

    def isCollision(self) -> bool:
        return bool(self._contacts)


class World:
    """Description of one simulated world; batched state lives in tensors, not here.

    reference: dart/simulation/World.cpp (defaults :75-87, addSkeleton :749-793,
    state/action API :2016-2185).
    """

    def __init__(self):
        self.skeletons: List[Skeleton] = []
        self.gravity = np.array([0.0, 0.0, -9.81])
        self.dt = 1e-3
        self.action_space: List[int] = []
        self.penetration_correction = False
        self.contact_clipping_depth = 0.03
        self.fallback_cfm = 1e-4
        self._version = 0  # bumped on every structural edit -> device model rebuilt lazily
        self._device_model = None
        # legacy single-world state (reference World is stateful)
        self._state = None
        self._lcp_cache = None

    # ----- (de)serialisation -----
    @staticmethod
    def from_raw(raw) -> "World":
        """Rebuild a World from a flattened RawModel (inverse of modelspec.flatten_world); used to ship model
        fixtures as JSON (tests/golden/models) without the original .urdf/.skel files."""
        from .modelspec import T_from_12

        w = World()
        w.gravity = np.array(raw.gravity, dtype=np.float64)
        w.dt = float(raw.dt)
        w.penetration_correction = bool(raw.penetration_correction)
        w.contact_clipping_depth = float(raw.contact_clipping_depth)
        w.fallback_cfm = float(raw.fallback_cfm)
        skels = {}
        bodies = []
        for i in range(raw.nb):
            sid = int(raw.skel_id[i])
            if sid not in skels:
                skels[sid] = Skeleton(f"skeleton_{sid}")
                skels[sid].mobile = bool(raw.mobile[i])
                skels[sid].self_collision = bool(raw.self_collision[i])
                skels[sid].adjacent_check = bool(raw.adjacent_check[i])
            sk = skels[sid]
            p = int(raw.parent[i])
            name = raw.body_names[i] if i < len(raw.body_names) else None
            j, b = sk._create(int(raw.jtype[i]), bodies[p] if p >= 0 else None, None, name)
            j.axis = np.array(raw.axis[i], dtype=np.float64)
            j.T_pj = T_from_12(raw.Tpj[i])
            j.T_cj = T_from_12(raw.Tcj[i])
            j.limit_enforced = bool(raw.limit_enforced[i])
            o = int(raw.dof_off[i])
            for k in ("damping", "spring", "rest", "pos_lo", "pos_hi", "vel_lo", "vel_hi", "force_lo", "force_hi",
                      "init_pos"):
                getattr(j, k)[:] = getattr(raw, k)[o:o + j.ndof]
            b.mass = float(raw.mass[i])
            b.com = np.array(raw.com[i], dtype=np.float64)
            m = raw.moment[i]
            b.moment = np.array([[m[0], m[3], m[4]], [m[3], m[1], m[5]], [m[4], m[5], m[2]]], dtype=np.float64)
            b.friction = float(raw.friction[i])
            b.restitution = float(raw.restitution[i])
            b.gravity_mode = bool(raw.gravity_mode[i])
            bodies.append(b)
        for s in range(raw.ns):
            sn = ShapeNode(Shape(int(raw.shape_type[s]), list(raw.shape_dims[s])), T_from_12(raw.shape_T[s]))
            sn.has_collision = True
            bodies[int(raw.shape_body[s])].shapes.append(sn)
        for sid in sorted(skels):
            w.skeletons.append(skels[sid])
            skels[sid]._world = w
        w.action_space = [int(a) for a in raw.action_map]
        return w

    # ----- structure -----
    def _touch(self):
        _edited()
        self._version += 1
        self._device_model = None

    def addSkeleton(self, skel: Skeleton):
        base = self.getNumDofs()
        self.skeletons.append(skel)
        skel._world = self
        # reference appends *every* dof (mobile or not) to the action space, World.cpp:779-785
        self.action_space.extend(range(base, base + skel.getNumDofs()))
        self._touch()
        return skel

    def loadSkeleton(self, path: str, base_position=None, base_euler=None):
        from .loader import load_skeleton

        skel = load_skeleton(path)
        if skel is None:
            return None
        if base_position is not None or base_euler is not None:
            raise NotImplementedError("loadSkeleton(base pose) is not supported yet")
        return self.addSkeleton(skel)

    def getSkeleton(self, i):
        return self.skeletons[i]

    def getNumSkeletons(self):
        return len(self.skeletons)

    # ----- parameters -----
    def setGravity(self, g):
        self.gravity = np.asarray(g, dtype=np.float64).copy()
        self._touch()

    def getGravity(self):
        return self.gravity.copy()

    def setTimeStep(self, dt):
        self.dt = float(dt)
        self._touch()

    def getTimeStep(self):
        return self.dt

    def setPenetrationCorrectionEnabled(self, v):
        self.penetration_correction = bool(v)
        self._touch()

    def setContactClippingDepth(self, d):
        self.contact_clipping_depth = float(d)
        self._touch()

    def setFallbackConstraintForceMixingConstant(self, c):
        self.fallback_cfm = float(c)
        self._touch()

    # ----- sizes -----
    def getNumDofs(self):
        return sum(s.getNumDofs() for s in self.skeletons)

    def getStateSize(self):
        return 2 * self.getNumDofs()

    def getActionSize(self):
        return len(self.action_space)

    def getActionSpace(self):
        return list(self.action_space)

    def setActionSpace(self, mapping):
        self.action_space = [int(i) for i in mapping]
        self._touch()

    def removeDofFromActionSpace(self, dof):
        if dof in self.action_space:
            self.action_space.remove(dof)
            self._touch()

    def addDofToActionSpace(self, dof):
        if dof not in self.action_space:
            self.action_space.append(int(dof))
            self._touch()

    # ----- tunable inertial parameters (dart/neural/WithRespectToMass.cpp; World.cpp:1013-1053, 1821-1825) -----
    def tuneMass(self, node, type, upperBound=None, lowerBound=None):
        """Register `node`'s inertial parameters of kind `type` (WrtMassBodyNodeEntryType) as part of the mass vector."""
        from .modelspec import WRT_MASS_DIMS

        if type not in WRT_MASS_DIMS:
            raise ValueError("unknown WrtMassBodyNodeEntryType")
        d = WRT_MASS_DIMS[type]
        ub = np.full(d, np.inf) if upperBound is None else np.asarray(upperBound, np.float64).reshape(d)
        lb = np.full(d, -np.inf) if lowerBound is None else np.asarray(lowerBound, np.float64).reshape(d)
        self._wrt_mass = [e for e in getattr(self, "_wrt_mass", []) if e[0] is not node] + [(node, int(type), ub, lb)]

    def clearTunableMassThisInstance(self):
        self._wrt_mass = []

    def getMassDims(self):
        from .modelspec import WRT_MASS_DIMS

        return sum(WRT_MASS_DIMS[t] for _, t, _, _ in getattr(self, "_wrt_mass", []))

    def getMassUpperLimits(self):
        return np.concatenate([ub for _, _, ub, _ in getattr(self, "_wrt_mass", [])] or [np.zeros(0)])

    def getMassLowerLimits(self):
        return np.concatenate([lb for _, _, _, lb in getattr(self, "_wrt_mass", [])] or [np.zeros(0)])

    @staticmethod
    def _mom6(b):
        I = b.moment
        return np.array([I[0, 0], I[1, 1], I[2, 2], I[0, 1], I[0, 2], I[1, 2]])

    def getMasses(self):
        from .modelspec import _mass_entry_value

        out = [_mass_entry_value(t, b.mass, b.com, self._mom6(b)) for b, t, _, _ in getattr(self, "_wrt_mass", [])]
        return np.concatenate(out) if out else np.zeros(0)

    def setMasses(self, masses):
        from .modelspec import WRT_MASS_DIMS, _apply_mass_entry

        masses = np.asarray(masses, dtype=np.float64).reshape(-1)
        self._mass_key = None  # (timestep() remembers which mass tensor the world holds; any direct call invalidates that)
        self._mass_P = None
        if masses.size != self.getMassDims():
            raise ValueError(f"World.setMasses() got size {masses.size}, expected getMassDims()={self.getMassDims()}")
        cur = 0
        for b, t, _, _ in getattr(self, "_wrt_mass", []):
            d = WRT_MASS_DIMS[t]
            m_, c_, mom = _apply_mass_entry(t, masses[cur:cur + d], b.mass, b.com, self._mom6(b))
            b.mass, b.com = float(m_), np.array(c_, dtype=np.float64)
            b.moment = np.array([[mom[0], mom[3], mom[4]], [mom[3], mom[1], mom[5]], [mom[4], mom[5], mom[2]]], dtype=np.float64)
            cur += d
        dm = self._device_model
        if dm is not None:
            dm.refresh_inertia(self)  # same tree, new inertias: no recompilation

    def _mass_entries(self):
        """[(raw body index, type)] in mass-vector order (raw bodies are numbered skeleton by skeleton, tree order)."""
        index = {}
        k = 0
        for sk in self.skeletons:
            for b in sk._ordered_bodies():
                index[id(b)] = k
                k += 1
        return [(index[id(b)], t) for b, t, _, _ in getattr(self, "_wrt_mass", [])]

    def getNumBodyNodes(self):
        return sum(s.getNumBodyNodes() for s in self.skeletons)

    def getBodyNodeByIndex(self, index):
        """World::getBodyNodeByIndex (World.cpp): bodies numbered skeleton by skeleton."""
        for s in self.skeletons:
            if index < s.getNumBodyNodes():
                return s._ordered_bodies()[index]
            index -= s.getNumBodyNodes()
        return None

    # ----- legacy stateful API (single world) -----
    def setAction(self, action):
        action = np.asarray(action, dtype=np.float64).reshape(-1)
        if action.size != self.getActionSize():
            raise ValueError(f"World.setAction() got size {action.size}, expected getActionSize()={self.getActionSize()}")
        self._action = action.copy()

    def getAction(self):
        a = getattr(self, "_action", None)
        return np.zeros(self.getActionSize()) if a is None else a.copy()

    def step(self):
        """World::step (World.cpp:221-254) of the single legacy world: advances the stored state with the stored action on
        the GPU, then clears the control forces like the reference (World.cpp:297-302).  Returns nothing."""
        import torch

        from .timestep import timestep

        with torch.no_grad():
            timestep(self, torch.tensor(self.getState(), dtype=torch.float64), torch.tensor(self.getAction(), dtype=torch.float64))
        self._action = None

    def clone(self) -> "World":
        """World::clone (dart/simulation/World.cpp:107-160; MultiShot gives every shot a clone, MultiShot.cpp:57-72): an independent copy of the
        model, the current state and the action; device buffers and the solver cache are NOT shared (the copy builds its own on first use)."""
        from .modelspec import flatten_world

        w = World.from_raw(flatten_world(self))
        w.action_space = list(self.action_space)
        if self._state is not None:
            w._state = self._state.copy()
        if getattr(self, "_action", None) is not None:
            w._action = self._action.copy()
        # tunable-mass registrations refer to BodyNode objects: re-point them at the copy's nodes (same order)
        mine = [b for sk in self.skeletons for b in sk._ordered_bodies()]
        theirs = [b for sk in w.skeletons for b in sk._ordered_bodies()]
        idx = {id(b): k for k, b in enumerate(mine)}
        w._wrt_mass = [(theirs[idx[id(node)]], t, ub.copy(), lb.copy()) for node, t, ub, lb in getattr(self, "_wrt_mass", []) if id(node) in idx]
        return w

    def getLastCollisionResult(self, world_index: int = 0) -> "CollisionResult":
        """World::getLastCollisionResult (pybind World.cpp:247-251): the contacts the constraint stage of the LAST timestep() / step() generated
        for one world of the batch (default: the first / the legacy single world), read back from the device cache.  Joint-limit rows are not
        contacts and are left out."""
        c = getattr(self, "_lcp_cache", None)
        if c is None:
            return CollisionResult([])
        nc = int(c["nc"][world_index].item())
        rows = c["cinfo"][world_index, :nc].cpu().numpy()
        names = [b.name for sk in self.skeletons for b in sk._ordered_bodies()]
        out = []
        for r in rows:
            if int(r[9]) >= 100:
                continue
            a, b = int(r[7]), int(r[8])
            out.append(Contact(point=r[0:3].astype(np.float64), normal=r[3:6].astype(np.float64), penetrationDepth=float(r[6]), type=int(r[9]),
                               bodyNodeA=names[a] if 0 <= a < len(names) else None, bodyNodeB=names[b] if 0 <= b < len(names) else None))
        return CollisionResult(out)

    def _legacy_jacobians(self):
        import torch

        from .jacobians import step_jacobians

        dev = torch.device("cuda", torch.cuda.current_device())
        s = torch.tensor(self.getState(), dtype=torch.float32, device=dev)[None]
        a = torch.tensor(self.getAction(), dtype=torch.float32, device=dev)[None]
        _, Js, Ja = step_jacobians(self, s, a)
        return Js[0].double().cpu().numpy(), Ja[0].double().cpu().numpy()

    def getStateJacobian(self):
        """[2n, 2n] d state_{t+1} / d state_t at the world's current state and action (World::getStateJacobian,
        BackpropSnapshot::getStateJacobian, dart/neural/BackpropSnapshot.cpp:1230-1241).  The world is not advanced."""
        return self._legacy_jacobians()[0]

    def getActionJacobian(self):
        """[2n, a] d state_{t+1} / d action_t (BackpropSnapshot::getActionJacobian, :1245-1260): like the reference's assembly the
        position rows are zero (lossWrtTorque = forceVel^T lossWrtVelocity, BackpropSnapshot.cpp:176) and the velocity rows hold the
        force-vel block restricted to the action space."""
        return self._legacy_jacobians()[1]

    def setState(self, state):
        state = np.asarray(state, dtype=np.float64).reshape(-1)
        if state.size != self.getStateSize():
            # reference prints to stderr and ignores the call (World.cpp:2027-2033);
            # we raise instead (documented deviation, SURVEY §5)
            raise ValueError(
                f"World.setState() got size {state.size}, expected getStateSize()={self.getStateSize()}")
        self._state = state.copy()

    def getState(self):
        if self._state is None:
            self._state = np.zeros(self.getStateSize())
            n = self.getNumDofs()
            self._state[:n] = self.getInitialPositions()
        return self._state.copy()

    def getPositions(self):
        return self.getState()[: self.getNumDofs()]

    def _mass_matrix(self, inverse):
        from .mass_matrix import _single_world

        return _single_world(self, "World.getInvMassMatrix()" if inverse else "World.getMassMatrix()", inverse)

    def getMassMatrix(self):
        """The world's mass matrix [n, n] at the current positions (numpy fp64, computed by the fp64 kernels at B = 1)."""
        return self._mass_matrix(False)

    def getInvMassMatrix(self):
        """M^-1 [n, n] at the current positions (numpy fp64, fp64 kernels)."""
        return self._mass_matrix(True)

    def getVelocities(self):
        return self.getState()[self.getNumDofs():]

    def getInitialPositions(self):
        out = []
        for s in self.skeletons:
            for b in s._ordered_bodies():
                out.append(b.parent_joint.init_pos)
        return np.concatenate(out) if out else np.zeros(0)

    def getPositionLowerLimits(self):
        return np.concatenate([s.getPositionLowerLimits() for s in self.skeletons] or [np.zeros(0)])

    def getPositionUpperLimits(self):
        return np.concatenate([s.getPositionUpperLimits() for s in self.skeletons] or [np.zeros(0)])
