"""Task-space mappings of a state: world poses / velocities of chosen body nodes, differentiable, on the GPU.

reference: dart/neural/IKMapping.{hpp,cpp} (IKMapping::addSpatialBodyNode / addLinearBodyNode / addAngularBodyNode, getPositionsInPlace
:146-181, getVelocitiesInPlace :183-237, getPosJacobian :371-417, getVelJacobian :429-474) and python/nimblephysics/mapping.py:23-114
(map_to_pos / map_to_vel autograd layers).  Same names and argument meaning; what changes: `state` may be a [B, 2n] CUDA tensor (B worlds
in one launch, gradients by the VJP kernel — no Jacobian matrix is formed), 1-D tensors keep the legacy single-world meaning.
The work is done by libnb2.so (include/nb2.h nb2_ik_*).  There is no CPU implementation.
"""
from __future__ import annotations

import ctypes
from typing import List, Tuple

import numpy as np
import torch

from . import _cabi
from .engine import device_model_for

SPATIAL, LINEAR, ANGULAR, COM = 0, 1, 2, 3


class IKMapping:
    """neural::IKMapping: an ordered list of (body node, what to report).  Entries are appended in call order and the mapped
    vectors are their concatenation (IKMapping.cpp:43-59)."""

    def __init__(self, world):
        self.world = world
        self.entries: List[Tuple[int, object]] = []
        self._handle = None
        self._key = None

    # ---- reference API
    def addSpatialBodyNode(self, node):
        self._add(SPATIAL, node)

    def addLinearBodyNode(self, node):
        self._add(LINEAR, node)

    def addAngularBodyNode(self, node):
        self._add(ANGULAR, node)

    def addSkeletonCOM(self, skel):
        """The COM entry type of IKMapping.hpp (Skeleton::getCOM / getCOMLinearVelocity, IKMapping.cpp:172-176, 224-228)."""
        self._add(COM, skel)

    def getPosDim(self) -> int:
        return sum(6 if t == SPATIAL else 3 for t, _ in self.entries)

    def getVelDim(self) -> int:
        return self.getPosDim()

    def getDim(self) -> int:
        return self.getPosDim()

    def getPositions(self, world=None) -> np.ndarray:
        w = world or self.world
        return map_to_pos(w, self, torch.tensor(w.getState(), dtype=torch.float64)).detach().cpu().numpy()

    def getVelocities(self, world=None) -> np.ndarray:
        w = world or self.world
        return map_to_vel(w, self, torch.tensor(w.getState(), dtype=torch.float64)).detach().cpu().numpy()

    def getRealPosToMappedPosJac(self, world=None) -> np.ndarray:
        """[getPosDim(), n] (IKMapping::getPosJacobian): rows are obtained by back-propagating the identity through the VJP kernel."""
        return self._jac(world or self.world, pos=True)

    def getRealVelToMappedVelJac(self, world=None) -> np.ndarray:
        return self._jac(world or self.world, pos=False)

    # ---- internals
    def _add(self, kind, obj):
        self.entries.append((kind, obj))
        self._handle = None

    def _jac(self, w, pos: bool) -> np.ndarray:
        dev = torch.device("cuda", torch.cuda.current_device())
        n = w.getNumDofs()
        d = self.getPosDim()
        s = torch.tensor(w.getState(), dtype=torch.float32, device=dev)[None].repeat(d, 1).requires_grad_(True)
        out = map_to_pos(w, self, s) if pos else map_to_vel(w, self, s)
        out.backward(torch.eye(d, device=dev))
        g = s.grad.double().cpu().numpy()
        return g[:, :n] if pos else g[:, n:]

    def device_handle(self, world):
        dm = device_model_for(world)
        key = (id(dm), dm.handle, len(self.entries))
        if self._handle is not None and self._key == key:
            return self._handle, dm
        if not self.entries:
            raise ValueError("IKMapping has no entries (addSpatialBodyNode / addLinearBodyNode / addAngularBodyNode)")
        index = {}
        k = 0
        for sk in world.skeletons:
            for b in sk._ordered_bodies():
                index[id(b)] = k
                k += 1
        cm = dm.cm
        types, bodies, Ts = [], [], []
        for kind, obj in self.entries:
            if kind == COM:
                roots = [b for b in obj._ordered_bodies() if b.parent_body is None]
                if not roots or id(roots[0]) not in index or cm.body_owner[index[id(roots[0])]] < 0:
                    raise ValueError("IKMapping COM entry: the skeleton is not a mobile tree of this world")
                owner = int(cm.body_owner[index[id(roots[0])]])
                while cm.parent[owner] >= 0:
                    owner = int(cm.parent[owner])
                types.append(COM); bodies.append(owner); Ts.append(np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], np.float64))
                continue
            if id(obj) not in index:
                raise ValueError(f"IKMapping: body node {getattr(obj, 'name', obj)!r} does not belong to this world")
            ri = index[id(obj)]
            T = np.asarray(cm.body_T[ri], np.float64)
            types.append(kind); bodies.append(int(cm.body_owner[ri]))
            Ts.append(np.concatenate([T[:3, :3].reshape(-1), T[:3, 3]]))
        t = np.asarray(types, np.int32); b = np.asarray(bodies, np.int32); T12 = np.ascontiguousarray(np.stack(Ts), np.float64)
        h = ctypes.c_void_p()
        _cabi.check(_cabi.lib().nb2_ik_create(dm.handle, len(types), t.ctypes.data, b.ctypes.data, T12.ctypes.data, ctypes.byref(h)))
        self._free()
        self._handle, self._key = h, key
        return h, dm

    def _free(self):
        if getattr(self, "_handle", None):
            try:
                _cabi.lib().nb2_ik_destroy(self._handle)
            except Exception:
                pass
            self._handle = None

    def __del__(self):
        self._free()


class _MapLayer(torch.autograd.Function):
    @staticmethod
    def forward(ctx, world, mapping, state, want_pos):
        h, dm = mapping.device_handle(world)
        n2 = 2 * dm.ndof
        legacy = state.dim() == 1
        s2 = state.detach().reshape(-1, n2)
        if not torch.cuda.is_available():
            raise RuntimeError("nimblephysics_b200.mapping needs a CUDA device; there is no CPU fallback")
        dev = s2.device if s2.is_cuda else torch.device("cuda", torch.cuda.current_device())
        sd = s2.to(device=dev, dtype=torch.float32).contiguous()
        B, dim = sd.shape[0], mapping.getPosDim()
        out = torch.empty((B, dim), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            st = torch.cuda.current_stream().cuda_stream
            _cabi.check(_cabi.lib().nb2_ik_forward(h, B, sd.data_ptr(), out.data_ptr() if want_pos else None, None if want_pos else out.data_ptr(), st))
        ctx.h, ctx.mapping, ctx.want_pos, ctx.legacy, ctx.B = h, mapping, want_pos, legacy, B
        ctx.in_device, ctx.in_dtype = state.device, state.dtype
        ctx.save_for_backward(sd)
        if legacy:
            return out[0].to(device=state.device, dtype=torch.float64)  # the reference returns fp64 (mapping.py:33)
        return out.to(device=state.device, dtype=state.dtype)

    @staticmethod
    def backward(ctx, grad_out):
        (sd,) = ctx.saved_tensors
        dev = sd.device
        g = grad_out.detach().reshape(ctx.B, -1).to(device=dev, dtype=torch.float32).contiguous()
        gs = torch.empty_like(sd)
        with torch.cuda.device(dev):
            st = torch.cuda.current_stream().cuda_stream
            _cabi.check(_cabi.lib().nb2_ik_backward(ctx.h, ctx.B, sd.data_ptr(), g.data_ptr() if ctx.want_pos else None,
                                                    None if ctx.want_pos else g.data_ptr(), gs.data_ptr(), st))
        if ctx.legacy:
            return None, None, gs[0].to(device=ctx.in_device, dtype=ctx.in_dtype), None
        return None, None, gs.to(device=ctx.in_device, dtype=ctx.in_dtype), None


def map_to_pos(world, map: IKMapping, state: torch.Tensor) -> torch.Tensor:
    """mapping.getPositions of the state, differentiable w.r.t. the position half of `state` (mapping.py:50-56)."""
    return _MapLayer.apply(world, map, state, True)


def map_to_vel(world, map: IKMapping, state: torch.Tensor) -> torch.Tensor:
    """mapping.getVelocities of the state, differentiable w.r.t. the velocity half of `state` (mapping.py:98-104)."""
    return _MapLayer.apply(world, map, state, False)
