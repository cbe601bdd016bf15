"""Kinematics by-products of the hot path's outward sweep, batched (SURVEY 8(f) rank 2).  Same names and meaning as the
reference, every quantity in the mechanism's root frame, 6-vectors as [angular; linear]:

    transform_to_root               -> transforms_to_root(_)             src/mechanism_state.jl:687-714
    center_of_mass                  -> center_of_mass                    src/mechanism_algorithms.jl:30-49
    kinetic_energy                  -> kinetic_energy                    src/mechanism_state.jl:886-888, 989-994
    gravitational_potential_energy  -> gravitational_potential_energy    src/mechanism_state.jl:897-903, 996-1000
    momentum / momentum_rate_bias   -> momentum / momentum_rate_bias     src/mechanism_state.jl:878-884, 975-987
    momentum_matrix!                -> momentum_matrix(_)                src/mechanism_algorithms.jl:313-327
    path + geometric_jacobian!      -> path, geometric_jacobian(_)       src/graphs/tree_path.jl, mechanism_algorithms.jl:80-100

All are one call of ``rbd_kinematics`` (include/rbd_b200.h) on the current CUDA stream; ``kinematics_`` exposes the fused
form (any subset of outputs from a single launch).  There is no CPU path.

Task-space kinematics -- quantities of chosen bodies relative to other bodies, in any body frame -- are one call of
``rbd_task_kinematics`` (DESIGN 4.17); ``task_kinematics_`` is its fused form for up to 32 ``TaskFrame``s:

    relative_transform(state, from, to)            -> relative_transform       src/mechanism_state.jl:1011-1014
    relative_twist(state, body, base)              -> relative_twist           src/mechanism_state.jl:1016-1038
    relative_acceleration(result, body, base)      -> relative_acceleration    src/mechanism_algorithms.jl:421-426
    point_jacobian!(Jp, state, path, point)        -> point_jacobian           src/mechanism_algorithms.jl:154-224
    point_velocity / point_acceleration            -> point_velocity, point_acceleration   src/spatial/spatialmotion.jl:346-363
    geometric_jacobian!(J, state, path), J.frame   -> geometric_jacobian(..., frame=)      src/mechanism_algorithms.jl:101-132
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import Dict, Optional, Sequence

import numpy as np
import torch

from . import _cabi
from .algorithms import DimensionMismatch, _stream
from .mechanism import Mechanism, RigidBody
from .state import MechanismState, _DT

__all__ = ["TreePath", "path", "kinematics_", "transforms_to_root", "transforms_to_root_", "center_of_mass", "kinetic_energy",
           "gravitational_potential_energy", "momentum", "momentum_rate_bias", "momentum_matrix", "momentum_matrix_",
           "geometric_jacobian", "geometric_jacobian_", "TaskFrame", "task_desc", "task_kinematics_", "relative_transform",
           "relative_twist", "relative_acceleration", "point_jacobian", "point_velocity", "point_acceleration"]

_ROWS = {"transforms_to_root": lambda s: 12 * len(s.mechanism.joints), "center_of_mass": lambda s: 3,
         "kinetic_energy": lambda s: 1, "gravitational_potential_energy": lambda s: 1, "momentum": lambda s: 6,
         "momentum_rate_bias": lambda s: 6, "momentum_matrix": lambda s: 6 * s.nv, "geometric_jacobian": lambda s: 6 * s.nv}
_NEEDS_V = ("kinetic_energy", "momentum", "momentum_rate_bias")


@dataclass
class TreePath:
    """``TreePath`` (src/graphs/tree_path.jl): the joints between ``source`` and ``target`` with their traversal
    directions, stored as one sign per tree joint: -1 = up (towards the root, source side), +1 = down, 0 = not on the path."""
    source: RigidBody
    target: RigidBody
    sign: np.ndarray            # int8 [number of tree joints]


def path(mechanism: Mechanism, source: RigidBody, target: RigidBody) -> TreePath:
    """``path(mechanism, from, to)`` (src/mechanism.jl:146-151 -> graphs/tree_path.jl:60-95): up from ``source`` to the
    lowest common ancestor, then down to ``target``."""
    index = {id(j.successor): i for i, j in enumerate(mechanism.joints)}

    def ancestors(body):                # joints from `body` up to the root
        out = []
        while body is not mechanism.root_body:
            i = index[id(body)]
            out.append(i)
            body = mechanism.joints[i].predecessor
        return out

    up, down = ancestors(source), ancestors(target)
    while up and down and up[-1] == down[-1]:      # drop the common part above the lowest common ancestor
        up.pop()
        down.pop()
    sign = np.zeros(len(mechanism.joints), np.int8)
    sign[up] = -1
    sign[down] = 1
    return TreePath(source, target, sign)


def kinematics_(state: MechanismState, path_: Optional[TreePath] = None, **outs: Optional[torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Fused form: fill any subset of {transforms_to_root, center_of_mass, kinetic_energy, gravitational_potential_energy,
    momentum, momentum_rate_bias, momentum_matrix, geometric_jacobian} ([rows, B] tensors of the state's dtype) with one
    kernel launch."""
    state.check_modcount()
    lib = _cabi.load_library()
    ko = _cabi.RbdKinematicsOut()
    for name, t in outs.items():
        if name not in _ROWS:
            raise TypeError(f"unknown kinematics output {name!r}")
        if t is None:
            continue
        rows = _ROWS[name](state)
        if t.dtype != state.dtype or t.device != state.q.device:
            raise TypeError(f"{name}: dtype/device must match the state")
        if t.dim() != 2 or t.shape[0] != rows or t.shape[1] != state.batch:
            raise DimensionMismatch(f"{name} has wrong size: expected ({rows}, {state.batch}), got {tuple(t.shape)}")
        if not t.is_contiguous():
            raise ValueError(f"{name} must be [rows, B] contiguous (batch index fastest)")
        setattr(ko, name, t.data_ptr())
    want_jac = outs.get("geometric_jacobian") is not None
    if want_jac and path_ is None:
        raise ValueError("geometric_jacobian needs a path")
    sign = None
    if want_jac:
        sign = np.ascontiguousarray(path_.sign, np.int8)
        if sign.shape != (len(state.mechanism.joints),):
            raise DimensionMismatch("path does not belong to this mechanism")
    _cabi.check(lib.rbd_kinematics(state.handle.ptr, _DT[state.dtype], state.batch, state.batch, state.q.data_ptr(),
                                   state.v.data_ptr(), None if sign is None else sign.ctypes.data_as(ctypes.c_void_p),
                                   ctypes.byref(ko), _stream()))
    return {k: t for k, t in outs.items() if t is not None}


def _alloc(state: MechanismState, name: str) -> torch.Tensor:
    return torch.empty((_ROWS[name](state), state.batch), dtype=state.dtype, device=state.q.device)


def _one(state: MechanismState, name: str, out: Optional[torch.Tensor] = None, path_: Optional[TreePath] = None):
    out = _alloc(state, name) if out is None else out
    kinematics_(state, path_, **{name: out})
    return out


def transforms_to_root_(out: torch.Tensor, state: MechanismState):
    """``transform_to_root(state, body)`` of every non-root body: rows 12 i .. 12 i + 11 = rotation (row-major 9) and
    translation (3) of the successor of tree joint i."""
    return _one(state, "transforms_to_root", out)


def transforms_to_root(state: MechanismState):
    return _one(state, "transforms_to_root")


def center_of_mass(state: MechanismState):
    return _one(state, "center_of_mass")


def kinetic_energy(state: MechanismState):
    return _one(state, "kinetic_energy")[0]


def gravitational_potential_energy(state: MechanismState):
    return _one(state, "gravitational_potential_energy")[0]


def momentum(state: MechanismState):
    return _one(state, "momentum")


def momentum_rate_bias(state: MechanismState):
    return _one(state, "momentum_rate_bias")


def momentum_matrix_(out: torch.Tensor, state: MechanismState):
    """``momentum_matrix!(A, state)``: [6 nv, B], column k of A at rows 6 k .. 6 k + 5."""
    return _one(state, "momentum_matrix", out)


def momentum_matrix(state: MechanismState):
    return _one(state, "momentum_matrix")


def geometric_jacobian_(out: torch.Tensor, state: MechanismState, path_: TreePath, frame: Optional[RigidBody] = None):
    """``geometric_jacobian!(J, state, path)``: [6 nv, B], column k at rows 6 k .. 6 k + 5, in the root frame (``rbd_kinematics``)
    or, with ``frame``, in that body's default frame (``rbd_task_kinematics``)."""
    if frame is None:
        return _one(state, "geometric_jacobian", out, path_)
    task_kinematics_(state, [TaskFrame(path_.target, path_.source, None, frame)], geometric_jacobian=out)
    return out


def geometric_jacobian(state: MechanismState, path_: TreePath, frame: Optional[RigidBody] = None):
    if frame is None:
        return _one(state, "geometric_jacobian", None, path_)
    return geometric_jacobian_(_task_alloc(state, "geometric_jacobian", 1), state, path_, frame)


# ---- task-space kinematics -------------------------------------------------------------------------------------------------
@dataclass
class TaskFrame:
    """One task of ``rbd_task_kinematics``: ``body`` relative to ``base`` (None = the root body), the point ``point`` fixed in
    ``body`` and given in its frame (None = its origin), results expressed in the default frame of ``frame`` (None = the root
    frame)."""
    body: RigidBody
    base: Optional[RigidBody] = None
    point: Optional[Sequence[float]] = None
    frame: Optional[RigidBody] = None


_TASK_ROWS = {"transform": lambda s: 12, "point": lambda s: 3, "twist": lambda s: 6, "point_velocity": lambda s: 3,
              "geometric_jacobian": lambda s: 6 * s.nv, "point_jacobian": lambda s: 3 * s.nv, "acceleration": lambda s: 6,
              "point_acceleration": lambda s: 3}
_TASK_NEEDS_V = ("twist", "point_velocity", "acceleration", "point_acceleration")


def task_desc(mechanism: Mechanism, tasks: Sequence[TaskFrame]):
    """The C struct ``rbd_task_desc`` for ``tasks``; returns (struct, keepalive arrays)."""
    index = {id(j.successor): i for i, j in enumerate(mechanism.joints)}

    def idx(body):
        if body is None or body is mechanism.root_body:
            return -1
        if id(body) not in index:
            raise ValueError(f"body {getattr(body, 'name', body)!r} does not belong to this mechanism")
        return index[id(body)]
    if len(tasks) > _cabi.RBD_MAX_TASKS:
        raise ValueError(f"at most {_cabi.RBD_MAX_TASKS} tasks per call")
    body = np.array([idx(t.body) for t in tasks], np.int32)
    base = np.array([idx(t.base) for t in tasks], np.int32)
    frame = np.array([idx(t.frame) for t in tasks], np.int32)
    point = np.zeros((len(tasks), 3))
    for k, t in enumerate(tasks):
        if t.point is not None:
            point[k] = np.asarray(t.point, np.float64).reshape(3)
    d = _cabi.RbdTaskDesc()
    d.ntasks = len(tasks)
    i32, f64 = ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_double)
    d.body, d.base, d.frame = (a.ctypes.data_as(i32) for a in (body, base, frame))
    d.point = point.ctypes.data_as(f64)
    return d, (body, base, frame, point)


def task_kinematics_(state: MechanismState, tasks: Sequence[TaskFrame], vd: Optional[torch.Tensor] = None,
                     **outs: Optional[torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Fused form: fill any subset of {transform, point, twist, point_velocity, geometric_jacobian, point_jacobian, acceleration,
    point_acceleration} ([rows * len(tasks), B] tensors of the state's dtype and device; task t owns rows t*rows .. (t+1)*rows - 1)
    with one kernel launch.  ``vd`` ([nv, B]) or None = zero joint accelerations: acceleration / point_acceleration are then the
    velocity-product terms J̇ v.  Gravity is in no output."""
    state.check_modcount()
    lib = _cabi.load_library()
    to = _cabi.RbdTaskOut()
    K = len(tasks)
    for name, t in outs.items():
        if name not in _TASK_ROWS:
            raise TypeError(f"unknown task kinematics output {name!r}")
        if t is None:
            continue
        rows = _TASK_ROWS[name](state) * K
        if t.dtype != state.dtype or t.device != state.q.device:
            raise TypeError(f"{name}: dtype/device must match the state")
        if t.dim() != 2 or t.shape[0] != rows or t.shape[1] != state.batch:
            raise DimensionMismatch(f"{name} has wrong size: expected ({rows}, {state.batch}), got {tuple(t.shape)}")
        if not t.is_contiguous():
            raise ValueError(f"{name} must be [rows, B] contiguous (batch index fastest)")
        setattr(to, name, t.data_ptr())
    if vd is not None:
        if vd.dtype != state.dtype or vd.device != state.q.device:
            raise TypeError("vd: dtype/device must match the state")
        if tuple(vd.shape) != (state.nv, state.batch):
            raise DimensionMismatch(f"vd has wrong size: expected ({state.nv}, {state.batch}), got {tuple(vd.shape)}")
        if not vd.is_contiguous():
            raise ValueError("vd must be [nv, B] contiguous (batch index fastest)")
    d, keep = task_desc(state.mechanism, tasks)
    _cabi.check(lib.rbd_task_kinematics(state.handle.ptr, _DT[state.dtype], state.batch, state.batch, state.q.data_ptr(),
                                        state.v.data_ptr(), None if vd is None else vd.data_ptr(), ctypes.byref(d),
                                        ctypes.byref(to), _stream()))
    return {k: t for k, t in outs.items() if t is not None}


def _task_alloc(state: MechanismState, name: str, ntasks: int) -> torch.Tensor:
    return torch.empty((_TASK_ROWS[name](state) * ntasks, state.batch), dtype=state.dtype, device=state.q.device)


def _task_one(state: MechanismState, name: str, task: TaskFrame, vd: Optional[torch.Tensor] = None) -> torch.Tensor:
    out = _task_alloc(state, name, 1)
    task_kinematics_(state, [task], vd, **{name: out})
    return out


def relative_transform(state: MechanismState, body: RigidBody, base: Optional[RigidBody] = None) -> torch.Tensor:
    """``relative_transform(state, default_frame(body), default_frame(base))`` = inv(T_base) T_body: [12, B], rotation
    row-major (9) then translation (3)."""
    return _task_one(state, "transform", TaskFrame(body, base))


def relative_twist(state: MechanismState, body: RigidBody, base: Optional[RigidBody] = None,
                   frame: Optional[RigidBody] = None) -> torch.Tensor:
    """``relative_twist(state, body, base)`` expressed in ``frame`` (None = root frame): [6, B], [angular; linear]."""
    return _task_one(state, "twist", TaskFrame(body, base, None, frame))


def relative_acceleration(state: MechanismState, body: RigidBody, base: Optional[RigidBody] = None,
                          vd: Optional[torch.Tensor] = None, frame: Optional[RigidBody] = None) -> torch.Tensor:
    """``relative_acceleration`` of the spatial accelerations at joint accelerations ``vd`` (None = zero), transformed to
    ``frame`` like ``transform(state, accel, frame)``: [6, B]."""
    return _task_one(state, "acceleration", TaskFrame(body, base, None, frame), vd)


def point_jacobian(state: MechanismState, path_: TreePath, point: Sequence[float], frame: Optional[RigidBody] = None) -> torch.Tensor:
    """``point_jacobian!(Jp, state, path, point)`` for a point fixed in ``path_.target`` and given in its frame, expressed in
    ``frame``: [3 nv, B], column k at rows 3 k .. 3 k + 2."""
    return _task_one(state, "point_jacobian", TaskFrame(path_.target, path_.source, point, frame))


def point_velocity(state: MechanismState, path_: TreePath, point: Sequence[float], frame: Optional[RigidBody] = None) -> torch.Tensor:
    """Velocity of the point (fixed in ``path_.target``, given in its frame) with respect to ``path_.source``, in ``frame``: [3, B]."""
    return _task_one(state, "point_velocity", TaskFrame(path_.target, path_.source, point, frame))


def point_acceleration(state: MechanismState, path_: TreePath, point: Sequence[float], vd: Optional[torch.Tensor] = None,
                       frame: Optional[RigidBody] = None) -> torch.Tensor:
    """``point_acceleration(twist, accel, point)`` of the point with respect to ``path_.source`` at joint accelerations ``vd``
    (None = zero: the velocity-product term J̇ v), all in ``frame``: [3, B]."""
    return _task_one(state, "point_acceleration", TaskFrame(path_.target, path_.source, point, frame), vd)
