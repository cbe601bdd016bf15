"""Closed-loop rollouts: joint-space PD and computed-torque feedback evaluated at every RK4 stage (rbd_integrate_pd, DESIGN 4.18).

The reference's ``simulate(state, final_time, control!)`` calls ``control!(τ, t, state)`` at every stage with that stage's state
(src/simulate.jl:36-55).  ``JointPD`` is the batched form of the two joint-space controllers its users write there, with the
reference's sign convention ``pd(gains, e, ė) = -k e - d ė`` (src/pdcontrol.jl:35) and e = local_coordinates!(q_ref, q):

    PD                τ = τ_ff - Kp e - Kd (v - v_ref)
    computed torque   τ = inverse_dynamics!(q, v, v̇_ref - Kp e - Kd (v - v_ref)) + τ_ff

each clamped to the effort bounds when they are given.  Pass one as ``controller=`` to ``simulate_`` / ``simulate_trajectory_``,
``simulate_contact_(trajectory_)`` or ``simulate_loops_(trajectory_)``; their ``torques`` argument is then τ_ff.

``TaskPD`` closes the loop in task space instead (rbd_integrate_task_pd, DESIGN 4.21): point and SE(3) PD on body frames, mapped
to the joints through J^T, optionally on top of a ``JointPD`` term; ``task_pd_torques`` evaluates its law at one state.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _cabi
from .state import MechanismState

__all__ = ["JointPD", "TaskPD", "task_pd_torques"]


class _RbdPdDesc(ctypes.Structure):
    _fields_ = [("mode", ctypes.c_int32), ("kp", ctypes.c_void_p), ("kd", ctypes.c_void_p), ("gain_ld", ctypes.c_int64),
                ("q_ref", ctypes.c_void_p), ("v_ref", ctypes.c_void_p), ("vd_ref", ctypes.c_void_p),
                ("q_ref_step_stride", ctypes.c_int64), ("v_ref_step_stride", ctypes.c_int64),
                ("effort_lo", ctypes.POINTER(ctypes.c_double)), ("effort_hi", ctypes.POINTER(ctypes.c_double))]


class _RbdPdBar(ctypes.Structure):
    _fields_ = [("kp", ctypes.c_void_p), ("kd", ctypes.c_void_p), ("q_ref", ctypes.c_void_p), ("v_ref", ctypes.c_void_p),
                ("vd_ref", ctypes.c_void_p)]


class JointPD:
    """Joint-space feedback for a closed-loop rollout.

    ``kp``, ``kd``: gains per velocity DoF, [nv] (shared by the batch) or [nv, B] (per sample).  ``q_ref`` [nq, B] (held over the
    call) or [nsteps, nq, B] (per step); its quaternions must be unit quaternions (they are not normalised).  ``v_ref``, and
    ``vd_ref`` (computed-torque mode only), [nv, B] or [nsteps, nv, B]; None = 0.  ``effort_bounds``: ``(lo, hi)`` arrays [nv] in
    velocity order, e.g. ``effort_bounds(mechanism)``; None = unbounded.  All tensors: the dtype and device of the state.

    ``autodiff.simulate`` / ``autodiff.simulate_contact`` take one as ``controller=`` too: gradients then also flow to those of
    ``kp``, ``kd``, ``q_ref``, ``v_ref`` and ``vd_ref`` that require grad (DESIGN 4.19); the effort bounds receive none."""

    def __init__(self, kp, kd, q_ref, v_ref=None, *, vd_ref=None, computed_torque: bool = False, effort_bounds=None):
        self.kp, self.kd, self.q_ref, self.v_ref, self.vd_ref = kp, kd, q_ref, v_ref, vd_ref
        self.computed_torque = bool(computed_torque)
        self.effort_bounds = effort_bounds
        if vd_ref is not None and not self.computed_torque:
            raise ValueError("JointPD: vd_ref is for computed-torque mode only")

    def _c_struct(self, state: MechanismState, nsteps: int, what: str):
        """(rbd_pd_desc, objects to keep alive over the call)."""
        from .algorithms import DimensionMismatch
        nq, nv, B = state.nq, state.nv, state.batch

        def tensor(t, name):
            if not isinstance(t, torch.Tensor) or t.dtype != state.dtype or t.device != state.q.device:
                raise TypeError(f"{what}: {name}: dtype/device must match the state ({state.dtype}, {state.q.device})")
            if not t.is_contiguous():
                raise TypeError(f"{what}: {name} must be contiguous")
            return t

        def ref(t, rows, name):          # -> (tensor, step stride in elements)
            if t is None:
                return None, 0
            tensor(t, name)
            if t.dim() == 2 and tuple(t.shape) == (rows, B):
                return t, 0
            if t.dim() == 3 and t.shape[0] >= nsteps and tuple(t.shape[1:]) == (rows, B):
                return t, rows * B
            raise DimensionMismatch(f"{what}: {name} has wrong size: expected ({rows}, {B}) or (nsteps, {rows}, {B}), "
                                    f"got {tuple(t.shape)}")

        kp, kd = tensor(self.kp, "kp"), tensor(self.kd, "kd")
        for t, name in ((kp, "kp"), (kd, "kd")):
            if tuple(t.shape) not in ((nv,), (nv, B)):
                raise DimensionMismatch(f"{what}: {name} has wrong size: expected ({nv},) or ({nv}, {B}), got {tuple(t.shape)}")
        if kp.shape != kd.shape:
            raise DimensionMismatch(f"{what}: kp and kd must have the same size")
        q_ref, qs = ref(self.q_ref, nq, "q_ref")
        if q_ref is None:
            raise ValueError(f"{what}: q_ref must be given")
        v_ref, vs = ref(self.v_ref, nv, "v_ref")
        vd_ref, vds = ref(self.vd_ref, nv, "vd_ref")
        if v_ref is not None and vd_ref is not None and vs != vds:
            raise DimensionMismatch(f"{what}: v_ref and vd_ref must both be held or both be per step")
        keep = [kp, kd, q_ref, v_ref, vd_ref]
        lo = hi = None
        if self.effort_bounds is not None:
            lo, hi = (np.ascontiguousarray(np.asarray(b, np.float64).reshape(-1)) for b in self.effort_bounds)
            if lo.shape != (nv,) or hi.shape != (nv,):
                raise DimensionMismatch(f"{what}: effort bounds must be two arrays of {nv} entries")
            keep += [lo, hi]
        dp = ctypes.POINTER(ctypes.c_double)
        ptr = lambda t: None if t is None else t.data_ptr()      # noqa: E731
        d = _RbdPdDesc(1 if self.computed_torque else 0, ptr(kp), ptr(kd), B if kp.dim() == 2 else 0, ptr(q_ref), ptr(v_ref),
                       ptr(vd_ref), qs, vs or vds, None if lo is None else lo.ctypes.data_as(dp),
                       None if hi is None else hi.ctypes.data_as(dp))
        return d, keep

    def _steps_from(self, first: int) -> "JointPD":
        """The controller of a rollout that starts at step ``first`` of this one (per-step references sliced)."""
        cut = lambda t: t if t is None or t.dim() == 2 else t[first:]      # noqa: E731
        return JointPD(self.kp, self.kd, cut(self.q_ref), cut(self.v_ref), vd_ref=cut(self.vd_ref), computed_torque=self.computed_torque,
                       effort_bounds=self.effort_bounds)


class _RbdTaskPdDesc(ctypes.Structure):
    _fields_ = [("mode", ctypes.c_int32), ("tasks", _cabi.RbdTaskDesc), ("kind", ctypes.POINTER(ctypes.c_int32)),
                ("kp", ctypes.c_void_p), ("kd", ctypes.c_void_p), ("gain_ld", ctypes.c_int64),
                ("x_ref", ctypes.c_void_p), ("x_ref_step_stride", ctypes.c_int64),
                ("xd_ref", ctypes.c_void_p), ("xd_ref_step_stride", ctypes.c_int64),
                ("joint", ctypes.POINTER(_RbdPdDesc)),
                ("effort_lo", ctypes.POINTER(ctypes.c_double)), ("effort_hi", ctypes.POINTER(ctypes.c_double))]


class _RbdTaskPdBar(ctypes.Structure):
    _fields_ = [("kp", ctypes.c_void_p), ("kd", ctypes.c_void_p), ("x_ref", ctypes.c_void_p), ("xd_ref", ctypes.c_void_p),
                ("joint", ctypes.POINTER(_RbdPdBar))]


_KINDS = {"point": 0, "pose": 1}


class TaskPD:
    """Task-space feedback for a closed-loop rollout: up to 32 tasks, each a ``TaskFrame`` and a kind, evaluated at every RK4 stage.

    ``kinds``: "point" (3 rows: the task's point relative to ``base``, in ``base`` coordinates, with gains per axis of the task's
    ``frame``) or "pose" (6 rows [angular; linear]: the frame at the task's point with the body's axes, relative to ``base``, with
    the reference's double-geodesic SE(3) PD and gains in that frame; ``frame`` must be None or the body).  Each task adds
    J_t^T f_t with f_t = -Kp e - Kd ė in its task frame.  ``kp``, ``kd``: [R] (shared) or [R, B] (per sample), R = Σ 3 | 6 in task
    order.  ``x_ref``: [X, B] (held) or [nsteps, X, B] (per step), X = Σ 3 | 12, a pose target in the layout of
    ``relative_transform`` (rotation row-major, then translation; the rotation must be orthonormal).  ``xd_ref``: [R, B] or
    [nsteps, R, B], None = 0 -- the target point velocity in ``base`` coordinates, or the target twist of the pose frame in that frame.
    ``joint``: a ``JointPD`` added in the same mode (its own ``effort_bounds`` must be None), e.g. posture or damping.
    ``computed_torque``: v̇_des = joint term + Σ J^T f, τ = inverse_dynamics!(q, v, v̇_des) + τ_ff; otherwise τ = τ_ff + joint term +
    Σ J^T f.  ``effort_bounds`` clamp the sum.

    ``autodiff.simulate`` / ``autodiff.simulate_contact`` take one as ``controller=`` too: gradients then also flow to those of
    ``kp``, ``kd``, ``x_ref``, ``xd_ref`` and of the joint term's arrays that require grad (DESIGN 4.22); the task points and the
    effort bounds receive none."""

    def __init__(self, tasks, kinds, kp, kd, x_ref, xd_ref=None, *, joint=None, computed_torque: bool = False, effort_bounds=None):
        self.tasks, self.kinds = list(tasks), list(kinds)
        self.kp, self.kd, self.x_ref, self.xd_ref = kp, kd, x_ref, xd_ref
        self.joint, self.computed_torque, self.effort_bounds = joint, bool(computed_torque), effort_bounds
        if len(self.kinds) != len(self.tasks):
            raise ValueError("TaskPD: one kind per task")
        for t, k in zip(self.tasks, self.kinds):
            if k not in _KINDS:
                raise ValueError(f"TaskPD: unknown task kind {k!r} (expected 'point' or 'pose')")
            if k == "pose" and t.frame is not None and t.frame is not t.body:
                raise ValueError("TaskPD: a pose task is expressed in its own body's frame (frame=None or the body)")
        if joint is not None:
            if not isinstance(joint, JointPD):
                raise TypeError("TaskPD: joint must be a JointPD")
            if joint.computed_torque != self.computed_torque:
                raise ValueError("TaskPD: the joint term must have the controller's mode")
            if joint.effort_bounds is not None:
                raise ValueError("TaskPD: the joint term's effort_bounds must be None (the controller's bounds clamp the sum)")

    def rows(self):
        """(R, X): gain / velocity rows and target rows."""
        return (sum(3 if k == "point" else 6 for k in self.kinds), sum(3 if k == "point" else 12 for k in self.kinds))

    def _c_struct(self, state: MechanismState, nsteps: int, what: str):
        """(rbd_task_pd_desc, objects to keep alive over the call)."""
        from .algorithms import DimensionMismatch
        from .kinematics import TaskFrame, task_desc
        B = state.batch
        R, X = self.rows()

        def ref(t, rows, name):          # -> (tensor, step stride in elements)
            if t is None:
                return None, 0
            if not isinstance(t, torch.Tensor) or t.dtype != state.dtype or t.device != state.q.device:
                raise TypeError(f"{what}: {name}: dtype/device must match the state ({state.dtype}, {state.q.device})")
            if not t.is_contiguous():
                raise TypeError(f"{what}: {name} must be contiguous")
            if t.dim() == 2 and tuple(t.shape) == (rows, B):
                return t, 0
            if t.dim() == 3 and t.shape[0] >= nsteps and tuple(t.shape[1:]) == (rows, B):
                return t, rows * B
            raise DimensionMismatch(f"{what}: {name} has wrong size: expected ({rows}, {B}) or (nsteps, {rows}, {B}), "
                                    f"got {tuple(t.shape)}")

        for t, name in ((self.kp, "kp"), (self.kd, "kd")):
            if not isinstance(t, torch.Tensor) or t.dtype != state.dtype or t.device != state.q.device:
                raise TypeError(f"{what}: {name}: dtype/device must match the state ({state.dtype}, {state.q.device})")
            if not t.is_contiguous():
                raise TypeError(f"{what}: {name} must be contiguous")
            if tuple(t.shape) not in ((R,), (R, B)):
                raise DimensionMismatch(f"{what}: {name} has wrong size: expected ({R},) or ({R}, {B}), got {tuple(t.shape)}")
        if self.kp.shape != self.kd.shape:
            raise DimensionMismatch(f"{what}: kp and kd must have the same size")
        x_ref, xs = ref(self.x_ref, X, "x_ref")
        if x_ref is None:
            raise ValueError(f"{what}: x_ref must be given")
        xd_ref, xds = ref(self.xd_ref, R, "xd_ref")
        # a pose task's frame is its body (None in the TaskFrame means the body here)
        tasks = [TaskFrame(t.body, t.base, t.point, t.body if k == "pose" else t.frame) for t, k in zip(self.tasks, self.kinds)]
        td, keep_t = task_desc(state.mechanism, tasks)
        kind = np.array([_KINDS[k] for k in self.kinds], np.int32)
        keep = [self.kp, self.kd, x_ref, xd_ref, keep_t, kind]
        joint = None
        if self.joint is not None:
            joint, keep_j = self.joint._c_struct(state, nsteps, what)
            keep += [joint, keep_j]
        lo = hi = None
        if self.effort_bounds is not None:
            lo, hi = (np.ascontiguousarray(np.asarray(b, np.float64).reshape(-1)) for b in self.effort_bounds)
            if lo.shape != (state.nv,) or hi.shape != (state.nv,):
                raise DimensionMismatch(f"{what}: effort bounds must be two arrays of {state.nv} entries")
            keep += [lo, hi]
        dp = ctypes.POINTER(ctypes.c_double)
        ptr = lambda t: None if t is None else t.data_ptr()      # noqa: E731
        d = _RbdTaskPdDesc(1 if self.computed_torque else 0, td, kind.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
                           ptr(self.kp), ptr(self.kd), B if self.kp.dim() == 2 else 0, ptr(x_ref), xs, ptr(xd_ref), xds,
                           None if joint is None else ctypes.pointer(joint), None if lo is None else lo.ctypes.data_as(dp),
                           None if hi is None else hi.ctypes.data_as(dp))
        return d, keep

    def _steps_from(self, first: int) -> "TaskPD":
        """The controller of a rollout that starts at step ``first`` of this one (per-step references sliced)."""
        cut = lambda t: t if t is None or t.dim() == 2 else t[first:]      # noqa: E731
        return TaskPD(self.tasks, self.kinds, self.kp, self.kd, cut(self.x_ref), cut(self.xd_ref),
                      joint=None if self.joint is None else self.joint._steps_from(first), computed_torque=self.computed_torque,
                      effort_bounds=self.effort_bounds)


def task_pd_torques(state: MechanismState, controller: TaskPD, torques=None, step: int = 0):
    """The torques ``controller`` applies at ``state`` (q, v) with the references of step ``step`` and feedforward ``torques``
    ([nv, B] or None): the batched ``control!`` of a task-space controller for callers that step their own loop (the reference's
    examples/4).  Returns a new [nv, B] tensor."""
    from .algorithms import _call, _check, _ptr, _require_tree, _stream
    from ._cabi import load_library
    from .state import _DT
    if not isinstance(controller, TaskPD):
        raise TypeError("task_pd_torques: controller must be a TaskPD")
    if controller.computed_torque:
        _require_tree(state, "task_pd_torques")
    state.check_modcount()
    _check(torques, state.nv, state, "torques")
    if step < 0:
        raise ValueError("task_pd_torques: step must be >= 0")
    d, keep = controller._c_struct(state, step + 1, "task_pd_torques")
    out = torch.empty_like(state.v)
    _call(load_library().rbd_task_pd_torques(state.handle.ptr, _DT[state.dtype], state.batch, state.batch, _ptr(state.q),
                                             _ptr(state.v), _ptr(torques), ctypes.byref(d), int(step), _ptr(out), _stream()))
    return out
