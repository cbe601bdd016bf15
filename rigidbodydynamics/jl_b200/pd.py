"""Closed-loop rollouts: joint-space PD and computed-torque feedback evaluated at every RK4 stage (rbd_integrate_pd, DESIGN 4.18).

The reference's ``simulate(state, final_time, control!)`` calls ``control!(τ, t, state)`` at every stage with that stage's state
(src/simulate.jl:36-55).  ``JointPD`` is the batched form of the two joint-space controllers its users write there, with the
reference's sign convention ``pd(gains, e, ė) = -k e - d ė`` (src/pdcontrol.jl:35) and e = local_coordinates!(q_ref, q):

    PD                τ = τ_ff - Kp e - Kd (v - v_ref)
    computed torque   τ = inverse_dynamics!(q, v, v̇_ref - Kp e - Kd (v - v_ref)) + τ_ff

each clamped to the effort bounds when they are given.  Pass one as ``controller=`` to ``simulate_`` / ``simulate_trajectory_``,
``simulate_contact_(trajectory_)`` or ``simulate_loops_(trajectory_)``; their ``torques`` argument is then τ_ff.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from .state import MechanismState

__all__ = ["JointPD"]


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
