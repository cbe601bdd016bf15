"""Reverse mode: vector-Jacobian products of ``dynamics!`` and ``inverse_dynamics!``, and ``torch.autograd`` functions built on them.

    dynamics_vjp_          ν̄ᵀ ∂v̇/∂(q, v, τ, w_ext)        rbd_dynamics_vjp          (include/rbd_b200.h, csrc/rbd_adjoint.cuh)
    inverse_dynamics_vjp_  τ̄ᵀ ∂τ/∂(q, v, v̇, w_ext)         rbd_inverse_dynamics_vjp
    integrate_vjp_         gradient of a recorded rollout       rbd_integrate_vjp         (csrc/rbd_integrate_adjoint.cuh)
    integrate_derivatives_ Jacobians ∂x_{s+1}/∂(x_s, τ_s) of every recorded step  rbd_integrate_derivatives  (csrc/rbd_integrate_deriv.cuh)
    integrate_contact_vjp_ gradient of a recorded contact rollout  rbd_integrate_contact_vjp  (csrc/rbd_contact_adjoint.cuh)
    integrate_pd_vjp_      gradient of a recorded closed-loop rollout  rbd_integrate_pd_vjp  (csrc/rbd_integrate_adjoint.cuh)
    integrate_task_pd_vjp_ gradient of a recorded task-space closed-loop rollout  rbd_integrate_task_pd_vjp  (csrc/rbd_task_pd_adjoint.cuh)
    task_pd_torques_vjp_   τ̄ᵀ ∂τ/∂(q, v, τ_ff, controller) of a TaskPD's torques at one state  rbd_task_pd_torques_vjp
    task_kinematics_vjp_   Σ ȳᵀ ∂y/∂(q, v, v̇) of task-space outputs  rbd_task_kinematics_vjp  (csrc/rbd_task_adjoint.cuh)
    kinematics_vjp_        Σ ȳᵀ ∂y/∂(q, v) of whole-body kinematics outputs  rbd_kinematics_vjp  (csrc/rbd_kin_adjoint.cuh)
    dynamics(mechanism, q, v, tau=None, externalwrenches=None)         differentiable v̇ = dynamics!(...)
    inverse_dynamics(mechanism, q, v, vd, externalwrenches=None)       differentiable τ = inverse_dynamics!(...)
    simulate(mechanism, q0, v0, torques=None, *, dt, nsteps, ...)     differentiable RK4 rollout (simulate)
    simulate_contact(mechanism, q0, v0, s0, torques=None, *, contact, dt, nsteps, ...)
                                                                       differentiable RK4 rollout with soft contact
    both with controller=JointPD(...) or TaskPD(...): closed loop, gradients also to the controller's gains and references
    task_kinematics(mechanism, q, v=None, vd=None, *, tasks, outputs=("point",))
                                                                       differentiable task-space kinematics (TaskFrame tasks)
    task_pd_torques(state, controller, torques=None, step=0)          differentiable torques of a TaskPD at one state
    kinematics(mechanism, q, v=None, *, outputs=("center_of_mass",), path=None)
                                                                       differentiable whole-body kinematics (centre of mass,
                                                                       energies, momentum, momentum matrix, ...)

One product costs one Articulated-Body solve (forward dynamics only) plus one outward and one inward sweep: O(n) per sample, no
nv x nv Jacobian is formed (``dynamics_derivatives_`` builds both full Jacobians instead).  Every tensor is ``[rows, B]``, contiguous,
CUDA, float32 or float64, batch index fastest.

Configuration gradients come in two coordinates.  ``q_bar_tan`` [nv, B] is the derivative along
``velocity_to_configuration_derivative(e_j)`` -- the convention of ``dynamics_derivatives_``'s ``dvd_dq`` columns.  ``q_bar_cfg``
[nq, B] is that covector mapped like the reference's ``configuration_derivative_to_velocity_adjoint!``
(mechanism_state.jl:912-918): ``q_bar_cfg · (N(q) u) == q_bar_tan · u`` for every u.  It is what autograd returns for ``q``.  For
quaternion joints it has no component along q itself: the derivative of the unnormalised rotation formula in that radial direction
depends on how the formula extends off the unit sphere, and a gradient should not depend on it.
"""
from __future__ import annotations

import ctypes
from types import SimpleNamespace
from typing import Dict, Optional, Sequence

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from . import _cabi
from .algorithms import DimensionMismatch, _check, _ptr, _require_tree
from .kinematics import _NEEDS_V, _ROWS, _TASK_NEEDS_V, _TASK_ROWS, TaskFrame, TreePath, task_desc
from .mechanism import Mechanism
from .state import _DT, MechanismState, _model_handle

__all__ = ["dynamics_vjp_", "inverse_dynamics_vjp_", "integrate_vjp_", "integrate_derivatives_", "integrate_derivatives", "integrate_contact_vjp_", "integrate_pd_vjp_", "integrate_task_pd_vjp_",
           "task_pd_torques_vjp_", "task_pd_torques", "dynamics",
           "inverse_dynamics", "simulate", "simulate_contact", "task_kinematics_vjp_", "task_kinematics", "kinematics_vjp_", "kinematics"]


def _stream(t: torch.Tensor):
    return torch.cuda.current_stream(t.device).cuda_stream


def dynamics_vjp_(state: MechanismState, vd: torch.Tensor, vd_bar: torch.Tensor, torques: Optional[torch.Tensor] = None,
                  externalwrenches: Optional[torch.Tensor] = None, *, q_bar_tan: Optional[torch.Tensor] = None,
                  q_bar_cfg: Optional[torch.Tensor] = None, v_bar: Optional[torch.Tensor] = None,
                  tau_bar: Optional[torch.Tensor] = None, wext_bar: Optional[torch.Tensor] = None):
    """The product ``ν̄ᵀ ∂v̇/∂(q, v, τ, w_ext)`` of ``dynamics!(result, state, torques, externalwrenches)`` for every sample.

    ``vd`` [nv, B] must be ``dynamics_``'s v̇ for the same state, torques and wrenches: the product is evaluated there and v̇ is not
    recomputed.  ``vd_bar`` [nv, B] is ν̄.  Outputs (each optional, filled in place): ``q_bar_tan`` [nv, B], ``q_bar_cfg`` [nq, B],
    ``v_bar`` [nv, B], ``tau_bar`` [nv, B] (= M⁻¹ν̄), ``wext_bar`` [6 nb, B] (rows 6i..6i+5: the root-frame twist [angular; linear] of
    the successor of tree joint i under the joint velocities M⁻¹ν̄)."""
    _require_tree(state, "dynamics_vjp_")
    state.check_modcount()
    lib = _cabi.load_library()
    nv, nq, nb6 = state.nv, state.nq, 6 * len(state.mechanism.joints)
    for t, rows, name in ((vd, nv, "vd"), (vd_bar, nv, "vd_bar"), (torques, nv, "torques"), (externalwrenches, nb6, "externalwrenches"),
                          (q_bar_tan, nv, "q_bar_tan"), (q_bar_cfg, nq, "q_bar_cfg"), (v_bar, nv, "v_bar"), (tau_bar, nv, "tau_bar"),
                          (wext_bar, nb6, "wext_bar")):
        _check(t, rows, state, name)
    if vd is None or vd_bar is None:
        raise ValueError("vd and vd_bar must be given")
    _cabi.check(lib.rbd_dynamics_vjp(state.handle.ptr, _DT[state.dtype], state.batch, state.batch, _ptr(state.q), _ptr(state.v),
                                     _ptr(torques), _ptr(externalwrenches), _ptr(vd), _ptr(vd_bar), _ptr(q_bar_tan), _ptr(q_bar_cfg),
                                     _ptr(v_bar), _ptr(tau_bar), _ptr(wext_bar), _stream(state.q)))


def inverse_dynamics_vjp_(state: MechanismState, vd: torch.Tensor, tau_bar: torch.Tensor,
                          externalwrenches: Optional[torch.Tensor] = None, *, q_bar_tan: Optional[torch.Tensor] = None,
                          q_bar_cfg: Optional[torch.Tensor] = None, v_bar: Optional[torch.Tensor] = None,
                          vd_bar: Optional[torch.Tensor] = None, wext_bar: Optional[torch.Tensor] = None):
    """The product ``τ̄ᵀ ∂τ/∂(q, v, v̇, w_ext)`` of ``inverse_dynamics!(τ, state, v̇, externalwrenches)`` for every sample.

    Outputs (each optional): ``q_bar_tan`` [nv, B], ``q_bar_cfg`` [nq, B], ``v_bar`` [nv, B], ``vd_bar`` [nv, B] (= M τ̄),
    ``wext_bar`` [6 nb, B] (MINUS the root-frame twist of each body under the joint velocities τ̄: wrenches are subtracted in
    ``newton_euler!``)."""
    _require_tree(state, "inverse_dynamics_vjp_")
    state.check_modcount()
    lib = _cabi.load_library()
    nv, nq, nb6 = state.nv, state.nq, 6 * len(state.mechanism.joints)
    for t, rows, name in ((vd, nv, "vd"), (tau_bar, nv, "tau_bar"), (externalwrenches, nb6, "externalwrenches"),
                          (q_bar_tan, nv, "q_bar_tan"), (q_bar_cfg, nq, "q_bar_cfg"), (v_bar, nv, "v_bar"), (vd_bar, nv, "vd_bar"),
                          (wext_bar, nb6, "wext_bar")):
        _check(t, rows, state, name)
    if vd is None or tau_bar is None:
        raise ValueError("vd and tau_bar must be given")
    _cabi.check(lib.rbd_inverse_dynamics_vjp(state.handle.ptr, _DT[state.dtype], state.batch, state.batch, _ptr(state.q),
                                             _ptr(state.v), _ptr(vd), _ptr(externalwrenches), _ptr(tau_bar), _ptr(q_bar_tan),
                                             _ptr(q_bar_cfg), _ptr(v_bar), _ptr(vd_bar), _ptr(wext_bar), _stream(state.q)))


# ----------------------------------------------------------------------------------------------------------------------
# torch.autograd
# ----------------------------------------------------------------------------------------------------------------------
def _inputs(mechanism: Mechanism, what: str, **tensors):
    """Checks of the differentiable functions: a tree mechanism, [rows, B] contiguous CUDA fp32 / fp64 tensors of one dtype and device.
    Returns (model handle, B)."""
    if mechanism.has_loops():
        raise _cabi.RbdError(_cabi.RBD_ELOOP, f"{what}: This method can currently only handle tree Mechanisms.")
    h = _model_handle(mechanism)
    rows = {"q": h.info.nq, "v": h.info.nv, "vd": h.info.nv, "tau": h.info.nv, "externalwrenches": 6 * h.info.nb}
    q = tensors["q"]
    if q.dtype not in _DT or not q.is_cuda:
        raise TypeError(f"{what}: q must be a float32 / float64 CUDA tensor")
    if q.dim() != 2:
        raise DimensionMismatch(f"{what}: q must be [nq, B]")
    B = q.shape[1]
    for name, t in tensors.items():
        if t is None:
            continue
        if t.dtype != q.dtype or t.device != q.device:
            raise TypeError(f"{what}: {name} must have the dtype and device of q")
        if t.dim() != 2 or tuple(t.shape) != (rows[name], B):
            raise DimensionMismatch(f"{what}: {name} has wrong size: expected ({rows[name]}, {B}), got {tuple(t.shape)}")
        if not t.is_contiguous():
            raise ValueError(f"{what}: {name} must be [rows, B] contiguous (batch index fastest)")
    return h, B


def _out(needed: bool, like: torch.Tensor, rows: int):
    return torch.empty((rows, like.shape[1]), dtype=like.dtype, device=like.device) if needed else None


class _Dynamics(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mechanism, q, v, tau, wext):
        h, B = _inputs(mechanism, "autodiff.dynamics", q=q, v=v, tau=tau, externalwrenches=wext)
        lib = _cabi.load_library()
        vd = torch.empty((h.info.nv, B), dtype=q.dtype, device=q.device)
        if B:
            _cabi.check(lib.rbd_dynamics(h.ptr, _DT[q.dtype], B, B, _ptr(q), _ptr(v), _ptr(tau), _ptr(wext), _ptr(vd), None, _stream(q)))
        ctx.handle, ctx.nb = h, h.info.nb
        ctx.save_for_backward(q, v, tau, wext, vd)
        return vd

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        q, v, tau, wext, vd = ctx.saved_tensors
        h = ctx.handle
        need = ctx.needs_input_grad
        g = g.contiguous()
        qb, vb = _out(need[1], q, q.shape[0]), _out(need[2], v, v.shape[0])
        tb = _out(need[3] and tau is not None, v, v.shape[0])
        wb = _out(need[4] and wext is not None, q, 6 * ctx.nb)
        B = q.shape[1]
        if B and any(t is not None for t in (qb, vb, tb, wb)):
            _cabi.check(_cabi.load_library().rbd_dynamics_vjp(h.ptr, _DT[q.dtype], B, B, _ptr(q), _ptr(v), _ptr(tau), _ptr(wext), _ptr(vd),
                                                              _ptr(g), None, _ptr(qb), _ptr(vb), _ptr(tb), _ptr(wb), _stream(q)))
        return None, qb, vb, tb, wb


class _InverseDynamics(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mechanism, q, v, vd, wext):
        h, B = _inputs(mechanism, "autodiff.inverse_dynamics", q=q, v=v, vd=vd, externalwrenches=wext)
        lib = _cabi.load_library()
        tau = torch.empty((h.info.nv, B), dtype=q.dtype, device=q.device)
        if B:
            _cabi.check(lib.rbd_inverse_dynamics(h.ptr, _DT[q.dtype], B, B, _ptr(q), _ptr(v), _ptr(vd), _ptr(wext), _ptr(tau), _stream(q)))
        ctx.handle, ctx.nb = h, h.info.nb
        ctx.save_for_backward(q, v, vd, wext)
        return tau

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        q, v, vd, wext = ctx.saved_tensors
        h = ctx.handle
        need = ctx.needs_input_grad
        g = g.contiguous()
        qb, vb, ab = _out(need[1], q, q.shape[0]), _out(need[2], v, v.shape[0]), _out(need[3], v, v.shape[0])
        wb = _out(need[4] and wext is not None, q, 6 * ctx.nb)
        B = q.shape[1]
        if B and any(t is not None for t in (qb, vb, ab, wb)):
            _cabi.check(_cabi.load_library().rbd_inverse_dynamics_vjp(h.ptr, _DT[q.dtype], B, B, _ptr(q), _ptr(v), _ptr(vd), _ptr(wext),
                                                                      _ptr(g), None, _ptr(qb), _ptr(vb), _ptr(ab), _ptr(wb), _stream(q)))
        return None, qb, vb, ab, wb


def dynamics(mechanism: Mechanism, q: torch.Tensor, v: torch.Tensor, tau: Optional[torch.Tensor] = None,
             externalwrenches: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Differentiable ``v̇ = dynamics!(result, state, tau, externalwrenches)`` for q [nq, B], v [nv, B], tau [nv, B] or None (zero),
    externalwrenches [6 nb, B] or None.  Backward runs ``rbd_dynamics_vjp`` for the inputs that need a gradient; the gradient of
    ``q`` is ``q_bar_cfg`` (see the module docstring).  Backward is not itself differentiable: a double backward raises."""
    return _Dynamics.apply(mechanism, q, v, tau, externalwrenches)


def inverse_dynamics(mechanism: Mechanism, q: torch.Tensor, v: torch.Tensor, vd: torch.Tensor,
                     externalwrenches: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Differentiable ``τ = inverse_dynamics!(τ, state, v̇, externalwrenches)``; backward runs ``rbd_inverse_dynamics_vjp``.  Not
    twice differentiable."""
    return _InverseDynamics.apply(mechanism, q, v, vd, externalwrenches)


# ----------------------------------------------------------------------------------------------------------------------
# task-space kinematics: rbd_task_kinematics / rbd_task_kinematics_vjp
# ----------------------------------------------------------------------------------------------------------------------
def _task_out(tensors: Dict[str, Optional[torch.Tensor]], K: int, nv: int, like: torch.Tensor, what: str) -> _cabi.RbdTaskOut:
    """rbd_task_out for {output: [rows * K, B] tensor or None}, checked against the dtype, device and batch of ``like``."""
    to = _cabi.RbdTaskOut()
    for name, t in tensors.items():
        if name not in _TASK_ROWS:
            raise TypeError(f"{what}: unknown task kinematics output {name!r}")
        if t is None:
            continue
        rows = _TASK_ROWS[name](SimpleNamespace(nv=nv))
        if t.dtype != like.dtype or t.device != like.device:
            raise TypeError(f"{what}: {name} must have the dtype and device of q")
        if t.dim() != 2 or tuple(t.shape) != (rows * K, like.shape[1]):
            raise DimensionMismatch(f"{what}: {name} has wrong size: expected ({rows * K}, {like.shape[1]}), got {tuple(t.shape)}")
        if not t.is_contiguous():
            raise ValueError(f"{what}: {name} must be [rows, B] contiguous (batch index fastest)")
        setattr(to, name, t.data_ptr())
    return to


def task_kinematics_vjp_(state: MechanismState, tasks: Sequence[TaskFrame], vd: Optional[torch.Tensor] = None, *, bars: dict,
                         q_bar_tan: Optional[torch.Tensor] = None, q_bar_cfg: Optional[torch.Tensor] = None,
                         v_bar: Optional[torch.Tensor] = None, vd_bar: Optional[torch.Tensor] = None):
    """The product ``Σ ȳᵀ ∂y/∂(q, v, v̇)`` of ``task_kinematics_(state, tasks, vd, ...)`` for every sample.

    ``bars``: {output name: ȳ} with each ȳ in that output's layout ([rows * len(tasks), B]); missing outputs have zero cotangent.
    Everything is recomputed from the state and ``vd`` (None = zero).  Outputs (each optional, overwritten): ``q_bar_tan`` [nv, B],
    ``q_bar_cfg`` [nq, B], ``v_bar`` [nv, B], ``vd_bar`` [nv, B] (see the module docstring for the two configuration covectors)."""
    state.check_modcount()
    lib = _cabi.load_library()
    to = _task_out(bars, len(tasks), state.nv, state.q, "task_kinematics_vjp_")
    for t, rows, name in ((vd, state.nv, "vd"), (q_bar_tan, state.nv, "q_bar_tan"), (q_bar_cfg, state.nq, "q_bar_cfg"),
                          (v_bar, state.nv, "v_bar"), (vd_bar, state.nv, "vd_bar")):
        _check(t, rows, state, name)
    d, keep = task_desc(state.mechanism, tasks)
    _cabi.check(lib.rbd_task_kinematics_vjp(state.handle.ptr, _DT[state.dtype], state.batch, state.batch, _ptr(state.q),
                                            _ptr(state.v), _ptr(vd), ctypes.byref(d), ctypes.byref(to), _ptr(q_bar_tan),
                                            _ptr(q_bar_cfg), _ptr(v_bar), _ptr(vd_bar), _stream(state.q)))


class _TaskKinematics(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mechanism, tasks, outputs, q, v, vd):
        h, B = _inputs(mechanism, "autodiff.task_kinematics", q=q, v=v, vd=vd)
        if v is None and any(k in _TASK_NEEDS_V for k in outputs):
            raise ValueError(f"autodiff.task_kinematics: {', '.join(k for k in outputs if k in _TASK_NEEDS_V)} need v")
        K, nv = len(tasks), h.info.nv
        outs = {k: torch.empty((_TASK_ROWS[k](SimpleNamespace(nv=nv)) * K, B), dtype=q.dtype, device=q.device) for k in outputs}
        to = _task_out(outs, K, nv, q, "autodiff.task_kinematics")
        d, keep = task_desc(mechanism, tasks)
        if B and K:
            _cabi.check(_cabi.load_library().rbd_task_kinematics(h.ptr, _DT[q.dtype], B, B, _ptr(q), _ptr(v), _ptr(vd), ctypes.byref(d),
                                                                 ctypes.byref(to), _stream(q)))
        ctx.handle, ctx.mechanism, ctx.tasks, ctx.outputs = h, mechanism, tasks, outputs
        ctx.save_for_backward(q, v, vd)
        return tuple(outs[k] for k in outputs)

    @staticmethod
    @once_differentiable
    def backward(ctx, *grads):
        q, v, vd = ctx.saved_tensors
        h = ctx.handle
        need = ctx.needs_input_grad
        qb = _out(need[3], q, q.shape[0])
        vb = _out(need[4] and v is not None, q, h.info.nv)
        ab = _out(need[5] and vd is not None, q, h.info.nv)
        bars = {k: g.contiguous() for k, g in zip(ctx.outputs, grads) if g is not None}
        B = q.shape[1]
        if B and any(t is not None for t in (qb, vb, ab)):
            to = _task_out(bars, len(ctx.tasks), h.info.nv, q, "autodiff.task_kinematics")
            d, keep = task_desc(ctx.mechanism, ctx.tasks)
            _cabi.check(_cabi.load_library().rbd_task_kinematics_vjp(h.ptr, _DT[q.dtype], B, B, _ptr(q), _ptr(v), _ptr(vd),
                                                                     ctypes.byref(d), ctypes.byref(to), None, _ptr(qb), _ptr(vb),
                                                                     _ptr(ab), _stream(q)))
        return None, None, None, qb, vb, ab


def task_kinematics(mechanism: Mechanism, q: torch.Tensor, v: Optional[torch.Tensor] = None, vd: Optional[torch.Tensor] = None, *,
                    tasks: Sequence[TaskFrame], outputs: Sequence[str] = ("point",)) -> Dict[str, torch.Tensor]:
    """Differentiable task-space kinematics: {name: [rows * len(tasks), B]} for the requested ``outputs`` (names and layout of
    ``task_kinematics_``) of q [nq, B], v [nv, B] (needed by twist / point_velocity / acceleration / point_acceleration) and vd
    [nv, B] or None (zero).  Forward is one ``rbd_task_kinematics`` call for all outputs; backward one ``rbd_task_kinematics_vjp``
    with the incoming gradients.  The gradient of ``q`` is ``q_bar_cfg`` (see the module docstring).  Not twice differentiable."""
    tasks, outputs = tuple(tasks), tuple(outputs)
    for k in outputs:
        if k not in _TASK_ROWS:
            raise TypeError(f"autodiff.task_kinematics: unknown task kinematics output {k!r}")
    if len(set(outputs)) != len(outputs):
        raise ValueError("autodiff.task_kinematics: outputs must be distinct")
    return dict(zip(outputs, _TaskKinematics.apply(mechanism, tasks, outputs, q, v, vd)))


# ----------------------------------------------------------------------------------------------------------------------
# whole-body kinematics: rbd_kinematics / rbd_kinematics_vjp
# ----------------------------------------------------------------------------------------------------------------------
def _kin_out(tensors: Dict[str, Optional[torch.Tensor]], nb: int, nv: int, like: torch.Tensor, what: str) -> _cabi.RbdKinematicsOut:
    """rbd_kinematics_out for {output: [rows, B] tensor or None}, checked against the dtype, device and batch of ``like``."""
    ko = _cabi.RbdKinematicsOut()
    dims = SimpleNamespace(nv=nv, mechanism=SimpleNamespace(joints=range(nb)))
    for name, t in tensors.items():
        if name not in _ROWS:
            raise TypeError(f"{what}: unknown kinematics output {name!r}")
        if t is None:
            continue
        rows = _ROWS[name](dims)
        if t.dtype != like.dtype or t.device != like.device:
            raise TypeError(f"{what}: {name} must have the dtype and device of q")
        if t.dim() != 2 or tuple(t.shape) != (rows, like.shape[1]):
            raise DimensionMismatch(f"{what}: {name} has wrong size: expected ({rows}, {like.shape[1]}), got {tuple(t.shape)}")
        if not t.is_contiguous():
            raise ValueError(f"{what}: {name} must be [rows, B] contiguous (batch index fastest)")
        setattr(ko, name, t.data_ptr())
    return ko


def _path_sign(path_: Optional[TreePath], want_jac: bool, nb: int):
    """The host int8 array of ``path_``'s signs, or None without a geometric Jacobian (the messages of ``kinematics_``)."""
    if not want_jac:
        return None
    if path_ is None:
        raise ValueError("geometric_jacobian needs a path")
    sign = np.ascontiguousarray(path_.sign, np.int8)
    if sign.shape != (nb,):
        raise DimensionMismatch("path does not belong to this mechanism")
    return sign


def _sign_ptr(sign):
    return None if sign is None else sign.ctypes.data_as(ctypes.c_void_p)


def kinematics_vjp_(state: MechanismState, path_: Optional[TreePath] = None, *, bars: dict, q_bar_tan: Optional[torch.Tensor] = None,
                    q_bar_cfg: Optional[torch.Tensor] = None, v_bar: Optional[torch.Tensor] = None):
    """The product ``Σ ȳᵀ ∂y/∂(q, v)`` of ``kinematics_(state, path_, ...)`` for every sample.

    ``bars``: {output name: ȳ} with the names and layouts of ``kinematics_``; missing outputs have zero cotangent, and a
    ``geometric_jacobian`` cotangent needs ``path_``.  Everything is recomputed from the state.  Outputs (each optional, overwritten):
    ``q_bar_tan`` [nv, B], ``q_bar_cfg`` [nq, B], ``v_bar`` [nv, B] (see the module docstring for the two configuration covectors)."""
    state.check_modcount()
    lib = _cabi.load_library()
    nb = len(state.mechanism.joints)
    ko = _kin_out(bars, nb, state.nv, state.q, "kinematics_vjp_")
    for t, rows, name in ((q_bar_tan, state.nv, "q_bar_tan"), (q_bar_cfg, state.nq, "q_bar_cfg"), (v_bar, state.nv, "v_bar")):
        _check(t, rows, state, name)
    sign = _path_sign(path_, bars.get("geometric_jacobian") is not None, nb)
    _cabi.check(lib.rbd_kinematics_vjp(state.handle.ptr, _DT[state.dtype], state.batch, state.batch, _ptr(state.q), _ptr(state.v),
                                       _sign_ptr(sign), ctypes.byref(ko), _ptr(q_bar_tan), _ptr(q_bar_cfg), _ptr(v_bar),
                                       _stream(state.q)))


class _Kinematics(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mechanism, outputs, sign, q, v):
        h, B = _inputs(mechanism, "autodiff.kinematics", q=q, v=v)
        if v is None and any(k in _NEEDS_V for k in outputs):
            raise ValueError(f"autodiff.kinematics: {', '.join(k for k in outputs if k in _NEEDS_V)} need v")
        nb, nv = h.info.nb, h.info.nv
        dims = SimpleNamespace(nv=nv, mechanism=SimpleNamespace(joints=range(nb)))
        outs = {k: torch.empty((_ROWS[k](dims), B), dtype=q.dtype, device=q.device) for k in outputs}
        ko = _kin_out(outs, nb, nv, q, "autodiff.kinematics")
        if B and outputs:
            _cabi.check(_cabi.load_library().rbd_kinematics(h.ptr, _DT[q.dtype], B, B, _ptr(q), _ptr(v), _sign_ptr(sign),
                                                            ctypes.byref(ko), _stream(q)))
        ctx.handle, ctx.outputs, ctx.sign = h, outputs, sign
        ctx.save_for_backward(q, v)
        return tuple(outs[k] for k in outputs)

    @staticmethod
    @once_differentiable
    def backward(ctx, *grads):
        q, v = ctx.saved_tensors
        h = ctx.handle
        need = ctx.needs_input_grad
        qb = _out(need[3], q, q.shape[0])
        vb = _out(need[4] and v is not None, q, h.info.nv)
        bars = {k: g.contiguous() for k, g in zip(ctx.outputs, grads) if g is not None}
        B = q.shape[1]
        if B and any(t is not None for t in (qb, vb)):
            ko = _kin_out(bars, h.info.nb, h.info.nv, q, "autodiff.kinematics")
            sign = ctx.sign if "geometric_jacobian" in bars else None
            _cabi.check(_cabi.load_library().rbd_kinematics_vjp(h.ptr, _DT[q.dtype], B, B, _ptr(q), _ptr(v), _sign_ptr(sign),
                                                                ctypes.byref(ko), None, _ptr(qb), _ptr(vb), _stream(q)))
        return None, None, None, qb, vb


def kinematics(mechanism: Mechanism, q: torch.Tensor, v: Optional[torch.Tensor] = None, *,
               outputs: Sequence[str] = ("center_of_mass",), path: Optional[TreePath] = None) -> Dict[str, torch.Tensor]:
    """Differentiable whole-body kinematics: {name: [rows, B]} for the requested ``outputs`` (names and layout of ``kinematics_``:
    transforms_to_root, center_of_mass, kinetic_energy, gravitational_potential_energy, momentum, momentum_rate_bias,
    momentum_matrix, geometric_jacobian) of q [nq, B] and v [nv, B] (needed by kinetic_energy / momentum / momentum_rate_bias);
    ``path`` is the geometric Jacobian's ``TreePath``.  Forward is one ``rbd_kinematics`` call for all outputs; backward one
    ``rbd_kinematics_vjp`` with the incoming gradients.  The gradient of ``q`` is ``q_bar_cfg`` (see the module docstring).  Not
    twice differentiable."""
    outputs = tuple(outputs)
    for k in outputs:
        if k not in _ROWS:
            raise TypeError(f"autodiff.kinematics: unknown kinematics output {k!r}")
    if len(set(outputs)) != len(outputs):
        raise ValueError("autodiff.kinematics: outputs must be distinct")
    sign = _path_sign(path, "geometric_jacobian" in outputs, len(mechanism.joints))
    return dict(zip(outputs, _Kinematics.apply(mechanism, outputs, sign, q, v)))


# ----------------------------------------------------------------------------------------------------------------------
# rollouts: rbd_integrate_trajectory / rbd_integrate_vjp
# ----------------------------------------------------------------------------------------------------------------------
def _rollout_inputs(mechanism: Mechanism, what: str, q: torch.Tensor, v: torch.Tensor, tau: Optional[torch.Tensor], nsteps: int):
    """Checks of a rollout: (model handle, B, step stride, stage stride) for q [nq, B], v [nv, B] and torques None / [nv, B] /
    [nsteps, nv, B] / [nsteps, 4, nv, B]."""
    h, B = _inputs(mechanism, what, q=q, v=v)
    nv = h.info.nv
    if nsteps < 0:
        raise ValueError(f"{what}: nsteps must be >= 0")
    if tau is None:
        return h, B, 0, 0
    if tau.dtype != q.dtype or tau.device != q.device or not tau.is_contiguous():
        raise TypeError(f"{what}: torques must be contiguous, with the dtype and device of q")
    blk = nv * B
    if tau.dim() == 2 and tuple(tau.shape) == (nv, B):
        return h, B, 0, 0
    if tau.dim() == 3 and tuple(tau.shape) == (nsteps, nv, B):
        return h, B, blk, 0
    if tau.dim() == 4 and tuple(tau.shape) == (nsteps, 4, nv, B):
        return h, B, 4 * blk, blk
    raise DimensionMismatch(f"{what}: torques must be [nv, B], [nsteps, nv, B] or [nsteps, 4, nv, B], got {tuple(tau.shape)}")


def integrate_vjp_(mechanism: Mechanism, q_traj: torch.Tensor, v_traj: torch.Tensor, torques: Optional[torch.Tensor] = None, *,
                   dt: float, q_traj_bar: Optional[torch.Tensor] = None, v_traj_bar: Optional[torch.Tensor] = None,
                   q0_bar_tan: Optional[torch.Tensor] = None, q0_bar_cfg: Optional[torch.Tensor] = None,
                   v0_bar: Optional[torch.Tensor] = None, tau_bar: Optional[torch.Tensor] = None):
    """Gradient of ``L = sum_s q_traj_bar[s] . q_traj[s] + v_traj_bar[s] . v_traj[s]`` over a trajectory recorded by
    ``simulate_trajectory_`` ([nsteps + 1, nq, B] / [nsteps + 1, nv, B]) with the same ``torques`` and ``dt``.  Outputs (each
    optional, filled in place): ``q0_bar_tan`` [nv, B], ``q0_bar_cfg`` [nq, B] (the coordinates of ``dynamics_vjp_``), ``v0_bar``
    [nv, B] and ``tau_bar`` (shape of ``torques``), to which the torque gradient is ADDED."""
    nsteps = q_traj.shape[0] - 1
    h, B, step, stage = _rollout_inputs(mechanism, "integrate_vjp_", q_traj[0], v_traj[0], torques, nsteps)
    _check_blocks("integrate_vjp_", q_traj, _rollout_vjp_rows("integrate_vjp_", h, B, torques, None, q_traj, v_traj, None, q_traj_bar,
                                                              v_traj_bar, None, q0_bar_tan, q0_bar_cfg, v0_bar, None, tau_bar))
    _cabi.check(_cabi.load_library().rbd_integrate_vjp(h.ptr, _DT[q_traj.dtype], B, _ptr(q_traj), _ptr(v_traj), _ptr(torques), step,
                                                       stage, float(dt), nsteps, _ptr(q_traj_bar), _ptr(v_traj_bar), _ptr(q0_bar_tan),
                                                       _ptr(q0_bar_cfg), _ptr(v0_bar), _ptr(tau_bar), _stream(q_traj)))


def integrate_derivatives_(mechanism: Mechanism, q_traj: torch.Tensor, v_traj: torch.Tensor, torques: Optional[torch.Tensor] = None, *,
                           dt: float, A_out: Optional[torch.Tensor] = None, B_out: Optional[torch.Tensor] = None):
    """Linearisation of every step of a trajectory recorded by ``simulate_trajectory_`` ([nsteps + 1, nq, B] / [nsteps + 1, nv, B])
    with the same ``torques`` (None, [nv, B] or [nsteps, nv, B]; a per-stage schedule raises) and ``dt``: ``A_out`` [nsteps, 4 nv^2, B]
    receives A_s = ∂x_{s+1}/∂x_s and ``B_out`` [nsteps, 2 nv^2, B] receives B_s = ∂x_{s+1}/∂τ_s, x = (q, v) with the configuration in
    the tangent space (columns along ``velocity_to_configuration_derivative(e_j)``, rows through
    ``configuration_derivative_to_velocity``), entry (i, j) at row i + j 2nv of a step's block.  Either may be None, not both."""
    what = "integrate_derivatives_"
    nsteps = q_traj.shape[0] - 1
    h, B, step, stage = _rollout_inputs(mechanism, what, q_traj[0], v_traj[0], torques, nsteps)
    if stage:
        raise ValueError(f"{what}: per-stage torque schedules are not supported")
    if A_out is None and B_out is None:
        raise ValueError(f"{what}: A_out and B_out must not both be None")
    nq, nv = h.info.nq, h.info.nv
    _check_blocks(what, q_traj, [(q_traj, (nsteps + 1, nq, B), "q_traj"), (v_traj, (nsteps + 1, nv, B), "v_traj"),
                                 (A_out, (nsteps, 4 * nv * nv, B), "A_out"), (B_out, (nsteps, 2 * nv * nv, B), "B_out")])
    _cabi.check(_cabi.load_library().rbd_integrate_derivatives(h.ptr, _DT[q_traj.dtype], B, _ptr(q_traj), _ptr(v_traj), _ptr(torques),
                                                               step, 0, float(dt), nsteps, _ptr(A_out), _ptr(B_out), _stream(q_traj)))


def integrate_derivatives(mechanism: Mechanism, q_traj: torch.Tensor, v_traj: torch.Tensor, torques: Optional[torch.Tensor] = None, *,
                          dt: float):
    """``integrate_derivatives_`` into new tensors; returns views ``A[s, i, j, b]`` [nsteps, 2nv, 2nv, B] and ``B[s, i, j, b]``
    [nsteps, 2nv, nv, B]."""
    nsteps, B = q_traj.shape[0] - 1, q_traj.shape[2]
    nv = v_traj.shape[1]
    A = torch.empty((max(nsteps, 0), 4 * nv * nv, B), dtype=q_traj.dtype, device=q_traj.device)
    Bm = torch.empty((max(nsteps, 0), 2 * nv * nv, B), dtype=q_traj.dtype, device=q_traj.device)
    integrate_derivatives_(mechanism, q_traj, v_traj, torques, dt=dt, A_out=A, B_out=Bm)
    return A.view(-1, 2 * nv, 2 * nv, B).transpose(1, 2), Bm.view(-1, nv, 2 * nv, B).transpose(1, 2)


def _trajectory(h, q0, v0, tau, s0, m, step, stage, dt):
    """rbd_integrate_trajectory over steps s0 .. s0 + m from (q0, v0) (not modified): [m + 1, rows, B] blocks."""
    B = q0.shape[1]
    q, v = q0.clone(), v0.clone()
    qt = torch.empty((m + 1,) + tuple(q0.shape), dtype=q0.dtype, device=q0.device)
    vt = torch.empty((m + 1,) + tuple(v0.shape), dtype=v0.dtype, device=v0.device)
    t = None if tau is None else (tau if tau.dim() == 2 else tau[s0:])
    _cabi.check(_cabi.load_library().rbd_integrate_trajectory(h.ptr, _DT[q0.dtype], B, B, _ptr(q), _ptr(v), _ptr(t), step, stage,
                                                              float(dt), m, _ptr(qt), _ptr(vt), _stream(q0)))
    return qt, vt


class _Simulate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mechanism, q0, v0, tau, dt, nsteps, trajectory, every):
        h, B, step, stage = _rollout_inputs(mechanism, "autodiff.simulate", q0, v0, tau, nsteps)
        ctx.handle, ctx.dt, ctx.nsteps, ctx.trajectory, ctx.step, ctx.stage = h, dt, nsteps, trajectory, step, stage
        if trajectory or B == 0:
            qt, vt = _trajectory(h, q0, v0, tau, 0, nsteps, step, stage, dt)
            ctx.every = nsteps
            ctx.save_for_backward(tau, qt, vt)
            return (qt, vt) if trajectory else (qt[-1].clone(), vt[-1].clone())
        # checkpoints every `every` steps; backward re-records each segment before its VJP
        every = max(1, min(every or nsteps, nsteps)) if nsteps else 1
        ctx.every = every
        q, v = q0, v0
        qs, vs = [q0], [v0]
        for s0 in range(0, nsteps, every):
            qt, vt = _trajectory(h, q, v, tau, s0, min(every, nsteps - s0), step, stage, dt)
            q, v = qt[-1].clone(), vt[-1].clone()
            qs.append(q); vs.append(v)
        ctx.save_for_backward(tau, torch.stack(qs[:-1]), torch.stack(vs[:-1]))
        return q, v

    @staticmethod
    @once_differentiable
    def backward(ctx, gq, gv):
        tau, qck, vck = ctx.saved_tensors
        h, dt, n = ctx.handle, ctx.dt, ctx.nsteps
        need = ctx.needs_input_grad
        q0, v0 = qck[0], vck[0]
        qc, vb = _out(need[1], q0, q0.shape[0]), torch.empty_like(v0)
        tb = torch.zeros_like(tau) if (need[3] and tau is not None) else None
        if q0.shape[1] == 0 or not (need[1] or need[2] or tb is not None):
            return None, qc, (vb if need[2] else None), tb, None, None, None, None
        if ctx.trajectory:
            _vjp_call(h, qck, vck, tau, ctx.step, ctx.stage, dt, n, gq.contiguous(), gv.contiguous(), qc, vb, tb)
            return None, qc, (vb if need[2] else None), tb, None, None, None, None
        # segments last to first; the adjoint of a segment's end state is its successor's q0_bar_cfg / v0_bar
        k = ctx.every
        qa, va = gq.contiguous(), gv.contiguous()
        starts = list(range(0, n, k)) if n else []
        if not starts:
            qc_ = torch.empty_like(q0)
            _vjp_call(h, qck, vck, tau, ctx.step, ctx.stage, dt, 0, qa[None], va[None], qc_, vb, tb)
            return None, (qc_ if need[1] else None), (vb if need[2] else None), tb, None, None, None, None
        for j in reversed(range(len(starts))):
            s0 = starts[j]
            m = min(k, n - s0)
            qt, vt = _trajectory(h, qck[j], vck[j], tau, s0, m, ctx.step, ctx.stage, dt)
            qtb = torch.zeros_like(qt); vtb = torch.zeros_like(vt)
            qtb[-1] = qa; vtb[-1] = va
            t = None if tau is None else (tau if tau.dim() == 2 else tau[s0:])
            tbs = None if tb is None else (tb if tb.dim() == 2 else tb[s0:])
            qa, va = torch.empty_like(q0), torch.empty_like(v0)
            _vjp_call(h, qt, vt, t, ctx.step, ctx.stage, dt, m, qtb, vtb, qa, va, tbs)
        return None, (qa if need[1] else None), (va if need[2] else None), tb, None, None, None, None


def _vjp_call(h, qt, vt, tau, step, stage, dt, n, qtb, vtb, qc, vb, tb):
    B = qt.shape[2]
    _cabi.check(_cabi.load_library().rbd_integrate_vjp(h.ptr, _DT[qt.dtype], B, _ptr(qt), _ptr(vt), _ptr(tau), step, stage, float(dt), n,
                                                       _ptr(qtb), _ptr(vtb), None, _ptr(qc), _ptr(vb), _ptr(tb), _stream(qt)))


def simulate(mechanism: Mechanism, q0: torch.Tensor, v0: torch.Tensor, torques: Optional[torch.Tensor] = None, *, dt: float,
             nsteps: int, trajectory: bool = True, checkpoint_every: Optional[int] = None, controller=None):
    """Differentiable ``nsteps`` Munthe-Kaas RK4 steps of ``simulate`` from q0 [nq, B], v0 [nv, B].  ``torques``: None (zero),
    constant [nv, B], per step [nsteps, nv, B] or per stage [nsteps, 4, nv, B].  Returns ``(q_traj, v_traj)`` ([nsteps + 1, rows, B],
    block 0 the initial state), or ``(q_final, v_final)`` when ``trajectory=False``.  Gradients flow to q0 (as ``q_bar_cfg``, see the
    module docstring), v0 and the torques; backward runs ``rbd_integrate_vjp``, which recomputes each step's stages from the recorded
    states.  With ``trajectory=False`` and ``checkpoint_every=k`` only every k-th state is kept, and backward re-records each
    segment of k steps before its VJP: peak memory O((nsteps / k + k) (nq + nv) B) instead of O(nsteps (nq + nv) B).  The gradients
    do not depend on k, bit for bit.  Not twice differentiable.

    ``controller``: a ``JointPD`` evaluated at every stage (``torques`` is then τ_ff), as ``simulate_(..., controller=)``.  Gradients
    then also flow to those of its ``kp``, ``kd``, ``q_ref``, ``v_ref`` and ``vd_ref`` that require grad (shared gains: summed over
    the batch); backward runs ``rbd_integrate_pd_vjp``.  Or a ``TaskPD``: gradients to its ``kp``, ``kd``, ``x_ref``, ``xd_ref`` and
    its joint term's arrays; backward runs ``rbd_integrate_task_pd_vjp``."""
    from .pd import TaskPD
    if isinstance(controller, TaskPD):
        return _simulate_task_pd(mechanism, q0, v0, None, torques, controller, None, dt, nsteps, trajectory, checkpoint_every,
                                 "autodiff.simulate")
    if controller is not None:
        return _simulate_pd(mechanism, q0, v0, None, torques, controller, None, dt, nsteps, trajectory, checkpoint_every,
                            "autodiff.simulate")
    return _Simulate.apply(mechanism, q0, v0, torques, float(dt), int(nsteps), bool(trajectory), checkpoint_every)


# ----------------------------------------------------------------------------------------------------------------------
# contact rollouts: rbd_integrate_contact (recording) / rbd_integrate_contact_vjp
# ----------------------------------------------------------------------------------------------------------------------
def _check_blocks(what: str, like: torch.Tensor, items):
    for t, shape, name in items:
        if t is None:
            continue
        if t.dtype != like.dtype or t.device != like.device or not t.is_contiguous():
            raise TypeError(f"{what}: {name} must be contiguous, with the dtype and device of q_traj")
        if shape is None or tuple(t.shape) != shape:
            raise DimensionMismatch(f"{what}: {name} has wrong size: expected {shape}, got {tuple(t.shape)}")


def _rollout_vjp_rows(what, h, B, torques, contact, q_traj, v_traj, s_traj, q_traj_bar, v_traj_bar, s_traj_bar, q0_bar_tan, q0_bar_cfg,
                      v0_bar, s0_bar, tau_bar):
    """The (tensor, shape, name) rows of ``_check_blocks`` that every rollout VJP shares: the trajectories, their adjoints and the
    state and torque outputs.  The contact state's arrays need ``contact``, and ``s_traj`` is needed with contact pairs."""
    nsteps = q_traj.shape[0] - 1
    nq, nv = h.info.nq, h.info.nv
    ns = 0 if contact is None else contact.nstates
    if contact is None and (s_traj is not None or s_traj_bar is not None or s0_bar is not None):
        raise ValueError(f"{what}: s_traj, s_traj_bar and s0_bar need contact")
    if ns > 0 and s_traj is None:
        raise ValueError(f"{what}: s_traj is needed with contact pairs")
    return [(q_traj, (nsteps + 1, nq, B), "q_traj"), (v_traj, (nsteps + 1, nv, B), "v_traj"), (s_traj, (nsteps + 1, ns, B), "s_traj"),
            (q_traj_bar, (nsteps + 1, nq, B), "q_traj_bar"), (v_traj_bar, (nsteps + 1, nv, B), "v_traj_bar"),
            (s_traj_bar, (nsteps + 1, ns, B), "s_traj_bar"), (q0_bar_tan, (nv, B), "q0_bar_tan"), (q0_bar_cfg, (nq, B), "q0_bar_cfg"),
            (v0_bar, (nv, B), "v0_bar"), (s0_bar, (ns, B), "s0_bar"),
            (tau_bar, None if torques is None else tuple(torques.shape), "tau_bar")]


def integrate_contact_vjp_(mechanism: Mechanism, q_traj: torch.Tensor, v_traj: torch.Tensor, s_traj: torch.Tensor,
                           torques: Optional[torch.Tensor] = None, *, contact, dt: float, q_traj_bar: Optional[torch.Tensor] = None,
                           v_traj_bar: Optional[torch.Tensor] = None, s_traj_bar: Optional[torch.Tensor] = None,
                           q0_bar_tan: Optional[torch.Tensor] = None, q0_bar_cfg: Optional[torch.Tensor] = None,
                           v0_bar: Optional[torch.Tensor] = None, s0_bar: Optional[torch.Tensor] = None,
                           tau_bar: Optional[torch.Tensor] = None):
    """Gradient of ``L = sum_s q_traj_bar[s] . q_traj[s] + v_traj_bar[s] . v_traj[s] + s_traj_bar[s] . s_traj[s]`` over a trajectory
    recorded by ``simulate_contact_trajectory_`` ([nsteps + 1, rows, B] each) with the same ``torques``, ``contact`` (a
    ``ContactDesc``) and ``dt``.  Outputs (each optional, filled in place) as ``integrate_vjp_``, plus ``s0_bar`` [num_contact_states,
    B]; ``tau_bar`` (shape of ``torques``) is ADDED TO."""
    nsteps = q_traj.shape[0] - 1
    h, B, step, stage = _rollout_inputs(mechanism, "integrate_contact_vjp_", q_traj[0], v_traj[0], torques, nsteps)
    _check_blocks("integrate_contact_vjp_", q_traj, _rollout_vjp_rows(
        "integrate_contact_vjp_", h, B, torques, contact, q_traj, v_traj, s_traj, q_traj_bar, v_traj_bar, s_traj_bar, q0_bar_tan,
        q0_bar_cfg, v0_bar, s0_bar, tau_bar))
    _contact_vjp_call(h, q_traj, v_traj, s_traj, torques, step, stage, contact, dt, nsteps, q_traj_bar, v_traj_bar, s_traj_bar,
                      q0_bar_tan, q0_bar_cfg, v0_bar, s0_bar, tau_bar)


def _contact_vjp_call(h, qt, vt, st, tau, step, stage, contact, dt, n, qtb, vtb, stb, q0t, qc, vb, sb, tb):
    import ctypes
    B = qt.shape[2]
    c, keep = contact.c_struct()
    _cabi.check(_cabi.load_library().rbd_integrate_contact_vjp(
        h.ptr, _DT[qt.dtype], B, _ptr(qt), _ptr(vt), _ptr(st), _ptr(tau), step, stage, ctypes.byref(c), float(dt), n, _ptr(qtb),
        _ptr(vtb), _ptr(stb), _ptr(q0t), _ptr(qc), _ptr(vb), _ptr(sb), _ptr(tb), _stream(qt)))
    del keep


def _contact_trajectory(h, q0, v0, s0, tau, first, m, step, stage, contact, dt):
    """rbd_integrate_contact recording steps first .. first + m from (q0, v0, s0) (not modified): [m + 1, rows, B] blocks."""
    import ctypes
    B = q0.shape[1]
    q, v, s = q0.clone(), v0.clone(), s0.clone()
    new = lambda x: torch.empty((m + 1,) + tuple(x.shape), dtype=x.dtype, device=x.device)   # noqa: E731
    qt, vt, st = new(q0), new(v0), new(s0)
    t = None if tau is None else (tau if tau.dim() == 2 else tau[first:])
    c, keep = contact.c_struct()
    _cabi.check(_cabi.load_library().rbd_integrate_contact(h.ptr, _DT[q0.dtype], B, B, _ptr(q), _ptr(v), _ptr(s), _ptr(t), step, stage,
                                                           ctypes.byref(c), float(dt), m, _ptr(qt), _ptr(vt), _ptr(st), _stream(q0)))
    del keep
    return qt, vt, st


class _SimulateContact(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mechanism, q0, v0, s0, tau, contact, dt, nsteps, trajectory, every):
        h, B, step, stage = _rollout_inputs(mechanism, "autodiff.simulate_contact", q0, v0, tau, nsteps)
        ns = contact.nstates
        if s0.dtype != q0.dtype or s0.device != q0.device or not s0.is_contiguous() or tuple(s0.shape) != (ns, B):
            raise DimensionMismatch(f"autodiff.simulate_contact: s0 must be a contiguous [{ns}, {B}] tensor with the dtype and device of q0")
        ctx.handle, ctx.contact, ctx.dt, ctx.nsteps, ctx.trajectory, ctx.step, ctx.stage = h, contact, dt, nsteps, trajectory, step, stage
        if trajectory or B == 0:
            qt, vt, st = _contact_trajectory(h, q0, v0, s0, tau, 0, nsteps, step, stage, contact, dt)
            ctx.every = nsteps
            ctx.save_for_backward(tau, qt, vt, st)
            return (qt, vt, st) if trajectory else (qt[-1].clone(), vt[-1].clone(), st[-1].clone())
        # checkpoints every `every` steps; backward re-records each segment before its VJP
        every = max(1, min(every or nsteps, nsteps)) if nsteps else 1
        ctx.every = every
        q, v, s = q0, v0, s0
        qs, vs, ss = [q0], [v0], [s0]
        for first in range(0, nsteps, every):
            qt, vt, st = _contact_trajectory(h, q, v, s, tau, first, min(every, nsteps - first), step, stage, contact, dt)
            q, v, s = qt[-1].clone(), vt[-1].clone(), st[-1].clone()
            qs.append(q); vs.append(v); ss.append(s)
        ctx.save_for_backward(tau, torch.stack(qs[:-1]), torch.stack(vs[:-1]), torch.stack(ss[:-1]))
        return q, v, s

    @staticmethod
    @once_differentiable
    def backward(ctx, gq, gv, gs):
        tau, qck, vck, sck = ctx.saved_tensors
        h, dt, n, cd = ctx.handle, ctx.dt, ctx.nsteps, ctx.contact
        need = ctx.needs_input_grad
        q0, v0, s0 = qck[0], vck[0], sck[0]
        tb = torch.zeros_like(tau) if (need[4] and tau is not None) else None
        if q0.shape[1] == 0 or not (need[1] or need[2] or need[3] or tb is not None):
            return (None, _out(need[1], q0, q0.shape[0]), _out(need[2], v0, v0.shape[0]), _out(need[3], s0, s0.shape[0]), tb,
                    None, None, None, None, None)
        if ctx.trajectory:
            qa, va, sa = torch.empty_like(q0), torch.empty_like(v0), torch.empty_like(s0)
            _contact_vjp_call(h, qck, vck, sck, tau, ctx.step, ctx.stage, cd, dt, n, gq.contiguous(), gv.contiguous(), gs.contiguous(),
                              None, qa, va, sa, tb)
        else:
            # segments last to first; the adjoint of a segment's end state is its successor's q0_bar_cfg / v0_bar / s0_bar
            k = ctx.every
            qa, va, sa = gq.contiguous(), gv.contiguous(), gs.contiguous()
            starts = list(range(0, n, k)) if n else []
            if not starts:
                qc_, vb_, sb_ = torch.empty_like(q0), torch.empty_like(v0), torch.empty_like(s0)
                _contact_vjp_call(h, qck, vck, sck, tau, ctx.step, ctx.stage, cd, dt, 0, qa[None], va[None], sa[None], None, qc_, vb_,
                                  sb_, tb)
                qa, va, sa = qc_, vb_, sb_
            for j in reversed(range(len(starts))):
                first = starts[j]
                m = min(k, n - first)
                qt, vt, st = _contact_trajectory(h, qck[j], vck[j], sck[j], tau, first, m, ctx.step, ctx.stage, cd, dt)
                qtb, vtb, stb = torch.zeros_like(qt), torch.zeros_like(vt), torch.zeros_like(st)
                qtb[-1] = qa; vtb[-1] = va; stb[-1] = sa
                t = None if tau is None else (tau if tau.dim() == 2 else tau[first:])
                tbs = None if tb is None else (tb if tb.dim() == 2 else tb[first:])
                qa, va, sa = torch.empty_like(q0), torch.empty_like(v0), torch.empty_like(s0)
                _contact_vjp_call(h, qt, vt, st, t, ctx.step, ctx.stage, cd, dt, m, qtb, vtb, stb, None, qa, va, sa, tbs)
        return (None, qa if need[1] else None, va if need[2] else None, sa if need[3] else None, tb, None, None, None, None, None)


def simulate_contact(mechanism: Mechanism, q0: torch.Tensor, v0: torch.Tensor, s0: torch.Tensor, torques: Optional[torch.Tensor] = None, *,
                     contact=None, dt: float, nsteps: int, trajectory: bool = True, checkpoint_every: Optional[int] = None,
                     controller=None):
    """Differentiable ``nsteps`` steps of ``simulate_contact_`` from q0 [nq, B], v0 [nv, B] and the contact state s0
    [num_contact_states, B].  ``contact``: a ``ContactDesc`` (the mechanism's ``contact_desc`` by default); ``torques`` as for
    ``simulate``.  Returns ``(q_traj, v_traj, s_traj)`` ([nsteps + 1, rows, B], block 0 the initial state), or the final
    ``(q, v, s)`` when ``trajectory=False``.  Gradients flow to q0 (as ``q_bar_cfg``), v0, s0 and the torques; backward runs
    ``rbd_integrate_contact_vjp``, which differentiates the contact force law on the branch each pair takes.  ``checkpoint_every``
    as for ``simulate``: the gradients do not depend on it, bit for bit.  ``controller`` as for ``simulate``.  Not twice
    differentiable."""
    from .contact import contact_desc
    if mechanism.has_loops():
        raise _cabi.RbdError(_cabi.RBD_ELOOP, "autodiff.simulate_contact: This method can currently only handle tree Mechanisms.")
    cd = contact if contact is not None else contact_desc(mechanism)
    from .pd import TaskPD
    if isinstance(controller, TaskPD):
        return _simulate_task_pd(mechanism, q0, v0, s0, torques, controller, cd, dt, nsteps, trajectory, checkpoint_every,
                                 "autodiff.simulate_contact")
    if controller is not None:
        return _simulate_pd(mechanism, q0, v0, s0, torques, controller, cd, dt, nsteps, trajectory, checkpoint_every,
                            "autodiff.simulate_contact")
    return _SimulateContact.apply(mechanism, q0, v0, s0, torques, cd, float(dt), int(nsteps), bool(trajectory), checkpoint_every)


# ----------------------------------------------------------------------------------------------------------------------
# closed-loop rollouts: rbd_integrate_pd (recording) / rbd_integrate_pd_vjp
# ----------------------------------------------------------------------------------------------------------------------
class _Batch:
    """What JointPD._c_struct / TaskPD._c_struct read from a state: sizes, dtype and device of a rollout's initial q0, the mechanism."""

    def __init__(self, h, q0: torch.Tensor, mechanism: Optional[Mechanism] = None):
        self.nq, self.nv, self.batch, self.dtype, self.q = h.info.nq, h.info.nv, q0.shape[1], q0.dtype, q0
        self.mechanism = mechanism


def _pd_struct(controller, h, q0, nsteps, what):
    from .pd import JointPD
    if not isinstance(controller, JointPD):
        raise TypeError(f"{what}: controller must be a JointPD")
    return controller._c_struct(_Batch(h, q0), nsteps, what)


def integrate_pd_vjp_(mechanism: Mechanism, q_traj: torch.Tensor, v_traj: torch.Tensor, torques: Optional[torch.Tensor] = None, *,
                      controller, dt: float, contact=None, s_traj: Optional[torch.Tensor] = None,
                      q_traj_bar: Optional[torch.Tensor] = None, v_traj_bar: Optional[torch.Tensor] = None,
                      s_traj_bar: Optional[torch.Tensor] = None, q0_bar_tan: Optional[torch.Tensor] = None,
                      q0_bar_cfg: Optional[torch.Tensor] = None, v0_bar: Optional[torch.Tensor] = None,
                      s0_bar: Optional[torch.Tensor] = None, tau_bar: Optional[torch.Tensor] = None,
                      kp_bar: Optional[torch.Tensor] = None, kd_bar: Optional[torch.Tensor] = None,
                      q_ref_bar: Optional[torch.Tensor] = None, v_ref_bar: Optional[torch.Tensor] = None,
                      vd_ref_bar: Optional[torch.Tensor] = None):
    """Gradient of ``L = sum_s q_traj_bar[s] . q_traj[s] + v_traj_bar[s] . v_traj[s] (+ s_traj_bar[s] . s_traj[s])`` over a
    trajectory recorded with ``controller`` (a ``JointPD``) by ``simulate_trajectory_`` or, with ``contact`` (a ``ContactDesc``)
    and ``s_traj``, by ``simulate_contact_trajectory_``, with the same ``torques`` (τ_ff) and ``dt``.  State and torque outputs as
    ``integrate_vjp_`` / ``integrate_contact_vjp_``.  Controller outputs, each optional and ADDED TO: ``kp_bar`` / ``kd_bar`` [nv, B]
    (per sample, also for shared gains: sum over the batch for theirs), ``q_ref_bar`` / ``v_ref_bar`` / ``vd_ref_bar`` with the shapes
    of ``q_ref`` / ``v_ref`` / ``vd_ref``.  Mechanisms with loops are refused (RBD_ELOOP)."""
    what = "integrate_pd_vjp_"
    nsteps = q_traj.shape[0] - 1
    h, B, step, stage = _rollout_inputs(mechanism, what, q_traj[0], v_traj[0], torques, nsteps)
    nv = h.info.nv
    pd, keep = _pd_struct(controller, h, q_traj[0], nsteps, what)
    shape = lambda t: None if t is None else tuple(t.shape)      # noqa: E731
    for bar, ref, name in ((v_ref_bar, controller.v_ref, "v_ref"), (vd_ref_bar, controller.vd_ref, "vd_ref")):
        if bar is not None and ref is None:
            raise ValueError(f"{what}: {name}_bar needs the controller's {name}")
    items = _rollout_vjp_rows(what, h, B, torques, contact, q_traj, v_traj, s_traj, q_traj_bar, v_traj_bar, s_traj_bar, q0_bar_tan,
                              q0_bar_cfg, v0_bar, s0_bar, tau_bar)
    _check_blocks(what, q_traj, items + [
        (kp_bar, (nv, B), "kp_bar"), (kd_bar, (nv, B), "kd_bar"), (q_ref_bar, shape(controller.q_ref), "q_ref_bar"),
        (v_ref_bar, shape(controller.v_ref), "v_ref_bar"), (vd_ref_bar, shape(controller.vd_ref), "vd_ref_bar")])
    _pd_vjp_call(h, q_traj, v_traj, s_traj, torques, step, stage, pd, contact, dt, nsteps, q_traj_bar, v_traj_bar, s_traj_bar,
                 q0_bar_tan, q0_bar_cfg, v0_bar, s0_bar, tau_bar, (kp_bar, kd_bar, q_ref_bar, v_ref_bar, vd_ref_bar))
    del keep


def _pd_vjp_call(h, qt, vt, st, tau, step, stage, pd, contact, dt, n, qtb, vtb, stb, q0t, qc, vb, sb, tb, bars):
    import ctypes
    from .pd import _RbdPdBar
    B = qt.shape[2]
    c, keep = contact.c_struct() if contact is not None else (None, None)
    pb = _RbdPdBar(*[_ptr(t) for t in bars])
    _cabi.check(_cabi.load_library().rbd_integrate_pd_vjp(
        h.ptr, _DT[qt.dtype], B, _ptr(qt), _ptr(vt), _ptr(st), _ptr(tau), step, stage, ctypes.byref(pd),
        None if c is None else ctypes.byref(c), float(dt), n, _ptr(qtb), _ptr(vtb), _ptr(stb), _ptr(q0t), _ptr(qc), _ptr(vb), _ptr(sb),
        _ptr(tb), ctypes.byref(pb), _stream(qt)))
    del keep


def _pd_trajectory(h, q0, v0, s0, tau, first, m, step, stage, ctl, contact, dt, what):
    """rbd_integrate_pd recording steps first .. first + m from (q0, v0[, s0]) (not modified): [m + 1, rows, B] blocks."""
    import ctypes
    B = q0.shape[1]
    q, v = q0.clone(), v0.clone()
    s = None if s0 is None else s0.clone()
    new = lambda x: torch.empty((m + 1,) + tuple(x.shape), dtype=x.dtype, device=x.device)   # noqa: E731
    qt, vt = new(q0), new(v0)
    st = None if s0 is None else new(s0)
    t = None if tau is None else (tau if tau.dim() == 2 else tau[first:])
    pd, keep = _pd_struct(ctl._steps_from(first), h, q0, m, what)
    c, keep2 = contact.c_struct() if contact is not None else (None, None)
    _cabi.check(_cabi.load_library().rbd_integrate_pd(
        h.ptr, _DT[q0.dtype], B, B, _ptr(q), _ptr(v), _ptr(s), _ptr(t), step, stage, ctypes.byref(pd), None,
        None if c is None else ctypes.byref(c), float(dt), m, _ptr(qt), _ptr(vt), _ptr(st), _stream(q0)))
    del keep, keep2
    return qt, vt, st


class _SimulatePD(torch.autograd.Function):
    """The closed-loop rollout; the controller's tensors are inputs (kp, kd, q_ref, v_ref, vd_ref), `spec` = (computed_torque,
    effort_bounds).  s0 / contact are None for the tree rollout."""

    @staticmethod
    def forward(ctx, mechanism, q0, v0, s0, tau, kp, kd, q_ref, v_ref, vd_ref, spec, contact, dt, nsteps, trajectory, every):
        from .pd import JointPD
        what = "autodiff.simulate" if contact is None else "autodiff.simulate_contact"
        h, B, step, stage = _rollout_inputs(mechanism, what, q0, v0, tau, nsteps)
        ctl = JointPD(kp, kd, q_ref, v_ref, vd_ref=vd_ref, computed_torque=spec[0], effort_bounds=spec[1])
        _pd_struct(ctl, h, q0, nsteps, what)          # the controller's checks, before any call
        if contact is not None:
            ns = contact.nstates
            if s0.dtype != q0.dtype or s0.device != q0.device or not s0.is_contiguous() or tuple(s0.shape) != (ns, B):
                raise DimensionMismatch(f"{what}: s0 must be a contiguous [{ns}, {B}] tensor with the dtype and device of q0")
        ctx.handle, ctx.ctl, ctx.contact, ctx.dt, ctx.nsteps, ctx.trajectory = h, ctl, contact, dt, nsteps, trajectory
        ctx.step, ctx.stage, ctx.what = step, stage, what
        if trajectory or B == 0:
            every = nsteps
        else:       # checkpoints every `every` steps; backward re-records each segment before its VJP
            every = max(1, min(every or nsteps, nsteps)) if nsteps else 1
        ctx.every = every
        q, v, s = q0, v0, s0
        qs, vs, ss = [q0], [v0], [s0]
        for first in range(0, max(nsteps, 1), every):
            m = min(every, nsteps - first)
            qt, vt, st = _pd_trajectory(h, q, v, s, tau, first, m, step, stage, ctl, contact, dt, what)
            if trajectory or B == 0:
                break
            q, v, s = qt[-1].clone(), vt[-1].clone(), None if st is None else st[-1].clone()
            qs.append(q); vs.append(v); ss.append(s)
        if trajectory or B == 0:
            ctx.save_for_backward(tau, qt, vt, st, kp, kd, q_ref, v_ref, vd_ref)
            out = (qt, vt) if contact is None else (qt, vt, st)
            return out if trajectory else tuple(x[-1].clone() for x in out)
        ctx.save_for_backward(tau, torch.stack(qs[:-1]), torch.stack(vs[:-1]), None if s0 is None else torch.stack(ss[:-1]), kp, kd,
                              q_ref, v_ref, vd_ref)
        return (q, v) if contact is None else (q, v, s)

    @staticmethod
    @once_differentiable
    def backward(ctx, *grads):
        tau, qck, vck, sck, kp, kd, q_ref, v_ref, vd_ref = ctx.saved_tensors
        h, dt, n, cd, ctl = ctx.handle, ctx.dt, ctx.nsteps, ctx.contact, ctx.ctl
        need = ctx.needs_input_grad
        gq, gv = grads[0].contiguous(), grads[1].contiguous()
        gs = grads[2].contiguous() if cd is not None else None
        q0, v0 = qck[0], vck[0]
        s0 = None if sck is None else sck[0]
        B = q0.shape[1]
        zero = lambda want, like: torch.zeros_like(like) if (want and like is not None) else None       # noqa: E731
        tb = zero(need[4], tau)
        kpb = torch.zeros_like(v0) if need[5] else None
        kdb = torch.zeros_like(v0) if need[6] else None
        qrb, vrb, vdrb = zero(need[7], q_ref), zero(need[8], v_ref), zero(need[9], vd_ref)
        qa, va = torch.zeros_like(q0), torch.zeros_like(v0)
        sa = None if s0 is None else torch.zeros_like(s0)
        nothing = (None,) * 6
        if B and any(need[1:10]):
            pd, keep = _pd_struct(ctl, h, q0, n, ctx.what)
            if ctx.trajectory:
                _pd_vjp_call(h, qck, vck, sck, tau, ctx.step, ctx.stage, pd, cd, dt, n, gq, gv, gs, None, qa, va, sa, tb,
                             (kpb, kdb, qrb, vrb, vdrb))
            else:
                # segments last to first; the adjoint of a segment's end state is its successor's q0_bar_cfg / v0_bar (/ s0_bar)
                k = ctx.every
                starts = list(range(0, n, k)) if n else [0]
                qa, va, sa = gq, gv, gs
                for j in reversed(range(len(starts))):
                    first = starts[j]
                    m = min(k, n - first)
                    qt, vt, st = _pd_trajectory(h, qck[j], vck[j], None if sck is None else sck[j], tau, first, m, ctx.step, ctx.stage,
                                                ctl, cd, dt, ctx.what)
                    bars = lambda x: torch.zeros_like(x)                      # noqa: E731
                    qtb, vtb = bars(qt), bars(vt)
                    qtb[-1] = qa; vtb[-1] = va
                    stb = None
                    if st is not None:
                        stb = bars(st)
                        stb[-1] = sa
                    seg = lambda t: t if t is None or t.dim() == 2 else t[first:]      # noqa: E731
                    pds, keep2 = _pd_struct(ctl._steps_from(first), h, q0, m, ctx.what)
                    qa, va = torch.empty_like(q0), torch.empty_like(v0)
                    sa = None if s0 is None else torch.empty_like(s0)
                    _pd_vjp_call(h, qt, vt, st, seg(tau), ctx.step, ctx.stage, pds, cd, dt, m, qtb, vtb, stb, None, qa, va, sa, seg(tb),
                                 (kpb, kdb, seg(qrb), seg(vrb), seg(vdrb)))
            del keep
        if kpb is not None and kp.dim() == 1:
            kpb = kpb.sum(1)
        if kdb is not None and kd.dim() == 1:
            kdb = kdb.sum(1)
        return (None, qa if need[1] else None, va if need[2] else None, sa if (need[3] and sa is not None) else None, tb, kpb, kdb, qrb,
                vrb, vdrb) + nothing


def _simulate_pd(mechanism, q0, v0, s0, torques, controller, contact, dt, nsteps, trajectory, every, what):
    from .pd import JointPD
    if not isinstance(controller, JointPD):
        raise TypeError(f"{what}: controller must be a JointPD or a TaskPD")
    c = controller
    return _SimulatePD.apply(mechanism, q0, v0, s0, torques, c.kp, c.kd, c.q_ref, c.v_ref, c.vd_ref, (c.computed_torque, c.effort_bounds),
                             contact, float(dt), int(nsteps), bool(trajectory), every)


# ----------------------------------------------------------------------------------------------------------------------
# task-space closed-loop rollouts: rbd_integrate_task_pd (recording) / rbd_integrate_task_pd_vjp
# ----------------------------------------------------------------------------------------------------------------------
def _task_struct(controller, mechanism, h, q0, nsteps, what):
    from .pd import TaskPD
    if not isinstance(controller, TaskPD):
        raise TypeError(f"{what}: controller must be a TaskPD")
    return controller._c_struct(_Batch(h, q0, mechanism), nsteps, what)


def integrate_task_pd_vjp_(mechanism: Mechanism, q_traj: torch.Tensor, v_traj: torch.Tensor, torques: Optional[torch.Tensor] = None, *,
                           controller, dt: float, contact=None, s_traj: Optional[torch.Tensor] = None,
                           q_traj_bar: Optional[torch.Tensor] = None, v_traj_bar: Optional[torch.Tensor] = None,
                           s_traj_bar: Optional[torch.Tensor] = None, q0_bar_tan: Optional[torch.Tensor] = None,
                           q0_bar_cfg: Optional[torch.Tensor] = None, v0_bar: Optional[torch.Tensor] = None,
                           s0_bar: Optional[torch.Tensor] = None, tau_bar: Optional[torch.Tensor] = None,
                           kp_bar: Optional[torch.Tensor] = None, kd_bar: Optional[torch.Tensor] = None,
                           x_ref_bar: Optional[torch.Tensor] = None, xd_ref_bar: Optional[torch.Tensor] = None,
                           joint_bars: Optional[Sequence[Optional[torch.Tensor]]] = None):
    """``integrate_pd_vjp_`` for a trajectory recorded with ``controller`` (a ``TaskPD``) by ``simulate_trajectory_`` or, with
    ``contact`` and ``s_traj``, by ``simulate_contact_trajectory_``.  Controller outputs, each optional and ADDED TO: ``kp_bar`` /
    ``kd_bar`` [R, B] (per sample, also for shared gains), ``x_ref_bar`` / ``xd_ref_bar`` with the shapes of ``x_ref`` / ``xd_ref``,
    and ``joint_bars`` = (kp, kd, q_ref, v_ref, vd_ref) bars of the joint term as in ``integrate_pd_vjp_``.  Mechanisms with loops
    are refused (RBD_ELOOP)."""
    what = "integrate_task_pd_vjp_"
    nsteps = q_traj.shape[0] - 1
    h, B, step, stage = _rollout_inputs(mechanism, what, q_traj[0], v_traj[0], torques, nsteps)
    nv = h.info.nv
    ctl, keep = _task_struct(controller, mechanism, h, q_traj[0], nsteps, what)
    R, _ = controller.rows()
    shape = lambda t: None if t is None else tuple(t.shape)      # noqa: E731
    if xd_ref_bar is not None and controller.xd_ref is None:
        raise ValueError(f"{what}: xd_ref_bar needs the controller's xd_ref")
    j = controller.joint
    jb = tuple(joint_bars) if joint_bars is not None else (None,) * 5
    if any(t is not None for t in jb) and j is None:
        raise ValueError(f"{what}: joint_bars need the controller's joint term")
    items = _rollout_vjp_rows(what, h, B, torques, contact, q_traj, v_traj, s_traj, q_traj_bar, v_traj_bar, s_traj_bar, q0_bar_tan,
                              q0_bar_cfg, v0_bar, s0_bar, tau_bar)
    items += [(kp_bar, (R, B), "kp_bar"), (kd_bar, (R, B), "kd_bar"), (x_ref_bar, shape(controller.x_ref), "x_ref_bar"),
              (xd_ref_bar, shape(controller.xd_ref), "xd_ref_bar")]
    if j is not None:
        for bar, ref, name in ((jb[3], j.v_ref, "v_ref"), (jb[4], j.vd_ref, "vd_ref")):
            if bar is not None and ref is None:
                raise ValueError(f"{what}: the joint term's {name} bar needs its {name}")
        items += [(jb[0], (nv, B), "joint kp_bar"), (jb[1], (nv, B), "joint kd_bar"), (jb[2], shape(j.q_ref), "joint q_ref_bar"),
                  (jb[3], shape(j.v_ref), "joint v_ref_bar"), (jb[4], shape(j.vd_ref), "joint vd_ref_bar")]
    _check_blocks(what, q_traj, items)
    _task_vjp_call(h, q_traj, v_traj, s_traj, torques, step, stage, ctl, contact, dt, nsteps, q_traj_bar, v_traj_bar, s_traj_bar,
                   q0_bar_tan, q0_bar_cfg, v0_bar, s0_bar, tau_bar, (kp_bar, kd_bar, x_ref_bar, xd_ref_bar), jb)
    del keep


def _task_vjp_call(h, qt, vt, st, tau, step, stage, ctl, contact, dt, n, qtb, vtb, stb, q0t, qc, vb, sb, tb, bars, joint_bars):
    from .pd import _RbdPdBar, _RbdTaskPdBar
    B = qt.shape[2]
    c, keep = contact.c_struct() if contact is not None else (None, None)
    jb = _RbdPdBar(*[_ptr(t) for t in joint_bars])
    tb_ = _RbdTaskPdBar(*[_ptr(t) for t in bars], ctypes.pointer(jb) if any(t is not None for t in joint_bars) else None)
    _cabi.check(_cabi.load_library().rbd_integrate_task_pd_vjp(
        h.ptr, _DT[qt.dtype], B, _ptr(qt), _ptr(vt), _ptr(st), _ptr(tau), step, stage, ctypes.byref(ctl),
        None if c is None else ctypes.byref(c), float(dt), n, _ptr(qtb), _ptr(vtb), _ptr(stb), _ptr(q0t), _ptr(qc), _ptr(vb), _ptr(sb),
        _ptr(tb), ctypes.byref(tb_), _stream(qt)))
    del keep


def _task_trajectory(h, mechanism, q0, v0, s0, tau, first, m, step, stage, ctl, contact, dt, what):
    """rbd_integrate_task_pd recording steps first .. first + m from (q0, v0[, s0]) (not modified): [m + 1, rows, B] blocks."""
    B = q0.shape[1]
    q, v = q0.clone(), v0.clone()
    s = None if s0 is None else s0.clone()
    new = lambda x: torch.empty((m + 1,) + tuple(x.shape), dtype=x.dtype, device=x.device)   # noqa: E731
    qt, vt = new(q0), new(v0)
    st = None if s0 is None else new(s0)
    t = None if tau is None else (tau if tau.dim() == 2 else tau[first:])
    d, keep = _task_struct(ctl._steps_from(first), mechanism, h, q0, m, what)
    c, keep2 = contact.c_struct() if contact is not None else (None, None)
    _cabi.check(_cabi.load_library().rbd_integrate_task_pd(
        h.ptr, _DT[q0.dtype], B, B, _ptr(q), _ptr(v), _ptr(s), _ptr(t), step, stage, ctypes.byref(d), None,
        None if c is None else ctypes.byref(c), float(dt), m, _ptr(qt), _ptr(vt), _ptr(st), _stream(q0)))
    del keep, keep2
    return qt, vt, st


class _SimulateTaskPD(torch.autograd.Function):
    """The task-space closed-loop rollout; the controller's tensors are inputs (kp, kd, x_ref, xd_ref, then the joint term's kp, kd,
    q_ref, v_ref, vd_ref), `ctl` the TaskPD they were taken from.  s0 / contact are None for the tree rollout."""

    @staticmethod
    def forward(ctx, mechanism, q0, v0, s0, tau, kp, kd, x_ref, xd_ref, jkp, jkd, jq_ref, jv_ref, jvd_ref, ctl, contact, dt, nsteps,
                trajectory, every):
        what = "autodiff.simulate" if contact is None else "autodiff.simulate_contact"
        h, B, step, stage = _rollout_inputs(mechanism, what, q0, v0, tau, nsteps)
        _task_struct(ctl, mechanism, h, q0, nsteps, what)          # the controller's checks, before any call
        if contact is not None:
            ns = contact.nstates
            if s0.dtype != q0.dtype or s0.device != q0.device or not s0.is_contiguous() or tuple(s0.shape) != (ns, B):
                raise DimensionMismatch(f"{what}: s0 must be a contiguous [{ns}, {B}] tensor with the dtype and device of q0")
        ctx.handle, ctx.mechanism, ctx.ctl, ctx.contact, ctx.dt, ctx.nsteps, ctx.trajectory = h, mechanism, ctl, contact, dt, nsteps, trajectory
        ctx.step, ctx.stage, ctx.what = step, stage, what
        if trajectory or B == 0:
            every = nsteps
        else:       # checkpoints every `every` steps; backward re-records each segment before its VJP
            every = max(1, min(every or nsteps, nsteps)) if nsteps else 1
        ctx.every = every
        q, v, s = q0, v0, s0
        qs, vs, ss = [q0], [v0], [s0]
        for first in range(0, max(nsteps, 1), every):
            m = min(every, nsteps - first)
            qt, vt, st = _task_trajectory(h, mechanism, q, v, s, tau, first, m, step, stage, ctl, contact, dt, what)
            if trajectory or B == 0:
                break
            q, v, s = qt[-1].clone(), vt[-1].clone(), None if st is None else st[-1].clone()
            qs.append(q); vs.append(v); ss.append(s)
        ctl_tensors = (kp, kd, x_ref, xd_ref, jkp, jkd, jq_ref, jv_ref, jvd_ref)
        if trajectory or B == 0:
            ctx.save_for_backward(tau, qt, vt, st, *ctl_tensors)
            out = (qt, vt) if contact is None else (qt, vt, st)
            return out if trajectory else tuple(x[-1].clone() for x in out)
        ctx.save_for_backward(tau, torch.stack(qs[:-1]), torch.stack(vs[:-1]), None if s0 is None else torch.stack(ss[:-1]), *ctl_tensors)
        return (q, v) if contact is None else (q, v, s)

    @staticmethod
    @once_differentiable
    def backward(ctx, *grads):
        tau, qck, vck, sck = ctx.saved_tensors[:4]      # the controller's tensors are saved to catch in-place changes; ctl holds them
        h, dt, n, cd, ctl, mech = ctx.handle, ctx.dt, ctx.nsteps, ctx.contact, ctx.ctl, ctx.mechanism
        need = ctx.needs_input_grad
        gq, gv = grads[0].contiguous(), grads[1].contiguous()
        gs = grads[2].contiguous() if cd is not None else None
        q0, v0 = qck[0], vck[0]
        s0 = None if sck is None else sck[0]
        B = q0.shape[1]
        R, _ = ctl.rows()
        j = ctl.joint
        zero = lambda want, like: torch.zeros_like(like) if (want and like is not None) else None       # noqa: E731
        per_sample = lambda want, rows: q0.new_zeros((rows, B)) if want else None                         # noqa: E731
        tb = zero(need[4], tau)
        bars = [per_sample(need[5], R), per_sample(need[6], R), zero(need[7], ctl.x_ref), zero(need[8], ctl.xd_ref)]
        jbars = [None] * 5
        if j is not None:
            jbars = [per_sample(need[9], v0.shape[0]), per_sample(need[10], v0.shape[0]), zero(need[11], j.q_ref),
                     zero(need[12], j.v_ref), zero(need[13], j.vd_ref)]
        qa, va = torch.zeros_like(q0), torch.zeros_like(v0)
        sa = None if s0 is None else torch.zeros_like(s0)
        if B and any(need[1:14]):
            seg_of = lambda t, first: t if t is None or t.dim() == 2 else t[first:]      # noqa: E731
            if ctx.trajectory:
                d, keep = _task_struct(ctl, mech, h, q0, n, ctx.what)
                _task_vjp_call(h, qck, vck, sck, tau, ctx.step, ctx.stage, d, cd, dt, n, gq, gv, gs, None, qa, va, sa, tb, bars, jbars)
                del keep
            else:
                # segments last to first; the adjoint of a segment's end state is its successor's q0_bar_cfg / v0_bar (/ s0_bar)
                k = ctx.every
                starts = list(range(0, n, k)) if n else [0]
                qa, va, sa = gq, gv, gs
                for jx in reversed(range(len(starts))):
                    first = starts[jx]
                    m = min(k, n - first)
                    qt, vt, st = _task_trajectory(h, mech, qck[jx], vck[jx], None if sck is None else sck[jx], tau, first, m, ctx.step,
                                                  ctx.stage, ctl, cd, dt, ctx.what)
                    qtb, vtb = torch.zeros_like(qt), torch.zeros_like(vt)
                    qtb[-1] = qa; vtb[-1] = va
                    stb = None
                    if st is not None:
                        stb = torch.zeros_like(st)
                        stb[-1] = sa
                    d, keep = _task_struct(ctl._steps_from(first), mech, h, q0, m, ctx.what)
                    qa, va = torch.empty_like(q0), torch.empty_like(v0)
                    sa = None if s0 is None else torch.empty_like(s0)
                    _task_vjp_call(h, qt, vt, st, seg_of(tau, first), ctx.step, ctx.stage, d, cd, dt, m, qtb, vtb, stb, None, qa, va, sa,
                                   seg_of(tb, first), [bars[0], bars[1], seg_of(bars[2], first), seg_of(bars[3], first)],
                                   [jbars[0], jbars[1], seg_of(jbars[2], first), seg_of(jbars[3], first), seg_of(jbars[4], first)])
                    del keep
        # shared gains: the per-sample bars summed over the batch
        for i, g in ((0, ctl.kp), (1, ctl.kd)):
            if bars[i] is not None and g.dim() == 1:
                bars[i] = bars[i].sum(1)
        for i, g in ((0, None if j is None else j.kp), (1, None if j is None else j.kd)):
            if jbars[i] is not None and g.dim() == 1:
                jbars[i] = jbars[i].sum(1)
        return ((None, qa if need[1] else None, va if need[2] else None, sa if (need[3] and sa is not None) else None, tb) + tuple(bars)
                + tuple(jbars) + (None,) * 6)


def _simulate_task_pd(mechanism, q0, v0, s0, torques, controller, contact, dt, nsteps, trajectory, every, what):
    if mechanism.has_loops():
        raise _cabi.RbdError(_cabi.RBD_ELOOP, f"{what}: This method can currently only handle tree Mechanisms.")
    c = controller
    j = c.joint
    jt = (None,) * 5 if j is None else (j.kp, j.kd, j.q_ref, j.v_ref, j.vd_ref)
    return _SimulateTaskPD.apply(mechanism, q0, v0, s0, torques, c.kp, c.kd, c.x_ref, c.xd_ref, *jt, c, contact, float(dt), int(nsteps),
                                 bool(trajectory), every)


# ----------------------------------------------------------------------------------------------------------------------
# the task-space law at one state: rbd_task_pd_torques / rbd_task_pd_torques_vjp
# ----------------------------------------------------------------------------------------------------------------------
def task_pd_torques_vjp_(state: MechanismState, controller, tau_out_bar: torch.Tensor, torques: Optional[torch.Tensor] = None,
                         step: int = 0, *, q_bar_tan: Optional[torch.Tensor] = None, q_bar_cfg: Optional[torch.Tensor] = None,
                         v_bar: Optional[torch.Tensor] = None, tau_bar: Optional[torch.Tensor] = None,
                         kp_bar: Optional[torch.Tensor] = None, kd_bar: Optional[torch.Tensor] = None,
                         x_ref_bar: Optional[torch.Tensor] = None, xd_ref_bar: Optional[torch.Tensor] = None,
                         joint_bars: Optional[Sequence[Optional[torch.Tensor]]] = None):
    """τ̄ᵀ ∂τ/∂(...) of ``task_pd_torques(state, controller, torques, step)`` for ``tau_out_bar`` [nv, B]: ``q_bar_tan`` [nv, B],
    ``q_bar_cfg`` [nq, B], ``v_bar`` [nv, B] and ``tau_bar`` (τ_ff, [nv, B]) are written; ``kp_bar`` / ``kd_bar`` [R, B] (per sample,
    also for shared gains), ``x_ref_bar`` / ``xd_ref_bar`` (shapes of x_ref / xd_ref) and ``joint_bars`` = (kp, kd, q_ref, v_ref,
    vd_ref) bars of the joint term ([nv, B] for the gains) are ADDED TO.  Each output is optional."""
    from .pd import TaskPD
    what = "task_pd_torques_vjp_"
    if not isinstance(controller, TaskPD):
        raise TypeError(f"{what}: controller must be a TaskPD")
    _require_tree(state, what)
    state.check_modcount()
    _check(torques, state.nv, state, "torques")
    _check(tau_out_bar, state.nv, state, "tau_out_bar")
    if step < 0:
        raise ValueError(f"{what}: step must be >= 0")
    if tau_bar is not None and torques is None:
        raise ValueError(f"{what}: tau_bar needs torques")
    if xd_ref_bar is not None and controller.xd_ref is None:
        raise ValueError(f"{what}: xd_ref_bar needs the controller's xd_ref")
    j = controller.joint
    jb = tuple(joint_bars) if joint_bars is not None else (None,) * 5
    if any(t is not None for t in jb) and j is None:
        raise ValueError(f"{what}: joint_bars need the controller's joint term")
    B, nq, nv = state.batch, state.nq, state.nv
    R, _ = controller.rows()
    shape = lambda t: None if t is None else tuple(t.shape)      # noqa: E731
    items = [(q_bar_tan, (nv, B), "q_bar_tan"), (q_bar_cfg, (nq, B), "q_bar_cfg"), (v_bar, (nv, B), "v_bar"), (tau_bar, (nv, B), "tau_bar"),
             (kp_bar, (R, B), "kp_bar"), (kd_bar, (R, B), "kd_bar"), (x_ref_bar, shape(controller.x_ref), "x_ref_bar"),
             (xd_ref_bar, shape(controller.xd_ref), "xd_ref_bar")]
    if j is not None:
        for bar, ref, name in ((jb[3], j.v_ref, "v_ref"), (jb[4], j.vd_ref, "vd_ref")):
            if bar is not None and ref is None:
                raise ValueError(f"{what}: the joint term's {name} bar needs its {name}")
        items += [(jb[0], (nv, B), "joint kp_bar"), (jb[1], (nv, B), "joint kd_bar"), (jb[2], shape(j.q_ref), "joint q_ref_bar"),
                  (jb[3], shape(j.v_ref), "joint v_ref_bar"), (jb[4], shape(j.vd_ref), "joint vd_ref_bar")]
    _check_blocks(what, state.q, items)
    d, keep = controller._c_struct(state, step + 1, what)
    _torques_vjp_call(state, d, torques, int(step), tau_out_bar.contiguous(), q_bar_tan, q_bar_cfg, v_bar, tau_bar,
                      (kp_bar, kd_bar, x_ref_bar, xd_ref_bar), jb)
    del keep


def _torques_vjp_call(state, d, torques, step, taub, qt, qc, vb, tb, bars, joint_bars):
    from .pd import _RbdPdBar, _RbdTaskPdBar
    jb = _RbdPdBar(*[_ptr(t) for t in joint_bars])
    tb_ = _RbdTaskPdBar(*[_ptr(t) for t in bars], ctypes.pointer(jb) if any(t is not None for t in joint_bars) else None)
    _cabi.check(_cabi.load_library().rbd_task_pd_torques_vjp(
        state.handle.ptr, _DT[state.dtype], state.batch, _ptr(state.q), _ptr(state.v), _ptr(torques), ctypes.byref(d), step, _ptr(taub),
        _ptr(qt), _ptr(qc), _ptr(vb), _ptr(tb), ctypes.byref(tb_), _stream(state.q)))


class _TaskPdTorques(torch.autograd.Function):
    """τ = task_pd_torques(state, ctl, torques, step) with q, v, τ_ff and the controller's tensors as inputs."""

    @staticmethod
    def forward(ctx, state, ctl, step, q, v, tau, kp, kd, x_ref, xd_ref, jkp, jkd, jq_ref, jv_ref, jvd_ref):
        from .pd import task_pd_torques
        ctx.state, ctx.ctl, ctx.step = state, ctl, step
        ctx.save_for_backward(q, v, tau, kp, kd, x_ref, xd_ref, jkp, jkd, jq_ref, jv_ref, jvd_ref)
        return task_pd_torques(state, ctl, tau, step)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        q, v, tau, kp, kd, x_ref, xd_ref, jkp, jkd, jq_ref, jv_ref, jvd_ref = ctx.saved_tensors
        state, ctl, step = ctx.state, ctx.ctl, ctx.step
        need = ctx.needs_input_grad
        B, nv = state.batch, state.nv
        R, _ = ctl.rows()
        z = lambda want, like: torch.zeros_like(like) if (want and like is not None) else None       # noqa: E731
        per_sample = lambda want, rows: q.new_zeros((rows, B)) if want else None                        # noqa: E731
        qc = torch.empty_like(q) if need[3] else None
        vb = torch.empty_like(v) if need[4] else None
        tb = torch.empty_like(v) if (need[5] and tau is not None) else None
        bars = [per_sample(need[6], R), per_sample(need[7], R), z(need[8], x_ref), z(need[9], xd_ref)]
        jbars = [per_sample(need[10], nv), per_sample(need[11], nv), z(need[12], jq_ref), z(need[13], jv_ref), z(need[14], jvd_ref)]
        if B and any(need[3:15]):
            d, keep = ctl._c_struct(state, step + 1, "autodiff.task_pd_torques")
            _torques_vjp_call(state, d, tau, step, g.contiguous(), None, qc, vb, tb, bars, jbars)
            del keep
        for i, t in ((0, kp), (1, kd)):
            if bars[i] is not None and t.dim() == 1:
                bars[i] = bars[i].sum(1)
        for i, t in ((0, jkp), (1, jkd)):
            if jbars[i] is not None and t.dim() == 1:
                jbars[i] = jbars[i].sum(1)
        return (None, None, None, qc, vb, tb) + tuple(bars) + tuple(jbars)


def task_pd_torques(state: MechanismState, controller, torques: Optional[torch.Tensor] = None, step: int = 0) -> torch.Tensor:
    """Differentiable ``task_pd_torques``: the torques ``controller`` (a ``TaskPD``) applies at ``state`` with the references of
    ``step`` and feedforward ``torques``.  Gradients flow to ``state.q`` (as ``q_bar_cfg``), ``state.v``, ``torques`` and the TaskPD's
    kp, kd, x_ref, xd_ref and its joint term's arrays, whichever require grad (shared gains: summed over the batch); backward runs
    ``rbd_task_pd_torques_vjp``.  Not twice differentiable."""
    from .pd import TaskPD
    if not isinstance(controller, TaskPD):
        raise TypeError("autodiff.task_pd_torques: controller must be a TaskPD")
    c, j = controller, controller.joint
    jt = (None,) * 5 if j is None else (j.kp, j.kd, j.q_ref, j.v_ref, j.vd_ref)
    return _TaskPdTorques.apply(state, c, int(step), state.q, state.v, torques, c.kp, c.kd, c.x_ref, c.xd_ref, *jt)
