"""Reverse mode: vector-Jacobian products of ``dynamics!`` and ``inverse_dynamics!``, and ``torch.autograd`` functions built on them.

    dynamics_vjp_          ν̄ᵀ ∂v̇/∂(q, v, τ, w_ext)        rbd_dynamics_vjp          (include/rbd_b200.h, csrc/rbd_adjoint.cuh)
    inverse_dynamics_vjp_  τ̄ᵀ ∂τ/∂(q, v, v̇, w_ext)         rbd_inverse_dynamics_vjp
    integrate_vjp_         gradient of a recorded rollout       rbd_integrate_vjp         (csrc/rbd_integrate_adjoint.cuh)
    dynamics(mechanism, q, v, tau=None, externalwrenches=None)         differentiable v̇ = dynamics!(...)
    inverse_dynamics(mechanism, q, v, vd, externalwrenches=None)       differentiable τ = inverse_dynamics!(...)
    simulate(mechanism, q0, v0, torques=None, *, dt, nsteps, ...)     differentiable RK4 rollout (simulate)

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

from typing import Optional

import torch
from torch.autograd.function import once_differentiable

from . import _cabi
from .algorithms import DimensionMismatch, _check, _ptr, _require_tree
from .mechanism import Mechanism
from .state import _DT, MechanismState, _model_handle

__all__ = ["dynamics_vjp_", "inverse_dynamics_vjp_", "integrate_vjp_", "dynamics", "inverse_dynamics", "simulate"]


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
    nq, nv = h.info.nq, h.info.nv
    for t, shape, name in ((q_traj, (nsteps + 1, nq, B), "q_traj"), (v_traj, (nsteps + 1, nv, B), "v_traj"),
                           (q_traj_bar, (nsteps + 1, nq, B), "q_traj_bar"), (v_traj_bar, (nsteps + 1, nv, B), "v_traj_bar"),
                           (q0_bar_tan, (nv, B), "q0_bar_tan"), (q0_bar_cfg, (nq, B), "q0_bar_cfg"), (v0_bar, (nv, B), "v0_bar"),
                           (tau_bar, None if torques is None else tuple(torques.shape), "tau_bar")):
        if t is None:
            continue
        if t.dtype != q_traj.dtype or t.device != q_traj.device or not t.is_contiguous():
            raise TypeError(f"integrate_vjp_: {name} must be contiguous, with the dtype and device of q_traj")
        if shape is None or tuple(t.shape) != shape:
            raise DimensionMismatch(f"integrate_vjp_: {name} has wrong size: expected {shape}, got {tuple(t.shape)}")
    _cabi.check(_cabi.load_library().rbd_integrate_vjp(h.ptr, _DT[q_traj.dtype], B, _ptr(q_traj), _ptr(v_traj), _ptr(torques), step,
                                                       stage, float(dt), nsteps, _ptr(q_traj_bar), _ptr(v_traj_bar), _ptr(q0_bar_tan),
                                                       _ptr(q0_bar_cfg), _ptr(v0_bar), _ptr(tau_bar), _stream(q_traj)))


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
             nsteps: int, trajectory: bool = True, checkpoint_every: Optional[int] = None):
    """Differentiable ``nsteps`` Munthe-Kaas RK4 steps of ``simulate`` from q0 [nq, B], v0 [nv, B].  ``torques``: None (zero),
    constant [nv, B], per step [nsteps, nv, B] or per stage [nsteps, 4, nv, B].  Returns ``(q_traj, v_traj)`` ([nsteps + 1, rows, B],
    block 0 the initial state), or ``(q_final, v_final)`` when ``trajectory=False``.  Gradients flow to q0 (as ``q_bar_cfg``, see the
    module docstring), v0 and the torques; backward runs ``rbd_integrate_vjp``, which recomputes each step's stages from the recorded
    states.  With ``trajectory=False`` and ``checkpoint_every=k`` only every k-th state is kept, and backward re-records each
    segment of k steps before its VJP: peak memory O((nsteps / k + k) (nq + nv) B) instead of O(nsteps (nq + nv) B).  The gradients
    do not depend on k, bit for bit.  Not twice differentiable."""
    return _Simulate.apply(mechanism, q0, v0, torques, float(dt), int(nsteps), bool(trajectory), checkpoint_every)
