"""The hot-path operators of the reference, batched: same names, argument meaning and error behaviour.

    dynamics!           -> dynamics_          src/mechanism_algorithms.jl:845-864 (ODE form :880-889)
    inverse_dynamics!   -> inverse_dynamics_  src/mechanism_algorithms.jl:542-553   (allocating: inverse_dynamics :560-572)
    mass_matrix!        -> mass_matrix_       src/mechanism_algorithms.jl:248-272   (allocating: mass_matrix :281)
    dynamics_bias!      -> dynamics_bias_     src/mechanism_algorithms.jl:484-498   (allocating: dynamics_bias :505-516)

Python has no ``!``; a trailing underscore marks the in-place (non-allocating) variants.  Every function is a thin call
into ``librbd_b200.so`` (C ABI, include/rbd_b200.h) on the current CUDA stream.  There is no CPU path: on a machine
without the built library or without a GPU these raise.
"""
from __future__ import annotations

import ctypes
from typing import Optional

import torch

from . import _cabi
from .pd import JointPD, TaskPD
from .state import DynamicsResult, MechanismState, _DT

__all__ = ["dynamics_", "dynamics_dual_", "dynamics_derivatives_", "dynamics_ode_", "simulate_", "simulate_trajectory_", "inverse_dynamics_", "inverse_dynamics", "mass_matrix_", "mass_matrix",
           "dynamics_bias_", "dynamics_bias", "DimensionMismatch"]


class DimensionMismatch(ValueError):
    """Julia's DimensionMismatch (mechanism_algorithms.jl:250-251)."""


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _check(t: Optional[torch.Tensor], rows: int, state: MechanismState, name: str):
    if t is None:
        return
    if t.dtype != state.dtype or t.device != state.q.device:
        raise TypeError(f"{name}: dtype/device must match the state ({state.dtype}, {state.q.device})")
    if t.dim() != 2 or t.shape[0] != rows or t.shape[1] != state.batch:
        raise DimensionMismatch(f"{name} has wrong size: expected ({rows}, {state.batch}), got {tuple(t.shape)}")
    if not t.is_contiguous():          # (strides of size-1 dimensions are irrelevant, which is_contiguous knows)
        raise ValueError(f"{name} must be [rows, B] contiguous (batch index fastest)")


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _call(status):
    _cabi.check(status)


def _require_tree(state: MechanismState, what: str):
    """Paths that cannot honour loop constraints refuse a mechanism with non-tree joints before anything is launched, with the
    reference's error (mechanism_algorithms.jl:549), instead of silently evaluating the spanning tree."""
    if state.mechanism.has_loops():
        raise _cabi.RbdError(_cabi.RBD_ELOOP, f"{what}: This method can currently only handle tree Mechanisms.")


def dynamics_(result: DynamicsResult, state: MechanismState, torques: Optional[torch.Tensor] = None,
              externalwrenches: Optional[torch.Tensor] = None, want_qd: bool = True, byproducts=()):
    """``dynamics!(result, state, torques, externalwrenches)``: fills ``result.vd`` (v̇) and ``result.qd`` (q̇).

    ``torques`` [nv, B] or None (zero, the ConstVector default); ``externalwrenches`` [6*nb, B] root-frame wrenches
    (rows 6i..6i+5 = [torque; force] on the successor of tree joint i) or None (the NullDict default).

    The reference's ``dynamics!`` also leaves ``result.massmatrix``, ``result.dynamicsbias`` (it solves M v̇ = tau - c) and, on
    request, ``result.accelerations`` / ``result.jointwrenches`` behind (dynamics_result.jl:11-85).  The Articulated-Body kernel
    needs none of them, so they are computed only when named in ``byproducts`` (any of "massmatrix", "dynamicsbias",
    "accelerations", "jointwrenches", or "all") -- a drop-in caller that reads those fields passes ``byproducts="all"``.

    A mechanism with loops goes to ``dynamics_loops_`` with the default stabilisation gains, as the reference's ``dynamics!`` does
    (mechanism_algorithms.jl:858-862); of the by-products it leaves ``massmatrix`` and ``dynamicsbias`` (spanning tree)."""
    state.check_modcount()
    if state.mechanism.has_loops():
        from .loops import dynamics_loops_
        want = {"massmatrix", "dynamicsbias"} if byproducts == "all" else set(byproducts or ())
        if want - {"massmatrix", "dynamicsbias"}:
            raise _cabi.RbdError(_cabi.RBD_ELOOP, "dynamics_: accelerations / jointwrenches of a mechanism with loops are not available")
        dynamics_loops_(result, state, torques, externalwrenches, want_qd=want_qd)
        if "massmatrix" in want:
            mass_matrix_(result, state)
        if "dynamicsbias" in want:
            dynamics_bias_(result, state, externalwrenches)
        return result
    lib = _cabi.load_library()
    _check(torques, state.nv, state, "torques")
    _check(externalwrenches, 6 * len(state.mechanism.joints), state, "externalwrenches")
    _check(result.vd, state.nv, state, "result.vd")
    want = {"massmatrix", "dynamicsbias", "accelerations", "jointwrenches"} if byproducts == "all" else set(byproducts or ())
    if not want:
        _call(lib.rbd_dynamics(state.handle.ptr, _DT[state.dtype], state.batch, state.batch, _ptr(state.q), _ptr(state.v),
                               _ptr(torques), _ptr(externalwrenches), _ptr(result.vd),
                               _ptr(result.qd) if want_qd else None, _stream()))
        return result
    _call(lib.rbd_dynamics_result(state.handle.ptr, _DT[state.dtype], state.batch, state.batch, _ptr(state.q), _ptr(state.v),
                                  _ptr(torques), _ptr(externalwrenches), _ptr(result.vd), _ptr(result.qd) if want_qd else None,
                                  _ptr(result.massmatrix) if "massmatrix" in want else None,
                                  _ptr(result.dynamicsbias) if "dynamicsbias" in want else None,
                                  _ptr(result.accelerations) if "accelerations" in want else None,
                                  _ptr(result.jointwrenches) if "jointwrenches" in want else None, _stream()))
    return result


def dynamics_dual_(vd_out: torch.Tensor, state: MechanismState, q: torch.Tensor, v: torch.Tensor,
                   torques: Optional[torch.Tensor] = None):
    """``dynamics!`` on ``ForwardDiff.Dual{Tag,Float64,6}`` inputs (BASELINE config 4; the reference reaches this through
    its generic-scalar path, examples/5 + src/caches.jl:46-64).  Arrays are float64 ``[rows, B, 7]`` = (value, 6 partials)
    per element, which is the memory layout of a Julia ``Matrix{Dual}(B, n)``.  ``state`` only supplies the model handle."""
    _require_tree(state, "dynamics_dual_")
    state.check_modcount()
    lib = _cabi.load_library()
    B = q.shape[1]
    for name, t, rows in (("q", q, state.nq), ("v", v, state.nv), ("torques", torques, state.nv), ("vd_out", vd_out, state.nv)):
        if t is None:
            continue
        if t.dtype != torch.float64 or not t.is_cuda or not t.is_contiguous():
            raise TypeError(f"{name}: expected a contiguous float64 CUDA tensor")
        if tuple(t.shape) != (rows, B, 7):
            raise DimensionMismatch(f"{name} has wrong size: expected ({rows}, {B}, 7), got {tuple(t.shape)}")
    _call(lib.rbd_dynamics(state.handle.ptr, _cabi.RBD_DUAL64X6, B, B, _ptr(q), _ptr(v), _ptr(torques), None,
                           _ptr(vd_out), None, _stream()))
    return vd_out


def dynamics_derivatives_(dvd_dq: torch.Tensor, dvd_dv: torch.Tensor, result: DynamicsResult, state: MechanismState,
                          torques: Optional[torch.Tensor] = None):
    """Jacobians of ``dynamics!`` with respect to the configuration (tangent space) and the velocity for every sample, in one call:
    the batched, analytic counterpart of ``ForwardDiff.jacobian`` over the reference's generic ``dynamics!`` (examples/5,
    test/test_mechanism_algorithms.jl:600-675).  ``dvd_dq`` / ``dvd_dv`` are [nv*nv, B], entry (i, j) at row i + j*nv (column-major
    like ``M.data``); ``dvd_dq[:, j]`` is the derivative along ``velocity_to_configuration_derivative(e_j)``, i.e.
    ``(d v̇/d q) * velocity_to_configuration_derivative_jacobian(state)``.  ``result.vd`` receives v̇."""
    _require_tree(state, "dynamics_derivatives_")
    state.check_modcount()
    lib = _cabi.load_library()
    _check(torques, state.nv, state, "torques")
    _check(result.vd, state.nv, state, "result.vd")
    _check(dvd_dq, state.nv * state.nv, state, "dvd_dq")
    _check(dvd_dv, state.nv * state.nv, state, "dvd_dv")
    if dvd_dq is None or dvd_dv is None:
        raise ValueError("dvd_dq and dvd_dv must be given")
    with torch.cuda.device(state.q.device):
        _call(lib.rbd_dynamics_derivatives(state.handle.ptr, _DT[state.dtype], state.batch, state.batch, _ptr(state.q), _ptr(state.v),
                                           _ptr(torques), _ptr(result.vd), _ptr(dvd_dq), _ptr(dvd_dv),
                                           torch.cuda.current_stream(state.q.device).cuda_stream))
    return dvd_dq, dvd_dv


def dynamics_ode_(xdot: torch.Tensor, result: DynamicsResult, state: MechanismState, x: torch.Tensor,
                  torques: Optional[torch.Tensor] = None, externalwrenches: Optional[torch.Tensor] = None):
    """ODE form ``dynamics!(ẋ, result, state, x, torques, externalwrenches)`` (mechanism_algorithms.jl:880-889):
    x = [q; v] -> ẋ = [q̇; v̇], all [*, B]."""
    state.copy_from_vector_(x)
    dynamics_(result, state, torques, externalwrenches)
    xdot[: state.nq].copy_(result.qd)
    xdot[state.nq:].copy_(result.vd)
    return xdot


def _torque_schedule(state: MechanismState, torques: torch.Tensor, nsteps: int):
    """Element strides (step, stage) of an open-loop torque schedule: [nsteps, nv, B] (zero-order hold over each step) or
    [nsteps, 4, nv, B] (one block per RK4 stage, the batched form of control!(torques, t, state) evaluated at t, t + dt/2, t + dt/2,
    t + dt)."""
    if torques.shape[0] < nsteps or torques.shape[-2:] != (state.nv, state.batch) or (torques.dim() == 4 and torques.shape[1] != 4):
        raise DimensionMismatch("torque schedule must be [nsteps, nv, B] or [nsteps, 4, nv, B]")
    if torques.dtype != state.dtype or torques.device != state.q.device or not torques.is_contiguous():
        raise TypeError("torque schedule: dtype / device must match the state, and it must be contiguous")
    blk = state.nv * state.batch
    return (4 * blk, blk) if torques.dim() == 4 else (blk, 0)


def _steps(final_time: float, dt: float) -> int:
    """The step count of the reference's `while t < final_time` loop (ode_integrators.jl:311)."""
    nsteps, t = 0, 0.0
    while t < final_time:
        t += dt
        nsteps += 1
    return nsteps


def _rollout(state: MechanismState, nsteps: int, torques: Optional[torch.Tensor], dt: float, what: str, record: bool = False,
             controller=None, loops=None, contact=None, contact_state: Optional[torch.Tensor] = None):
    """``nsteps`` RK4 steps of the state (leading dimension B) in one call of the library's rollout: the tree rollout, or with the
    prebuilt descriptors ``loops`` / ``contact`` the loop / contact rollout, with ``controller`` evaluated at every stage.  Returns
    ``(q_traj, v_traj, s_traj)`` when ``record`` (s_traj None without contact, and for the loop rollout without contact states),
    else three Nones."""
    state.check_modcount()
    if nsteps < 0:
        raise ValueError("nsteps must be >= 0")
    lib = _cabi.load_library()
    ns = contact.nstates if contact is not None else 0
    if contact_state is None and ns > 0:
        raise ValueError(f"{what}: contact_state [{ns}, B] must be given (the mechanism has contact points)")
    _check(contact_state, ns, state, "contact_state")
    step = stage = 0
    if torques is not None and torques.dim() in (3, 4):
        step, stage = _torque_schedule(state, torques, nsteps)
    else:
        _check(torques, state.nv, state, "torques")
    traj = (None, None, None)
    if record:
        new = lambda rows: torch.empty((nsteps + 1, rows, state.batch), dtype=state.dtype, device=state.q.device)   # noqa: E731
        traj = (new(state.nq), new(state.nv), None if contact is None or (loops is not None and ns == 0) else new(ns))
    lst, keep_l = loops.c_struct() if loops is not None else (None, None)          # keep_*: arrays alive over the call
    cst, keep_c = contact.c_struct() if contact is not None else (None, None)
    ref = lambda st: None if st is None else ctypes.byref(st)                     # noqa: E731
    head = (state.handle.ptr, _DT[state.dtype], state.batch, state.batch, _ptr(state.q), _ptr(state.v))
    steps = (float(dt), nsteps)
    out = tuple(_ptr(t) for t in traj)
    if isinstance(controller, TaskPD):
        tpd, keep_tpd = controller._c_struct(state, nsteps, what)
        _call(lib.rbd_integrate_task_pd(*head, _ptr(contact_state), _ptr(torques), step, stage, ctypes.byref(tpd), ref(lst), ref(cst),
                                        *steps, *out, _stream()))
    elif controller is not None:
        if not isinstance(controller, JointPD):
            raise TypeError(f"{what}: controller must be a JointPD")
        pd, keep_pd = controller._c_struct(state, nsteps, what)
        _call(lib.rbd_integrate_pd(*head, _ptr(contact_state), _ptr(torques), step, stage, ctypes.byref(pd), ref(lst), ref(cst),
                                   *steps, *out, _stream()))
    elif loops is not None:
        _call(lib.rbd_integrate_loops(*head, _ptr(contact_state), _ptr(torques), step, stage, ref(lst), ref(cst), *steps, *out,
                                      _stream()))
    elif contact is not None:
        _call(lib.rbd_integrate_contact(*head, _ptr(contact_state), _ptr(torques), step, stage, ref(cst), *steps, *out, _stream()))
    elif record:
        _call(lib.rbd_integrate_trajectory(*head, _ptr(torques), step, stage, *steps, *out[:2], _stream()))
    else:
        _call(lib.rbd_integrate_schedule(*head, _ptr(torques), step, stage, *steps, _stream()))
    return traj


def simulate_trajectory_(state: MechanismState, nsteps: int, torques: Optional[torch.Tensor] = None, dt: float = 1e-4, *,
                         controller=None):
    """``nsteps`` Munthe-Kaas RK4 steps like ``simulate_``, recording the trajectory: returns ``(q_traj, v_traj)``,
    [nsteps + 1, nq, B] and [nsteps + 1, nv, B], block 0 the initial state and block s the state after step s.  ``state`` is advanced
    in place exactly as ``simulate_`` advances it.  ``torques``: None, constant [nv, B], per step [nsteps, nv, B] or per stage
    [nsteps, 4, nv, B].  ``controller``: a ``JointPD`` evaluated at every stage (``torques`` is then its feedforward), as in
    ``simulate_``.  The recorded trajectory of an open-loop rollout is what ``autodiff.integrate_vjp_`` differentiates."""
    _require_tree(state, "simulate_trajectory_")
    return _rollout(state, nsteps, torques, dt, "simulate_trajectory_", record=True, controller=controller)[:2]


def simulate_(state: MechanismState, final_time: float, torques: Optional[torch.Tensor] = None, dt: float = 1e-4, *,
              controller=None) -> int:
    """``simulate(state0, final_time, control!; Δt)`` (src/simulate.jl:36-55) for the whole batch, on the GPU: Munthe-Kaas RK4
    steps (src/ode_integrators.jl:233-300) until ``t >= final_time``; ``state.q`` / ``state.v`` are advanced in place.  The
    control is the default passive one (``torques=None``), a constant torque array [nv, B] (zero-order hold over the call) or an
    open-loop schedule ([nsteps, nv, B] or [nsteps, 4, nv, B]).  ``controller``: a ``JointPD`` (joint-space PD or computed-torque
    feedback) evaluated at every RK4 stage on that stage's state, with ``torques`` as its feedforward.  Returns the number of steps
    taken."""
    _require_tree(state, "simulate_")
    nsteps = _steps(final_time, dt)
    _rollout(state, nsteps, torques, dt, "simulate_", controller=controller)
    return nsteps


def inverse_dynamics_(torquesout: torch.Tensor, state: MechanismState, vd: torch.Tensor,
                      externalwrenches: Optional[torch.Tensor] = None, jointwrenchesout: Optional[torch.Tensor] = None,
                      accelerations: Optional[torch.Tensor] = None):
    """``inverse_dynamics!(torquesout, jointwrenchesout, accelerations, state, v̇, externalwrenches)`` (mechanism_algorithms.jl:542-553):
    tau = M(q) v̇ + c(q, v, w_ext).  ``jointwrenchesout`` / ``accelerations`` [6*nb, B] (optional) receive the reference's per-body
    outputs, root frame, rows 6i..6i+5 for the successor of tree joint i."""
    _require_tree(state, "inverse_dynamics_")
    state.check_modcount()
    lib = _cabi.load_library()
    nb6 = 6 * len(state.mechanism.joints)
    _check(vd, state.nv, state, "v̇")
    _check(torquesout, state.nv, state, "torquesout")
    _check(externalwrenches, nb6, state, "externalwrenches")
    _check(jointwrenchesout, nb6, state, "jointwrenchesout")
    _check(accelerations, nb6, state, "accelerations")
    _call(lib.rbd_inverse_dynamics(state.handle.ptr, _DT[state.dtype], state.batch, state.batch, _ptr(state.q),
                                   _ptr(state.v), _ptr(vd), _ptr(externalwrenches), _ptr(torquesout), _stream()))
    if jointwrenchesout is not None or accelerations is not None:
        _call(lib.rbd_inverse_dynamics_bodies(state.handle.ptr, _DT[state.dtype], state.batch, state.batch, _ptr(state.q),
                                              _ptr(state.v), _ptr(vd), _ptr(externalwrenches), _ptr(accelerations),
                                              _ptr(jointwrenchesout), _stream()))
    return torquesout


def inverse_dynamics(state: MechanismState, vd: torch.Tensor, externalwrenches: Optional[torch.Tensor] = None):
    return inverse_dynamics_(torch.empty_like(state.v), state, vd, externalwrenches)


def dynamics_bias_(result_or_out, state: MechanismState, externalwrenches: Optional[torch.Tensor] = None):
    """``dynamics_bias!(result, state)`` / 5-argument form: c(q, v, w_ext)."""
    state.check_modcount()
    lib = _cabi.load_library()
    out = result_or_out.dynamicsbias if isinstance(result_or_out, DynamicsResult) else result_or_out
    _check(out, state.nv, state, "dynamicsbias")
    _check(externalwrenches, 6 * len(state.mechanism.joints), state, "externalwrenches")
    _call(lib.rbd_dynamics_bias(state.handle.ptr, _DT[state.dtype], state.batch, state.batch, _ptr(state.q),
                                _ptr(state.v), _ptr(externalwrenches), _ptr(out), _stream()))
    return out


def dynamics_bias(state: MechanismState, externalwrenches: Optional[torch.Tensor] = None):
    return dynamics_bias_(torch.empty_like(state.v), state, externalwrenches)


def mass_matrix_(result_or_out, state: MechanismState, uplo: str = "full"):
    """``mass_matrix!(M, state)`` / ``mass_matrix!(result, state)``: [nv*nv, B], entry (i, j) at row i + j*nv.
    ``uplo="L"``: only the lower triangle (row >= column) is written, like the reference's ``Symmetric(:L)`` storage."""
    state.check_modcount()
    lib = _cabi.load_library()
    out = result_or_out.massmatrix if isinstance(result_or_out, DynamicsResult) else result_or_out
    if out.dim() != 2 or out.shape[0] != state.nv * state.nv or out.shape[1] != state.batch:
        raise DimensionMismatch("mass matrix has wrong size")                 # mechanism_algorithms.jl:250
    _check(out, state.nv * state.nv, state, "mass matrix")
    if uplo not in ("full", "L"):
        raise ValueError("uplo must be 'full' or 'L'")                      # mechanism_algorithms.jl:251 (uplo == 'L')
    _call(lib.rbd_mass_matrix_uplo(state.handle.ptr, _DT[state.dtype], state.batch, state.batch, _ptr(state.q), _ptr(out),
                                   1 if uplo == "L" else 0, _stream()))
    return out


def mass_matrix(state: MechanismState):
    out = torch.empty((state.nv * state.nv, state.batch), dtype=state.dtype, device=state.q.device)
    return mass_matrix_(out, state)
