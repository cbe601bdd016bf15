"""Mechanisms with kinematic loops, batched: the constraint side of the reference's ``dynamics!`` (SURVEY 8(f) rank 4).

    PDGains, SE3PDGains                           src/pdcontrol.jl:30-35, :80-90
    default_constraint_stabilization_gains        src/mechanism_algorithms.jl:610-612 (k = 100, d = 20, angular and linear)
    constraint_wrench_subspace(joint_type)        fixed.jl:42, revolute.jl:91, prismatic.jl:96, planar.jl:95,
                                                  quaternion_spherical.jl:60, sin_cos_revolute.jl:125; none for floating joints
    dynamics!(result, state, ...) with loops      mechanism_algorithms.jl:845-864 (constraint_jacobian! :574-598,
                                                  constraint_bias! :630-673, dynamics_solve! :747-822)   -> dynamics_loops_
    simulate(state, final_time; Δt, stabilization_gains) with loops (simulate.jl:36-55), with or without contact points
                                                  -> simulate_loops_, simulate_loops_trajectory_

A ``Mechanism``'s spanning tree is its q / v order and its model handle; the non-tree joints travel with every call as an
``rbd_loop_desc`` (include/rbd_b200.h).  All compute is one CUDA kernel behind ``rbd_dynamics_loops`` (per RK4 stage behind
``rbd_integrate_loops``); there is no CPU path.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from . import _cabi
from .algorithms import _call, _check, _ptr, _rollout, _steps, _stream
from .contact import ContactDesc, contact_desc
from .joint_types import Fixed, Planar, Prismatic, QuaternionSpherical, Revolute
from .mechanism import Mechanism
from .spatial import rotation_between
from .state import DynamicsResult, MechanismState, _DT

__all__ = ["PDGains", "SE3PDGains", "default_constraint_stabilization_gains", "constraint_wrench_subspace", "num_constraints",
           "LoopDesc", "loop_desc", "dynamics_loops_", "simulate_loops_", "simulate_loops_trajectory_"]


@dataclass
class PDGains:
    """pdcontrol.jl:30-35: pd(gains, e, ė) = -k e - d ė."""
    k: float
    d: float


@dataclass
class SE3PDGains:
    """pdcontrol.jl:80-90: gains for the angular and the linear part of an SE(3) error."""
    angular: PDGains
    linear: PDGains


def default_constraint_stabilization_gains() -> SE3PDGains:
    """Critically damped Baumgarte gains, T_stab = 0.1 in Featherstone (2008) 8.3 (mechanism_algorithms.jl:610-612)."""
    return SE3PDGains(PDGains(100.0, 20.0), PDGains(100.0, 20.0))


_DEFAULT = object()      # sentinel: "the default gains", distinct from None (= stabilisation off)


def constraint_wrench_subspace(joint_type) -> np.ndarray:
    """The constant basis T of the wrenches a joint transmits, as a [6, 6 - nv] array whose columns are [torque; force] in the
    frame after the joint, in the reference's column order.  1-DoF joints use ``rotation_from_z_aligned = rotation_between(z,
    axis)``; for them only the span of T is pinned by the reference, because Rotations.jl's rotation_between is not part of it."""
    def cols(ang, lin):
        return np.vstack([np.asarray(ang, float).reshape(3, -1), np.asarray(lin, float).reshape(3, -1)])
    z3 = np.zeros((3, 3))
    if isinstance(joint_type, Fixed):                                       # fixed.jl:42-47
        return np.eye(6)
    if isinstance(joint_type, Prismatic):                                   # prismatic.jl:96-103
        R = rotation_between([0.0, 0.0, 1.0], joint_type.axis)
        return cols(np.hstack([R, np.zeros((3, 2))]), np.hstack([z3, R[:, :2]]))
    if isinstance(joint_type, Revolute):                                    # revolute.jl:91-98, sin_cos_revolute.jl:125-132
        R = rotation_between([0.0, 0.0, 1.0], joint_type.axis)
        return cols(np.hstack([R[:, :2], z3]), np.hstack([np.zeros((3, 2)), R]))
    if isinstance(joint_type, Planar):                                      # planar.jl:95-100
        return cols(np.column_stack([np.zeros(3), joint_type.x_axis, joint_type.y_axis]),
                    np.column_stack([joint_type.rot_axis, np.zeros(3), np.zeros(3)]))
    if isinstance(joint_type, QuaternionSpherical):                         # quaternion_spherical.jl:60-65
        return cols(z3, np.eye(3))
    if joint_type.isfloating:                                               # quaternion_floating.jl:93, spquat_floating.jl:91
        return np.zeros((6, 0))
    raise TypeError(f"no constraint wrench subspace for {joint_type!r}")


def num_constraints(mechanism: Mechanism) -> int:
    """Rows of the constraint Jacobian: sum over the non-tree joints of 6 - nv."""
    return sum(6 - j.nv for j in mechanism.non_tree_joints)


class _RbdLoopDesc(ctypes.Structure):
    _fields_ = [("nloops", ctypes.c_int32), ("predecessor", ctypes.c_void_p), ("successor", ctypes.c_void_p),
                ("joint_to_predecessor", ctypes.c_void_p), ("joint_to_successor", ctypes.c_void_p),
                ("nconstraints", ctypes.c_void_p), ("wrench_basis", ctypes.c_void_p), ("gains", ctypes.c_void_p)]


@dataclass
class LoopDesc:
    """Plain-array form == the fields of ``rbd_loop_desc``, in non_tree_joints order."""
    predecessor: np.ndarray            # int32 [nl]   tree-joint index whose successor is the body, -1 = root
    successor: np.ndarray              # int32 [nl]
    joint_to_predecessor: np.ndarray   # float64 [nl, 12]  R row-major, p
    joint_to_successor: np.ndarray     # float64 [nl, 12]
    nconstraints: np.ndarray           # int32 [nl]
    wrench_basis: np.ndarray           # float64 [nc, 6]   [torque; force], frame after the joint
    gains: Optional[np.ndarray]        # float64 [nl, 4]   angular k, d, linear k, d;  None = no stabilisation

    @property
    def nloops(self):
        return len(self.predecessor)

    @property
    def nc(self):
        return int(self.nconstraints.sum())

    def c_struct(self):
        keep = [np.ascontiguousarray(self.predecessor, np.int32), np.ascontiguousarray(self.successor, np.int32),
                np.ascontiguousarray(self.joint_to_predecessor, np.float64), np.ascontiguousarray(self.joint_to_successor, np.float64),
                np.ascontiguousarray(self.nconstraints, np.int32), np.ascontiguousarray(self.wrench_basis, np.float64),
                None if self.gains is None else np.ascontiguousarray(self.gains, np.float64)]
        p = [None if a is None or a.size == 0 else a.ctypes.data for a in keep]
        return _RbdLoopDesc(self.nloops, *p), keep


def _gains_row(g: SE3PDGains):
    return [g.angular.k, g.angular.d, g.linear.k, g.linear.d]


def loop_desc(mechanism: Mechanism, stabilization_gains=_DEFAULT) -> LoopDesc:
    """Collect the non-tree joints.  ``stabilization_gains``: the default gains (omitted), ``None`` (no Baumgarte stabilisation),
    one ``SE3PDGains`` for every joint, or a dict from non-tree ``Joint`` (or its name) to ``SE3PDGains``."""
    index = {id(j.successor): i for i, j in enumerate(mechanism.joints)}
    body = lambda b: -1 if b is mechanism.root_body else index[id(b)]
    nt = mechanism.non_tree_joints
    bases = [constraint_wrench_subspace(j.joint_type) for j in nt]
    if stabilization_gains is _DEFAULT:
        stabilization_gains = default_constraint_stabilization_gains()
    if stabilization_gains is None:
        gains = None
    elif isinstance(stabilization_gains, SE3PDGains):
        gains = np.array([_gains_row(stabilization_gains) for _ in nt], float).reshape(-1, 4)
    else:
        def lookup(j):
            if j in stabilization_gains:
                return stabilization_gains[j]
            return stabilization_gains[j.name]
        gains = np.array([_gains_row(lookup(j)) for j in nt], float).reshape(-1, 4)
    return LoopDesc(predecessor=np.array([body(j.predecessor) for j in nt], np.int32),
                    successor=np.array([body(j.successor) for j in nt], np.int32),
                    joint_to_predecessor=np.array([j.joint_to_predecessor.flat12() for j in nt], float).reshape(-1, 12),
                    joint_to_successor=np.array([j.joint_to_successor.flat12() for j in nt], float).reshape(-1, 12),
                    nconstraints=np.array([b.shape[1] for b in bases], np.int32),
                    wrench_basis=(np.concatenate([b.T for b in bases], 0) if bases else np.zeros((0, 6))).reshape(-1, 6),
                    gains=gains)


def dynamics_loops_(result: DynamicsResult, state: MechanismState, torques: Optional[torch.Tensor] = None,
                    externalwrenches: Optional[torch.Tensor] = None, stabilization_gains=_DEFAULT, want_qd: bool = True,
                    loops: Optional[LoopDesc] = None):
    """``dynamics!(result, state, torques, externalwrenches; stabilization_gains)`` for a mechanism with loops: fills ``result.vd``
    (v̇), ``result.qd`` (q̇), ``result.lam`` (λ, [nl, B]), ``result.constraintjacobian`` (K, [nl*nv, B], entry (c, j) at row
    c + j*nl) and ``result.constraintbias`` (k, [nl, B]).  ``loops``: a prebuilt ``loop_desc(mechanism, gains)`` (else built here)."""
    state.check_modcount()
    lib = _cabi.load_library()
    ld = loops if loops is not None else loop_desc(state.mechanism, stabilization_gains)
    nl = ld.nc
    _check(torques, state.nv, state, "torques")
    _check(externalwrenches, 6 * len(state.mechanism.joints), state, "externalwrenches")
    _check(result.vd, state.nv, state, "result.vd")
    lam, K, k = result.lam, result.constraintjacobian, result.constraintbias
    _check(lam, nl, state, "result.lam")
    _check(K, nl * state.nv, state, "result.constraintjacobian")
    _check(k, nl, state, "result.constraintbias")
    st, keep = ld.c_struct()
    _call(lib.rbd_dynamics_loops(state.handle.ptr, _DT[state.dtype], state.batch, state.batch, _ptr(state.q), _ptr(state.v),
                                 _ptr(torques), _ptr(externalwrenches), ctypes.byref(st), _ptr(result.vd),
                                 _ptr(result.qd) if want_qd else None, _ptr(lam), _ptr(K), _ptr(k), _stream()))
    del keep
    return result


def simulate_loops_trajectory_(state: MechanismState, nsteps: int, torques: Optional[torch.Tensor] = None, dt: float = 1e-4,
                               stabilization_gains=_DEFAULT, loops: Optional[LoopDesc] = None,
                               contact_state: Optional[torch.Tensor] = None, contact: Optional[ContactDesc] = None, *,
                               controller=None):
    """``nsteps`` steps of ``simulate_loops_``, recording the trajectory: returns ``(q_traj, v_traj, s_traj)``, [nsteps + 1, nq, B],
    [nsteps + 1, nv, B] and [nsteps + 1, num_contact_states, B] (None without contact states), block 0 the initial state and block s
    the state after step s.  ``state`` and ``contact_state`` are advanced in place exactly as ``simulate_loops_`` advances them.
    ``controller``: a ``JointPD`` evaluated at every stage, as in ``simulate_loops_`` (``torques`` is then its feedforward; PD mode
    only when the mechanism has loops)."""
    ld = loops if loops is not None else loop_desc(state.mechanism, stabilization_gains)
    cd = contact if contact is not None else contact_desc(state.mechanism)
    return _rollout(state, nsteps, torques, dt, "simulate_loops_trajectory_", record=True, controller=controller, loops=ld, contact=cd,
                    contact_state=contact_state)


def simulate_loops_(state: MechanismState, final_time: float, torques: Optional[torch.Tensor] = None, dt: float = 1e-4,
                    stabilization_gains=_DEFAULT, loops: Optional[LoopDesc] = None, contact_state: Optional[torch.Tensor] = None,
                    contact: Optional[ContactDesc] = None, *, controller=None) -> int:
    """``simulate(state, final_time; Δt, stabilization_gains)`` (src/simulate.jl:36-55) for a mechanism with non-tree joints, all on
    the GPU: Munthe-Kaas RK4 steps until ``t >= final_time`` (the step count of ``simulate_``) whose every stage runs ``dynamics!``
    as ``dynamics_loops_`` does -- with contact points, contact_dynamics! first and its wrenches as the external wrenches
    (mechanism_algorithms.jl:845-864).  ``state.q``, ``state.v`` and ``contact_state`` ([num_contact_states, B], required when the
    mechanism has contact points) are advanced in place; the contact state follows ``simulate_contact_`` (integrated, never reset,
    carried across calls).  ``torques``: None, constant [nv, B], per step [nsteps, nv, B] or per stage [nsteps, 4, nv, B].
    ``stabilization_gains``: as ``loop_desc`` (default gains, None = off, or per joint); ``loops`` / ``contact``: prebuilt
    descriptors (default: the mechanism's).  A tree mechanism is accepted (the KKT path without constraint rows).  ``controller``: a
    ``JointPD`` evaluated at every stage, as in ``simulate_`` (PD mode only when the mechanism has loops: computed-torque mode needs
    inverse_dynamics!, which refuses loops with RBD_ELOOP).  Returns the number of steps taken."""
    nsteps = _steps(final_time, dt)
    ld = loops if loops is not None else loop_desc(state.mechanism, stabilization_gains)
    cd = contact if contact is not None else contact_desc(state.mechanism)
    _rollout(state, nsteps, torques, dt, "simulate_loops_", controller=controller, loops=ld, contact=cd, contact_state=contact_state)
    return nsteps
