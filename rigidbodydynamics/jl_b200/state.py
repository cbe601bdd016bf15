"""Batched ``MechanismState`` / ``DynamicsResult``: the reference's state and result holders, one column per sample.

Reference: ``MechanismState`` src/mechanism_state.jl:35-78 (q, v, and the dirty-flag caches), ``DynamicsResult``
src/dynamics_result.jl:11-85.  Here the caches do not exist (every batched call recomputes, which is what
``setdirty!`` before each call does in perf/runbenchmarks.jl:37-67) and q / v are ``[n, B]`` torch tensors on the GPU
with the batch index fastest -- the layout of a Julia ``Matrix{T}(B, n)`` -- so kernels read them coalesced.
PyTorch is used only as the owner of device memory and streams.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from . import _cabi
from .mechanism import Mechanism

_DT = {torch.float32: _cabi.RBD_F32, torch.float64: _cabi.RBD_F64}


def _model_handle(mechanism: Mechanism) -> "_cabi.ModelHandle":
    """Flatten once per (mechanism, modcount): the analogue of constructing a MechanismState
    (mechanism_state.jl:79-172).  A modified mechanism gets a fresh handle; stale states are caught by
    ``rbd_model_check_modcount`` (ModificationCountMismatch, src/util.jl:56-72).  The handle describes the spanning tree only;
    the non-tree joints of a mechanism with loops are passed per call by ``dynamics_loops_`` (loops.py)."""
    cache = getattr(mechanism, "_rbd_handle", None)
    if cache is None or cache[0] != mechanism.modcount:
        desc = mechanism.flatten()
        h = _cabi.ModelHandle(desc, num_non_tree_joints=0)
        mechanism._rbd_handle = (mechanism.modcount, h, desc)
    return mechanism._rbd_handle[1]


class MechanismState:
    """State of ``batch`` independent copies of one Mechanism: ``q`` is ``[nq, B]``, ``v`` is ``[nv, B]``."""

    def __init__(self, mechanism: Mechanism, batch: int = 1, dtype: torch.dtype = torch.float64,
                 device: Optional[torch.device] = None):
        if dtype not in _DT:
            raise TypeError("the GPU path supports float32 and float64; other scalar types must use the reference "
                            "implementation itself (SURVEY 8(b) 'Scalar types / fallback')")
        self.mechanism = mechanism
        self.handle = _model_handle(mechanism)
        self.modcount = mechanism.modcount
        self.batch = int(batch)
        self.dtype = dtype
        self.device = torch.device("cuda") if device is None else torch.device(device)
        self.nq = mechanism.num_positions()
        self.nv = mechanism.num_velocities()
        self.q = torch.zeros((self.nq, self.batch), dtype=dtype, device=self.device)
        self.v = torch.zeros((self.nv, self.batch), dtype=dtype, device=self.device)
        zero_configuration_(self)

    def num_positions(self):
        return self.nq

    def num_velocities(self):
        return self.nv

    def check_modcount(self):
        """@modcountcheck (src/util.jl:56-72).  Every operator calls this first, so it also checks that the state's tensors
        live on the CURRENT CUDA device: the library launches on the current device and stream, and pointers into another
        GPU's memory would fault (or silently cross NVLink)."""
        self.handle.check_modcount(self.mechanism.modcount)
        if self.q.is_cuda and self.q.device.index != torch.cuda.current_device():
            raise ValueError(f"MechanismState lives on {self.q.device} but the current CUDA device is "
                             f"cuda:{torch.cuda.current_device()}; wrap the call in `with torch.cuda.device(state.q.device):`")

    def to_vector(self) -> torch.Tensor:
        """``Vector(state)`` = [q; v] per sample (mechanism_state.jl:482-506) -> [nq + nv, B]."""
        return torch.cat([self.q, self.v], 0)

    def copy_from_vector_(self, x: torch.Tensor):
        """``copyto!(state, x)`` (mechanism_state.jl:450-480)."""
        if x.shape != (self.nq + self.nv, self.batch):
            raise ValueError("DimensionMismatch: state vector has wrong size")
        self.q.copy_(x[: self.nq])
        self.v.copy_(x[self.nq:])
        return self


def _segments(mechanism: Mechanism):
    qs = vs = 0
    for j in mechanism.joints:
        yield j, qs, vs
        qs += j.nq
        vs += j.nv


def zero_configuration_(state: MechanismState):
    """zero_configuration! (mechanism_state.jl:286-300): identity joint transforms."""
    q0 = torch.as_tensor(state.mechanism.zero_configuration(), dtype=state.dtype, device=state.device)
    state.q.copy_(q0[:, None].expand(-1, state.batch))
    return state


def zero_velocity_(state: MechanismState):
    state.v.zero_()
    return state


def zero_(state: MechanismState):
    zero_configuration_(state)
    return zero_velocity_(state)


def rand_configuration_(state: MechanismState, rng: np.random.Generator):
    """rand_configuration! (mechanism_state.jl:318-324), vectorised over the batch on the host in fp64
    (SURVEY 8(d) 'Synthetic inputs'), then cast and uploaded."""
    from .joint_types import (Planar, Prismatic, QuaternionFloating, QuaternionSpherical, Revolute,
                              SinCosRevolute, SPQuatFloating)
    B = state.batch
    q = np.zeros((state.nq, B))
    for j, qs, _ in _segments(state.mechanism):
        jt = j.joint_type
        if isinstance(jt, SinCosRevolute):
            x = rng.standard_normal((2, B))
            q[qs:qs + 2] = x / np.linalg.norm(x, axis=0)
        elif isinstance(jt, (Revolute, Prismatic)):
            q[qs] = rng.standard_normal(B)
        elif isinstance(jt, Planar):
            q[qs:qs + 2] = rng.random((2, B)) - 0.5
            q[qs + 2] = rng.standard_normal(B)
        elif isinstance(jt, (QuaternionFloating, QuaternionSpherical)):
            x = rng.standard_normal((4, B))
            q[qs:qs + 4] = x / np.linalg.norm(x, axis=0)
            if isinstance(jt, QuaternionFloating):
                q[qs + 4:qs + 7] = rng.random((3, B)) - 0.5
        elif isinstance(jt, SPQuatFloating):
            x = rng.standard_normal((4, B))
            x /= np.linalg.norm(x, axis=0)
            x *= np.where(x[0] < 0, -1.0, 1.0)
            q[qs:qs + 3] = x[1:] / (1 + x[0])
            q[qs + 3:qs + 6] = rng.random((3, B)) - 0.5
    state.q.copy_(torch.from_numpy(q).to(state.dtype))
    return state


def rand_velocity_(state: MechanismState, rng: np.random.Generator):
    """rand_velocity! (mechanism_state.jl:342-346): v ~ U[0, 1)."""
    state.v.copy_(torch.from_numpy(rng.random((state.nv, state.batch))).to(state.dtype))
    return state


def rand_(state: MechanismState, rng: np.random.Generator):
    """rand!(state)."""
    rand_configuration_(state, rng)
    return rand_velocity_(state, rng)


class DynamicsResult:
    """dynamics_result.jl:11-85, batched: ``vd`` (v̇) [nv, B], ``qd`` (q̇) [nq, B], ``massmatrix`` [nv*nv, B]
    (entry (i, j) at row i + j*nv, both triangles), ``dynamicsbias`` [nv, B]; for mechanisms with loops also ``lam`` (λ) [nl, B],
    ``constraintjacobian`` [nl*nv, B] (entry (c, j) at row c + j*nl) and ``constraintbias`` [nl, B]."""

    def __init__(self, mechanism: Mechanism, batch: int = 1, dtype: torch.dtype = torch.float64,
                 device: Optional[torch.device] = None, with_massmatrix: bool = False):
        device = torch.device("cuda") if device is None else torch.device(device)
        nq, nv = mechanism.num_positions(), mechanism.num_velocities()
        self.mechanism = mechanism
        self.batch = int(batch)
        self.vd = torch.empty((nv, batch), dtype=dtype, device=device)
        self.qd = torch.empty((nq, batch), dtype=dtype, device=device)
        self.dynamicsbias = torch.empty((nv, batch), dtype=dtype, device=device)
        self._mm = torch.empty((nv * nv, batch), dtype=dtype, device=device) if with_massmatrix else None
        self._mm_args = (nv, batch, dtype, device)
        self._nb6 = 6 * len(mechanism.joints)
        self._nl = sum(6 - j.nv for j in mechanism.non_tree_joints)      # constraint rows (loops.num_constraints)
        self._acc = self._jw = None
        self._lam = self._K = self._k = None

    @property
    def accelerations(self) -> torch.Tensor:
        """result.accelerations (dynamics_result.jl): [6*nb, B], root frame, allocated on first use."""
        if self._acc is None:
            _, batch, dtype, device = self._mm_args
            self._acc = torch.empty((self._nb6, batch), dtype=dtype, device=device)
        return self._acc

    @property
    def jointwrenches(self) -> torch.Tensor:
        """result.jointwrenches: [6*nb, B], root frame, allocated on first use."""
        if self._jw is None:
            _, batch, dtype, device = self._mm_args
            self._jw = torch.empty((self._nb6, batch), dtype=dtype, device=device)
        return self._jw

    def _rows(self, rows):
        _, batch, dtype, device = self._mm_args
        return torch.empty((rows, batch), dtype=dtype, device=device)

    @property
    def lam(self) -> torch.Tensor:
        """result.λ: constraint forces [nl, B], allocated on first use."""
        if self._lam is None:
            self._lam = self._rows(self._nl)
        return self._lam

    @property
    def constraintjacobian(self) -> torch.Tensor:
        """result.constraintjacobian K: [nl*nv, B], entry (c, j) at row c + j*nl, allocated on first use."""
        if self._K is None:
            self._K = self._rows(self._nl * self._mm_args[0])
        return self._K

    @property
    def constraintbias(self) -> torch.Tensor:
        """result.constraintbias k: [nl, B], allocated on first use."""
        if self._k is None:
            self._k = self._rows(self._nl)
        return self._k

    @property
    def massmatrix(self) -> torch.Tensor:
        if self._mm is None:      # nv^2 * B scalars: allocated on first use only
            nv, batch, dtype, device = self._mm_args
            self._mm = torch.empty((nv * nv, batch), dtype=dtype, device=device)
        return self._mm

    def to_vector(self) -> torch.Tensor:
        """``copyto!(ẋ, result)`` = [q̇; v̇] (dynamics_result.jl:89-98)."""
        return torch.cat([self.qd, self.vd], 0)
