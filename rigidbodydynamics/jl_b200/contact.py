"""Soft point contact with half-spaces, batched: the host mirror of the reference's ``Contact`` module (src/contact.jl) and of
``contact_dynamics!`` (src/mechanism_algorithms.jl:680-723).  SURVEY 8(f) rank 4.

    HuntCrossleyModel / hunt_crossley_hertz      contact.jl:130-146
    ViscoelasticCoulombModel                     contact.jl:152-206
    SoftContactModel, ContactPoint               contact.jl:35-102
    HalfSpace3D, ContactEnvironment              contact.jl:219-250
    add_contact_point!(body, point)              rigid_body.jl:173-179
    add_environment_primitive!(mechanism, hs)    mechanism_modification.jl:375
    contact_dynamics!(result, state)             mechanism_algorithms.jl:680-723     -> contact_dynamics_
    dynamics!(result, state, tau, wext) with contact points (contact wrenches added to the external ones, :850-856)
                                                                                      -> dynamics_contact_

The additional state ``s`` of a ``MechanismState`` (3 tangential-displacement entries per (contact point, half-space) pair, in
body / point / half-space order, mechanism_state.jl:140-153) is a ``[num_contact_states, B]`` tensor here.  All compute is one
CUDA kernel behind ``rbd_contact_dynamics`` (include/rbd_b200.h); there is no CPU path.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import List, Optional

import numpy as np
import torch

from . import _cabi
from .algorithms import DimensionMismatch, _call, _check, _ptr, _require_tree, _stream, dynamics_
from .state import DynamicsResult, MechanismState, _DT

__all__ = ["HuntCrossleyModel", "hunt_crossley_hertz", "ViscoelasticCoulombModel", "SoftContactModel", "ContactPoint", "HalfSpace3D",
           "add_contact_point", "contact_points", "add_environment_primitive", "environment", "num_contact_states", "ContactDesc",
           "contact_desc", "contact_dynamics_", "dynamics_contact_"]


@dataclass
class HuntCrossleyModel:
    """f = lambda z^n zdot + k z^n  (contact.jl:130-146)."""
    k: float
    lam: float
    n: float


def hunt_crossley_hertz(k: float = 50e3, alpha: float = 0.2) -> HuntCrossleyModel:
    return HuntCrossleyModel(k, 1.5 * alpha * k, 1.5)        # contact.jl:137-140, (12) in Marhefka & Orin


@dataclass
class ViscoelasticCoulombModel:
    """Featherstone RBDA 11.8 (contact.jl:152-206); 3 states (tangential displacement)."""
    mu: float
    k: float
    b: float


@dataclass
class SoftContactModel:
    normal: HuntCrossleyModel
    friction: ViscoelasticCoulombModel


@dataclass
class ContactPoint:
    """``location`` in the body's default frame (= frame after its joint once attached, as add_contact_point! stores it)."""
    location: np.ndarray
    model: SoftContactModel


class HalfSpace3D:
    """Point + outward normal in the root frame; the normal is normalised on construction (contact.jl:219-227)."""

    def __init__(self, point, outward_normal):
        self.point = np.asarray(point, float).reshape(3).copy()
        n = np.asarray(outward_normal, float).reshape(3)
        self.outward_normal = n / np.linalg.norm(n)


def add_contact_point(body, point: ContactPoint):
    if not hasattr(body, "contact_points"):
        body.contact_points = []
    point.location = np.asarray(point.location, float).reshape(3).copy()
    body.contact_points.append(point)


def contact_points(body) -> List[ContactPoint]:
    return getattr(body, "contact_points", [])


def add_environment_primitive(mechanism, halfspace: HalfSpace3D):
    if not hasattr(mechanism, "environment"):
        mechanism.environment = []
    mechanism.environment.append(halfspace)


def environment(mechanism) -> List[HalfSpace3D]:
    return getattr(mechanism, "environment", [])


def num_contact_states(mechanism) -> int:
    """num_additional_states (mechanism.jl:143-149): 3 per (contact point, half-space)."""
    npts = sum(len(contact_points(j.successor)) for j in mechanism.joints)
    return 3 * npts * len(environment(mechanism))


class _RbdContactDesc(ctypes.Structure):
    _fields_ = [("npoints", ctypes.c_int32), ("body", ctypes.c_void_p), ("location", ctypes.c_void_p),
                ("normal_model", ctypes.c_void_p), ("friction_model", ctypes.c_void_p), ("nhalfspaces", ctypes.c_int32),
                ("halfspace", ctypes.c_void_p)]


@dataclass
class ContactDesc:
    """Plain-array form == the fields of ``rbd_contact_desc``."""
    body: np.ndarray           # int32 [np]   tree joint index of the carrying body
    location: np.ndarray       # float64 [np, 3]
    normal_model: np.ndarray   # float64 [np, 3]  k, lambda, n
    friction_model: np.ndarray  # float64 [np, 3]  mu, k, b
    halfspace: np.ndarray      # float64 [nh, 6]  point, outward normal

    @property
    def npoints(self):
        return len(self.body)

    @property
    def nhalfspaces(self):
        return len(self.halfspace)

    @property
    def nstates(self):
        return 3 * self.npoints * self.nhalfspaces

    def c_struct(self):
        keep = [np.ascontiguousarray(self.body, np.int32), np.ascontiguousarray(self.location, np.float64),
                np.ascontiguousarray(self.normal_model, np.float64), np.ascontiguousarray(self.friction_model, np.float64),
                np.ascontiguousarray(self.halfspace, np.float64)]
        p = [a.ctypes.data if a.size else None for a in keep]
        return _RbdContactDesc(self.npoints, p[0], p[1], p[2], p[3], self.nhalfspaces, p[4]), keep


def contact_desc(mechanism) -> ContactDesc:
    """Collect the contact points (body / point order, like the reference's state layout) and the environment."""
    body, loc, hc, fr = [], [], [], []
    for i, j in enumerate(mechanism.joints):
        for c in contact_points(j.successor):
            body.append(i)
            loc.append(np.asarray(c.location, float).reshape(3))
            hc.append([c.model.normal.k, c.model.normal.lam, c.model.normal.n])
            fr.append([c.model.friction.mu, c.model.friction.k, c.model.friction.b])
    hs = [np.concatenate([h.point, h.outward_normal]) for h in environment(mechanism)]
    return ContactDesc(np.asarray(body, np.int32), np.asarray(loc, float).reshape(-1, 3), np.asarray(hc, float).reshape(-1, 3),
                       np.asarray(fr, float).reshape(-1, 3), np.asarray(hs, float).reshape(-1, 6))


def contact_dynamics_(state: MechanismState, contactwrenches: torch.Tensor, contact_state: Optional[torch.Tensor] = None,
                      contact_state_derivatives: Optional[torch.Tensor] = None, contact: Optional[ContactDesc] = None):
    """``contact_dynamics!(result, state)``: fills ``contactwrenches`` [6*nb, B] (root frame, per body) and
    ``contact_state_derivatives`` [num_contact_states, B]; ``contact_state`` (same shape; None = zeros) is reset to zero for the
    pairs that are not in contact, as the reference does."""
    state.check_modcount()
    lib = _cabi.load_library()
    cd = contact if contact is not None else contact_desc(state.mechanism)
    _check(contactwrenches, 6 * len(state.mechanism.joints), state, "contactwrenches")
    if contactwrenches is None:
        raise ValueError("contactwrenches must be given")
    _check(contact_state, cd.nstates, state, "contact_state")
    _check(contact_state_derivatives, cd.nstates, state, "contact_state_derivatives")
    st, keep = cd.c_struct()
    _call(lib.rbd_contact_dynamics(state.handle.ptr, _DT[state.dtype], state.batch, state.batch, _ptr(state.q), _ptr(state.v),
                                   ctypes.byref(st), _ptr(contact_state), _ptr(contact_state_derivatives), _ptr(contactwrenches),
                                   _stream()))
    del keep
    return contactwrenches


def dynamics_contact_(result: DynamicsResult, state: MechanismState, torques: Optional[torch.Tensor] = None,
                      externalwrenches: Optional[torch.Tensor] = None, contact_state: Optional[torch.Tensor] = None,
                      contact_state_derivatives: Optional[torch.Tensor] = None, contact: Optional[ContactDesc] = None,
                      want_qd: bool = True):
    """``dynamics!`` for a mechanism with contact points (mechanism_algorithms.jl:845-866): contact_dynamics!, then the contact
    wrench of every body is added to its external wrench and the forward dynamics run on the sum.  Leaves
    ``result.contactwrenches`` and ``result.totalwrenches`` ([6*nb, B]) behind like the reference's DynamicsResult."""
    _require_tree(state, "dynamics_contact_")
    nb6 = 6 * len(state.mechanism.joints)
    _check(externalwrenches, nb6, state, "externalwrenches")
    cw = getattr(result, "contactwrenches", None)
    if cw is None or cw.shape != (nb6, state.batch) or cw.dtype != state.dtype or cw.device != state.q.device:
        cw = torch.empty((nb6, state.batch), dtype=state.dtype, device=state.q.device)
        result.contactwrenches = cw
    contact_dynamics_(state, cw, contact_state, contact_state_derivatives, contact)
    if externalwrenches is not None:
        tw = getattr(result, "totalwrenches", None)
        if tw is None or tw.shape != cw.shape or tw.dtype != cw.dtype or tw.device != cw.device:
            tw = torch.empty_like(cw)
        torch.add(cw, externalwrenches, out=tw)
    else:
        tw = cw
    result.totalwrenches = tw
    return dynamics_(result, state, torques, tw, want_qd=want_qd)
