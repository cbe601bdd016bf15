"""Host-side model: RigidBody / Joint / Mechanism, mirroring the reference's user-facing types.

Reference (all under the reference's src/, RigidBodyDynamics.jl v2.5.0):
  RigidBody                 rigid_body.jl:12-29
  Joint                     joint.jl:43-67   (joint_to_predecessor :49, joint_to_successor :50)
  Mechanism                 mechanism.jl:10-34, default gravity (0,0,-9.81) mechanism.jl:1
  attach!                   mechanism_modification.jl:21-46
  remove_fixed_tree_joints! mechanism_modification.jl:260-317
  maximal_coordinates       mechanism_modification.jl:335-362
  rand_*_mechanism          mechanism_modification.jl:382-426

A ``Mechanism`` is immutable while a batch is being evaluated; ``flatten()`` turns it into the plain
arrays of ``rbd_model_desc`` (include/rbd_b200.h) in the reference's tree-joint order, which is
the q/v/τ index order (mechanism_state.jl:101-104).  Frames are implicit: a body's frame IS the
frame after its parent joint (mechanism.jl:250-260, canonicalize_frame_definitions!).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, List, Optional, Sequence

import numpy as np

from .joint_types import Fixed, JointType, QuaternionFloating
from .spatial import SpatialInertia, Transform3D

DEFAULT_GRAVITATIONAL_ACCELERATION = (0.0, 0.0, -9.81)     # mechanism.jl:1


class RigidBody:
    """rigid_body.jl:12-29. ``inertia`` is expressed in the body's default frame; ``None`` for the world."""

    def __init__(self, name_or_inertia=None, inertia: Optional[SpatialInertia] = None):
        if isinstance(name_or_inertia, SpatialInertia):
            inertia, name = name_or_inertia, None
        else:
            name = name_or_inertia
        self.name = name
        self.inertia = inertia

    def has_defined_inertia(self):
        return self.inertia is not None

    def __repr__(self):
        return f"RigidBody({self.name!r})"


@dataclass(frozen=True)
class Bounds:
    """Bounds{T} (src/bounds.jl): a closed interval, (-inf, inf) by default."""
    lower: float = -np.inf
    upper: float = np.inf


class Joint:
    """joint.jl:43-67.  ``position_bounds`` ([nq]), ``velocity_bounds`` and ``effort_bounds`` ([nv]): lists of ``Bounds``, infinite
    unless given (joint.jl:51-58, parsed from URDF <limit> by parse_urdf)."""

    def __init__(self, name: str, joint_type: JointType, *, position_bounds: Optional[Sequence[Bounds]] = None,
                 velocity_bounds: Optional[Sequence[Bounds]] = None, effort_bounds: Optional[Sequence[Bounds]] = None):
        self.name = name
        self.joint_type = joint_type
        self.position_bounds = list(position_bounds) if position_bounds is not None else [Bounds()] * joint_type.nq
        self.velocity_bounds = list(velocity_bounds) if velocity_bounds is not None else [Bounds()] * joint_type.nv
        self.effort_bounds = list(effort_bounds) if effort_bounds is not None else [Bounds()] * joint_type.nv
        if len(self.position_bounds) != joint_type.nq or len(self.velocity_bounds) != joint_type.nv or \
                len(self.effort_bounds) != joint_type.nv:
            raise ValueError("joint bounds: nq position bounds and nv velocity / effort bounds")
        self.joint_to_predecessor = Transform3D.identity()   # frame before joint -> predecessor body frame
        # frame after joint -> successor body frame: the identity for tree joints (the body frame IS the frame after the joint),
        # inv(successor_pose) for non-tree joints (mechanism_modification.jl:34)
        self.joint_to_successor = Transform3D.identity()
        self.predecessor: Optional[RigidBody] = None
        self.successor: Optional[RigidBody] = None

    @property
    def nq(self):
        return self.joint_type.nq

    @property
    def nv(self):
        return self.joint_type.nv

    def __repr__(self):
        return f"Joint({self.name!r}, {self.joint_type!r})"


@dataclass
class ModelDesc:
    """Plain-array form of a tree Mechanism == the fields of ``rbd_model_desc`` (include/rbd_b200.h)."""
    nb: int
    nq: int
    nv: int
    parent: np.ndarray      # int32 [nb]  index of the joint whose successor is this joint's predecessor; -1 = world
    jtype: np.ndarray       # int32 [nb]
    qstart: np.ndarray      # int32 [nb]
    vstart: np.ndarray      # int32 [nb]
    X_tree: np.ndarray      # float64 [nb,12]  joint_to_predecessor: R row-major, p
    jparam: np.ndarray      # float64 [nb,9]
    inertia: np.ndarray     # float64 [nb,13]  moment row-major, cross_part, mass (frame after joint)
    gravity: np.ndarray     # float64 [3]
    modcount: int = 0
    joint_names: List[str] = field(default_factory=list)
    body_names: List[str] = field(default_factory=list)


class Mechanism:
    """mechanism.jl:10-34.  ``joints`` is the spanning tree (the q/v order); non-tree (loop) joints are kept in
    ``non_tree_joints`` with their attachment transforms and enter dynamics! as constraints (loops.py)."""

    def __init__(self, root_body: Optional[RigidBody] = None, gravity=DEFAULT_GRAVITATIONAL_ACCELERATION):
        self.root_body = root_body if root_body is not None else RigidBody("world")
        self.root_body.inertia = None
        self.bodies: List[RigidBody] = [self.root_body]
        self.joints: List[Joint] = []            # tree joints, in tree order (== q/v order)
        self.non_tree_joints: List[Joint] = []
        self.gravitational_acceleration = np.asarray(gravity, float).reshape(3).copy()
        self.modcount = 0

    # -- queries --------------------------------------------------------------------------------
    def tree_joints(self):
        return self.joints

    def non_root_bodies(self):
        return self.bodies[1:]

    def has_loops(self):                                      # mechanism.jl:88
        return len(self.non_tree_joints) > 0

    def num_positions(self):
        return sum(j.nq for j in self.joints)

    def num_velocities(self):
        return sum(j.nv for j in self.joints)

    def findbody(self, name):
        m = [b for b in self.bodies if b.name == name]
        if len(m) != 1:
            raise KeyError(f"body {name!r}: {len(m)} matches")
        return m[0]

    def findjoint(self, name):
        m = [j for j in self.joints + self.non_tree_joints if j.name == name]
        if len(m) != 1:
            raise KeyError(f"joint {name!r}: {len(m)} matches")
        return m[0]

    def joint_to_parent(self, body):
        for j in self.joints:
            if j.successor is body:
                return j
        raise KeyError(body)

    def mass(self):
        return sum(b.inertia.mass for b in self.non_root_bodies())

    # -- construction ---------------------------------------------------------------------------
    def attach(self, predecessor: RigidBody, successor: RigidBody, joint: Joint,
               joint_pose: Optional[Transform3D] = None, successor_pose: Optional[Transform3D] = None):
        """mechanism_modification.jl:21-46.  ``joint_pose``: frame before joint -> predecessor frame;
        ``successor_pose``: successor's current default frame -> frame after joint."""
        if predecessor not in self.bodies:
            raise ValueError("predecessor must already be part of the mechanism")
        if joint in self.joints or joint in self.non_tree_joints:
            raise ValueError("joint already attached")
        joint.joint_to_predecessor = joint_pose if joint_pose is not None else Transform3D.identity()
        joint.predecessor, joint.successor = predecessor, successor
        if successor in self.bodies:
            # loop joint: the successor keeps its frame, the joint records where it attaches (mechanism_modification.jl:34)
            joint.joint_to_successor = successor_pose.inv() if successor_pose is not None else Transform3D.identity()
            self.non_tree_joints.append(joint)
        else:
            joint.joint_to_successor = Transform3D.identity()
            if successor.inertia is None:
                successor.inertia = SpatialInertia.zero()
            if successor_pose is not None:
                # canonicalize_frame_definitions! (mechanism.jl:250-260): the body frame becomes
                # frame_after(joint); the inertia is re-expressed there (rigid_body.jl change_default_frame!)
                successor.inertia = successor.inertia.transform(successor_pose)
            self.bodies.append(successor)
            self.joints.append(joint)
        self.modcount += 1
        return self

    def remove_fixed_tree_joints(self):
        """mechanism_modification.jl:260-317: weld successors of Fixed tree joints into their predecessors.
        Non-fixed joints keep their relative order (:265-266,308); bodies welded to the world lose
        their inertia because the world has none (:286)."""
        fixed = [j for j in self.joints if isinstance(j.joint_type, Fixed)]
        for fj in fixed:
            pred, succ = fj.predecessor, fj.successor
            to_pred = fj.joint_to_predecessor            # Fixed joint transform is the identity (fixed.jl:18-22)
            if pred.has_defined_inertia():
                pred.inertia = pred.inertia + succ.inertia.transform(to_pred)
            for j in self.joints + self.non_tree_joints:
                if j is fj:
                    continue
                if j.predecessor is succ:
                    j.predecessor = pred
                    j.joint_to_predecessor = to_pred * j.joint_to_predecessor
                if j.successor is succ:                   # only possible for non-tree joints
                    j.successor = pred
                    j.joint_to_successor = to_pred * j.joint_to_successor
            self.bodies.remove(succ)
            self.joints.remove(fj)
        self.modcount += 1
        return self

    # -- flattening -----------------------------------------------------------------------------
    def flatten(self) -> ModelDesc:
        """Plain arrays in tree-joint order (== SegmentedVector layout, mechanism_state.jl:101-104)."""
        nb = len(self.joints)
        succ_index = {id(j.successor): i for i, j in enumerate(self.joints)}
        parent = np.empty(nb, np.int32)
        jtype = np.empty(nb, np.int32)
        qstart = np.empty(nb, np.int32)
        vstart = np.empty(nb, np.int32)
        X_tree = np.empty((nb, 12))
        jparam = np.empty((nb, 9))
        inertia = np.empty((nb, 13))
        nq = nv = 0
        for i, j in enumerate(self.joints):
            parent[i] = -1 if j.predecessor is self.root_body else succ_index[id(j.predecessor)]
            if parent[i] >= i:
                raise ValueError("tree joints are not in topological order")
            jtype[i] = j.joint_type.code
            qstart[i], vstart[i] = nq, nv
            nq += j.nq
            nv += j.nv
            X_tree[i] = j.joint_to_predecessor.flat12()
            jparam[i] = j.joint_type.params9()
            inertia[i] = j.successor.inertia.flat13()
        return ModelDesc(nb=nb, nq=nq, nv=nv, parent=parent, jtype=jtype, qstart=qstart, vstart=vstart,
                         X_tree=X_tree, jparam=jparam, inertia=inertia,
                         gravity=self.gravitational_acceleration.copy(), modcount=self.modcount,
                         joint_names=[j.name for j in self.joints],
                         body_names=[j.successor.name for j in self.joints])

    # -- state helpers shared by the oracle tests and MechanismState ----------------------------
    def rand_configuration(self, rng) -> np.ndarray:
        """One sample of rand_configuration!(state) (mechanism_state.jl:318-324)."""
        parts = [j.joint_type.rand_configuration(rng) for j in self.joints]
        return np.concatenate(parts) if parts else np.zeros(0)

    def zero_configuration(self) -> np.ndarray:
        parts = [j.joint_type.zero_configuration() for j in self.joints]
        return np.concatenate(parts) if parts else np.zeros(0)

    def __repr__(self):
        return (f"Mechanism({len(self.bodies) - 1} bodies, nq={self.num_positions()}, "
                f"nv={self.num_velocities()})")


def maximal_coordinates(mechanism: Mechanism, floating_joint_type: type = QuaternionFloating, bodymap: Optional[dict] = None,
                        jointmap: Optional[dict] = None) -> Mechanism:
    """mechanism_modification.jl:335-362: every non-root body is attached to the root by a floating joint and every joint of
    ``mechanism`` (tree and non-tree) becomes a non-tree joint between the copies.  ``bodymap`` / ``jointmap`` (optional dicts)
    receive original -> copy, like the reference's keyword arguments."""
    import copy
    if not floating_joint_type.isfloating:
        raise ValueError("floating_joint_type must be a floating joint type")
    bodymap = {} if bodymap is None else bodymap
    jointmap = {} if jointmap is None else jointmap
    bodymap.clear()
    jointmap.clear()
    root = bodymap[mechanism.root_body] = RigidBody(mechanism.root_body.name)
    ret = Mechanism(root, gravity=mechanism.gravitational_acceleration)
    for src in mechanism.non_root_bodies():
        body = bodymap[src] = RigidBody(src.name, src.inertia.copy())
        ret.attach(root, body, Joint(str(src.name), floating_joint_type()))
    for src in mechanism.joints + mechanism.non_tree_joints:             # _copyjoint! (:48-63)
        joint = jointmap[src] = Joint(src.name, copy.deepcopy(src.joint_type), position_bounds=src.position_bounds,
                                      velocity_bounds=src.velocity_bounds, effort_bounds=src.effort_bounds)
        ret.attach(bodymap[src.predecessor], bodymap[src.successor], joint, joint_pose=src.joint_to_predecessor,
                   successor_pose=src.joint_to_successor.inv())
    return ret


# -------------------------------------------------------------------------------------------------
# random test fixtures (mechanism_modification.jl:382-426)
# -------------------------------------------------------------------------------------------------
def rand_tree_mechanism(rng, joint_types: Sequence[type], parentselector: Optional[Callable] = None) -> Mechanism:
    """Each new body is attached to a parent chosen by ``parentselector(mechanism, rng)`` (default: any
    existing body including the world, like ``rand(bodies(mechanism))``)."""
    if parentselector is None:
        parentselector = lambda m, r: m.bodies[int(r.integers(len(m.bodies)))]
    mech = Mechanism(RigidBody("world"))
    parent = mech.root_body
    for i, jt in enumerate(joint_types, start=1):
        joint = Joint(f"joint{i}", jt.rand(rng))
        body = RigidBody(f"body{i}", SpatialInertia.rand(rng))
        mech.attach(parent, body, joint, joint_pose=Transform3D.rand(rng))
        parent = parentselector(mech, rng)
    return mech


def rand_chain_mechanism(rng, joint_types: Sequence[type]) -> Mechanism:
    return rand_tree_mechanism(rng, joint_types, lambda m, r: m.bodies[-1])


def rand_floating_tree_mechanism(rng, nonfloating_joint_types: Sequence[type]) -> Mechanism:
    def sel(m, r):
        nr = m.non_root_bodies()
        return m.root_body if not nr else nr[int(r.integers(len(nr)))]
    return rand_tree_mechanism(rng, [QuaternionFloating, *nonfloating_joint_types], sel)


def effort_bounds(mechanism: "Mechanism"):
    """The tree joints' effort bounds in velocity order: ``(lo, hi)``, two float64 arrays [nv] -- the saturation of a ``JointPD``."""
    b = [e for j in mechanism.joints for e in j.effort_bounds]
    return np.array([x.lower for x in b], float), np.array([x.upper for x in b], float)
