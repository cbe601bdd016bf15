"""URDF -> Mechanism with the reference's exact ordering rules (src/urdf/parse.jl:162-221).

Rules that decide the q/v/τ index order (get one wrong and every batched array is scrambled):
  * only DIRECT children <link>/<joint> of <robot> are read (parse.jl:184-185) -- transmissions
    contain nested <joint> tags that must be ignored;
  * the spanning tree is breadth-first from the unique root link, children in document order of the
    <joint> elements (parse.jl:187-206, graphs/spanning_tree.jl:45-83);
  * the root link is attached to the world by "<rootlink>_to_world", QuaternionFloating iff
    ``floating`` else Fixed (parse.jl:121-127);
  * fixed tree joints are then removed, the others keep their relative order (parse.jl:216-218);
  * <origin rpy> -> Rz(yaw) Ry(pitch) Rx(roll) (parse.jl:46-51); <inertia> is about the COM in the
    <inertial><origin> frame and is transformed into the link frame (parse.jl:104-112);
  * <dynamics damping>, <limit>, <mimic> do not enter the dynamics (parse.jl:74-95); <limit> gives the joint bounds
    (parse.jl:75-91): lower / upper the position bounds, velocity="v" / effort="e" the bounds (-v, v) / (-e, e).
"""
from __future__ import annotations

import xml.etree.ElementTree as ET
from collections import deque
from typing import Dict, Optional

import numpy as np

from .joint_types import (Fixed, JointType, Planar, Prismatic, QuaternionFloating, Revolute)
from .mechanism import DEFAULT_GRAVITATIONAL_ACCELERATION, Bounds, Joint, Mechanism, RigidBody
from .spatial import SpatialInertia, Transform3D, rot_rpy, rotation_between


def default_urdf_joint_types() -> Dict[str, type]:
    """parse.jl:6-15."""
    return {"revolute": Revolute, "continuous": Revolute, "prismatic": Prismatic,
            "floating": QuaternionFloating, "fixed": Fixed, "planar": Planar}


def _vec(e: Optional[ET.Element], name: str, default: str):
    s = default if e is None or e.get(name) is None else e.get(name)
    return np.array([float(x) for x in s.split()])


def _scalar(e: Optional[ET.Element], name: str, default: str = "0"):
    s = default if e is None or e.get(name) is None else e.get(name)
    return float(s)


def parse_pose(xml_pose: Optional[ET.Element]):
    """parse.jl:40-51."""
    if xml_pose is None:
        return np.eye(3), np.zeros(3)
    rpy = _vec(xml_pose, "rpy", "0 0 0")
    return rot_rpy(rpy[0], rpy[1], rpy[2]), _vec(xml_pose, "xyz", "0 0 0")


def _pose_dict(xml_pose: Optional[ET.Element]):
    if xml_pose is None:
        return None
    return {"xyz": _vec(xml_pose, "xyz", "0 0 0").tolist(), "rpy": _vec(xml_pose, "rpy", "0 0 0").tolist()}


def read_urdf(filename: str) -> dict:
    """URDF file -> plain "robot description" dict holding exactly what the reference's parser reads:
    links (name, optional inertial: mass / origin / 6 inertia entries) and joints (name, type, parent, child, origin,
    axis, limit: the attributes lower / upper / velocity / effort present on its <limit> elements) in DOCUMENT order, direct
    children of <robot> only (parse.jl:184-185)."""
    xroot = ET.parse(filename).getroot()
    if xroot.tag != "robot":
        raise ValueError("URDF root element must be <robot>")
    links, joints = [], []
    for xl in xroot.findall("link"):
        xi = xl.find("inertial")
        inertial = None
        if xi is not None:
            e = xi.find("inertia")
            inertial = {
                "mass": _scalar(xi.find("mass"), "value", "0"),
                "origin": _pose_dict(xi.find("origin")),
                "inertia": [_scalar(e, k) for k in ("ixx", "ixy", "ixz", "iyy", "iyz", "izz")],
            }
        links.append({"name": xl.get("name"), "inertial": inertial})
    for xj in xroot.findall("joint"):
        ax = xj.find("axis")
        limit = {}
        for xlim in xj.findall("limit"):          # later elements override earlier ones, attribute by attribute (parse.jl:78-91)
            limit.update({k: float(xlim.get(k)) for k in ("lower", "upper", "velocity", "effort") if xlim.get(k) is not None})
        joints.append({
            "limit": limit,
            "name": xj.get("name"), "type": xj.get("type"),
            "parent": xj.find("parent").get("link"), "child": xj.find("child").get("link"),
            "origin": _pose_dict(xj.find("origin")),
            "axis": None if ax is None or ax.get("xyz") is None else _vec(ax, "xyz", "1 0 0").tolist(),
        })
    return {"name": xroot.get("name"), "links": links, "joints": joints}


def load_description(path: str) -> dict:
    """Robot description stored as JSON (see ``read_urdf`` for the schema; written by tools/make_fixtures.py)."""
    import json
    with open(path) as f:
        return json.load(f)


def _pose(p):
    if p is None:
        return np.eye(3), np.zeros(3)
    rpy = p.get("rpy", [0, 0, 0])
    return rot_rpy(rpy[0], rpy[1], rpy[2]), np.asarray(p.get("xyz", [0, 0, 0]), float)


def _joint_type_from(j: dict, joint_types: Dict[str, type]) -> JointType:
    """parse.jl:53-72."""
    t = j["type"]
    if t not in joint_types:
        raise ValueError(f"joint type {t} not recognized")
    cls = joint_types[t]
    axis = np.asarray(j["axis"] if j.get("axis") is not None else [1.0, 0, 0], float)
    if t in ("revolute", "continuous", "prismatic"):
        return cls(axis)
    if t in ("floating", "fixed"):
        return cls()
    if t == "planar":
        R = rotation_between([0.0, 0.0, 1.0], axis)          # plane perpendicular to the URDF axis
        return cls(R @ np.array([1.0, 0, 0]), R @ np.array([0, 1.0, 0]))
    raise ValueError(f"joint type {t} not recognized")


def _joint_bounds(j: dict, jt: JointType):
    """parse_joint_bounds (parse.jl:75-91): (position, velocity, effort) bounds; descriptions without <limit> get infinite ones."""
    lim = j.get("limit") or {}
    pos = Bounds(lim.get("lower", -np.inf), lim.get("upper", np.inf))
    vel = Bounds(-lim["velocity"], lim["velocity"]) if "velocity" in lim else Bounds()
    eff = Bounds(-lim["effort"], lim["effort"]) if "effort" in lim else Bounds()
    return dict(position_bounds=[pos] * jt.nq, velocity_bounds=[vel] * jt.nv, effort_bounds=[eff] * jt.nv)


def _body_from(link: dict) -> RigidBody:
    """parse.jl:104-119: inertia about the COM in the <inertial><origin> frame, moved to the link frame;
    links without <inertial> get zero inertia."""
    xi = link.get("inertial")
    if xi is None:
        inertia = SpatialInertia.zero()
    else:
        ixx, ixy, ixz, iyy, iyz, izz = xi["inertia"]
        moment = np.array([[ixx, ixy, ixz], [ixy, iyy, iyz], [ixz, iyz, izz]])
        rot, trans = _pose(xi.get("origin"))
        inertia = SpatialInertia(moment, np.zeros(3), xi["mass"]).transform(Transform3D(rot, trans))
    return RigidBody(link["name"], inertia)


def mechanism_from_description(desc: dict, *, floating: bool = False, joint_types: Optional[Dict[str, type]] = None,
                               root_joint_type: Optional[JointType] = None, remove_fixed_tree_joints: bool = True,
                               gravity=DEFAULT_GRAVITATIONAL_ACCELERATION) -> Mechanism:
    """The body of ``parse_urdf`` (parse.jl:162-221) on an already-read robot description."""
    jt = default_urdf_joint_types() if joint_types is None else joint_types
    if root_joint_type is None:
        root_joint_type = jt["floating" if floating else "fixed"]()
    if floating and not root_joint_type.isfloating:
        raise ValueError("Ambiguous input arguments: `floating` specified, but `root_joint_type` is not a "
                         "floating joint type.")                                    # parse.jl:177-179
    name_to_link = {l["name"]: l for l in desc["links"]}
    out_edges = {n: [] for n in name_to_link}   # document order == add_edge! order
    has_parent = set()
    for j in desc["joints"]:
        out_edges[j["parent"]].append(j)
        has_parent.add(j["child"])
    roots = [n for n in name_to_link if n not in has_parent]
    if len(roots) != 1:
        raise ValueError("Can only handle a single root")                          # parse.jl:204

    # breadth-first spanning tree, FIFO over edges (graphs/spanning_tree.jl:45-83 with next_edge = first)
    tree_edges = []
    visited = {roots[0]}
    frontier = deque(out_edges[roots[0]])
    while frontier:
        e = frontier.popleft()
        if e["child"] in visited:
            continue                             # a second path to an already-placed link (loop): skipped
        visited.add(e["child"])
        tree_edges.append(e)
        frontier.extend(out_edges[e["child"]])
    if len(visited) != len(name_to_link):
        raise ValueError("Graph is not connected.")

    mech = Mechanism(RigidBody("world"), gravity=gravity)
    bodies = {}
    body = _body_from(name_to_link[roots[0]])
    bodies[roots[0]] = body
    mech.attach(mech.root_body, body, Joint(f"{body.name}_to_world", root_joint_type))   # parse.jl:121-127
    for e in tree_edges:
        parent = bodies[e["parent"]]
        joint_type = _joint_type_from(e, jt)
        joint = Joint(e["name"], joint_type, **_joint_bounds(e, joint_type))
        rot, trans = _pose(e.get("origin"))
        body = _body_from(name_to_link[e["child"]])
        bodies[e["child"]] = body
        mech.attach(parent, body, joint, joint_pose=Transform3D(rot, trans))             # parse.jl:129-140
    if remove_fixed_tree_joints:
        mech.remove_fixed_tree_joints()
    return mech


def parse_urdf(filename: str, *, floating: bool = False, joint_types: Optional[Dict[str, type]] = None,
               root_joint_type: Optional[JointType] = None, remove_fixed_tree_joints: bool = True,
               gravity=DEFAULT_GRAVITATIONAL_ACCELERATION) -> Mechanism:
    """Mirror of ``parse_urdf(filename; floating, joint_types, root_joint_type, remove_fixed_tree_joints,
    gravity)`` (parse.jl:162-221).  ``scalar_type`` is not a parameter: the host model is always fp64 and
    the batch dtype is chosen per call (SURVEY appendix: promotion rule mechanism_state.jl:179-182)."""
    return mechanism_from_description(read_urdf(filename), floating=floating, joint_types=joint_types,
                                      root_joint_type=root_joint_type,
                                      remove_fixed_tree_joints=remove_fixed_tree_joints, gravity=gravity)


_MODELS_DIR = __import__("os").path.join(__import__("os").path.dirname(__import__("os").path.abspath(__file__)), "models")


def load_model(name: str, **kwargs) -> Mechanism:
    """Load one of the robot descriptions shipped in ``models/`` (``<name>.json`` or ``<name>.urdf``)."""
    import os
    pj = os.path.join(_MODELS_DIR, name + ".json")
    if os.path.exists(pj):
        return mechanism_from_description(load_description(pj), **kwargs)
    pu = os.path.join(_MODELS_DIR, name + ".urdf")
    if os.path.exists(pu):
        return parse_urdf(pu, **kwargs)
    raise FileNotFoundError(f"no model named {name!r} in {_MODELS_DIR}")
