"""Host-side (numpy, fp64) 3-vector / transform / spatial-inertia helpers.

These are used ONLY to build and flatten a model on the host (URDF parsing, fixed-joint
merging, frame canonicalisation).  The batched dynamics never run through this file: they
run in the CUDA kernels behind the C-ABI (``csrc/``).

Conventions follow the reference (all citations relative to the root of RigidBodyDynamics.jl v2.5.0):
  * 6-vectors are [angular; linear]                      -- src/spatial/common.jl:13
  * ``Transform3D`` maps coordinates FROM one frame TO another: x_to = R x_from + p
                                                          -- src/spatial/transform3d.jl:7-69
  * ``SpatialInertia`` = (moment about the frame origin, cross_part = m*com, mass)
                                                          -- src/spatial/motion_force_interaction.jl:28-37
"""
from __future__ import annotations

import numpy as np

__all__ = [
    "Transform3D", "SpatialInertia", "rot_x", "rot_y", "rot_z", "rot_rpy", "rot_angle_axis",
    "rot_quat", "rot_mrp", "hat", "rotation_between", "random_rotation", "random_unit_quaternion",
    "quat_to_mrp",
]


def hat(v):
    """3-vector -> skew-symmetric matrix (src/spatial/util.jl:56-61)."""
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def rot_x(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[1, 0, 0], [0, c, -s], [0, s, c]], dtype=float)


def rot_y(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]], dtype=float)


def rot_z(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]], dtype=float)


def rot_rpy(roll, pitch, yaw):
    """URDF rpy -> R = Rz(yaw) Ry(pitch) Rx(roll)  (src/urdf/parse.jl:46-51; goldens test/test_urdf.jl:79-102)."""
    return rot_z(yaw) @ rot_y(pitch) @ rot_x(roll)


def rot_angle_axis(theta, axis):
    """Rodrigues formula in the element order the reference restates at
    src/joint_types/sin_cos_revolute.jl:69-96 (axis must be unit length)."""
    x, y, z = axis
    s, c = np.sin(theta), np.cos(theta)
    c1 = 1.0 - c
    return np.array([
        [1 - c1 * y * y - c1 * z * z, c1 * x * y - s * z, c1 * x * z + s * y],
        [c1 * x * y + s * z, 1 - c1 * x * x - c1 * z * z, c1 * y * z - s * x],
        [c1 * x * z - s * y, c1 * y * z + s * x, 1 - c1 * x * x - c1 * y * y],
    ])


def rot_quat(w, x, y, z):
    """Quaternion [w x y z] -> rotation matrix, NOT normalised (quaternion_floating.jl:29-32,81-83).
    For unit quaternions every standard formula agrees to rounding (SURVEY 8(c))."""
    return np.array([
        [1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
        [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
        [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)],
    ])


def rot_mrp(x, y, z):
    """Modified Rodrigues parameters -> rotation (spquat_floating.jl:30-32): the stereographic
    projection of the unit quaternion, p = vec/(1+w)."""
    n2 = x * x + y * y + z * z
    w = (1 - n2) / (1 + n2)
    f = 2 / (1 + n2)
    return rot_quat(w, f * x, f * y, f * z)


def quat_to_mrp(q):
    w, x, y, z = q
    return np.array([x, y, z]) / (1 + w)


def rotation_between(u, v):
    """A rotation R with R u/|u| = v/|v| (used for the z-alignment of 1-DoF joint axes on the host)."""
    u = np.asarray(u, float) / np.linalg.norm(u)
    v = np.asarray(v, float) / np.linalg.norm(v)
    c = float(u @ v)
    if c > 1 - 1e-15:
        return np.eye(3)
    if c < -1 + 1e-15:
        # 180 degrees about any axis orthogonal to u
        a = np.cross(u, [1.0, 0, 0])
        if np.linalg.norm(a) < 1e-8:
            a = np.cross(u, [0, 1.0, 0])
        a /= np.linalg.norm(a)
        return 2 * np.outer(a, a) - np.eye(3)
    w = np.cross(u, v)
    K = hat(w)
    return np.eye(3) + K + K @ K / (1 + c)


def random_unit_quaternion(rng):
    q = rng.standard_normal(4)
    return q / np.linalg.norm(q)


def random_rotation(rng):
    return rot_quat(*random_unit_quaternion(rng))


class Transform3D:
    """x_to = rot @ x_from + trans  (src/spatial/transform3d.jl:7-69; frames are implicit here)."""

    __slots__ = ("rot", "trans")

    def __init__(self, rot=None, trans=None):
        self.rot = np.eye(3) if rot is None else np.asarray(rot, float).reshape(3, 3).copy()
        self.trans = np.zeros(3) if trans is None else np.asarray(trans, float).reshape(3).copy()

    @staticmethod
    def identity():
        return Transform3D()

    def __mul__(self, other: "Transform3D") -> "Transform3D":      # transform3d.jl:60-64
        return Transform3D(self.rot @ other.rot, self.rot @ other.trans + self.trans)

    def inv(self) -> "Transform3D":                                 # transform3d.jl:66-69
        rt = self.rot.T
        return Transform3D(rt, -(rt @ self.trans))

    def mat(self):
        m = np.eye(4)
        m[:3, :3] = self.rot
        m[:3, 3] = self.trans
        return m

    def flat12(self):
        """Row-major R (9) followed by p (3): the layout of rbd_model_desc.X_tree."""
        return np.concatenate([self.rot.reshape(9), self.trans])

    @staticmethod
    def rand(rng):                                                  # transform3d.jl rand
        return Transform3D(random_rotation(rng), rng.random(3))

    def __repr__(self):
        return f"Transform3D(rot={self.rot.tolist()}, trans={self.trans.tolist()})"


class SpatialInertia:
    """(moment about frame origin, cross_part = m*com, mass)  (motion_force_interaction.jl:28-37)."""

    __slots__ = ("moment", "cross_part", "mass")

    def __init__(self, moment=None, cross_part=None, mass=0.0, *, com=None, moment_about_com=None):
        if moment_about_com is not None:
            # motion_force_interaction.jl:50-58: moment = moment_about_com - m * hat(com)^2
            com = np.asarray(com, float)
            h = hat(com)
            moment = np.asarray(moment_about_com, float) - mass * (h @ h)
            cross_part = mass * com
        elif com is not None:
            cross_part = mass * np.asarray(com, float)
        self.moment = np.zeros((3, 3)) if moment is None else np.asarray(moment, float).reshape(3, 3).copy()
        self.cross_part = np.zeros(3) if cross_part is None else np.asarray(cross_part, float).reshape(3).copy()
        self.mass = float(mass)

    @staticmethod
    def zero():
        return SpatialInertia()

    def copy(self):
        return SpatialInertia(self.moment, self.cross_part, self.mass)

    def __add__(self, other):                                       # motion_force_interaction.jl:147-153
        return SpatialInertia(self.moment + other.moment, self.cross_part + other.cross_part,
                              self.mass + other.mass)

    def transform(self, t: Transform3D) -> "SpatialInertia":
        """motion_force_interaction.jl:160-176, same operation order."""
        J, mc, m = self.moment, self.cross_part, self.mass
        R, p = t.rot, t.trans
        Rmc = R @ mc
        mp = m * p
        mcnew = Rmc + mp
        X = np.outer(Rmc, p)
        Y = X + X.T + np.outer(mp, p)
        Jnew = R @ J @ R.T - Y + np.trace(Y) * np.eye(3)
        return SpatialInertia(Jnew, mcnew, m)

    def center_of_mass(self):
        return self.cross_part / self.mass

    def mat6(self):
        """6x6 [J c^; c^T m1]  (motion_force_interaction.jl:102-107)."""
        M = np.zeros((6, 6))
        M[:3, :3] = self.moment
        M[:3, 3:] = hat(self.cross_part)
        M[3:, :3] = hat(self.cross_part).T
        M[3:, 3:] = self.mass * np.eye(3)
        return M

    def flat13(self):
        """Row-major moment (9), cross_part (3), mass (1): the layout of rbd_model_desc.inertia."""
        return np.concatenate([self.moment.reshape(9), self.cross_part, [self.mass]])

    @staticmethod
    def rand(rng):
        """Random physical inertia, same recipe as motion_force_interaction.jl:178-197."""
        ixx = rng.random() / 10.0
        iyy = rng.random() / 10.0
        lb, ub = abs(ixx - iyy), ixx + iyy
        izz = rng.random() * (ub - lb) + lb
        R = random_rotation(rng)
        mcom = R @ np.diag([ixx, iyy, izz]) @ R.T
        com = rng.random(3) - 0.5
        mass = rng.random()
        return SpatialInertia(mass=mass, com=com, moment_about_com=mcom)

    def __repr__(self):
        return f"SpatialInertia(mass={self.mass}, cross_part={self.cross_part.tolist()})"
