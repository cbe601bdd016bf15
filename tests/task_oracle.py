"""TEST INFRASTRUCTURE -- fp64 restatement of the reference's task-space kinematics in numpy, on top of the CPU oracle.

Built from the oracle's root-frame outputs (transforms and path Jacobians from ``Oracle.kinematics``, body accelerations from
``Oracle.inverse_dynamics_bodies``) and the reference's formulas:
  relative_transform(state, from, to) = inv(T_to) T_from                        src/mechanism_state.jl:1011-1014
  relative_twist(state, body, base)   = twist_wrt_world(body) - twist_wrt_world(base), root frame   :1016-1038
  transform(twist, T)                 = Ad(T) twist                             src/spatial/spatialmotion.jl
  geometric_jacobian!(J, state, path) column = Ad(inv(T_F)) (±S_k)              src/mechanism_algorithms.jl:80-132
  point_jacobian!: column = -p̂ w_S + v_S in J.frame                             :154-224
  point_velocity(twist, point)        = w x p + v                               spatialmotion.jl:346-349
  relative_acceleration               = a_body - a_base (root frame, gravity in both)   mechanism_algorithms.jl:421-426
  transform(state, accel, to)         = Ad(old_to_new) (a + v_{old wrt new} x v_{body wrt base})   mechanism_state.jl:1049-1056,
                                                                                 spatialmotion.jl:375-401
  point_acceleration(twist, accel, p) = w' x p + a_lin + w x (w x p + v_lin)     spatialmotion.jl:351-363
Arrays are [rows, B]; 6-vectors [angular; linear].  Tasks are ``TaskFrame``s (rigidbodydynamics.jl_b200.kinematics).
"""
from __future__ import annotations

import numpy as np

import rigidbodydynamics.jl_b200 as rbd
from oracle import Oracle

OUTPUTS = ("transform", "point", "twist", "point_velocity", "geometric_jacobian", "point_jacobian", "acceleration",
           "point_acceleration")


def cross(a, b):
    """cross product along axis 0 of [3, ...] arrays"""
    return np.stack([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])


def motion_cross(m1, m2):
    """se3_commutator: [w1 x w2; w1 x v2 + v1 x w2]"""
    return np.concatenate([cross(m1[:3], m2[:3]), cross(m1[:3], m2[3:]) + cross(m1[3:], m2[:3])])


def rotT(R, x):
    """R^T x for R [3, 3, B], x [3, ...B]"""
    return np.einsum("jib,j...b->i...b", R, x)


def rot(R, x):
    return np.einsum("ijb,j...b->i...b", R, x)


def to_frame(R, p, m):
    """root-frame motion vector(s) m [6, ...B] -> the frame with root pose (R, p): Ad(inv(T))"""
    w, l = m[:3], m[3:]
    pb = p.reshape((3,) + (1,) * (w.ndim - 2) + (p.shape[-1],))
    return np.concatenate([rotT(R, w), rotT(R, l + cross(w, np.broadcast_to(pb, w.shape)))])


def from_frame(R, p, m):
    """motion vector m [6, B] in the frame with root pose (R, p) -> root frame: Ad(T)"""
    w = rot(R, m[:3])
    return np.concatenate([w, rot(R, m[3:]) + cross(p, w)])


class TaskOracle:
    """Root-frame state of every body of one batch (q, v, v̇), and the task outputs built from it."""

    def __init__(self, mech, q, v=None, vd=None):
        self.mech = mech
        self.desc = desc = mech.flatten()
        self.orc = Oracle(desc)
        self.q = np.asarray(q, np.float64)
        self.B = self.q.shape[1]
        self.v = None if v is None else np.asarray(v, np.float64)
        self.vd = np.zeros((desc.nv, self.B)) if vd is None else np.asarray(vd, np.float64)
        self.index = {id(j.successor): i for i, j in enumerate(mech.joints)}
        T = self.orc.kinematics(self.q, None, want=("transforms",))["transforms"].reshape(desc.nb, 12, self.B)
        self.R = {i: T[i, :9].reshape(3, 3, self.B) for i in range(desc.nb)}
        self.p = {i: T[i, 9:] for i in range(desc.nb)}
        self.R[-1] = np.broadcast_to(np.eye(3)[:, :, None], (3, 3, self.B)).copy()
        self.p[-1] = np.zeros((3, self.B))
        if self.v is not None:
            self.tw = {-1: np.zeros((6, self.B))}
            for i in range(desc.nb):
                self.tw[i] = np.einsum("kcb,kb->cb", self.J(-1, i), self.v)
            acc, _ = self.orc.inverse_dynamics_bodies(self.q, self.v, self.vd)
            self.acc = {i: acc[6 * i:6 * i + 6] for i in range(desc.nb)}
            self.acc[-1] = np.zeros((6, self.B))
            self.acc[-1][3:] = -np.asarray(desc.gravity, np.float64)[:, None]          # a_root = -g, spatial_accelerations!

    def idx(self, body):
        return -1 if body is None or body is self.mech.root_body else self.index[id(body)]

    def J(self, base, body):
        """root-frame geometric Jacobian of path(mechanism, base, body): [nv, 6, B]"""
        b0 = self.mech.root_body if base < 0 else self.mech.joints[base].successor
        b1 = self.mech.root_body if body < 0 else self.mech.joints[body].successor
        sign = rbd.path(self.mech, b0, b1).sign
        if not sign.any():
            return np.zeros((self.desc.nv, 6, self.B))
        return self.orc.kinematics(self.q, None, sign, want=("J",))["J"].reshape(self.desc.nv, 6, self.B)

    def accel_in(self, a_root, f, body, base):
        """transform(state, accel, default_frame(f)) of a root-frame acceleration of `body` w.r.t. `base` (indices)"""
        if f < 0:
            return a_root
        rel = self.tw[body] - self.tw[base]
        return to_frame(self.R[f], self.p[f], a_root - motion_cross(self.tw[f], rel))

    def accel_to_root(self, a_f, f, body, base):
        """the inverse: transform(state, accel expressed in default_frame(f), root frame)"""
        if f < 0:
            return a_f
        rel = self.tw[body] - self.tw[base]
        return from_frame(self.R[f], self.p[f], a_f) + motion_cross(self.tw[f], rel)

    def task(self, t):
        """dict of the eight outputs of one TaskFrame (velocity-dependent ones only when v was given)"""
        b, a, f = self.idx(t.body), self.idx(t.base), self.idx(t.frame)
        pt = np.zeros(3) if t.point is None else np.asarray(t.point, np.float64).reshape(3)
        Rb, pb, Ra, pa, RF, pF = self.R[b], self.p[b], self.R[a], self.p[a], self.R[f], self.p[f]
        out = {}
        Rr = np.einsum("jib,jkb->ikb", Ra, Rb)
        out["transform"] = np.concatenate([Rr.reshape(9, self.B), rotT(Ra, pb - pa)])
        proot = pb + rot(Rb, np.broadcast_to(pt[:, None], (3, self.B)))
        pf = rotT(RF, proot - pF)
        out["point"] = pf
        J = self.J(a, b).transpose(1, 0, 2)                                    # [6, nv, B]
        out["geometric_jacobian"] = to_frame(RF, pF, J).transpose(1, 0, 2).reshape(6 * self.desc.nv, self.B)
        Jp = rotT(RF, J[3:] + cross(J[:3], np.broadcast_to(proot[:, None], J[:3].shape)))
        out["point_jacobian"] = Jp.transpose(1, 0, 2).reshape(3 * self.desc.nv, self.B)
        if self.v is None:
            return out
        rel = self.tw[b] - self.tw[a]
        twf = to_frame(RF, pF, rel)
        out["twist"] = twf
        pv = cross(twf[:3], pf) + twf[3:]
        out["point_velocity"] = pv
        af = self.accel_in(self.acc[b] - self.acc[a], f, b, a)
        out["acceleration"] = af
        out["point_acceleration"] = cross(af[:3], pf) + af[3:] + cross(twf[:3], pv)
        return out

    def tasks(self, tasks, want=OUTPUTS):
        """outputs of several tasks stacked like rbd_task_kinematics: task t at rows t*R .. (t+1)*R - 1"""
        per = [self.task(t) for t in tasks]
        return {k: np.concatenate([p[k] for p in per]) for k in want if k in per[0]}
