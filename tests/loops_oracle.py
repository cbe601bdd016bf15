"""TEST INFRASTRUCTURE -- the reference's dynamics! for mechanisms with loops, restated on the host (numpy / scipy) over the CPU oracle.

The tree quantities come from oracle/ (world-frame restatement of the reference): transforms to root, geometric Jacobians, body
accelerations, M and c.  On top of them this module restates, for the non-tree joints in non_tree_joints order:
  non-tree joint transform      mechanism_state.jl:703-711     inv(T_pred X_pred) (T_succ X_succ)
  wrench subspaces              mechanism_state.jl:786-793     basis (frame after the joint) moved to the root frame
  constraint_jacobian!          mechanism_algorithms.jl:574-598  K = T^T J(path(pred, succ))   (J has the -1 / +1 path signs)
  constraint_bias!              mechanism_algorithms.jl:630-673  k = T^T (v_s x v_p + b_s - b_p - stab), SE3 PD linearised
  dynamics_solve! (BLAS branch) mechanism_algorithms.jl:747-822  Cholesky, triangular solves, LAPACK gelsy with rcond 1e-10
and the fixtures of the loop tests (four-bar linkage, Atlas in double support, maximal-coordinate trees) and a ctypes binding of
tests/hostsim/hostsim_loops.cpp (the kernel's per-sample function compiled for the CPU).
"""
from __future__ import annotations

import ctypes
import functools

import numpy as np
import scipy.linalg as sla

import rigidbodydynamics.jl_b200 as rbd
from oracle import Oracle
from rigidbodydynamics.jl_b200._cabi import RbdModelDesc, make_desc
from rigidbodydynamics.jl_b200.loops import _DEFAULT, constraint_wrench_subspace, loop_desc
from rigidbodydynamics.jl_b200.spatial import SpatialInertia, Transform3D
from tests import hostsim

RCOND = 1e-10       # singular_value_zero_tolerance, mechanism_algorithms.jl:804


def _motion_cross(a, b):
    """[w; l] x [w'; l'] (spatialmotion.jl)."""
    return np.concatenate([np.cross(a[:3], b[:3]), np.cross(a[:3], b[3:]) + np.cross(a[3:], b[:3])])


def _pose(tr, i, b):
    if i < 0:
        return np.eye(3), np.zeros(3)
    return tr[12 * i:12 * i + 9, b].reshape(3, 3), tr[12 * i + 9:12 * i + 12, b]


class LoopOracle:
    """dynamics! with loops for one Mechanism (spanning tree on the CPU oracle)."""

    def __init__(self, mechanism):
        self.mech = mechanism
        self.desc = mechanism.flatten()
        self.oracle = Oracle(self.desc)
        self.nv, self.nq, self.nb = self.desc.nv, self.desc.nq, self.desc.nb
        self.g = np.asarray(mechanism.gravitational_acceleration, float)
        self.index = {id(j.successor): i for i, j in enumerate(mechanism.joints)}

    def body(self, b):
        return -1 if b is self.mech.root_body else self.index[id(b)]

    def _sign(self, src, dst):
        return rbd.path(self.mech, src, dst).sign

    def constraints(self, q, v, stabilization_gains=_DEFAULT):
        """K [B, nl, nv] and k [B, nl] (items 1-4 of the contract)."""
        q = np.asarray(q, float).reshape(self.nq, -1)
        v = np.asarray(v, float).reshape(self.nv, -1)
        B = q.shape[1]
        ld = loop_desc(self.mech, stabilization_gains)
        tr = self.oracle.kinematics(q, want=("transforms",))["transforms"]
        acc, _ = self.oracle.inverse_dynamics_bodies(q, v)            # v̇ = 0: bias accelerations with the root at -g
        g6 = np.concatenate([np.zeros(3), -self.g])
        nl = ld.nc
        K = np.zeros((B, nl, self.nv))
        k = np.zeros((B, nl))
        c0 = 0
        for l, j in enumerate(self.mech.non_tree_joints):
            P, S = self.body(j.predecessor), self.body(j.successor)
            Jp = self.oracle.kinematics(q, sign=self._sign(j.predecessor, j.successor), want=("J",))["J"]   # [6 nv, B]
            Jroot_p = None if P < 0 else self.oracle.kinematics(q, sign=self._sign(self.mech.root_body, j.predecessor), want=("J",))["J"]
            Jroot_s = None if S < 0 else self.oracle.kinematics(q, sign=self._sign(self.mech.root_body, j.successor), want=("J",))["J"]
            basis = constraint_wrench_subspace(j.joint_type)                  # [6, n]
            n = basis.shape[1]
            for b in range(B):
                Rpb, ppb = _pose(tr, P, b)
                Rsb, psb = _pose(tr, S, b)
                Xp, Xs = j.joint_to_predecessor, j.joint_to_successor
                Rp, pp = Rpb @ Xp.rot, Rpb @ Xp.trans + ppb                   # frame before the joint -> root
                Rs, ps = Rsb @ Xs.rot, Rsb @ Xs.trans + psb                   # frame after the joint -> root
                T = np.zeros((6, n))
                T[3:] = Rs @ basis[3:]
                T[:3] = Rs @ basis[:3] + np.cross(ps, T[3:].T).T
                Jcols = Jp[:, b].reshape(self.nv, 6).T                         # [6, nv]
                K[b, c0:c0 + n] = T.T @ Jcols
                vp = np.zeros(6) if P < 0 else Jroot_p[:, b].reshape(self.nv, 6).T @ v[:, b]
                vs = np.zeros(6) if S < 0 else Jroot_s[:, b].reshape(self.nv, 6).T @ v[:, b]
                bp = np.zeros(6) if P < 0 else acc[6 * P:6 * P + 6, b] - g6
                bs = np.zeros(6) if S < 0 else acc[6 * S:6 * S + 6, b] - g6
                a = _motion_cross(vs, vp) + (bs - bp)
                if ld.gains is not None:
                    ka, da, kl, dl = ld.gains[l]
                    Re, pe = Rp.T @ Rs, Rp.T @ (ps - pp)                        # joint transform, after -> before
                    jt = vs - vp
                    ew = Rs.T @ jt[:3]
                    el = Rs.T @ (jt[3:] - np.cross(ps, jt[:3]))
                    psi = 0.5 * np.array([Re[2, 1] - Re[1, 2], Re[0, 2] - Re[2, 0], Re[1, 0] - Re[0, 1]])
                    sa = -ka * psi - da * ew
                    sl = -kl * (Re.T @ pe) - dl * el
                    wa = Rs @ sa
                    a = a - np.concatenate([wa, Rs @ sl + np.cross(ps, wa)])
                k[b, c0:c0 + n] = T.T @ a
            c0 += n
        return K, k

    def dynamics(self, q, v, tau=None, wext=None, stabilization_gains=_DEFAULT, rcond=RCOND):
        """Returns dict(vd [nv, B], lam [nl, B], K [nl*nv, B] (row c + j nl), k [nl, B], A [B, nl, nl])."""
        q = np.asarray(q, float).reshape(self.nq, -1)
        v = np.asarray(v, float).reshape(self.nv, -1)
        B = q.shape[1]
        tau = np.zeros((self.nv, B)) if tau is None else np.asarray(tau, float).reshape(self.nv, B)
        K, k = self.constraints(q, v, stabilization_gains)
        Mm = self.oracle.mass_matrix(q)
        c = self.oracle.dynamics_bias(q, v, wext)
        nl = K.shape[1]
        vd, lam, A = np.zeros((self.nv, B)), np.zeros((nl, B)), np.zeros((B, nl, nl))
        for b in range(B):
            M = Mm[:, b].reshape(self.nv, self.nv, order="F")
            L = sla.cholesky(M, lower=True)
            tb = tau[:, b] - c[:, b]
            if nl:
                Y = sla.solve_triangular(L, K[b].T, lower=True).T                # Y = K L^-T
                z = sla.solve_triangular(L, tb, lower=True)
                A[b] = Y @ Y.T
                rhs = Y @ z + k[b]
                lam[:, b] = sla.lstsq(A[b], rhs, cond=rcond, lapack_driver="gelsy")[0]
                tb = tb - K[b].T @ lam[:, b]
            vd[:, b] = sla.cho_solve((L, True), tb)
        Kc = K.transpose(0, 2, 1).reshape(B, self.nv * nl).T.copy()          # entry (c, j) at row c + j nl
        return dict(vd=vd, lam=lam, K=Kc, Kb=K, k=k.T.copy(), A=A, M=Mm, c=c)


# ------------------------------------------------------------------------------------------------------------------------------
# fixtures
# ------------------------------------------------------------------------------------------------------------------------------
FOUR_BAR_Q0 = np.array([1.6707963267948966, -1.4591054166649482, 1.5397303602625536])     # test_simulate.jl:190-197


def four_bar():
    """The four-bar linkage of test/test_simulate.jl:127-188 (all axes along -y, loop joint4 between link2 and link3)."""
    g = -9.81
    l_0, l_1, l_2, l_3 = 1.10, 0.5, 1.20, 0.75
    m_1, m_2, m_3 = 0.5, 1.0, 0.75
    c_1, c_2, c_3 = 0.25, 0.60, 0.375
    I_1, I_2, I_3 = 0.333, 0.537, 0.4
    axis = np.array([0.0, -1.0, 0.0])
    world = rbd.RigidBody("world")
    mech = rbd.Mechanism(world, gravity=(0.0, 0.0, g))
    inertia = lambda I, m: SpatialInertia(mass=m, com=np.zeros(3), moment_about_com=I * np.outer(axis, axis))
    link1, link2, link3 = (rbd.RigidBody(n, inertia(I, m)) for n, I, m in (("link1", I_1, m_1), ("link2", I_2, m_2), ("link3", I_3, m_3)))
    j1, j2, j3, j4 = (rbd.Joint(f"joint{i}", rbd.Revolute(axis)) for i in range(1, 5))
    tr = lambda x: Transform3D(trans=(x, 0.0, 0.0))
    mech.attach(world, link1, j1, joint_pose=Transform3D.identity(), successor_pose=tr(c_1))
    mech.attach(link1, link2, j2, joint_pose=tr(l_1), successor_pose=tr(c_2))
    mech.attach(world, link3, j3, joint_pose=tr(l_0), successor_pose=tr(c_3))
    mech.attach(link2, link3, j4, joint_pose=tr(l_2), successor_pose=tr(-l_3))
    return mech


def closure_distance(lo, q):
    """|point(frame_before(loop joint)) - point(frame_after(loop joint))| in the root frame, per sample, first loop joint."""
    q = np.asarray(q, float).reshape(lo.nq, -1)
    j = lo.mech.non_tree_joints[0]
    tr = lo.oracle.kinematics(q, want=("transforms",))["transforms"]
    out = []
    for b in range(q.shape[1]):
        Rp, pp = _pose(tr, lo.body(j.predecessor), b)
        Rs, ps = _pose(tr, lo.body(j.successor), b)
        out.append(np.linalg.norm((Rp @ j.joint_to_predecessor.trans + pp) - (Rs @ j.joint_to_successor.trans + ps)))
    return np.array(out)


def energy(lo, q, v):
    kin = lo.oracle.kinematics(np.asarray(q, float).reshape(lo.nq, -1), np.asarray(v, float).reshape(lo.nv, -1), want=("ke", "pe"))
    return kin["ke"][0] + kin["pe"][0]


def atlas_double_support():
    """Atlas (floating base) with both feet welded to the world by Fixed loop joints at their configuration-independent
    reference poses: nl = 12."""
    mech = rbd.load_model("atlas", floating=True)
    for name, y in (("l_foot", 0.12), ("r_foot", -0.12)):
        foot = mech.findbody(name)
        mech.attach(mech.root_body, foot, rbd.Joint(f"{name}_weld", rbd.Fixed()),
                    joint_pose=Transform3D(trans=(0.0, y, 0.0)), successor_pose=Transform3D.identity())
    return mech


MC_JOINT_TYPES = (rbd.Revolute, rbd.Prismatic, rbd.Planar, rbd.QuaternionSpherical, rbd.SinCosRevolute, rbd.Fixed)


def maximal_coordinate_pair(seed, nbodies=12):
    """A random tree with a floating root and every joint type, and its maximal-coordinate twin (every body floating, every
    tree joint a loop joint): test/test_mechanism_modification.jl:274-318.  Returns (tree, mc, bodymap)."""
    rng = np.random.default_rng(seed)
    types = [MC_JOINT_TYPES[i % len(MC_JOINT_TYPES)] for i in range(nbodies - 1)]
    tree = rbd.rand_floating_tree_mechanism(rng, types)
    bodymap = {}
    mc = rbd.maximal_coordinates(tree, bodymap=bodymap)
    return tree, mc, bodymap


def mc_state_from_tree(tree, mc, bodymap, q, v):
    """q / v of the maximal-coordinate mechanism equivalent to the tree state (q, v) (one column): each floating joint carries
    the body's pose and its twist in the body frame."""
    lo = LoopOracle(tree)
    tr = lo.oracle.kinematics(q.reshape(-1, 1), want=("transforms",))["transforms"][:, 0]
    qm, vm = np.zeros(mc.num_positions()), np.zeros(mc.num_velocities())
    qs = vs = 0
    for jm in mc.joints:
        body = next(b for b, c in bodymap.items() if c is jm.successor)
        i = lo.index[id(body)]
        R, p = tr[12 * i:12 * i + 9].reshape(3, 3), tr[12 * i + 9:12 * i + 12]
        sign = rbd.path(tree, tree.root_body, body).sign
        Jc = lo.oracle.kinematics(q.reshape(-1, 1), sign=sign, want=("J",))["J"][:, 0].reshape(lo.nv, 6).T
        tw = Jc @ v
        w_b = R.T @ tw[:3]
        l_b = R.T @ (tw[3:] + np.cross(tw[:3], p))          # body-frame linear velocity of the body origin
        qm[qs:qs + 7] = np.concatenate([_rot_to_quat(R), p])
        vm[vs:vs + 6] = np.concatenate([w_b, l_b])
        qs += 7
        vs += 6
    return qm, vm


def _rot_to_quat(R):
    w = np.sqrt(max(0.0, 1 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    x = np.sqrt(max(0.0, 1 + R[0, 0] - R[1, 1] - R[2, 2])) / 2
    y = np.sqrt(max(0.0, 1 - R[0, 0] + R[1, 1] - R[2, 2])) / 2
    z = np.sqrt(max(0.0, 1 - R[0, 0] - R[1, 1] + R[2, 2])) / 2
    x = np.copysign(x, R[2, 1] - R[1, 2])
    y = np.copysign(y, R[0, 2] - R[2, 0])
    z = np.copysign(z, R[1, 0] - R[0, 1])
    qq = np.array([w, x, y, z])
    return qq / np.linalg.norm(qq)


def body_accelerations(lo, q, v, vd):
    """Spatial accelerations of the bodies relative to the root (gravity removed), root frame, [6 nb, B]."""
    acc, _ = lo.oracle.inverse_dynamics_bodies(np.asarray(q, float), np.asarray(v, float), np.asarray(vd, float))
    g6 = np.concatenate([np.zeros(3), -lo.g])
    return acc - np.tile(g6, lo.nb)[:, None]


# ------------------------------------------------------------------------------------------------------------------------------
# loops_sample on the CPU (tests/hostsim/hostsim_loops.cpp, compiled and loaded by hostsim.shim)
# ------------------------------------------------------------------------------------------------------------------------------
@functools.cache
def _hostsim_loops():
    lib = hostsim.shim("hostsim_loops")
    lib.hostsim_dynamics_loops.argtypes = [ctypes.POINTER(RbdModelDesc), ctypes.c_void_p, ctypes.c_int, ctypes.c_int64] + \
        [ctypes.c_void_p] * 9
    return lib


def hostsim_dynamics_loops(mech, q, v, tau=None, wext=None, stabilization_gains=_DEFAULT, ld=None, want=("qd", "lam", "K", "k")):
    """loops_sample on the CPU; q's dtype selects fp32 / fp64.  Returns (status, dict(vd, qd, lam, K, k)); outputs not in ``want``
    are passed as NULL and come back as None."""
    desc = mech.flatten()
    ld = loop_desc(mech, stabilization_gains) if ld is None else ld
    d, keep = make_desc(desc)
    st, keep2 = ld.c_struct()
    dt = q.dtype
    q = np.ascontiguousarray(q)
    B = q.shape[1]
    v = np.ascontiguousarray(v, dt)
    tau = None if tau is None else np.ascontiguousarray(tau, dt)
    wext = None if wext is None else np.ascontiguousarray(wext, dt)
    nl = ld.nc
    out = dict(vd=np.full((desc.nv, B), np.nan, dt), qd=np.full((desc.nq, B), np.nan, dt), lam=np.full((nl, B), np.nan, dt),
               K=np.full((nl * desc.nv, B), np.nan, dt), k=np.full((nl, B), np.nan, dt))
    for key in ("qd", "lam", "K", "k"):
        if key not in want:
            out[key] = None
    p = lambda a: None if a is None or a.size == 0 else a.ctypes.data
    rc = _hostsim_loops().hostsim_dynamics_loops(ctypes.byref(d), ctypes.byref(st), 0 if dt == np.float32 else 1, B, p(q), p(v), p(tau),
                                                 p(wext), p(out["vd"]), p(out["qd"]), p(out["lam"]), p(out["K"]), p(out["k"]))
    return rc, out
