"""Task-space feedback (DESIGN 4.21): rbd_integrate_task_pd / ``controller=TaskPD(...)`` and rbd_task_pd_torques.

The fp64 numpy law below builds u_task = Σ_t J_t^T f_t from explicit matrices -- TaskOracle's point and geometric Jacobians
(tests/task_oracle.py) -- with the SE(3) part a line-by-line restatement of the reference's double-geodesic PD
(src/pdcontrol.jl:85-107).  The device code (csrc/rbd_task_pd.cuh, compiled for the host by tests/hostsim/hostsim_task_pd.cpp)
must agree with it, and the GPU rollouts with tests/test_pd_rollout.py's host integrator running this law at every stage.
"""
import ctypes
import hashlib
import math
import os
import subprocess
import tempfile
import zlib

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import rigidbodydynamics.jl_b200 as rbd
from oracle import Oracle
from rigidbodydynamics.jl_b200 import _cabi
from rigidbodydynamics.jl_b200._cabi import RbdModelDesc, make_desc
from rigidbodydynamics.jl_b200.kinematics import TaskFrame
from rigidbodydynamics.jl_b200.pd import _RbdPdDesc, _RbdTaskPdDesc
from tests.task_oracle import TaskOracle, rot, rotT, to_frame
from tests.test_pd_rollout import Ctrl, _col, _controller, _model, _pad, _state, _tau_at, integrate_pd, law
from tests.test_task_kinematics import task_set
from tests.util import config_distance, rand_inputs, randmech, ref_urdf, rel_err

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "..", "rigidbodydynamics", "jl_b200", "csrc")
_lib = None
TOL64 = 1e-9
# fp32 rollout against the fp64 host integrator (Atlas, 5 steps at dt = 1e-3, fp32-representable inputs).  Measured on an NVIDIA
# H100 80GB HBM3 at 700 W: q 1.4e-6 / v 1.8e-4 (torque mode), q 3.3e-7 / v 2.4e-6 (computed torque); each bound is about 5x the
# largest error of its mode (DESIGN 4.21)
TOL32 = {"pd": 1e-3, "ct": 1.5e-5}


# ------------------------------------------------------------------------------------------------------------------
# the law in numpy
# ------------------------------------------------------------------------------------------------------------------
def _rows(kind):
    return (3, 3) if kind == "point" else (6, 12)


def se3_pd_double_geodesic(kw, dw, kv, dv, x_R, x_p, xdes_R, xdes_p, T, Tdes):
    """pd(SE3PDGains, x, xdes, T, Tdes) with SE3PDMethod{:DoubleGeodesic} (src/pdcontrol.jl:25-27, 83-107), batched: x_R / xdes_R
    [3, 3, B], x_p / xdes_p [3, B], T / Tdes [6, B] ([angular; linear], in the body frame), gains [3] or [3, B] in the body frame."""
    R = np.einsum("jib,jkb->ikb", xdes_R, x_R)            # group_error(x, xdes) = inv(xdes) * x          (:25)
    p = rotT(xdes_R, x_p - xdes_p)
    edot = -Tdes + T                                       # pd(gains, x, xdes, ẋ, ẋdes) = pd(gains, e, -ẋdes + ẋ)   (:27)
    psi = Rotation.from_matrix(R.transpose(2, 0, 1)).as_rotvec().T     # ψ = RotationVec(R)                      (:99)
    ang = -_col(kw) * psi - _col(dw) * edot[:3]            # pd(angular(gains), ψ, angular(ė))            (:101)
    lin = -_col(kv) * rotT(R, p) - _col(dv) * edot[3:]     # pd(linear(gains), R' * p, linear(ė))         (:102)
    return np.concatenate([ang, lin])


def task_terms(mech, q, v, tasks, kinds, kp, kd, xref, xdref=None):
    """(u_task [nv, B], Σ_t |J_t|^T |f_t| [nv, B] -- the scale of u's rounding)."""
    to = TaskOracle(mech, q, v)
    nv, B = mech.num_velocities(), q.shape[1]
    kp, kd = _col(np.asarray(kp, float)), _col(np.asarray(kd, float))
    u, mag = np.zeros((nv, B)), np.zeros((nv, B))
    r = x = 0
    for t, k in zip(tasks, kinds):
        nr, nx = _rows(k)
        xr = xref[x:x + nx]
        xd = np.zeros((nr, B)) if xdref is None else xdref[r:r + nr]
        if k == "point":
            o = to.task(TaskFrame(t.body, t.base, t.point, t.frame))
            xb = to.task(TaskFrame(t.body, t.base, t.point, t.base))["point"]            # transform(state, point, base)
            RFb = np.einsum("jib,jkb->ikb", to.R[to.idx(t.frame)], to.R[to.idx(t.base)])   # R_F<-base
            e = rot(RFb, xb - xr)
            ed = o["point_velocity"] - rot(RFb, xd)
            f = -kp[r:r + 3] * e - kd[r:r + 3] * ed
            J = o["point_jacobian"].reshape(nv, 3, B).transpose(1, 0, 2)                 # [3, nv, B]
        else:
            o = to.task(TaskFrame(t.body, t.base, t.point, None))
            Rb, pC = to.R[to.idx(t.body)], o["point"]                                   # the frame C, root frame
            J = to_frame(Rb, pC, o["geometric_jacobian"].reshape(nv, 6, B).transpose(1, 0, 2))
            T = to_frame(Rb, pC, o["twist"])
            xp = to.task(TaskFrame(t.body, t.base, t.point, t.base))["point"]
            f = se3_pd_double_geodesic(kp[r:r + 3], kd[r:r + 3], kp[r + 3:r + 6], kd[r + 3:r + 6], o["transform"][:9].reshape(3, 3, B),
                                       xp, xr[:9].reshape(3, 3, B), xr[9:], T, xd)
        u += np.einsum("ckb,cb->kb", J, f)
        mag += np.einsum("ckb,cb->kb", np.abs(J), np.abs(f))
        r, x = r + nr, x + nx
    return u, mag


class TaskCtrl:
    """The host form of a TaskPD, with the interface of test_pd_rollout.Ctrl (torque(orc, n, q, v, tau_ff)) so that
    test_pd_rollout.integrate_pd runs it at every stage.  x_ref / xd_ref [rows, B] or [nsteps, rows, B]; joint: a Ctrl or None."""

    def __init__(self, mech, tasks, kinds, kp, kd, x_ref, xd_ref=None, joint=None, ct=False, bounds=None):
        self.mech, self.tasks, self.kinds = mech, tasks, kinds
        self.kp, self.kd, self.x_ref, self.xd_ref, self.joint, self.ct, self.bounds = kp, kd, x_ref, xd_ref, joint, ct, bounds

    def at(self, a, n):
        return None if a is None else (a[n] if a.ndim == 3 else a)

    def command(self, orc, n, q, v, tau_ff):
        """τ (torque mode) or v̇_des (computed-torque mode) before the inverse dynamics and the clamp."""
        u, _ = task_terms(self.mech, q, v, self.tasks, self.kinds, self.kp, self.kd, self.at(self.x_ref, n), self.at(self.xd_ref, n))
        j = self.joint
        if j is not None:
            base = law(orc.desc, q, v, j.at(j.q_ref, n), j.at(j.v_ref, n), j.at(j.vd_ref, n) if self.ct else tau_ff, j.kp, j.kd)
        else:
            base = 0 if (self.ct or tau_ff is None) else tau_ff
        return base + u

    def torque(self, orc, n, q, v, tau_ff):
        c = self.command(orc, n, q, v, tau_ff)
        tau = orc.inverse_dynamics(q, v, c) + (0 if tau_ff is None else tau_ff) if self.ct else c
        if self.bounds is None:
            return tau
        return np.clip(tau, np.asarray(self.bounds[0])[:, None], np.asarray(self.bounds[1])[:, None])

    def torch(self, dtype):
        import torch
        t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dtype).cuda()    # noqa: E731
        j = self.joint
        joint = None if j is None else rbd.JointPD(t(j.kp), t(j.kd), t(j.q_ref), t(j.v_ref), vd_ref=t(j.vd_ref), computed_torque=self.ct)
        return rbd.TaskPD(self.tasks, self.kinds, t(self.kp), t(self.kd), t(self.x_ref), t(self.xd_ref), joint=joint,
                          computed_torque=self.ct, effort_bounds=self.bounds)


# ------------------------------------------------------------------------------------------------------------------
# tasks and targets
# ------------------------------------------------------------------------------------------------------------------
def task_mix(mech, seed, npoint=7):
    """task_set's point tasks (base = root, base != root, body = base, body = root, F = body / base / a third body, points on and off
    the origin) and pose tasks (base = root, base != root, body = base, body = root)."""
    pts = task_set(mech, seed)[:npoint]
    rng = np.random.default_rng(seed + 100)
    bodies = [j.successor for j in mech.joints]
    b1, b2 = bodies[int(rng.integers(len(bodies)))], bodies[-1]
    pt = lambda: rng.standard_normal(3)                                # noqa: E731
    pose = [TaskFrame(b1, None, pt()), TaskFrame(b2, b1, pt()), TaskFrame(b1, b1, None), TaskFrame(mech.root_body, b2, pt())]
    return pts + pose, ["point"] * len(pts) + ["pose"] * len(pose)


def targets(mech, q, tasks, kinds, rng, mode="random"):
    """x_ref [X, B] around the current task values; mode "near_pi": every pose error's angle within 1e-3 of pi; "zero": the pose
    targets are the current poses."""
    to = TaskOracle(mech, q)
    B = q.shape[1]
    out = []
    for t, k in zip(tasks, kinds):
        cur = to.task(TaskFrame(t.body, t.base, t.point, t.base))["point"]
        if k == "point":
            out.append(cur + 0.3 * rng.standard_normal((3, B)))
            continue
        Rx = to.task(TaskFrame(t.body, t.base))["transform"][:9].reshape(3, 3, B)
        if mode == "zero":
            Rr, pr = Rx, cur
        else:
            if mode == "near_pi":
                ax = rng.standard_normal((3, B))
                ax /= np.linalg.norm(ax, axis=0)
                d = Rotation.from_rotvec((ax * (math.pi - 1e-3 * rng.random(B))).T).as_matrix().transpose(1, 2, 0)
            else:
                d = Rotation.from_rotvec(rng.standard_normal((B, 3)) * 0.8).as_matrix().transpose(1, 2, 0)
            Rr = np.einsum("ijb,jkb->ikb", Rx, d)          # R_e = R_ref^T R_x = d^T
            pr = cur + 0.3 * rng.standard_normal((3, B))
        out.append(np.concatenate([Rr.reshape(9, B), pr]))
    return np.concatenate(out)


# ------------------------------------------------------------------------------------------------------------------
# the device law on the CPU
# ------------------------------------------------------------------------------------------------------------------
def _shim():
    """tests/hostsim/hostsim_task_pd.cpp, compiled on first use into a temporary directory."""
    global _lib
    if _lib is not None:
        return _lib
    srcs = [os.path.join(_HERE, "hostsim", "hostsim_task_pd.cpp")] + sorted(
        os.path.join(_CSRC, f) for f in os.listdir(_CSRC) if f.endswith((".cuh", ".h")) or f == "rbd_model.cpp")
    srcs.append(os.path.join(_HERE, "..", "include", "rbd_b200.h"))
    h = hashlib.sha1(b"".join(open(s, "rb").read() for s in srcs)).hexdigest()[:16]
    d = os.path.join(tempfile.gettempdir(), f"rbd_hostsim_task_pd_{os.getuid()}")
    os.makedirs(d, exist_ok=True)
    so = os.path.join(d, f"hostsim_task_pd_{h}.so")
    if not os.path.exists(so):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so + f".{os.getpid()}",
                               srcs[0], os.path.join(_CSRC, "rbd_model.cpp")])
        os.replace(so + f".{os.getpid()}", so)
    lib = ctypes.CDLL(so)
    vp = ctypes.c_void_p
    lib.hostsim_task_pd_law.argtypes = [ctypes.POINTER(RbdModelDesc), ctypes.POINTER(_RbdTaskPdDesc), ctypes.c_int, ctypes.c_int64,
                                        vp, vp, vp, vp]
    _lib = lib
    return lib


def _task_struct(mech, tasks, kinds, ct, arrays, joint_arrays=None, bounds=None, gain_ld=0):
    """rbd_task_pd_desc over numpy arrays (host pointers); arrays = (kp, kd, x_ref, xd_ref)."""
    from rigidbodydynamics.jl_b200.kinematics import task_desc
    tasks = [TaskFrame(t.body, t.base, t.point, t.body if k == "pose" else t.frame) for t, k in zip(tasks, kinds)]
    td, keep = task_desc(mech, tasks)
    kind = np.array([0 if k == "point" else 1 for k in kinds], np.int32)
    p = lambda a: None if a is None else a.ctypes.data                 # noqa: E731
    dp = ctypes.POINTER(ctypes.c_double)
    joint = None
    if joint_arrays is not None:
        jkp, jkd, jq, jv, jvd = joint_arrays
        joint = _RbdPdDesc(int(ct), p(jkp), p(jkd), gain_ld if jkp.ndim == 2 else 0, p(jq), p(jv), p(jvd), 0, 0, None, None)
    lo, hi = (None, None) if bounds is None else (np.ascontiguousarray(b, np.float64) for b in bounds)
    kp, kd, xr, xd = arrays
    d = _RbdTaskPdDesc(int(ct), td, kind.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), p(kp), p(kd), gain_ld if kp.ndim == 2 else 0,
                       p(xr), 0, p(xd), 0, None if joint is None else ctypes.pointer(joint),
                       None if lo is None else lo.ctypes.data_as(dp), None if hi is None else hi.ctypes.data_as(dp))
    return d, (keep, kind, joint, lo, hi, arrays, joint_arrays)


def hostsim_task_law(mech, tasks, kinds, q, v, kp, kd, xref, xdref=None, ff=None, joint=None, ct=False, bounds=None):
    """The device law on the CPU (dtype of q): torques (torque mode) or v̇_des (computed-torque mode)."""
    dt = q.dtype
    c = lambda a: None if a is None else np.ascontiguousarray(a, dt)      # noqa: E731
    B = q.shape[1]
    arrays = tuple(c(a) for a in (kp, kd, xref, xdref))
    ja = None if joint is None else tuple(c(a) for a in (joint.kp, joint.kd, joint.q_ref, joint.v_ref, joint.vd_ref))
    d, keep = _task_struct(mech, tasks, kinds, ct, arrays, ja, bounds, gain_ld=B)
    q, v, ff = c(q), c(v), c(ff)
    out = np.full((mech.num_velocities(), B), np.nan, dt)
    md, keep2 = make_desc(mech.flatten())
    p = lambda a: None if a is None else a.ctypes.data                    # noqa: E731
    rc = _shim().hostsim_task_pd_law(ctypes.byref(md), ctypes.byref(d), 0 if dt == np.float32 else 1, B, p(q), p(v), p(ff), p(out))
    assert rc == 0, rc
    return out


def _gains(rng, kinds, B, per_sample, scale=1.0):
    R = sum(_rows(k)[0] for k in kinds)
    shape = (R, B) if per_sample else (R,)
    return rng.uniform(5, 40, shape) * scale, rng.uniform(0.5, 4, shape) * scale


def _cpu_models():
    return [("atlas", rbd.load_model("atlas", floating=True)), ("valkyrie", rbd.load_model("valkyrie", floating=True)),
            ("iiwa14", rbd.load_model("iiwa14")), ("double_pendulum", rbd.load_model("double_pendulum")),
            ("randmech0", randmech(0)), ("randmech1", randmech(1)), ("randmech2", randmech(2)), ("randmech3", randmech(3))]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("which", ["atlas", "valkyrie", "iiwa14", "double_pendulum", "randmech0", "randmech1", "randmech2", "randmech3"])
def test_hostsim_law_matches_numpy(which, dtype):
    """task_pd_sample + pd_joint against the numpy law: point and pose tasks (base != root, body = base, F != base, points off the
    origin), shared and per-sample gains, pose errors within 1e-3 of pi and at 0, a joint term in both modes, active clamps."""
    mech = dict(_cpu_models())[which]
    d = mech.flatten()
    B = 12
    seed = zlib.crc32(which.encode())
    rng = np.random.default_rng(seed)
    q, v, tau, _, _ = rand_inputs(mech, B, seed % 1000)
    tasks, kinds = task_mix(mech, seed % 97)
    r = lambda a: None if a is None else a.astype(dtype).astype(np.float64)     # noqa: E731   inputs representable in dtype
    q, v, tau = r(q), r(v), r(tau)
    tol = 1e-11 if dtype == np.float64 else 2e-5
    R = sum(_rows(k)[0] for k in kinds)
    for case, mode in enumerate(("random", "near_pi", "zero")):
        xref = targets(mech, q, tasks, kinds, rng, mode)
        if dtype == np.float32:      # the rotation targets stay orthonormal to fp32 rounding; re-measure the fp64 law on them
            xref = r(xref)
        xdref = r(rng.standard_normal((R, B))) if case != 1 else None
        kp, kd = (r(g) for g in _gains(rng, kinds, B, per_sample=case == 1))
        for ct in (False, True):
            joint = _controller(mech, q, rng, ct=ct, per_sample=case == 0)
            joint.kp, joint.kd, joint.q_ref, joint.v_ref, joint.vd_ref = (r(a) for a in (joint.kp, joint.kd, joint.q_ref, joint.v_ref,
                                                                                         joint.vd_ref))
            for jt in (None, joint):
                u, mag = task_terms(mech, q, v, tasks, kinds, kp, kd, xref, xdref)
                ff = None if ct else tau
                base = 0 if jt is None and (ct or ff is None) else (ff if jt is None else
                                                                    law(d, q, v, jt.q_ref, jt.v_ref, jt.vd_ref if ct else ff, jt.kp, jt.kd))
                ref = base + u
                scale = np.maximum(1.0, (mag + np.abs(ref)).max(0))
                got = hostsim_task_law(mech, tasks, kinds, q.astype(dtype), v.astype(dtype), kp, kd, xref, xdref, ff, jt, ct)
                assert (np.abs(got - ref).max(0) / scale).max() < tol, (mode, ct, jt is None)
                if not ct and jt is not None:      # clamps on the sum: bounds at about half the range
                    lo, hi = -np.abs(ref).mean(1) * 0.5, np.abs(ref).mean(1) * 0.4
                    refc = np.clip(ref, lo[:, None], hi[:, None])
                    assert np.any(refc == hi[:, None]) and np.any(refc == lo[:, None])
                    gotc = hostsim_task_law(mech, tasks, kinds, q.astype(dtype), v.astype(dtype), kp, kd, xref, xdref, ff, jt, ct, (lo, hi))
                    assert (np.abs(gotc - refc).max(0) / scale).max() < tol
    if which == "atlas":
        # the near-pi targets do reach the branch they are meant for
        to = TaskOracle(mech, q)
        t = tasks[-4]
        Rx = to.task(TaskFrame(t.body, t.base))["transform"][:9].reshape(3, 3, B)
        xr = targets(mech, q, tasks, kinds, np.random.default_rng(1), "near_pi")
        x0 = sum(_rows(k)[1] for k in kinds[:-4])
        Re = np.einsum("jib,jkb->ikb", xr[x0:x0 + 9].reshape(3, 3, B), Rx)
        assert np.all(np.linalg.norm(Rotation.from_matrix(Re.transpose(2, 0, 1)).as_rotvec(), axis=1) > math.pi - 2e-3)


def test_x_axis_rotation():
    """test/test_pd_control.jl "x-axis rotation": a pose error that is a rotation by θ about x with angular velocity ω about x gives
    the angular row -k θ - d ω on x and zeros elsewhere (one QuaternionFloating body attached without an offset: its Jacobian in the
    body frame is I, so the torques are the law's output)."""
    rng = np.random.default_rng(56)
    mech = rbd.Mechanism(rbd.RigidBody("world"))
    body = rbd.RigidBody("body", rbd.SpatialInertia.rand(rng))
    mech.attach(mech.root_body, body, rbd.Joint("floating", rbd.QuaternionFloating.rand(rng)))
    B = 9
    th = np.linspace(-3.0, 3.0, B)
    w = rng.standard_normal(B)
    q = np.zeros((7, B))
    q[0], q[1] = np.cos(th / 2), np.sin(th / 2)
    v = np.zeros((6, B))
    v[0] = w
    xref = np.concatenate([np.eye(3).reshape(9, 1).repeat(B, 1), np.zeros((3, B))])
    k, dgain = 10.0, 2.0
    kp, kd = np.array([k] * 3 + [0.0] * 3), np.array([dgain] * 3 + [0.0] * 3)
    got = hostsim_task_law(mech, [TaskFrame(body)], ["pose"], q, v, kp, kd, xref)
    assert np.abs(got[0] - (-k * th - dgain * w)).max() < 1e-12
    assert np.abs(got[1:]).max() < 1e-12


def test_host_integrator_with_zero_task_gains_is_the_joint_space_one():
    """integrate_pd with the task law at every stage and all task gains 0 equals integrate_pd with the joint term alone."""
    mech = rbd.load_model("iiwa14")
    orc = Oracle(mech.flatten())
    B, n = 4, 3
    rng = np.random.default_rng(6)
    q, v, tau, _, _ = rand_inputs(mech, B, 8)
    tasks, kinds = task_mix(mech, 5, npoint=3)
    R = sum(_rows(k)[0] for k in kinds)
    xref = targets(mech, q, tasks, kinds, rng)
    for ct in (False, True):
        joint = _controller(mech, q, rng, ct=ct)
        tc = TaskCtrl(mech, tasks, kinds, np.zeros(R), np.zeros(R), xref, joint=joint, ct=ct)
        qa, va, _ = integrate_pd(orc, q, v, tc, tau, dt=1e-3, nsteps=n)
        qb, vb, _ = integrate_pd(orc, q, v, joint, tau, dt=1e-3, nsteps=n)
        assert config_distance(mech, qa, qb) < 1e-12 and rel_err(va, vb) < 1e-12


# ------------------------------------------------------------------------------------------------------------------
# argument checks (host only, nothing launched)
# ------------------------------------------------------------------------------------------------------------------
def test_argument_checks(built):
    from tests.loops_oracle import four_bar
    lib = rbd.load_library()
    mech = rbd.load_model("iiwa14")
    h = _cabi.ModelHandle(mech.flatten())
    fake = 64                                          # never dereferenced by the checks below
    F64 = _cabi.RBD_F64
    body = [j.successor for j in mech.joints]
    tasks, kinds = [TaskFrame(body[6], None, [0.0, 0.0, 0.1]), TaskFrame(body[3], body[1])], ["point", "pose"]
    dp = ctypes.POINTER(ctypes.c_double)
    lo_ok, hi_ok = (np.ascontiguousarray(b) for b in rbd.effort_bounds(mech))

    def desc(*, mode=0, kind=None, frame=None, joint=None, **kw):
        from rigidbodydynamics.jl_b200.kinematics import task_desc
        td, keep = task_desc(mech, [TaskFrame(t.body, t.base, t.point, t.body if k == "pose" else t.frame)
                                    for t, k in zip(tasks, kinds)])
        if frame is not None:
            keep = keep + (np.array(frame, np.int32),)
            td.frame = keep[-1].ctypes.data_as(ctypes.POINTER(ctypes.c_int32))
        kd_ = np.array(kind if kind is not None else [0, 1], np.int32)
        f = dict(kp=fake, kd=fake, gain_ld=0, x_ref=fake, x_ref_step_stride=0, xd_ref=None, xd_ref_step_stride=0,
                 effort_lo=lo_ok.ctypes.data_as(dp), effort_hi=hi_ok.ctypes.data_as(dp))
        f.update(kw)
        d = _RbdTaskPdDesc(mode=mode, tasks=td, kind=kd_.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
                           joint=None if joint is None else ctypes.pointer(joint), **f)
        d._keep = (keep, kd_, joint)
        return d

    def jd(**kw):
        f = dict(mode=0, kp=fake, kd=fake, gain_ld=0, q_ref=fake, v_ref=None, vd_ref=None, q_ref_step_stride=0, v_ref_step_stride=0,
                 effort_lo=None, effort_hi=None)
        f.update(kw)
        return _RbdPdDesc(**f)

    def roll(c, B=4, ld=4, handle=h, loops=None, dtype=F64):
        return lib.rbd_integrate_task_pd(handle.ptr, dtype, B, ld, fake, fake, None, None, 0, 0,
                                         None if c is None else ctypes.byref(c), loops, None, 1e-3, 1, None, None, None, None)

    def once(c, B=4, ld=4, step=0, dtype=F64):
        return lib.rbd_task_pd_torques(h.ptr, dtype, B, ld, fake, fake, None, None if c is None else ctypes.byref(c), step, fake, None)

    def status(rc, code=_cabi.RBD_EINVAL, text=None):
        assert rc == code, rc
        if text:
            assert text.encode() in lib.rbd_last_error(), lib.rbd_last_error()

    for call in (roll, once):
        status(call(None), text="ctrl must not be NULL")
        status(call(desc(mode=2)), text="unknown mode")
        status(call(desc(kind=[0, 7])), text="unknown task kind")
        status(call(desc(frame=[-1, -1])), text="frame[t] == body[t]")
        status(call(desc(kp=None)), text="must not be NULL")
        status(call(desc(x_ref=None)), text="must not be NULL")
        status(call(desc(gain_ld=3)), text="gain_ld")
        status(call(desc(x_ref_step_stride=-1)), text="strides")
        status(call(desc(xd_ref_step_stride=-1)), text="strides")
        status(call(desc(effort_hi=None)), text="both")
        bad = lo_ok.copy()
        bad[2] = 1e9
        status(call(desc(effort_lo=bad.ctypes.data_as(dp))), text="lo <= hi")
        status(call(desc(joint=jd(mode=1))), text="the controller's mode")
        status(call(desc(joint=jd(effort_lo=lo_ok.ctypes.data_as(dp), effort_hi=hi_ok.ctypes.data_as(dp)))), text="effort bounds must be NULL")
        status(call(desc(joint=jd(q_ref=None))), text="kp, kd and q_ref must not be NULL")
        status(call(desc(joint=jd(vd_ref=fake))), text="computed-torque mode only")
        assert call(desc(), B=8, ld=4) == _cabi.RBD_EDIM
        assert call(desc(), dtype=_cabi.RBD_DUAL64X6) == _cabi.RBD_EUNSUPPORTED
        assert call(desc(), B=0, ld=0) == _cabi.RBD_OK
    # rbd_task_desc's own checks, with their codes
    tasks.append(TaskFrame(body[0]))
    kinds.append("point")
    status(roll(desc(kind=[0, 1, 0], frame=[-1, 3, 64])), text="index")
    tasks[:] = [TaskFrame(body[6])]
    kinds[:] = ["point"]
    many = desc(kind=[0])
    many.tasks.ntasks = 33                             # more than RBD_MAX_TASKS: refused before any entry is read
    status(roll(many), _cabi.RBD_EUNSUPPORTED)
    status(once(desc(kind=[0]), step=-1), text="step")
    # computed-torque mode with loops
    fb = four_bar()
    hf = rbd.MechanismState(fb, 1, device="cpu").handle
    lst, keep = rbd.loop_desc(fb).c_struct()
    b1 = fb.joints[0].successor
    mech_saved, mech = mech, fb
    tasks[:] = [TaskFrame(b1)]
    ct = desc(mode=1, kind=[0], effort_lo=None, effort_hi=None)
    assert roll(ct, handle=hf, loops=ctypes.byref(lst)) == _cabi.RBD_ELOOP
    assert roll(desc(kind=[0], effort_lo=None, effort_hi=None), handle=hf, loops=ctypes.byref(lst), B=0, ld=0) == _cabi.RBD_OK
    h.close()


def test_python_argument_checks():
    """TaskPD's own checks, its shape / dtype checks before any call into the library, and autodiff's refusal."""
    import torch
    mech = rbd.load_model("iiwa14")
    body = mech.joints[-1].successor
    st = rbd.MechanismState(mech, 3, device="cpu")
    z = lambda *s, dtype=torch.float64: torch.zeros(*s, dtype=dtype)          # noqa: E731
    with pytest.raises(ValueError):
        rbd.TaskPD([TaskFrame(body)], ["line"], z(3), z(3), z(3, 3))
    with pytest.raises(ValueError):
        rbd.TaskPD([TaskFrame(body, None, None, mech.joints[0].successor)], ["pose"], z(6), z(6), z(12, 3))
    with pytest.raises(ValueError):
        rbd.TaskPD([TaskFrame(body)], ["point"], z(3), z(3), z(3, 3), joint=rbd.JointPD(z(7), z(7), z(7, 3), computed_torque=True))
    with pytest.raises(ValueError):
        rbd.TaskPD([TaskFrame(body)], ["point"], z(3), z(3), z(3, 3), joint=rbd.JointPD(z(7), z(7), z(7, 3), effort_bounds=(z(7), z(7))))
    ok = dict(kp=z(3), kd=z(3), x_ref=z(3, 3))
    cases = [(dict(ok, kp=z(4)), rbd.DimensionMismatch), (dict(ok, kd=z(3, 3)), rbd.DimensionMismatch),
             (dict(ok, x_ref=z(12, 3)), rbd.DimensionMismatch), (dict(ok, x_ref=z(3, 3, dtype=torch.float32)), TypeError),
             (dict(ok, xd_ref=z(6, 3)), rbd.DimensionMismatch)]
    for kw, err in cases:
        c = rbd.TaskPD([TaskFrame(body)], ["point"], kw["kp"], kw["kd"], kw["x_ref"], kw.get("xd_ref"))
        with pytest.raises(err):
            rbd.simulate_(st, 2e-3, dt=1e-3, controller=c)
        with pytest.raises(err):
            rbd.task_pd_torques(st, c)
    c = rbd.TaskPD([TaskFrame(body)], ["point"], z(3), z(3), z(3, 3))
    with pytest.raises(TypeError):
        rbd.autodiff.simulate(mech, st.q, st.v, None, 1e-3, 2, controller=c)


# ------------------------------------------------------------------------------------------------------------------
# GPU tier
# ------------------------------------------------------------------------------------------------------------------
def _cabi_rollout(mech, q, v, tc, tau, dtype, dt, nsteps, ld, *, cd=None, s=None, loops=False, record=False):
    """rbd_integrate_task_pd through the C ABI, every array with leading dimension ld (> B: NaN padding that must stay untouched)."""
    import torch
    B = q.shape[1]
    st = rbd.MechanismState(mech, batch=1, dtype=dtype)
    qd, vd = _pad(q, ld, dtype), _pad(v, ld, dtype)
    sd = None if s is None else _pad(s, ld, dtype)
    td = None if tau is None else _pad(tau, ld, dtype)
    nv, nq = mech.num_velocities(), mech.num_positions()
    step, stage = (0, 0) if tau is None or tau.ndim == 2 else ((nv * ld, 0) if tau.ndim == 3 else (4 * nv * ld, nv * ld))
    R = sum(_rows(k)[0] for k in tc.kinds)
    X = sum(_rows(k)[1] for k in tc.kinds)
    dev = lambda a, per: None if a is None else (_pad(a, ld, dtype) if per else torch.from_numpy(a).to(dtype).cuda())  # noqa: E731
    kp, kd = dev(tc.kp, tc.kp.ndim == 2), dev(tc.kd, tc.kd.ndim == 2)
    xr, xd = dev(tc.x_ref, True), dev(tc.xd_ref, True)
    rs = lambda a, rows: 0 if a is None or a.ndim == 2 else rows * ld        # noqa: E731
    p = lambda t: None if t is None else t.data_ptr()                        # noqa: E731
    j = tc.joint
    jt = None
    if j is not None:
        jkp, jkd = dev(j.kp, j.kp.ndim == 2), dev(j.kd, j.kd.ndim == 2)
        jr = [dev(a, True) for a in (j.q_ref, j.v_ref, j.vd_ref)]
        jt = (jkp, jkd, jr)
        jdesc = _RbdPdDesc(int(tc.ct), p(jkp), p(jkd), ld if j.kp.ndim == 2 else 0, p(jr[0]), p(jr[1]), p(jr[2]), rs(j.q_ref, nq),
                           rs(j.v_ref if j.v_ref is not None else j.vd_ref, nv), None, None)
    from rigidbodydynamics.jl_b200.kinematics import task_desc
    tdsc, keep = task_desc(mech, [TaskFrame(t.body, t.base, t.point, t.body if k == "pose" else t.frame)
                                  for t, k in zip(tc.tasks, tc.kinds)])
    kind = np.array([0 if k == "point" else 1 for k in tc.kinds], np.int32)
    dp = ctypes.POINTER(ctypes.c_double)
    lo, hi = (None, None) if tc.bounds is None else (np.ascontiguousarray(b, np.float64) for b in tc.bounds)
    d = _RbdTaskPdDesc(int(tc.ct), tdsc, kind.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), p(kp), p(kd),
                       ld if tc.kp.ndim == 2 else 0, p(xr), rs(tc.x_ref, X), p(xd), rs(tc.xd_ref, R),
                       None if j is None else ctypes.pointer(jdesc), None if lo is None else lo.ctypes.data_as(dp),
                       None if hi is None else hi.ctypes.data_as(dp))
    lst, keep_l = rbd.loop_desc(mech).c_struct() if loops else (None, None)
    cst, keep_c = cd.c_struct() if cd is not None else (None, None)
    traj = (None, None, None)
    if record:
        traj = tuple(torch.empty((nsteps + 1, rows, B), dtype=dtype, device="cuda") for rows in (nq, nv, 0 if cd is None else cd.nstates))
        if cd is None or cd.nstates == 0:
            traj = traj[:2] + (None,)
    _cabi.check(rbd.load_library().rbd_integrate_task_pd(
        st.handle.ptr, _cabi.RBD_F32 if dtype == torch.float32 else _cabi.RBD_F64, B, ld, p(qd), p(vd), p(sd), p(td), step, stage,
        ctypes.byref(d), None if lst is None else ctypes.byref(lst), None if cst is None else ctypes.byref(cst), dt, nsteps,
        *[p(t) for t in traj], torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    for t in (qd, vd) + (() if sd is None else (sd,)):
        assert bool(torch.isnan(t[:, B:]).all())
    out = tuple(t[:, :B].double().cpu().numpy() for t in (qd, vd))
    out = out + (None if sd is None else sd[:, :B].double().cpu().numpy(),)
    if record:
        assert torch.equal(traj[0][-1].cpu(), qd[:, :B].cpu()) and torch.equal(traj[1][-1].cpu(), vd[:, :B].cpu())
    return out


def _task_ctrl(mech, q, rng, *, ct=False, per_step=0, per_sample=False, clamp=False, joint=True, xd=True, npoint=2, scale=1.0):
    tasks, kinds = task_mix(mech, int(rng.integers(1000)), npoint=npoint)
    tasks, kinds = tasks[:npoint] + tasks[-2:], kinds[:npoint] + kinds[-2:]
    B = q.shape[1]
    R = sum(_rows(k)[0] for k in kinds)
    kp, kd = _gains(rng, kinds, B, per_sample, 0.2 * scale)
    xref = targets(mech, q, tasks, kinds, rng) if not per_step else np.stack([targets(mech, q, tasks, kinds, rng) for _ in range(per_step)])
    xdref = None
    if xd:
        xdref = rng.standard_normal((R, B) if not per_step else (per_step, R, B)) * 0.2
    jc = _controller(mech, q, rng, ct=ct, per_step=per_step, per_sample=per_sample, scale=0.3 * scale) if joint else None
    bounds = None
    if clamp:
        lim = rng.uniform(5, 30, mech.num_velocities())
        bounds = (-lim, lim * 0.8)
    return TaskCtrl(mech, tasks, kinds, kp, kd, xref, xdref, jc, ct, bounds)


@pytest.mark.gpu
@pytest.mark.parametrize("which,mode,per_step,per_sample,clamp,joint,tau_kind,nsteps", [
    ("atlas", "pd", 0, False, True, True, "none", 4), ("atlas", "ct", 4, True, True, True, "step", 4),
    ("atlas", "pd", 4, True, True, False, "stage", 4), ("valkyrie", "ct", 0, False, False, False, "const", 3),
    ("iiwa14", "pd", 6, True, True, True, "const", 6), ("iiwa14", "ct", 0, False, True, False, "none", 6),
    ("double_pendulum", "pd", 0, False, False, False, "stage", 10), ("double_pendulum", "ct", 10, True, False, True, "const", 10),
    ("randmech0", "pd", 3, True, True, True, "step", 3), ("randmech3", "ct", 0, False, False, True, "stage", 3)])
def test_gpu_rollout_matches_host_integrator_fp64(built, which, mode, per_step, per_sample, clamp, joint, tau_kind, nsteps):
    import torch
    mech = _model(which)
    rng = np.random.default_rng(zlib.crc32(f"{which}{mode}{nsteps}".encode()))
    B = 19
    q, v, tau, _, _ = rand_inputs(mech, B, 21)
    v *= 0.3
    tc = _task_ctrl(mech, q, rng, ct=mode == "ct", per_step=per_step, per_sample=per_sample, clamp=clamp, joint=joint)
    taus = {"none": None, "const": tau, "step": tau[None] * rng.uniform(0.5, 1.5, (nsteps, 1, 1)),
            "stage": tau[None, None] * rng.uniform(0.5, 1.5, (nsteps, 4, 1, 1))}[tau_kind]
    orc = Oracle(mech.flatten())
    qr, vr, _ = integrate_pd(orc, q, v, tc, taus, dt=1e-3, nsteps=nsteps)
    if clamp:                                   # the clamp on the sum is active on some samples at the first stage, not on all
        t0 = tc.torque(orc, 0, q, v, _tau_at(taus, 0, 0))
        sat = (t0 == tc.bounds[0][:, None]) | (t0 == tc.bounds[1][:, None])
        assert sat.any() and not sat.all()
    qg, vg, _ = _cabi_rollout(mech, q, v, tc, taus, torch.float64, 1e-3, nsteps, ld=B + 5, record=per_step > 0)
    assert config_distance(mech, qg, qr) < TOL64
    assert rel_err(vg, vr) < TOL64


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["pd", "ct"])
def test_gpu_rollout_fp32(built, mode):
    import torch
    mech = _model("atlas")
    rng = np.random.default_rng(5)
    B = 33
    q, v, tau, _, _ = rand_inputs(mech, B, 23)
    v *= 0.3
    r = lambda a: None if a is None else a.astype(np.float32).astype(np.float64)    # noqa: E731
    q, v, tau = r(q), r(v), r(tau)
    tc = _task_ctrl(mech, q, rng, ct=mode == "ct", per_sample=True, clamp=True)
    tc.kp, tc.kd, tc.x_ref, tc.xd_ref = (r(a) for a in (tc.kp, tc.kd, tc.x_ref, tc.xd_ref))
    j = tc.joint
    j.kp, j.kd, j.q_ref, j.v_ref, j.vd_ref = (r(a) for a in (j.kp, j.kd, j.q_ref, j.v_ref, j.vd_ref))
    qr, vr, _ = integrate_pd(Oracle(mech.flatten()), q, v, tc, tau, dt=1e-3, nsteps=5)
    qg, vg, _ = _cabi_rollout(mech, q, v, tc, tau, torch.float32, 1e-3, 5, ld=B)
    eq, ev = config_distance(mech, qg, qr), rel_err(vg, vr)
    print(f"task_pd fp32 {mode}: q {eq:.3e} v {ev:.3e}")
    assert eq < TOL32[mode] and ev < TOL32[mode]


@pytest.mark.gpu
def test_gpu_torques_match_host_law_and_composition(built):
    """rbd_task_pd_torques against the numpy law (fp64, both modes, a joint term, bounds), and -- torque mode without a joint term
    -- against the composition rbd_task_kinematics -> the law in torch -> rbd_task_kinematics_vjp's v_bar (= J^T f)."""
    import torch
    for which in ("atlas", "iiwa14", "randmech2"):
        mech = _model(which)
        rng = np.random.default_rng(zlib.crc32(which.encode()))
        B = 29
        q, v, tau, _, _ = rand_inputs(mech, B, 3)
        st = _state(mech, q, v, torch.float64)
        orc = Oracle(mech.flatten())
        for ct in (False, True):
            tc = _task_ctrl(mech, q, rng, ct=ct, per_sample=True, clamp=not ct, npoint=4)
            got = rbd.task_pd_torques(st, tc.torch(torch.float64), torch.from_numpy(tau).cuda()).cpu().numpy()
            ref = tc.torque(orc, 0, q, v, tau)
            assert rel_err(got, ref) < 1e-10, (which, ct)
        tc = _task_ctrl(mech, q, rng, joint=False, npoint=4)
        c = tc.torch(torch.float64)
        got = rbd.task_pd_torques(st, c).cpu().numpy()
        comp = composed_task_torques(st, c).cpu().numpy()
        assert rel_err(got, comp) < 1e-10, which


def _rotvec_torch(R):
    """rotation vectors of rotation matrices [3, 3, B] (quaternion with the largest pivot, then 2 atan2(|xyz|, w))."""
    import torch
    tr = R[0, 0] + R[1, 1] + R[2, 2]
    w = 0.5 * torch.sqrt(torch.clamp(1 + tr, min=0))
    x = 0.5 * torch.sqrt(torch.clamp(1 + R[0, 0] - R[1, 1] - R[2, 2], min=0))
    y = 0.5 * torch.sqrt(torch.clamp(1 - R[0, 0] + R[1, 1] - R[2, 2], min=0))
    z = 0.5 * torch.sqrt(torch.clamp(1 - R[0, 0] - R[1, 1] + R[2, 2], min=0))
    piv = torch.stack([w, x, y, z]).argmax(0)
    qw = torch.stack([w, (R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w)])
    qx = torch.stack([(R[2, 1] - R[1, 2]) / (4 * x), x, (R[0, 1] + R[1, 0]) / (4 * x), (R[0, 2] + R[2, 0]) / (4 * x)])
    qy = torch.stack([(R[0, 2] - R[2, 0]) / (4 * y), (R[0, 1] + R[1, 0]) / (4 * y), y, (R[1, 2] + R[2, 1]) / (4 * y)])
    qz = torch.stack([(R[1, 0] - R[0, 1]) / (4 * z), (R[0, 2] + R[2, 0]) / (4 * z), (R[1, 2] + R[2, 1]) / (4 * z), z])
    qq = torch.where(piv == 0, qw, torch.where(piv == 1, qx, torch.where(piv == 2, qy, qz)))
    qq = qq * torch.where(qq[0] < 0, -1.0, 1.0).to(qq.dtype)
    s = torch.linalg.vector_norm(qq[1:], dim=0)
    th = 2 * torch.atan2(s, qq[0])
    k = torch.where(s > 1e-12, th / torch.clamp(s, min=1e-300), 2.0 + s * s / 3)
    return qq[1:] * k


def composed_task_torques(state, c):
    """u_task of a TaskPD (torque mode, no joint term, no bounds, τ_ff = 0) from the pieces a user has without it: one
    rbd_task_kinematics call (transform, point, twist, point_velocity of helper tasks), the law in torch, one
    rbd_task_kinematics_vjp call whose v_bar is Σ J^T f."""
    import torch
    from rigidbodydynamics.jl_b200.autodiff import task_kinematics_vjp_
    B, dt, dev = state.batch, state.dtype, state.q.device
    aux = []
    for t, k in zip(c.tasks, c.kinds):
        if k == "point":      # x in base coordinates; the point velocity in F (its cotangent is f); R_base<-F
            aux += [TaskFrame(t.body, t.base, t.point, t.base), TaskFrame(t.body, t.base, t.point, t.frame), TaskFrame(t.frame, t.base)]
        else:                 # the point C in base coordinates; the body's transform and twist in its own frame
            aux += [TaskFrame(t.body, t.base, t.point, t.base), TaskFrame(t.body, t.base, None, t.body)]
    K = len(aux)
    outs = {n: torch.empty((r * K, B), dtype=dt, device=dev) for n, r in (("transform", 12), ("point", 3), ("twist", 6), ("point_velocity", 3))}
    rbd.task_kinematics_(state, aux, **outs)
    tr = outs["transform"].view(K, 12, B)
    pt, tw, pv = outs["point"].view(K, 3, B), outs["twist"].view(K, 6, B), outs["point_velocity"].view(K, 3, B)
    bars = {"twist": torch.zeros_like(outs["twist"]), "point_velocity": torch.zeros_like(outs["point_velocity"])}
    btw, bpv = bars["twist"].view(K, 6, B), bars["point_velocity"].view(K, 3, B)
    kp = c.kp if c.kp.dim() == 2 else c.kp[:, None]
    kd = c.kd if c.kd.dim() == 2 else c.kd[:, None]
    xdr = torch.zeros((c.rows()[0], B), dtype=dt, device=dev) if c.xd_ref is None else c.xd_ref
    a = r = x = 0
    for t, k in zip(c.tasks, c.kinds):
        if k == "point":
            RbF = tr[a + 2, :9].view(3, 3, B)                 # R_base<-F; R_F<-base is its transpose
            e = torch.einsum("jib,jb->ib", RbF, pt[a] - c.x_ref[x:x + 3])
            ed = pv[a + 1] - torch.einsum("jib,jb->ib", RbF, xdr[r:r + 3])
            bpv[a + 1] = -kp[r:r + 3] * e - kd[r:r + 3] * ed
            a, r, x = a + 3, r + 3, x + 3
        else:
            Rx = tr[a + 1, :9].view(3, 3, B)
            px = pt[a]
            Rr, pr = c.x_ref[x:x + 9].view(3, 3, B), c.x_ref[x + 9:x + 12]
            Re = torch.einsum("jib,jkb->ikb", Rr, Rx)
            pe = torch.einsum("jib,jb->ib", Rr, px - pr)
            psi = _rotvec_torch(Re)
            pl = torch.as_tensor(np.zeros(3) if t.point is None else np.asarray(t.point, np.float64), dtype=dt, device=dev)[:, None]
            w = tw[a + 1, :3]
            vC = tw[a + 1, 3:] + torch.cross(w, pl.expand(3, B), dim=0)     # the twist of C in C
            ang = -kp[r:r + 3] * psi - kd[r:r + 3] * (w - xdr[r:r + 3])
            lin = -kp[r + 3:r + 6] * torch.einsum("jib,jb->ib", Re, pe) - kd[r + 3:r + 6] * (vC - xdr[r + 3:r + 6])
            btw[a + 1, :3] = ang + torch.cross(pl.expand(3, B), lin, dim=0)   # f . T_C as a cotangent on the body twist
            btw[a + 1, 3:] = lin
            a, r, x = a + 2, r + 6, x + 12
    v_bar = torch.empty_like(state.v)
    task_kinematics_vjp_(state, aux, bars=bars, v_bar=v_bar)
    return v_bar


@pytest.mark.gpu
def test_gpu_zero_task_gains_bit_identical(built):
    """Task gains 0: bit-identical to rbd_integrate_pd with the joint term alone, and without a joint term to the open-loop
    rollout with the same τ_ff schedule (fp32 at B = 4096: the vectorised stage kernels; fp64 at B = 37)."""
    import torch
    for dtype, B in ((torch.float32, 4096), (torch.float64, 37)):
        mech = rbd.load_model("atlas", floating=True)
        rng = np.random.default_rng(1)
        q, v, tau, _, _ = rand_inputs(mech, B, 2)
        n = 3
        taus = torch.from_numpy(tau[None, None] * rng.uniform(0.5, 1.5, (n, 4, 1, 1))).to(dtype).cuda()
        tc = _task_ctrl(mech, q, rng, per_sample=True)
        R = tc.kp.shape[0]
        for ct in (False, True):
            j = _controller(mech, q, rng, ct=ct)
            jt = j.torch(dtype)
            zero = torch.zeros(R, dtype=dtype, device="cuda")
            x_ref = torch.from_numpy(tc.x_ref).to(dtype).cuda()
            for joint in (jt, None):
                if joint is None and ct:
                    continue
                c = rbd.TaskPD(tc.tasks, tc.kinds, zero, zero, x_ref, joint=joint, computed_torque=ct)
                a, b = _state(mech, q, v, dtype), _state(mech, q, v, dtype)
                rbd.simulate_(a, n * 1e-3 - 1e-9, taus, dt=1e-3, controller=joint)
                rbd.simulate_(b, n * 1e-3 - 1e-9, taus, dt=1e-3, controller=c)
                assert torch.equal(a.q, b.q) and torch.equal(a.v, b.v), (dtype, ct, joint is None)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["orientation", "pose"])
def test_gpu_reference_pd_control_in_task_space(built, which):
    """test/test_pd_control.jl "orientation control" / "pose control" as written, in task space: rand_floating_tree_mechanism, a pose
    task on the body w.r.t. the world, gains 100 / 20 (0 on the translation for "orientation"), computed torque, Δt = 1e-3, 3 s, 64
    random targets.  R R_des^T = I and ω = 0 to 1e-8; for "pose" the transform and twist to 1e-6."""
    import torch
    rng = np.random.default_rng(61 if which == "orientation" else 62)
    mech = rbd.rand_floating_tree_mechanism(rng, [])
    body = mech.joints[0].successor
    B = 64
    st = rbd.MechanismState(mech, B, torch.float64)
    rbd.rand_(st, rng)
    Rd = Rotation.random(B, random_state=7).as_matrix().transpose(1, 2, 0)
    pd_ = rng.standard_normal((3, B))
    xref = np.concatenate([Rd.reshape(9, B), pd_])
    kp = np.array([100.0] * 6)
    kd = np.array([20.0] * 6)
    if which == "orientation":
        kp[3:] = kd[3:] = 0.0
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()          # noqa: E731
    c = rbd.TaskPD([TaskFrame(body)], ["pose"], t(kp), t(kd), t(xref), computed_torque=True)
    n = rbd.simulate_(st, 3.0, dt=1e-3, controller=c)
    assert n >= 3000
    tr = rbd.relative_transform(st, body).cpu().numpy()
    tw = rbd.relative_twist(st, body, None, body).cpu().numpy()
    R = tr[:9].reshape(3, 3, B)
    assert np.abs(np.einsum("ijb,kjb->ikb", R, Rd) - np.eye(3)[:, :, None]).max() < 1e-8 and np.abs(tw[:3]).max() < 1e-8
    if which == "pose":
        assert np.abs(tr[9:] - pd_).max() < 1e-6 and np.abs(tw).max() < 1e-6


@pytest.mark.gpu
def test_gpu_example4_circle(built, tmp_path):
    """examples/4 on Acrobot.urdf: the point (0, 0, -2) of lower_link follows a circle under v̇ = Kp J^T Δp - Kd v,
    τ = inverse_dynamics(v̇): a point task with Kp = 200, a joint term with kp = 0, kd = 20, computed torque, per-step circle
    targets, Δt = 1e-3, 10 s.  The first 100 steps match the host integrator; after a 3 s transient the tracking error stays small."""
    import torch
    mech = rbd.parse_urdf(ref_urdf("Acrobot", tmp_path))
    lower = mech.findbody("lower_link")
    B, dt, nsteps = 8, 1e-3, 10000
    rng = np.random.default_rng(4)
    q0 = rng.uniform(-0.3, 0.3, (2, B))
    v0 = np.zeros((2, B))
    task = TaskFrame(lower, None, [0.0, 0.0, -2.0])
    p0 = TaskOracle(mech, q0).task(task)["point"]
    tt = np.arange(nsteps) * dt
    center = np.array([0.5, 0.0, -2.0])
    rad = 0.5
    xref = np.empty((nsteps, 3, B))
    xref[:, 0] = center[0] + rad * np.cos(tt)[:, None]
    xref[:, 1] = p0[1][None]                     # the plane the Acrobot moves in
    xref[:, 2] = center[2] + rad * np.sin(tt)[:, None]
    joint = Ctrl(np.zeros(2), np.full(2, 20.0), q0, ct=True)
    tc = TaskCtrl(mech, [task], ["point"], np.full(3, 200.0), np.zeros(3), xref, joint=joint, ct=True)
    qr, vr, _ = integrate_pd(Oracle(mech.flatten()), q0, v0, tc, None, dt=dt, nsteps=100)
    tc100 = TaskCtrl(mech, [task], ["point"], tc.kp, tc.kd, xref[:100], joint=joint, ct=True)
    qg, vg, _ = _cabi_rollout(mech, q0, v0, tc100, None, torch.float64, dt, 100, ld=B + 1)
    assert config_distance(mech, qg, qr) < TOL64 and rel_err(vg, vr) < TOL64
    st = _state(mech, q0, v0, torch.float64)
    qt, vt = rbd.simulate_trajectory_(st, nsteps, dt=dt, controller=tc.torch(torch.float64))
    after = range(3000, nsteps, 250)
    err = max(np.abs(TaskOracle(mech, qt[k].cpu().numpy()).task(task)["point"] - xref[k - 1]).max() for k in after)
    print(f"example 4 circle: max tracking error after 3 s {err:.3e} m")
    assert err < 0.1


@pytest.mark.gpu
def test_gpu_contact_and_loops(built):
    """Atlas standing on the floor with a pelvis pose task holding its height (contact rollout), and the four-bar with a point task
    (loop rollout), both PD mode, against the host integrator."""
    import torch
    from tests.loops_oracle import LoopOracle
    from tests.test_loops_rollout import _case, atlas_on_floor, atlas_states, stage_dynamics
    mech, cd = atlas_on_floor()
    B = 24
    q, v, tau = atlas_states(mech, B, 44)
    s0 = np.random.default_rng(3).standard_normal((cd.nstates, B)) * 1e-3
    pelvis = mech.joints[0].successor
    task = TaskFrame(pelvis)
    to = TaskOracle(mech, q)
    x0 = np.concatenate([to.task(task)["transform"][:9], to.task(task)["point"]])
    x0[11] += 0.02                                  # hold the pelvis a little higher
    kp, kd = np.array([200.0] * 3 + [500.0] * 3), np.array([20.0] * 3 + [50.0] * 3)
    tc = TaskCtrl(mech, [task], ["pose"], kp, kd, x0, bounds=(np.full(mech.num_velocities(), -300.0), np.full(mech.num_velocities(), 300.0)))
    orc = Oracle(mech.flatten())
    qr, vr, sr = integrate_pd(orc, q, v, tc, tau, dt=1e-3, nsteps=5, contact=cd, s=s0)
    assert np.any(sr != s0)
    qg, vg, sg = _cabi_rollout(mech, q, v, tc, tau, torch.float64, 1e-3, 5, ld=B + 3, cd=cd, s=s0, record=True)
    assert config_distance(mech, qg, qr) < TOL64 and rel_err(vg, vr) < 1e-8
    assert float(np.abs(sg - sr).max() / max(1.0, np.abs(sr).max())) < 1e-8
    mech, cd, q, v, tau, s = _case("four_bar", 21, 32)
    lo = LoopOracle(mech)
    link = mech.findbody("link2")
    task = TaskFrame(link, None, [0.3, 0.0, 0.0])
    x0 = TaskOracle(mech, q).task(task)["point"] + 0.05
    tc = TaskCtrl(mech, [task], ["point"], np.full(3, 30.0), np.full(3, 3.0), x0)
    sd = lambda qs, vs, ss, t: (stage_dynamics(lo, qs, vs, ss, cd, t)[0], np.zeros_like(ss))    # noqa: E731
    qr, vr, _ = integrate_pd(lo.oracle, q, v, tc, tau, dt=1e-3, nsteps=5, stage_dynamics=sd)
    qg, vg, _ = _cabi_rollout(mech, q, v, tc, tau, torch.float64, 1e-3, 5, ld=23, loops=True)
    assert config_distance(mech, qg, qr) < TOL64 and rel_err(vg, vr) < TOL64


@pytest.mark.gpu
def test_gpu_launch_count(built):
    """One kernel more per stage than rbd_integrate_pd with the same joint term, in both modes; rbd_task_pd_torques is one kernel in
    torque mode."""
    import torch
    mech = rbd.load_model("atlas", floating=True)
    B = 4096
    q, v, tau, _, _ = rand_inputs(mech, B, 2)
    rng = np.random.default_rng(0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()          # noqa: E731
    st = _state(mech, q, v, torch.float64)
    for ct in (False, True):
        tc = _task_ctrl(mech, q, rng, ct=ct)
        c = tc.torch(torch.float64)
        rbd.simulate_(st, 2e-3 - 1e-9, t(tau), dt=1e-3, controller=c.joint)
        base = rbd.launch_info().kernels_launched
        rbd.simulate_(st, 2e-3 - 1e-9, t(tau), dt=1e-3, controller=c)
        assert rbd.launch_info().kernels_launched == base + 2 * 4
    rbd.task_pd_torques(st, _task_ctrl(mech, q, rng).torch(torch.float64))
    assert rbd.launch_info().kernels_launched == 1


@pytest.mark.gpu
def test_gpu_atlas_fp32_large_batch(built):
    """Atlas fp32 at 2^20 with four tasks (hands as points, feet as poses), both modes: finite results."""
    import torch
    mech = rbd.load_model("atlas", floating=True)
    B = 1 << 20
    st = rbd.MechanismState(mech, B, torch.float32)
    rbd.rand_(st, np.random.default_rng(0))
    st.v.mul_(0.2)
    st.q[4:7].zero_()
    st.q[6] = 0.9
    tasks = [TaskFrame(mech.findbody("l_hand"), None, [0.0, 0.1, 0.0]), TaskFrame(mech.findbody("r_hand"), None, [0.0, -0.1, 0.0]),
             TaskFrame(mech.findbody("l_foot")), TaskFrame(mech.findbody("r_foot"))]
    kinds = ["point", "point", "pose", "pose"]
    xr = rbd.relative_transform(st, tasks[2].body)
    xl = rbd.relative_transform(st, tasks[3].body)
    x_ref = torch.cat([torch.zeros(6, B, device="cuda"), xr, xl]).contiguous()
    g = torch.full((18,), 10.0, device="cuda")
    for ct in (False, True):
        a = rbd.MechanismState(mech, B, torch.float32)
        a.q.copy_(st.q)
        a.v.copy_(st.v)
        rbd.simulate_(a, 5e-3 - 1e-9, dt=1e-3, controller=rbd.TaskPD(tasks, kinds, g, g * 0.1, x_ref, computed_torque=ct))
        assert bool(torch.isfinite(a.q).all()) and bool(torch.isfinite(a.v).all())
