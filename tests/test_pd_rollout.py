"""Closed-loop rollouts (DESIGN 4.18): rbd_integrate_pd / ``controller=JointPD(...)`` on simulate_*, and the URDF joint bounds.

The host integrator below is the Munthe-Kaas RK4 step of tests/contact_oracle.py with the feedback law evaluated at every stage on
that stage's state, as the reference's simulate calls control!(τ, t, state) (src/simulate.jl:36-55):
    e = local(q_ref, q_s)            numpy restatement of local_coordinates! (local_error below)
    PD               τ = τ_ff - Kp e - Kd (v_s - v_ref)
    computed torque  τ = Oracle.inverse_dynamics(q_s, v_s, v̇_ref - Kp e - Kd (v_s - v_ref)) + τ_ff
then clamped to the effort bounds.  It is pinned on the CPU by Oracle.integrate / integrate_contact at zero gains; the device law
(csrc/rbd_pd.cuh, compiled for the host by tests/hostsim/hostsim_pd.cpp) must agree with local_error / the law, and the GPU rollouts
with the host integrator.
"""
import ctypes
import functools
import math
import zlib

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from oracle import Oracle
from rigidbodydynamics.jl_b200 import _cabi
from rigidbodydynamics.jl_b200._cabi import RbdModelDesc, make_desc
from tests import hostsim
from tests.contact_oracle import (K_QFLOAT, K_QSPH, K_SINCOS, NQ, RK4_A, RK4_B, _conj, _mtv, _quat_mul,
                                  _quat_to_rotvec, _rot, _rotvec_to_quat, global_coordinates, integrate_contact, local_rate)
from tests.util import config_distance, rand_inputs, randmech, ref_urdf, rel_err


TOL64 = 1e-9          # GPU rollout against the fp64 host integrator, relative (the other rollouts' bound)
# fp32 rollout against the fp64 host integrator, 5 steps at dt = 1e-3 from fp32-representable inputs, per mode.  Measured on an H100:
# q 4.2e-7 / v 2.1e-5 (Atlas, PD), 3.0e-7 / 2.8e-6 (Atlas, computed torque), 4.4e-7 / 4.3e-7 (iiwa14, computed torque), 3.4e-7 /
# 1.5e-6 (random tree, PD); at B = 1024 through the vectorised stage kernel 2.5e-7 / 1.8e-5 (Atlas, PD) and 2.6e-7 / 1.2e-6 (Atlas,
# computed torque); each bound is about 5x the largest error of its mode.
TOL32 = {"pd": 1e-4, "ct": 1.5e-5}


# ------------------------------------------------------------------------------------------------------------------
# the host integrator
# ------------------------------------------------------------------------------------------------------------------
def _cross(a, b):
    return np.cross(a, b, axis=0)


def local_error(desc, qref, q):
    """e = local_coordinates!(q_ref, q) of every joint, [nv, B] (fp64 numpy restatement of rbd_pd.cuh's joint_error)."""
    e = np.zeros((desc.nv, q.shape[1]))
    for i, jt in enumerate(desc.jtype):
        qs, vs = desc.qstart[i], desc.vstart[i]
        a, b = qref[qs:qs + NQ[jt]], q[qs:qs + NQ[jt]]
        if jt == K_QFLOAT:                       # log of the relative transform (spatialmotion.jl:226-252)
            psi, th = _quat_to_rotvec(_quat_mul(_conj(a[:4]), b[:4]))
            p = _mtv(_rot(a), b[4:7] - a[4:7])
            small = th < 1e-4
            ths = np.where(small, 1.0, th)
            g = np.where(small, 1 / 12 + th ** 2 / 720, (1 - ths / 2 / np.tan(ths / 2)) / ths ** 2)
            e[vs:vs + 3] = psi
            e[vs + 3:vs + 6] = p - 0.5 * _cross(psi, p) + g * _cross(psi, _cross(psi, p))
        elif jt == K_QSPH:
            e[vs:vs + 3] = _quat_to_rotvec(_quat_mul(_conj(a), b))[0]
        elif jt == K_SINCOS:
            e[vs] = np.arctan2(a[1] * b[0] - a[0] * b[1], a[1] * b[1] + a[0] * b[0])
        elif NQ[jt]:
            e[vs:vs + NQ[jt]] = b - a
    return e


def _col(x):
    return x[:, None] if x.ndim == 1 else x


def law(desc, q, v, qref, vref, ff, kp, kd, lo=None, hi=None):
    """ff - Kp e - Kd (v - v_ref), clamped to [lo, hi] when given; kp / kd [nv] or [nv, B]; vref / ff None = 0."""
    u = (0 if ff is None else ff) - _col(kp) * local_error(desc, qref, q) - _col(kd) * (v - (0 if vref is None else vref))
    return u if lo is None else np.clip(u, np.asarray(lo)[:, None], np.asarray(hi)[:, None])


class Ctrl:
    """The host form of a JointPD: numpy arrays; q_ref / v_ref / vd_ref [rows, B] or [nsteps, rows, B]."""

    def __init__(self, kp, kd, q_ref, v_ref=None, vd_ref=None, ct=False, bounds=None):
        self.kp, self.kd, self.q_ref, self.v_ref, self.vd_ref, self.ct, self.bounds = kp, kd, q_ref, v_ref, vd_ref, ct, bounds

    def at(self, a, n):
        return None if a is None else (a[n] if a.ndim == 3 else a)

    def torque(self, orc, n, q, v, tau_ff):
        lo, hi = self.bounds if self.bounds is not None else (None, None)
        qr, vr = self.at(self.q_ref, n), self.at(self.v_ref, n)
        if not self.ct:
            return law(orc.desc, q, v, qr, vr, tau_ff, self.kp, self.kd, lo, hi)
        vdd = law(orc.desc, q, v, qr, vr, self.at(self.vd_ref, n), self.kp, self.kd)
        tau = orc.inverse_dynamics(q, v, vdd) + (0 if tau_ff is None else tau_ff)
        return tau if lo is None else np.clip(tau, np.asarray(lo)[:, None], np.asarray(hi)[:, None])

    def torch(self, dtype):
        """The JointPD of this controller."""
        import torch
        t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dtype).cuda()    # noqa: E731
        return rbd.JointPD(t(self.kp), t(self.kd), t(self.q_ref), t(self.v_ref), vd_ref=t(self.vd_ref), computed_torque=self.ct,
                           effort_bounds=self.bounds)


def _tau_at(tau, n, i):
    if tau is None or tau.ndim == 2:
        return tau
    return tau[n] if tau.ndim == 3 else tau[n, i]


def integrate_pd(orc, q, v, ctrl, tau=None, *, dt=1e-4, nsteps=1, contact=None, s=None, stage_dynamics=None):
    """``nsteps`` closed-loop Munthe-Kaas RK4 steps; tau (τ_ff): None, [nv, B], [nsteps, nv, B] or [nsteps, 4, nv, B].  With
    ``contact`` the contact state s is integrated as in contact_oracle.integrate_contact; ``stage_dynamics(q, v, s, tau) -> (v̇, ṡ)``
    replaces the tree / contact dynamics (the loop rollout).  Returns (q, v, s)."""
    desc = orc.desc
    q, v = np.array(q, float), np.array(v, float)
    ns = 0 if contact is None else 3 * len(contact.body) * len(contact.halfspace)
    s = np.zeros((ns, q.shape[1])) if s is None else np.array(s, float)
    tau = None if tau is None else np.asarray(tau, float)
    for n in range(nsteps):
        q0, v0, s0 = q, v, s
        phid, vd, sd = [None] * 4, [None] * 4, [None] * 4
        for i in range(4):
            wa = dt * RK4_A[i]
            qs = global_coordinates(desc, q0, wa * phid[i - 1] if i else np.zeros_like(v0))
            vs = v0 + wa * vd[i - 1] if i else v0.copy()
            ss = s0 + wa * sd[i - 1] if i else s0.copy()
            t = ctrl.torque(orc, n, qs, vs, _tau_at(tau, n, i))
            if stage_dynamics is not None:
                vd[i], sd[i] = stage_dynamics(qs, vs, ss, t)
                qd = orc.dynamics(qs, vs, t, want_qd=True)[1]
            else:
                wr = None
                sd[i] = np.zeros_like(s0)
                if ns:
                    wr, sd[i], _ = orc.contact_dynamics(qs, vs, contact, ss)
                vd[i], qd = orc.dynamics(qs, vs, t, wr, want_qd=True)
            phid[i] = local_rate(desc, q0, qs, vs, qd)
        q = global_coordinates(desc, q0, dt * sum(RK4_B[i] * phid[i] for i in range(4)))
        v = v0 + dt * sum(RK4_B[i] * vd[i] for i in range(4))
        s = s0 + dt * sum(RK4_B[i] * sd[i] for i in range(4))
    return q, v, s


# ------------------------------------------------------------------------------------------------------------------
# CPU tier: URDF bounds
# ------------------------------------------------------------------------------------------------------------------
def test_urdf_joint_bounds(tmp_path):
    """test/test_urdf.jl:2-18: the six asserts on Acrobot and Acrobot_with_limits."""
    inf = float("inf")
    acro = rbd.parse_urdf(ref_urdf("Acrobot", tmp_path), remove_fixed_tree_joints=False)
    lim = rbd.parse_urdf(ref_urdf("Acrobot_with_limits", tmp_path), remove_fixed_tree_joints=False)
    find = lambda m, name: next(j for j in m.joints if j.name == name)     # noqa: E731
    for name in ("shoulder", "elbow"):
        j = find(acro, name)
        assert j.position_bounds == [rbd.Bounds(-inf, inf)]
        assert j.velocity_bounds == [rbd.Bounds(-inf, inf)]
        assert j.effort_bounds == [rbd.Bounds(-inf, inf)]
    for name, e in (("shoulder", 0.0), ("elbow", 5.0)):
        j = find(lim, name)
        assert j.position_bounds == [rbd.Bounds(-6.28, 6.28)]
        assert j.velocity_bounds == [rbd.Bounds(-10, 10)]
        assert j.effort_bounds == [rbd.Bounds(-e, e)]
    lo, hi = rbd.effort_bounds(lim)
    assert lo.tolist() == [-0.0, -5.0] and hi.tolist() == [0.0, 5.0]


def test_maximal_coordinates_keeps_joint_bounds():
    """maximal_coordinates copies every joint with its bounds, as the reference's _copyjoint! does."""
    m = rbd.load_model("iiwa14")
    mc = rbd.maximal_coordinates(m)
    assert [j.effort_bounds for j in mc.non_tree_joints] == [j.effort_bounds for j in m.joints]
    assert [j.position_bounds for j in mc.non_tree_joints] == [j.position_bounds for j in m.joints]


def test_effort_bounds_of_bundled_models():
    lo, hi = rbd.effort_bounds(rbd.load_model("iiwa14"))
    assert hi.tolist() == [320, 320, 176, 176, 110, 40, 40] and lo.tolist() == [-320, -320, -176, -176, -110, -40, -40]
    lo, hi = rbd.effort_bounds(rbd.load_model("atlas", floating=True))     # a JSON description without limits
    assert lo.shape == (36,) and np.isinf(lo).all() and np.isinf(hi).all() and (lo < 0).all()


# ------------------------------------------------------------------------------------------------------------------
# CPU tier: the device law compiled for the host
# ------------------------------------------------------------------------------------------------------------------
@functools.cache
def _shim():
    """tests/hostsim/hostsim_pd.cpp, compiled and loaded by hostsim.shim."""
    lib = hostsim.shim("hostsim_pd")
    vp = ctypes.c_void_p
    lib.hostsim_pd_law.argtypes = [ctypes.POINTER(RbdModelDesc), ctypes.c_int, ctypes.c_int64] + [vp] * 7 + [ctypes.c_int, vp, vp, vp]
    return lib


def hostsim_law(desc, q, v, qref, vref, ff, kp, kd, lo=None, hi=None):
    dt = q.dtype
    c = lambda a: None if a is None else np.ascontiguousarray(a, dt)           # noqa: E731
    p = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)     # noqa: E731
    B = q.shape[1]
    out = np.full((desc.nv, B), np.nan, dt)
    d, keep = make_desc(desc)
    q, v, qref, vref, ff, kp, kd = (c(a) for a in (q, v, qref, vref, ff, kp, kd))
    lo, hi = (None if a is None else np.ascontiguousarray(a, np.float64) for a in (lo, hi))
    assert _shim().hostsim_pd_law(ctypes.byref(d), 0 if dt == np.float32 else 1, B, p(q), p(v), p(qref), p(vref), p(ff), p(kp), p(kd),
                                  int(kp.ndim == 2), p(lo), p(hi), p(out)) == 0
    return out


def _rotate_by(q4, axis_angle):
    """q4 [4, B] times the unit quaternion of the rotation vectors axis_angle [3, B]."""
    return _quat_mul(q4, _rotvec_to_quat(axis_angle))


def _targets(mech, q, rng, near_pi=False):
    """q_ref: a random perturbation of every joint's coordinates, staying on the joints' manifolds; with near_pi the quaternion
    joints' relative rotations are within 1e-3 of pi."""
    d = mech.flatten()
    qref = np.array(q)
    B = q.shape[1]
    for i, jt in enumerate(d.jtype):
        a = qref[d.qstart[i]:d.qstart[i] + NQ[jt]]
        if jt in (K_QFLOAT, K_QSPH):
            r = rng.standard_normal((3, B))
            r /= np.linalg.norm(r, axis=0)
            ang = (math.pi - 1e-3 * rng.random(B)) if near_pi else rng.random(B) * 2.5
            a[:4] = _rotate_by(a[:4], r * ang)
            if jt == K_QFLOAT:
                a[4:7] += rng.standard_normal((3, B))
        elif jt == K_SINCOS:
            th = np.arctan2(a[0], a[1]) + rng.uniform(-3, 3, B)
            a[0], a[1] = np.sin(th), np.cos(th)
        else:
            a += rng.standard_normal(a.shape)
    return qref


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("case", ["randmech0", "randmech1", "randmech2", "randmech3", "atlas", "near_pi"])
def test_hostsim_law_matches_numpy(case, dtype):
    """pd_joint on every joint type against local_error + law in fp64: per-sample and shared gains, feedforward and v_ref present
    and absent, active clamps, and quaternion errors near pi."""
    rng = np.random.default_rng(7)
    mech = rbd.load_model("atlas", floating=True) if case == "atlas" else randmech(3 if case == "near_pi" else int(case[-1]))
    d = mech.flatten()
    B = 24
    q, v, tau, _, _ = rand_inputs(mech, B, 11)
    qref = _targets(mech, q, rng, near_pi=case == "near_pi")
    vref = rng.standard_normal(v.shape)
    r = lambda a: a.astype(dtype).astype(np.float64)                     # noqa: E731   inputs representable in dtype
    q, v, qref, vref, tau = r(q), r(v), r(qref), r(vref), r(tau)
    kp_s, kd_s = r(rng.uniform(0, 50, d.nv)), r(rng.uniform(0, 5, d.nv))
    kp_b, kd_b = r(rng.uniform(0, 50, (d.nv, B))), r(rng.uniform(0, 5, (d.nv, B)))
    tol = 1e-12 if dtype == np.float64 else 1e-5
    for kp, kd, vr, ff in ((kp_s, kd_s, vref, tau), (kp_b, kd_b, None, None), (kp_b, kd_b, vref, tau)):
        ref = law(d, q, v, qref, vr, ff, kp, kd)
        got = hostsim_law(d, q.astype(dtype), v.astype(dtype), qref.astype(dtype), None if vr is None else vr.astype(dtype),
                          None if ff is None else ff.astype(dtype), kp.astype(dtype), kd.astype(dtype))
        scale = np.abs(ref).max(0) + (np.abs(_col(kp)) * (1 + np.abs(local_error(d, qref, q)))).max(0)
        assert (np.abs(got - ref).max(0) / scale).max() < tol
        # clamps: bounds at about half the torque range, so that most DoFs saturate on some samples
        lo, hi = -np.abs(ref).mean(1) * 0.5, np.abs(ref).mean(1) * 0.4
        refc = law(d, q, v, qref, vr, ff, kp, kd, lo, hi)
        gotc = hostsim_law(d, q.astype(dtype), v.astype(dtype), qref.astype(dtype), None if vr is None else vr.astype(dtype),
                           None if ff is None else ff.astype(dtype), kp.astype(dtype), kd.astype(dtype), lo, hi)
        assert np.any(refc == hi[:, None]) and np.any(refc == lo[:, None]) and np.any((refc > lo[:, None]) & (refc < hi[:, None]))
        assert (np.abs(gotc - refc).max(0) / scale).max() < tol
    if case == "near_pi":
        th = [np.linalg.norm(local_error(d, qref, q)[d.vstart[i]:d.vstart[i] + 3], axis=0)
              for i, jt in enumerate(d.jtype) if jt in (K_QFLOAT, K_QSPH)]
        assert th and all(np.all(t > math.pi - 2e-3) for t in th)


def test_local_error_of_the_target_itself_is_zero():
    mech = randmech(1)
    d = mech.flatten()
    q, _, _, _, _ = rand_inputs(mech, 6, 3)
    assert np.abs(local_error(d, q, q)).max() < 1e-12
    assert np.abs(hostsim_law(d, q, np.zeros((d.nv, 6)), q, None, None, np.ones(d.nv), np.ones(d.nv))).max() < 1e-12


# ------------------------------------------------------------------------------------------------------------------
# CPU tier: the host integrator
# ------------------------------------------------------------------------------------------------------------------
def test_host_integrator_with_zero_gains_is_the_open_loop_rollout():
    """Kp = Kd = 0 and a per-step τ_ff: the closed-loop integrator equals Oracle.integrate step by step and, with contact,
    contact_oracle.integrate_contact."""
    mech = rbd.load_model("atlas", floating=True)
    d = mech.flatten()
    orc = Oracle(d)
    B, n = 5, 3
    q, v, tau, _, _ = rand_inputs(mech, B, 4)
    taus = tau[None] * np.linspace(0.5, 1.5, n)[:, None, None]
    ctrl = Ctrl(np.zeros(d.nv), np.zeros(d.nv), q)
    qc, vc, _ = integrate_pd(orc, q, v, ctrl, taus, dt=1e-3, nsteps=n)
    qo, vo = q, v
    for k in range(n):
        qo, vo = orc.integrate(qo, vo, taus[k], dt=1e-3, nsteps=1)
    assert config_distance(mech, qc, qo) < 1e-12 and rel_err(vc, vo) < 1e-12
    from tests.test_loops_rollout import atlas_on_floor, atlas_states
    mech, cd = atlas_on_floor()
    orc = Oracle(mech.flatten())
    q, v, tau = atlas_states(mech, B, 5)
    s0 = np.random.default_rng(1).standard_normal((cd.nstates, B)) * 1e-3
    ctrl = Ctrl(np.zeros(mech.num_velocities()), np.zeros(mech.num_velocities()), q)
    qc, vc, sc = integrate_pd(orc, q, v, ctrl, tau, dt=1e-3, nsteps=2, contact=cd, s=s0)
    qo, vo, so = integrate_contact(orc, q, v, s0, cd, tau, dt=1e-3, nsteps=2)
    assert np.any(so != s0)
    assert config_distance(mech, qc, qo) < 1e-12 and rel_err(vc, vo) < 1e-12 and rel_err(sc, so) < 1e-12


# ------------------------------------------------------------------------------------------------------------------
# CPU tier: C-ABI argument checks (host only, nothing launched)
# ------------------------------------------------------------------------------------------------------------------
class _PdDesc(ctypes.Structure):
    _fields_ = [("mode", ctypes.c_int32), ("kp", ctypes.c_void_p), ("kd", ctypes.c_void_p), ("gain_ld", ctypes.c_int64),
                ("q_ref", ctypes.c_void_p), ("v_ref", ctypes.c_void_p), ("vd_ref", ctypes.c_void_p),
                ("q_ref_step_stride", ctypes.c_int64), ("v_ref_step_stride", ctypes.c_int64),
                ("effort_lo", ctypes.POINTER(ctypes.c_double)), ("effort_hi", ctypes.POINTER(ctypes.c_double))]


def test_integrate_pd_argument_checks(built):
    from tests.loops_oracle import four_bar
    from tests.test_loops_rollout import atlas_on_floor
    lib = rbd.load_library()
    mech = rbd.load_model("iiwa14")
    h = _cabi.ModelHandle(mech.flatten())
    fake = 64                                         # never dereferenced by the checks below
    F32, F64 = _cabi.RBD_F32, _cabi.RBD_F64
    lo_ok, hi_ok = (np.ascontiguousarray(b) for b in rbd.effort_bounds(mech))
    dp = ctypes.POINTER(ctypes.c_double)

    def desc(**kw):
        f = dict(mode=0, kp=fake, kd=fake, gain_ld=0, q_ref=fake, v_ref=None, vd_ref=None, q_ref_step_stride=0, v_ref_step_stride=0,
                 effort_lo=lo_ok.ctypes.data_as(dp), effort_hi=hi_ok.ctypes.data_as(dp))
        f.update(kw)
        return _PdDesc(**f)

    def call(pd, dtype=F64, B=4, ld=4, step=0, stage=0, dt=1e-3, n=1, handle=h, loops=None, contact=None, s=None,
             traj=(None, None, None)):
        return lib.rbd_integrate_pd(handle.ptr, dtype, B, ld, fake, fake, s, None, step, stage,
                                    None if pd is None else ctypes.byref(pd), loops, contact, dt, n, *traj, None)

    def status(rc, text=None):
        assert rc == _cabi.RBD_EINVAL, rc
        if text:
            assert text.encode() in lib.rbd_last_error(), lib.rbd_last_error()
    status(call(None), "pd must not be NULL")
    for k in ("kp", "kd", "q_ref"):
        status(call(desc(**{k: None})), "must not be NULL")
    status(call(desc(mode=2)), "unknown mode")
    status(call(desc(mode=-1)), "unknown mode")
    status(call(desc(vd_ref=fake)), "computed-torque mode only")
    status(call(desc(q_ref_step_stride=-1)), "strides")
    status(call(desc(v_ref_step_stride=-7)), "strides")
    status(call(desc(), step=-1), "strides")
    status(call(desc(), stage=-1), "strides")
    status(call(desc(gain_ld=3)), "gain_ld")
    status(call(desc(effort_hi=None)), "both")
    bad_lo = lo_ok.copy()
    bad_lo[3] = 1e9
    status(call(desc(effort_lo=bad_lo.ctypes.data_as(dp))), "lo <= hi")
    nan_hi = hi_ok.copy()
    nan_hi[0] = np.nan
    status(call(desc(effort_hi=nan_hi.ctypes.data_as(dp))), "lo <= hi")
    status(call(desc(), n=-1))
    status(call(desc(), dt=0.0))
    status(call(desc(), traj=(fake, None, None)), "all NULL or all set")
    assert call(desc(), dtype=_cabi.RBD_DUAL64X6) == _cabi.RBD_EUNSUPPORTED
    assert call(desc(), B=8, ld=4) == _cabi.RBD_EDIM
    assert call(desc(), B=0, ld=0) == _cabi.RBD_OK                         # empty batch: nothing to do
    assert call(desc(gain_ld=4), dtype=F32, B=0, ld=4) == _cabi.RBD_OK
    # computed-torque mode on a mechanism with loops: the reference's inverse_dynamics! refuses loops
    fb = four_bar()
    hf = rbd.MechanismState(fb, 1, device="cpu").handle
    lst, keep = rbd.loop_desc(fb).c_struct()
    ct = desc(mode=1, effort_lo=None, effort_hi=None)
    assert call(ct, handle=hf, loops=ctypes.byref(lst)) == _cabi.RBD_ELOOP
    assert call(desc(effort_lo=None, effort_hi=None), handle=hf, loops=ctypes.byref(lst), B=0, ld=0) == _cabi.RBD_OK
    # contact: s is required with contact pairs
    am, cd = atlas_on_floor()
    ha = _cabi.ModelHandle(am.flatten())
    cst, keep2 = cd.c_struct()
    nolim = desc(effort_lo=None, effort_hi=None)
    status(call(nolim, handle=ha, contact=ctypes.byref(cst)), "s must not be NULL")
    status(call(nolim, handle=ha, contact=ctypes.byref(cst), s=fake, traj=(fake, fake, None)), "all NULL or all set")
    for x in (h, ha):
        x.close()


def test_python_argument_checks():
    """JointPD's shape / dtype / device checks run before any call into the library (CPU tensors: nothing reaches the GPU)."""
    import torch
    mech = rbd.load_model("iiwa14")
    st = rbd.MechanismState(mech, 3, device="cpu")
    nv, nq = st.nv, st.nq
    z = lambda *s, dtype=torch.float64: torch.zeros(*s, dtype=dtype)          # noqa: E731
    ok = dict(kp=z(nv), kd=z(nv), q_ref=z(nq, 3))
    with pytest.raises(ValueError):
        rbd.JointPD(z(nv), z(nv), z(nq, 3), vd_ref=z(nv, 3))
    cases = [(dict(ok, kp=z(nv + 1)), rbd.DimensionMismatch), (dict(ok, kd=z(nv, 3)), rbd.DimensionMismatch),
             (dict(ok, q_ref=z(nq, 4)), rbd.DimensionMismatch), (dict(ok, q_ref=z(1, nq, 3)), rbd.DimensionMismatch),
             (dict(ok, kp=z(nv, dtype=torch.float32)), TypeError), (dict(ok, q_ref=z(3, nq).t()), TypeError),
             (dict(ok, v_ref=z(nv, 2)), rbd.DimensionMismatch), (dict(ok, effort_bounds=(np.zeros(2), np.zeros(2))), rbd.DimensionMismatch)]
    for kw, err in cases:
        c = rbd.JointPD(kw["kp"], kw["kd"], kw["q_ref"], kw.get("v_ref"), effort_bounds=kw.get("effort_bounds"))
        with pytest.raises(err):
            rbd.simulate_(st, 2e-3, dt=1e-3, controller=c)
    with pytest.raises(TypeError):
        rbd.simulate_(st, 2e-3, dt=1e-3, controller=object())


# ------------------------------------------------------------------------------------------------------------------
# GPU tier
# ------------------------------------------------------------------------------------------------------------------
def _pad(a, ld, dtype, misalign=False):
    """[..., ld] device copy of a [..., B] with NaN padding; misalign: the data starts one element past a 16-byte boundary."""
    import torch
    shape = a.shape[:-1] + (ld,)
    n = int(np.prod(shape))
    t = torch.full((n + 1,), float("nan"), dtype=dtype, device="cuda")[int(misalign):n + int(misalign)].view(shape)
    t[..., :a.shape[-1]] = torch.from_numpy(np.ascontiguousarray(a)).to(dtype)
    return t


def _cabi_rollout(mech, q, v, ctrl, tau, dtype, dt, nsteps, ld, *, cd=None, s=None, loops=False, record=False, misalign=None):
    """rbd_integrate_pd through the C ABI on arrays with leading dimension ld (> B: NaN padding that must stay untouched);
    misalign: "q_ref" or "kp" -- that controller array starts one element past a 16-byte boundary."""
    import torch
    B = q.shape[1]
    st = rbd.MechanismState(mech, batch=1, dtype=dtype)
    qd, vd = _pad(q, ld, dtype), _pad(v, ld, dtype)
    sd = None if s is None else _pad(s, ld, dtype)
    td = None if tau is None else _pad(tau, ld, dtype)
    nv, nq = mech.num_velocities(), mech.num_positions()
    step, stage = (0, 0) if tau is None or tau.ndim == 2 else ((nv * ld, 0) if tau.ndim == 3 else (4 * nv * ld, nv * ld))
    per_sample = ctrl.kp.ndim == 2
    kp = _pad(ctrl.kp, ld, dtype, misalign == "kp") if per_sample else torch.from_numpy(ctrl.kp).to(dtype).cuda()
    kd = _pad(ctrl.kd, ld, dtype) if per_sample else torch.from_numpy(ctrl.kd).to(dtype).cuda()
    refs = [None if a is None else _pad(a, ld, dtype, misalign == "q_ref" and k == 0)
            for k, a in enumerate((ctrl.q_ref, ctrl.v_ref, ctrl.vd_ref))]
    rs = lambda a, rows: 0 if a is None or a.ndim == 2 else rows * ld        # noqa: E731
    dp = ctypes.POINTER(ctypes.c_double)
    lo, hi = (None, None) if ctrl.bounds is None else (np.ascontiguousarray(b, np.float64) for b in ctrl.bounds)
    p = lambda t: None if t is None else t.data_ptr()                        # noqa: E731
    d = _PdDesc(int(ctrl.ct), p(kp), p(kd), ld if per_sample else 0, p(refs[0]), p(refs[1]), p(refs[2]), rs(ctrl.q_ref, nq),
                rs(ctrl.v_ref if ctrl.v_ref is not None else ctrl.vd_ref, nv), None if lo is None else lo.ctypes.data_as(dp),
                None if hi is None else hi.ctypes.data_as(dp))
    lst, keep = rbd.loop_desc(mech).c_struct() if loops else (None, None)
    cst, keep2 = cd.c_struct() if cd is not None else (None, None)
    traj = (None, None, None)
    if record:
        traj = tuple(torch.empty((nsteps + 1, rows, B), dtype=dtype, device="cuda") for rows in (nq, nv, 0 if cd is None else cd.nstates))
        if cd is None or cd.nstates == 0:
            traj = traj[:2] + (None,)
    _cabi.check(rbd.load_library().rbd_integrate_pd(
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
        assert np.array_equal(traj[0][0].double().cpu().numpy(), q.astype(np.float32 if dtype == torch.float32 else np.float64))
    return out


def _model(which):
    if which == "atlas":
        return rbd.load_model("atlas", floating=True)
    if which == "valkyrie":
        return rbd.load_model("valkyrie", floating=True)
    if which in ("iiwa14", "double_pendulum"):
        return rbd.load_model(which)
    return randmech(int(which[-1]))


def _controller(mech, q, rng, *, ct=False, per_step=0, per_sample=False, clamp=False, vref=True, scale=1.0):
    d = mech.flatten()
    B = q.shape[1]
    kp = rng.uniform(5, 40, (d.nv, B) if per_sample else d.nv) * scale
    kd = rng.uniform(0.5, 4, (d.nv, B) if per_sample else d.nv) * scale
    qref = _targets(mech, q, rng) if not per_step else np.stack([_targets(mech, q, rng) for _ in range(per_step)])
    vshape = (d.nv, B) if not per_step else (per_step, d.nv, B)
    vr = rng.standard_normal(vshape) * 0.3 if vref else None
    vdr = rng.standard_normal(vshape) if ct else None
    bounds = None
    if clamp:
        lim = rng.uniform(5, 30, d.nv)
        bounds = (-lim, lim * 0.8)
    return Ctrl(kp, kd, qref, vr, vdr, ct, bounds)


@pytest.mark.gpu
@pytest.mark.parametrize("which,mode,per_step,per_sample,clamp,tau_kind,nsteps", [
    ("atlas", "pd", 0, False, True, "none", 5), ("atlas", "ct", 5, True, True, "step", 5),
    ("atlas", "pd", 5, True, True, "stage", 5), ("valkyrie", "ct", 0, False, False, "const", 3),
    ("valkyrie", "pd", 3, True, True, "step", 3), ("iiwa14", "pd", 0, True, True, "const", 10),
    ("iiwa14", "ct", 10, False, True, "none", 10), ("double_pendulum", "pd", 0, False, False, "stage", 20),
    ("double_pendulum", "ct", 20, True, False, "const", 20), ("randmech0", "pd", 4, True, True, "step", 4),
    ("randmech1", "ct", 0, False, False, "none", 4), ("randmech2", "pd", 0, False, True, "const", 4),
    ("randmech3", "ct", 4, True, True, "stage", 4)])
def test_gpu_rollout_matches_host_integrator_fp64(built, which, mode, per_step, per_sample, clamp, tau_kind, nsteps):
    import torch
    mech = _model(which)
    rng = np.random.default_rng(zlib.crc32(f"{which}{mode}{nsteps}".encode()))
    B = 37
    q, v, tau, _, _ = rand_inputs(mech, B, 21)
    v *= 0.3
    ctrl = _controller(mech, q, rng, ct=mode == "ct", per_step=per_step, per_sample=per_sample, clamp=clamp)
    taus = {"none": None, "const": tau, "step": tau[None] * rng.uniform(0.5, 1.5, (nsteps, 1, 1)),
            "stage": tau[None, None] * rng.uniform(0.5, 1.5, (nsteps, 4, 1, 1))}[tau_kind]
    orc = Oracle(mech.flatten())
    dt = 1e-3
    qr, vr, _ = integrate_pd(orc, q, v, ctrl, taus, dt=dt, nsteps=nsteps)
    if clamp:                                   # the clamp is active on some samples at the first stage, not on all
        t0 = ctrl.torque(orc, 0, q, v, _tau_at(taus, 0, 0))
        lo, hi = ctrl.bounds
        sat = (t0 == lo[:, None]) | (t0 == hi[:, None])
        assert sat.any() and not sat.all()
    qg, vg, _ = _cabi_rollout(mech, q, v, ctrl, taus, torch.float64, dt, nsteps, ld=B + 11, record=per_step > 0)
    assert config_distance(mech, qg, qr) < TOL64
    assert rel_err(vg, vr) < TOL64


@pytest.mark.gpu
@pytest.mark.parametrize("which,mode", [("atlas", "pd"), ("atlas", "ct"), ("iiwa14", "ct"), ("randmech2", "pd")])
def test_gpu_rollout_fp32(built, which, mode):
    import torch
    mech = _model(which)
    rng = np.random.default_rng(5)
    B = 33
    q, v, tau, _, _ = rand_inputs(mech, B, 23)
    v *= 0.3
    ctrl = _controller(mech, q, rng, ct=mode == "ct", per_sample=True, clamp=True)
    r = lambda a: None if a is None else a.astype(np.float32).astype(np.float64)    # noqa: E731
    q, v, tau = r(q), r(v), r(tau)
    ctrl.kp, ctrl.kd, ctrl.q_ref, ctrl.v_ref, ctrl.vd_ref = (r(a) for a in (ctrl.kp, ctrl.kd, ctrl.q_ref, ctrl.v_ref, ctrl.vd_ref))
    qr, vr, _ = integrate_pd(Oracle(mech.flatten()), q, v, ctrl, tau, dt=1e-3, nsteps=5)
    qg, vg, _ = _cabi_rollout(mech, q, v, ctrl, tau, torch.float32, 1e-3, 5, ld=B)
    eq, ev = config_distance(mech, qg, qr), rel_err(vg, vr)
    print(f"fp32 {which} {mode}: q {eq:.2e}  v {ev:.2e}")
    assert eq < TOL32[mode] and ev < TOL32[mode]


def _subset(ctrl, idx):
    """The controller of the columns idx."""
    cut = lambda a: None if a is None else a[..., idx]                       # noqa: E731
    return Ctrl(ctrl.kp if ctrl.kp.ndim == 1 else ctrl.kp[:, idx], ctrl.kd if ctrl.kd.ndim == 1 else ctrl.kd[:, idx], cut(ctrl.q_ref),
                cut(ctrl.v_ref), cut(ctrl.vd_ref), ctrl.ct, ctrl.bounds)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name,mode,per_sample", [("float64", "pd", False), ("float64", "pd", True), ("float64", "ct", True),
                                                        ("float32", "pd", True), ("float32", "ct", False)])
def test_gpu_vectorised_stage_kernel(built, dtype_name, mode, per_sample):
    """The law in integrate_stage_linear_kernel, the path of every batch with B >= 1024 and whole vectors per row: Atlas (revolute
    joints in the vectorised kernel, the floating base in the per-(sample, joint) one) at B = 1024, nonzero gains, per-step q_ref and
    v_ref (and v̇_ref), active clamps, a per-step τ_ff.  A column subset against the host integrator; the whole batch against the same
    call at ld = B + 1 (every joint in the per-(sample, joint) kernel) to rounding; a misaligned q_ref or per-sample Kp falls back to
    that kernel for the revolute rows with the same result.  The launch counts show which kernels ran."""
    import torch
    dtype = getattr(torch, dtype_name)
    mech = rbd.load_model("atlas", floating=True)
    B, n, dt = 1024, 3, 1e-3
    rng = np.random.default_rng(zlib.crc32(f"{dtype_name}{mode}{per_sample}".encode()))
    q, v, tau, _, _ = rand_inputs(mech, B, 31)
    v *= 0.3
    ctrl = _controller(mech, q, rng, ct=mode == "ct", per_step=n, per_sample=per_sample, clamp=True)
    taus = tau[None] * rng.uniform(0.5, 1.5, (n, 1, 1))
    if dtype == torch.float32:                  # fp32-representable inputs for the host integrator
        r = lambda a: None if a is None else a.astype(np.float32).astype(np.float64)    # noqa: E731
        q, v, taus = r(q), r(v), r(taus)
        ctrl.kp, ctrl.kd, ctrl.q_ref, ctrl.v_ref, ctrl.vd_ref = (r(a) for a in (ctrl.kp, ctrl.kd, ctrl.q_ref, ctrl.v_ref, ctrl.vd_ref))
    lo, hi = ctrl.bounds
    t0 = ctrl.torque(Oracle(mech.flatten()), 0, q, v, taus[0])
    sat = (t0 == lo[:, None]) | (t0 == hi[:, None])
    assert sat[6:].any() and not sat[6:].all()                # clamps active on some revolute DoFs and samples
    run = lambda ld, mis=None: (_cabi_rollout(mech, q, v, ctrl, taus, dtype, dt, n, ld, misalign=mis),   # noqa: E731
                                rbd.launch_info().kernels_launched)
    (qg, vg, _), k_vec = run(B)
    (qs, vs, _), k_scalar = run(B + 1)
    assert k_vec - k_scalar == 5 * n           # per stage the vectorised kernel, per step the vectorised finishing kernel
    idx = np.arange(3, B, 61)[:16]
    qr, vr, _ = integrate_pd(Oracle(mech.flatten()), q[:, idx], v[:, idx], _subset(ctrl, idx), taus[..., idx], dt=dt, nsteps=n)
    eq, ev = config_distance(mech, qg[:, idx], qr), rel_err(vg[:, idx], vr)
    tol = TOL64 if dtype == torch.float64 else TOL32[mode]
    print(f"vectorised {dtype_name} {mode} per_sample={per_sample}: q {eq:.2e}  v {ev:.2e}")
    assert eq < tol and ev < tol
    # the two kernels may round the law's last bit differently; fp64 shows it to 1e-12.  In fp32 Atlas' light links amplify one ulp
    # of torque through the feedback to the fp32 rollout's own error level (measured on an H100: v 2.0e-5 between the two paths in
    # PD mode, next to 1.8e-5 against the fp64 host integrator), so there the paths are held to the fp32 bound
    same = 1e-12 if dtype == torch.float64 else TOL32[mode]
    assert config_distance(mech, qg, qs) < same and rel_err(vg, vs) < same
    for mis in ("q_ref",) + (("kp",) if per_sample else ()):
        (qm, vm, _), k_mis = run(B, mis)
        assert k_vec - k_mis == 4 * n, mis        # the stage kernels fall back; the finishing kernels stay vectorised
        assert config_distance(mech, qm, qs) < same and rel_err(vm, vs) < same, mis


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["pd", "ct"])
def test_gpu_contact_rollout(built, mode):
    """Atlas on the floor holding a posture (targets = the initial configuration): the contact rollout with the controller against
    the host integrator, fp64, contact state included, recording on."""
    import torch
    from tests.test_loops_rollout import atlas_on_floor, atlas_states
    mech, cd = atlas_on_floor()
    B = 40
    q, v, tau = atlas_states(mech, B, 44)
    s0 = np.random.default_rng(3).standard_normal((cd.nstates, B)) * 1e-3
    rng = np.random.default_rng(9)
    ctrl = _controller(mech, q, rng, ct=mode == "ct", per_sample=mode == "pd", clamp=True, vref=False)
    ctrl.q_ref = q.copy()
    orc = Oracle(mech.flatten())
    qr, vr, sr = integrate_pd(orc, q, v, ctrl, tau, dt=1e-3, nsteps=5, contact=cd, s=s0)
    assert np.any(sr != s0)
    qg, vg, sg = _cabi_rollout(mech, q, v, ctrl, tau, torch.float64, 1e-3, 5, ld=B + 3, cd=cd, s=s0, record=True)
    # the stiff contacts amplify rounding: measured on an H100, v 1.04e-9 relative in PD mode with per-sample gains
    assert config_distance(mech, qg, qr) < TOL64 and rel_err(vg, vr) < 1e-8
    assert float(np.abs(sg - sr).max() / max(1.0, np.abs(sr).max())) < 1e-8


@pytest.mark.gpu
def test_gpu_loops_rollout_pd(built):
    """The four-bar and Atlas double support (loop rollout) in PD mode against the host integrator with LoopOracle's dynamics."""
    import torch
    from tests.loops_oracle import LoopOracle
    from tests.test_loops_rollout import _case, stage_dynamics
    for which in ("four_bar", "atlas_ds"):
        B = 21
        mech, cd, q, v, tau, s = _case(which, B, 32)
        lo = LoopOracle(mech)
        rng = np.random.default_rng(4)
        ctrl = _controller(mech, q, rng, per_sample=True, clamp=True, scale=0.2)
        sd = lambda qs, vs, ss, t: (stage_dynamics(lo, qs, vs, ss, cd, t)[0], np.zeros_like(ss))    # noqa: E731
        qr, vr, _ = integrate_pd(lo.oracle, q, v, ctrl, tau, dt=1e-3, nsteps=5, stage_dynamics=sd)
        qg, vg, _ = _cabi_rollout(mech, q, v, ctrl, tau, torch.float64, 1e-3, 5, ld=B + 2, loops=True)
        assert config_distance(mech, qg, qr) < TOL64 and rel_err(vg, vr) < TOL64, which


def _state(m, q, v, dtype):
    import torch
    st = rbd.MechanismState(m, q.shape[1], dtype)
    st.q.copy_(torch.from_numpy(np.ascontiguousarray(q)))
    st.v.copy_(torch.from_numpy(np.ascontiguousarray(v)))
    return st


@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name,B", [("float64", 37), ("float32", 4096), ("float64", 2048)])
def test_gpu_zero_gains_bit_identical_to_open_loop(built, dtype_name, B):
    """PD mode with Kp = Kd = 0 and a τ_ff schedule is bit-identical to the open-loop rollouts with the same torques: tree
    (rbd_integrate_schedule), contact (rbd_integrate_contact) and loops (rbd_integrate_loops); B = 4096 / 2048 take the vectorised
    stage kernels."""
    import torch
    from tests.test_loops_rollout import _case, atlas_on_floor, atlas_states
    dtype = getattr(torch, dtype_name)
    rng = np.random.default_rng(1)
    n = 3
    for which in ("tree", "contact", "loops"):
        if which == "tree":
            mech = rbd.load_model("atlas", floating=True)
            q, v, tau, _, _ = rand_inputs(mech, B, 2)
            cd, s = None, None
        elif which == "contact":
            mech, cd = atlas_on_floor()
            q, v, tau = atlas_states(mech, B, 3)
            s = rng.standard_normal((cd.nstates, B)) * 1e-3
        else:
            mech, cd, q, v, tau, s = _case("atlas_ds", B, 5)
        nv = mech.num_velocities()
        taus = torch.from_numpy(tau[None, None] * rng.uniform(0.5, 1.5, (n, 4, 1, 1))).to(dtype).cuda()
        zero = torch.zeros(nv, dtype=dtype, device="cuda")
        a, b = _state(mech, q, v, dtype), _state(mech, q, v, dtype)
        ctl = rbd.JointPD(zero, zero, torch.from_numpy(q).to(dtype).cuda() + 0.25, torch.ones_like(a.v))
        sa = None if s is None else torch.from_numpy(s).to(dtype).cuda()
        sb = None if s is None else sa.clone()
        if which == "tree":
            rbd.simulate_(a, n * 1e-3 - 1e-9, taus, dt=1e-3)
            rbd.simulate_(b, n * 1e-3 - 1e-9, taus, dt=1e-3, controller=ctl)
        elif which == "contact":
            rbd.simulate_contact_(a, n * 1e-3 - 1e-9, sa, taus, dt=1e-3)
            rbd.simulate_contact_(b, n * 1e-3 - 1e-9, sb, taus, dt=1e-3, controller=ctl)
        else:
            rbd.simulate_loops_(a, n * 1e-3 - 1e-9, taus, dt=1e-3)
            rbd.simulate_loops_(b, n * 1e-3 - 1e-9, taus, dt=1e-3, controller=ctl)
        assert torch.equal(a.q, b.q) and torch.equal(a.v, b.v), which
        assert not torch.equal(a.q, torch.from_numpy(q).to(dtype).cuda())
        if which == "contact":
            assert torch.equal(sa, sb)


@pytest.mark.gpu
def test_gpu_computed_torque_closed_forms(built):
    """Fixed-base revolute chain, computed-torque mode, fp64: zero gains and v̇_ref give q(t) = q0 + v0 t + v̇_ref t^2 / 2 (RK4 is
    exact on it); gains with a constant target and v_ref = v̇_ref = 0 give ë + Kd ė + Kp e = 0 per DoF, matched against the
    analytic solution to RK4 accuracy."""
    import torch
    rng = np.random.default_rng(3)
    mech = rbd.rand_chain_mechanism(rng, [rbd.Revolute] * 6)
    nv, B = 6, 64
    q0 = rng.uniform(-1, 1, (nv, B))
    v0 = rng.uniform(-1, 1, (nv, B))
    acc = rng.uniform(-2, 2, (nv, B))
    T, dt = 0.5, 1e-3
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()          # noqa: E731
    st = _state(mech, q0, v0, torch.float64)
    zero = torch.zeros(nv, dtype=torch.float64, device="cuda")
    n = rbd.simulate_(st, T - 1e-9, dt=dt, controller=rbd.JointPD(zero, zero, t(q0), vd_ref=t(acc), computed_torque=True))
    tt = n * dt
    assert rel_err(st.q.cpu().numpy(), q0 + v0 * tt + 0.5 * acc * tt * tt) < 1e-10
    assert rel_err(st.v.cpu().numpy(), v0 + acc * tt) < 1e-10
    # second-order error dynamics: underdamped, critically damped and overdamped DoFs
    kp = np.array([100.0, 100.0, 25.0, 400.0, 16.0, 64.0])
    kd = np.array([4.0, 20.0, 10.0, 10.0, 12.0, 2.0])
    qref = rng.uniform(-1, 1, (nv, B))
    st = _state(mech, q0, v0, torch.float64)
    n = rbd.simulate_(st, T - 1e-9, dt=dt, controller=rbd.JointPD(t(kp), t(kd), t(qref), computed_torque=True))
    tt = n * dt
    e0, de0 = q0 - qref, v0
    e = np.empty_like(e0)
    de = np.empty_like(e0)
    for k in range(nv):
        r = np.roots([1.0, kd[k], kp[k]])
        if abs(r[0] - r[1]) < 1e-12:                     # critical: (c1 + c2 t) exp(r t)
            a_ = r[0].real
            c1, c2 = e0[k], de0[k] - a_ * e0[k]
            e[k] = (c1 + c2 * tt) * np.exp(a_ * tt)
            de[k] = (c2 + a_ * (c1 + c2 * tt)) * np.exp(a_ * tt)
        else:
            M = np.array([[1, 1], [r[0], r[1]]])
            c = np.linalg.solve(M, np.stack([e0[k], de0[k]]).astype(complex))
            e[k] = (c[0] * np.exp(r[0] * tt) + c[1] * np.exp(r[1] * tt)).real
            de[k] = (c[0] * r[0] * np.exp(r[0] * tt) + c[1] * r[1] * np.exp(r[1] * tt)).real
    assert np.abs(st.q.cpu().numpy() - qref - e).max() < 1e-8
    assert np.abs(st.v.cpu().numpy() - de).max() < 1e-7


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["orientation", "pose"])
def test_gpu_reference_pd_control(built, which):
    """test/test_pd_control.jl "orientation control" / "pose control" on rand_floating_tree_mechanism (one floating body): computed
    torque with gains 100 / 20, Δt = 1e-3, 3 s, fp64, over a batch of random targets -- in joint space, whose error for the
    floating joint is the SE(3) log of q_ref^-1 q.  Orientation: the target's rotation only (translation free, gains 0 on it),
    R R_des^T = I and ω = 0 to 1e-8; pose: the whole transform and twist to 1e-6."""
    import torch
    rng = np.random.default_rng(57 if which == "orientation" else 58)
    mech = rbd.rand_floating_tree_mechanism(rng, [])
    assert len(mech.joints) == 1 and type(mech.joints[0].joint_type) is rbd.QuaternionFloating
    B = 64
    st = rbd.MechanismState(mech, B, torch.float64)
    rbd.rand_(st, rng)
    qref = np.empty((7, B))
    r = rng.standard_normal((4, B))
    qref[:4] = r / np.linalg.norm(r, axis=0)
    qref[4:] = rng.standard_normal((3, B))
    kp = np.array([100.0] * 6)
    kd = np.array([20.0] * 6)
    if which == "orientation":
        kp[3:] = kd[3:] = 0.0
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()          # noqa: E731
    n = rbd.simulate_(st, 3.0, dt=1e-3, controller=rbd.JointPD(t(kp), t(kd), t(qref), computed_torque=True))
    assert n >= 3000                                  # the reference's `while t < final_time` loop on floating-point t
    q, v = st.q.cpu().numpy(), st.v.cpu().numpy()
    R, Rd = _rot(q), _rot(qref)
    orient = np.abs(np.einsum("ijb,kjb->ikb", R, Rd) - np.eye(3)[:, :, None]).max()
    assert orient < 1e-8 and np.abs(v[:3]).max() < 1e-8
    if which == "pose":
        assert np.abs(q[4:] - qref[4:]).max() < 1e-6 and np.abs(v).max() < 1e-6


@pytest.mark.gpu
def test_gpu_energy_with_feedback(built):
    """Fixed-base 1-DoF chain, PD mode, v_ref = 0, constant q_ref, no feedforward: E_kin + E_pot + Kp e^2 / 2 is non-increasing over
    the rollout within the integration error; its rate in continuous time is -Kd v^2."""
    import torch
    rng = np.random.default_rng(12)
    mech = rbd.rand_chain_mechanism(rng, [rbd.Revolute])
    B, dt, n = 32, 1e-3, 400
    q0 = rng.uniform(-2, 2, (1, B))
    v0 = rng.uniform(-2, 2, (1, B))
    qref = rng.uniform(-1, 1, (1, B))
    kp, kd = 30.0, 0.8
    st = _state(mech, q0, v0, torch.float64)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float64)).cuda()     # noqa: E731
    qt, vt = rbd.simulate_trajectory_(st, n, dt=dt, controller=rbd.JointPD(t([kp]), t([kd]), t(qref)))
    E = []
    for k in range(n + 1):
        kin = rbd.kinetic_energy(_state(mech, qt[k].cpu().numpy(), vt[k].cpu().numpy(), torch.float64)).cpu().numpy()
        pot = rbd.gravitational_potential_energy(_state(mech, qt[k].cpu().numpy(), vt[k].cpu().numpy(), torch.float64)).cpu().numpy()
        e = qt[k].cpu().numpy() - qref
        E.append(kin.reshape(-1) + pot.reshape(-1) + 0.5 * kp * (e * e).sum(0))
    E = np.array(E)
    dE = np.diff(E, axis=0)
    assert (dE <= 1e-9 * np.maximum(1.0, np.abs(E[:-1]))).all()
    # the rate: E(t + dt) - E(t) = -Kd v^2 dt, here against the trapezoidal rule on the recorded v (its own error is O(dt^3): 5.9e-5
    # of the largest step on the fp64 host integrator); over the whole rollout the energy lost is Kd times the integral of v^2
    v = vt.cpu().numpy()[:, 0]
    rate = -kd * 0.5 * (v[:-1] ** 2 + v[1:] ** 2) * dt
    assert np.abs(dE - rate).max() < 2e-4 * np.abs(rate).max()
    assert np.abs((E[-1] - E[0]) - rate.sum(0)).max() < 1e-4 * np.abs(rate.sum(0)).max()
    assert E[-1].mean() < 0.2 * E[0].mean()


@pytest.mark.gpu
def test_gpu_saturation(built, tmp_path):
    """Acrobot_with_limits (shoulder effort 0: unactuated) under PD with its effort bounds: the shoulder gets no torque -- the rollout
    equals the open-loop rollout with the elbow torque alone; bounds lo = hi = 0 everywhere reproduce the passive rollout."""
    import torch
    mech = rbd.parse_urdf(ref_urdf("Acrobot_with_limits", tmp_path))
    B, dt = 16, 1e-3
    rng = np.random.default_rng(2)
    q0, v0 = rng.uniform(-1, 1, (2, B)), rng.uniform(-1, 1, (2, B))
    qref = rng.uniform(-1, 1, (2, B))
    kp, kd = np.array([50.0, 50.0]), np.array([5.0, 5.0])
    ctrl = Ctrl(kp, kd, qref, bounds=rbd.effort_bounds(mech))
    qr, vr, _ = integrate_pd(Oracle(mech.flatten()), q0, v0, ctrl, dt=dt, nsteps=50)
    st = _state(mech, q0, v0, torch.float64)
    rbd.simulate_(st, 50 * dt - 1e-9, dt=dt, controller=ctrl.torch(torch.float64))
    assert config_distance(mech, st.q.cpu().numpy(), qr) < TOL64 and rel_err(st.v.cpu().numpy(), vr) < TOL64
    # the host integrator's shoulder torque is 0 at every stage: check it directly at the start
    assert np.all(ctrl.torque(Oracle(mech.flatten()), 0, q0, v0, None)[0] == 0)
    a, b = _state(mech, q0, v0, torch.float64), _state(mech, q0, v0, torch.float64)
    zero = (np.zeros(2), np.zeros(2))
    rbd.simulate_(a, 50 * dt - 1e-9, dt=dt)
    rbd.simulate_(b, 50 * dt - 1e-9, dt=dt, controller=Ctrl(kp, kd, qref, bounds=zero).torch(torch.float64))
    assert config_distance(mech, b.q.cpu().numpy(), a.q.cpu().numpy()) < 1e-13 and rel_err(b.v.cpu().numpy(), a.v.cpu().numpy()) < 1e-13


@pytest.mark.gpu
@pytest.mark.parametrize("which,B", [("atlas", 4096), ("atlas", 777), ("iiwa14", 4096), ("contact", 4096), ("loops", 4096)])
def test_gpu_launch_count(built, which, B):
    """PD mode launches exactly the kernels of the open-loop rollout; computed-torque mode two more per stage (fp64: the inverse
    dynamics is one kernel)."""
    import torch
    from tests.test_loops_rollout import _case, atlas_on_floor, atlas_states
    cd = s = None
    if which == "contact":
        mech, cd = atlas_on_floor()
        q, v, tau = atlas_states(mech, B, 3)
        s = torch.zeros((cd.nstates, B), dtype=torch.float64, device="cuda")
    elif which == "loops":
        mech, cd, q, v, tau, _ = _case("atlas_ds", B, 5)
    else:
        mech = _model(which)
        q, v, tau, _, _ = rand_inputs(mech, B, 2)
    nv = mech.num_velocities()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()          # noqa: E731
    gains = torch.ones(nv, dtype=torch.float64, device="cuda")
    st = _state(mech, q, v, torch.float64)
    run = {"contact": lambda c: rbd.simulate_contact_(st, 2e-3 - 1e-9, s, t(tau), dt=1e-3, controller=c),
           "loops": lambda c: rbd.simulate_loops_(st, 2e-3 - 1e-9, t(tau), dt=1e-3, controller=c)}.get(
        which, lambda c: rbd.simulate_(st, 2e-3 - 1e-9, t(tau), dt=1e-3, controller=c))
    run(None)
    base = rbd.launch_info().kernels_launched
    run(rbd.JointPD(gains, gains, t(q)))
    assert rbd.launch_info().kernels_launched == base
    if which != "loops":
        run(rbd.JointPD(gains, gains, t(q), computed_torque=True))
        assert rbd.launch_info().kernels_launched == base + 2 * 4 * 2
