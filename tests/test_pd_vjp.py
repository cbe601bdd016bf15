"""Reverse mode through closed-loop rollouts (DESIGN 4.19): rbd_integrate_pd_vjp, ``integrate_pd_vjp_`` and ``controller=`` on
``autodiff.simulate`` / ``autodiff.simulate_contact``.

CPU tier: the law's adjoint (csrc/rbd_integrate_adjoint.cuh's pd_adj_joint, compiled for the host by tests/hostsim/hostsim_pd_vjp.cpp)
against central differences of the law on every joint type, and the C ABI's argument checks.  GPU tier: the whole backward pass
against central differences of the fp64 GPU rollout, bit-identity with the open-loop VJPs at zero gains, the vectorised phase kernel
against its per-(sample, joint) fallback, autograd against the direct call and across checkpoint segments, launch counts, and a
gradient-descent use case.
"""
import ctypes
import hashlib
import os
import subprocess
import tempfile
import zlib

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from rigidbodydynamics.jl_b200 import _cabi
from tests.contact_oracle import K_PLANAR, K_PRIS, K_QFLOAT, K_QSPH, K_REV, K_SINCOS, K_SPQFLOAT, NQ, _quat_mul, _rotvec_to_quat
from oracle import Oracle
from rigidbodydynamics.jl_b200._cabi import RbdModelDesc, make_desc
from tests.test_integrate_vjp import EPS_FD, TOL64, TOL_FD, host_ivjp
from tests.test_pd_rollout import Ctrl, _PdDesc, _controller, _model, _tau_at, integrate_pd
from tests.util import rand_inputs, rel_err

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "..", "rigidbodydynamics", "jl_b200", "csrc")
_lib = None
NV = {K_REV: 1, K_PRIS: 1, K_PLANAR: 3, K_QFLOAT: 6, K_SPQFLOAT: 6, K_QSPH: 3, K_SINCOS: 1}


class _PdBar(ctypes.Structure):
    _fields_ = [("kp", ctypes.c_void_p), ("kd", ctypes.c_void_p), ("q_ref", ctypes.c_void_p), ("v_ref", ctypes.c_void_p),
                ("vd_ref", ctypes.c_void_p)]


# ------------------------------------------------------------------------------------------------------------------
# CPU tier: the law's adjoint compiled for the host
# ------------------------------------------------------------------------------------------------------------------
def _shim():
    """tests/hostsim/hostsim_pd_vjp.cpp, compiled on first use into a temporary directory."""
    global _lib
    if _lib is not None:
        return _lib
    srcs = [os.path.join(_HERE, "hostsim", "hostsim_pd_vjp.cpp")] + sorted(
        os.path.join(_CSRC, f) for f in os.listdir(_CSRC) if f.endswith((".cuh", ".h")) or f == "rbd_model.cpp")
    h = hashlib.sha1(b"".join(open(s, "rb").read() for s in srcs)).hexdigest()[:16]
    d = os.path.join(tempfile.gettempdir(), f"rbd_hostsim_pd_vjp_{os.getuid()}")
    os.makedirs(d, exist_ok=True)
    so = os.path.join(d, f"hostsim_pd_vjp_{h}.so")
    if not os.path.exists(so):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so + f".{os.getpid()}",
                               srcs[0], os.path.join(_CSRC, "rbd_model.cpp")])
        os.replace(so + f".{os.getpid()}", so)
    lib = ctypes.CDLL(so)
    vp = ctypes.c_void_p
    lib.hostsim_joint_error.argtypes = [ctypes.c_int, vp, vp, vp]
    lib.hostsim_pd_adj_joint.argtypes = [ctypes.c_int] + [vp] * 19
    i64, ci = ctypes.c_int64, ctypes.c_int
    ctl = [ci, vp, vp, i64, vp, vp, vp, i64, i64, vp, vp, vp, i64, i64, ctypes.c_double, ci]
    lib.hostsim_pd_traj.argtypes = [ctypes.POINTER(RbdModelDesc), ci, i64, vp, vp] + ctl
    lib.hostsim_pd_vjp.argtypes = [ctypes.POINTER(RbdModelDesc), ci, i64, vp, vp] + ctl + [vp] * 7
    _lib = lib
    return lib


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _err(kind, qref, q):
    e = np.zeros(NV[kind])
    _shim().hostsim_joint_error(kind, _p(np.ascontiguousarray(qref, float)), _p(np.ascontiguousarray(q, float)), _p(e))
    return e


def _joint_config(kind, rng, near_pi=False):
    """(q, q_ref) of one joint: unit quaternions / sin-cos pairs; with near_pi the relative rotation is within 1e-3 of pi (not at)."""
    q = rng.standard_normal(NQ[kind])
    if kind in (K_QFLOAT, K_QSPH):
        q[:4] /= np.linalg.norm(q[:4])
        r = rng.standard_normal(3)
        r /= np.linalg.norm(r)
        ang = np.pi - 1e-3 * (0.2 + 0.8 * rng.random()) if near_pi else 2.5 * rng.random()
        qref = q.copy()
        qref[:4] = _quat_mul(q[:4, None], _rotvec_to_quat((r * ang)[:, None]))[:, 0]
        if kind == K_QFLOAT:
            qref[4:] += rng.standard_normal(3)
        return q, qref
    if kind == K_SINCOS:
        th, tr = rng.uniform(-3, 3, 2)
        return np.array([np.sin(th), np.cos(th)]), np.array([np.sin(tr), np.cos(tr)])
    return q, q + rng.standard_normal(NQ[kind])


@pytest.mark.parametrize("kind", [K_REV, K_PRIS, K_PLANAR, K_SPQFLOAT, K_SINCOS, K_QSPH, K_QFLOAT])
@pytest.mark.parametrize("mode", ["pd", "pd_clamp", "ct", "near_pi"])
def test_law_adjoint_matches_central_differences(kind, mode):
    """pd_adj_joint against central differences (eps 1e-5, 1e-6 relative) of the law on one joint, fp64: the seeds' products with
    the law's derivatives with respect to q_s (configuration coordinates), v_s, q_ref (all coordinates, as given), v_ref, Kp, Kd and
    τ_ff (PD) / v̇_ref (computed torque).  pd_clamp: bounds active on some rows (away from them by a margin) and not on others."""
    if mode == "near_pi" and kind not in (K_QSPH, K_QFLOAT):
        pytest.skip("quaternion joints only")
    rng = np.random.default_rng(zlib.crc32(f"{kind}{mode}".encode()))
    nq, nv = NQ[kind], NV[kind]
    ct = mode == "ct"
    for trial in range(4):
        q, qref = _joint_config(kind, rng, mode == "near_pi")
        v, vref, ff = rng.standard_normal((3, nv))
        kp, kd = rng.uniform(5, 40, nv), rng.uniform(0.5, 4, nv)
        seed = rng.standard_normal(nv)         # τ̄ (PD) or v̇̄_des (computed torque)

        def law(q_, v_, qr_, vr_, kp_, kd_, ff_):
            return ff_ - kp_ * _err(kind, qr_, q_) - kd_ * (v_ - vr_)

        lo = hi = tau = None
        if mode == "pd_clamp":
            u = law(q, v, qref, vref, kp, kd, ff)
            lo, hi = u - 1.0, u + 1.0
            cut = rng.random(nv) < 0.5
            cut[0] = True
            hi[cut] = u[cut] - 0.5            # saturated at hi, 0.5 away
            if nv > 1:
                cut[-1] = False
                hi[-1] = u[-1] + 1.0
            tau = np.clip(u, lo, hi)

        def L(x):
            u = law(*x)
            return float(seed @ (u if lo is None else np.clip(u, lo, hi)))

        x0 = [q, v, qref, vref, kp, kd, ff]
        cq, cv, m = np.zeros(nq), np.zeros(nv), np.zeros(nv)
        kpb, kdb, qrb, vrb, vdrb = np.zeros(nv), np.zeros(nv), np.zeros(nq), np.zeros(nv), np.zeros(nv)
        c = lambda a: None if a is None else np.ascontiguousarray(a, float)     # noqa: E731
        _shim().hostsim_pd_adj_joint(kind, _p(c(q)), _p(c(v)), _p(c(qref)), _p(c(vref)), _p(c(kp)), _p(c(kd)),
                                     _p(c(np.zeros(nv) if ct else seed)), _p(c(tau)), _p(c(lo)), _p(c(hi)), _p(c(seed) if ct else None),
                                     _p(cq), _p(cv), _p(m), _p(kpb), _p(kdb), _p(qrb), _p(vrb), _p(vdrb))
        # the adjoint of each input; with a seed on v̇_des, the "ff" slot is v̇_ref (vdrb), and m is the zero τ̄ passed through
        grads = [cq, cv, qrb, vrb, kpb, kdb, vdrb if ct else m]
        for idx, (x, gr) in enumerate(zip(x0, grads)):
            for k in range(len(x)):
                xp = [a.copy() for a in x0]
                xm = [a.copy() for a in x0]
                xp[idx][k] += 1e-5
                xm[idx][k] -= 1e-5
                fd = (L(xp) - L(xm)) / 2e-5
                assert abs(fd - gr[k]) <= 1e-6 * max(1.0, abs(fd)), (trial, idx, k, fd, gr[k])
        if ct:
            assert np.all(m == 0)
        if mode == "pd_clamp":
            sat = (tau == lo) | (tau == hi)
            assert sat.any() and np.all(m[sat] == 0) and np.all(m[~sat] == seed[~sat])


# ------------------------------------------------------------------------------------------------------------------
# CPU tier: the whole backward pass on the CPU
# ------------------------------------------------------------------------------------------------------------------
def _ctl_args(ctrl, dtype, B, taus):
    """(keep-alive list, the shim's controller arguments) for a host Ctrl and τ_ff (None, [nv, B], [n, nv, B] or [n, 4, nv, B])."""
    c = lambda a: None if a is None else np.ascontiguousarray(a, dtype)        # noqa: E731
    arrs = [c(a) for a in (ctrl.kp, ctrl.kd, ctrl.q_ref, ctrl.v_ref, ctrl.vd_ref, taus)]
    lo, hi = (None, None) if ctrl.bounds is None else (np.ascontiguousarray(b, np.float64) for b in ctrl.bounds)
    nq, nv = ctrl.q_ref.shape[-2], ctrl.kp.shape[0]
    rs = lambda a, rows: 0 if a is None or a.ndim == 2 else rows * B        # noqa: E731
    t = arrs[5]
    step, stage = (0, 0) if t is None or t.ndim == 2 else ((nv * B, 0) if t.ndim == 3 else (4 * nv * B, nv * B))
    vr = ctrl.v_ref if ctrl.v_ref is not None else ctrl.vd_ref
    args = [int(ctrl.ct), _p(arrs[0]), _p(arrs[1]), B if ctrl.kp.ndim == 2 else 0, _p(arrs[2]), _p(arrs[3]), _p(arrs[4]),
            rs(ctrl.q_ref, nq), rs(vr, nv), _p(lo), _p(hi), _p(t), step, stage]
    return arrs + [lo, hi], args


def host_pd_traj(desc, q, v, ctrl, taus, n, dt=1e-3):
    """The closed-loop trajectory of the device code run on the CPU: [n + 1, rows, B] fp64 / fp32 (the dtype of q)."""
    dt_, B = q.dtype, q.shape[1]
    qt = np.zeros((n + 1, desc.nq, B), dt_); vt = np.zeros((n + 1, desc.nv, B), dt_)
    qt[0], vt[0] = q, v
    keep, args = _ctl_args(ctrl, dt_, B, taus)
    d, keep2 = make_desc(desc)
    assert _shim().hostsim_pd_traj(ctypes.byref(d), 0 if dt_ == np.float32 else 1, B, _p(qt), _p(vt), *args, dt, n) == 0
    return qt, vt


def host_pd_vjp(desc, qt, vt, ctrl, taus, qtb, vtb, dt=1e-3):
    """The CPU run of rbd_integrate_pd_vjp: dict q0t, q0c, v0b, taub and kp / kd / q_ref / v_ref / vd_ref gradients."""
    dt_ = qt.dtype
    n, B = qt.shape[0] - 1, qt.shape[2]
    keep, args = _ctl_args(ctrl, dt_, B, taus)
    z = lambda a: None if a is None else np.zeros(np.shape(a), dt_)          # noqa: E731
    out = {"q0t": np.full((desc.nv, B), np.nan, dt_), "q0c": np.full((desc.nq, B), np.nan, dt_), "v0b": np.full((desc.nv, B), np.nan, dt_),
           "taub": z(taus), "kp": np.zeros((desc.nv, B), dt_), "kd": np.zeros((desc.nv, B), dt_), "q_ref": z(ctrl.q_ref),
           "v_ref": z(ctrl.v_ref), "vd_ref": z(ctrl.vd_ref)}
    bars = (ctypes.c_void_p * 5)(*[None if out[k] is None else out[k].ctypes.data for k in ("kp", "kd", "q_ref", "v_ref", "vd_ref")])
    c = lambda a: np.ascontiguousarray(a, dt_)                                  # noqa: E731
    qt, vt, qtb, vtb = c(qt), c(vt), c(qtb), c(vtb)
    d, keep2 = make_desc(desc)
    assert _shim().hostsim_pd_vjp(ctypes.byref(d), 0 if dt_ == np.float32 else 1, B, _p(qt), _p(vt), *args, dt, n, _p(qtb), _p(vtb),
                                  _p(out["q0t"]), _p(out["q0c"]), _p(out["v0b"]), _p(out["taub"]), bars) == 0
    return out


def _cpu_model(which):
    if which == "randtree":          # every joint type
        from tests.util import randmech
        return randmech(1)
    return _model(which)


@pytest.mark.parametrize("which,mode,n,per_step,per_sample,clamp,tau_kind", [
    ("atlas", "pd", 5, 0, False, True, "const"), ("atlas", "ct", 5, 5, True, True, "step"), ("atlas", "pd", 1, 1, True, False, "none"),
    ("randtree", "pd", 5, 5, True, True, "stage"), ("randtree", "ct", 1, 0, False, False, "const"),
    ("randtree", "ct", 5, 0, True, True, "none"), ("double_pendulum", "pd", 5, 0, False, True, "step"),
    ("double_pendulum", "ct", 5, 5, False, True, "stage"), ("double_pendulum", "pd", 1, 0, True, False, "const")])
def test_cpu_backward_matches_host_integrator(which, mode, n, per_step, per_sample, clamp, tau_kind):
    """The whole backward pass on the CPU against central differences (eps 1e-5, 1e-6) of the fp64 host closed-loop integrator
    (test_pd_rollout.integrate_pd) along random directions of q0 (tangent), v0, τ_ff, Kp, Kd, q_ref, v_ref and v̇_ref; held and
    per-step targets, shared and per-sample gains, no / constant / per-step / per-stage feedforward, clamps active on some samples."""
    mech = _cpu_model(which)
    d = mech.flatten()
    dt, B = 1e-3, 3
    q, v, taus, ctrl, rng = _fd_case(mech, B, n, mode, per_step, per_sample, clamp, tau_kind, zlib.crc32(f"{which}{mode}{n}".encode()))
    orc = Oracle(d)
    if clamp:                                       # active on some samples at the first stage, not on all
        t0 = ctrl.torque(orc, 0, q, v, _tau_at(taus, 0, 0))
        lo, hi = ctrl.bounds
        sat = (t0 == lo[:, None]) | (t0 == hi[:, None])
        assert sat.any() and not sat.all()
    qt, vt = host_pd_traj(d, q, v, ctrl, taus, n, dt)
    qr, vr, _ = integrate_pd(orc, q, v, ctrl, taus, dt=dt, nsteps=n)
    # the CPU run steps like the host integrator, to the rollout bound of tests/test_pd_rollout.py (the feedback amplifies rounding)
    assert rel_err(qt[-1], qr) < 1e-9 and rel_err(vt[-1], vr) < 1e-9
    wq, wv = rng.standard_normal(qt.shape), rng.standard_normal(vt.shape)
    r = host_pd_vjp(d, qt, vt, ctrl, taus, wq, wv, dt)
    base = dict(q0=q, v0=v, tau=taus, kp=ctrl.kp, kd=ctrl.kd, q_ref=ctrl.q_ref, v_ref=ctrl.v_ref, vd_ref=ctrl.vd_ref)
    grads = dict(q0=r["q0c"], v0=r["v0b"], tau=r["taub"], kp=r["kp"] if ctrl.kp.ndim == 2 else r["kp"].sum(1),
                 kd=r["kd"] if ctrl.kd.ndim == 2 else r["kd"].sum(1), q_ref=r["q_ref"], v_ref=r["v_ref"], vd_ref=r["vd_ref"])

    def loss(x):
        c = Ctrl(x["kp"], x["kd"], x["q_ref"], x["v_ref"], x["vd_ref"], ctrl.ct, ctrl.bounds)
        L, qq, vv = 0.0, x["q0"], x["v0"]
        L += float((wq[0] * qq).sum() + (wv[0] * vv).sum())
        for s in range(n):                          # step by step, with the step's slice of every per-step array
            cs = Ctrl(c.kp, c.kd, *(None if a is None else (a[s:] if a.ndim == 3 else a) for a in (c.q_ref, c.v_ref, c.vd_ref)),
                      ct=c.ct, bounds=c.bounds)
            t = x["tau"]
            t = None if t is None else (t if t.ndim == 2 else t[s:s + 1] if t.ndim == 4 else t[s])
            qq, vv, _ = integrate_pd(orc, qq, vv, cs, t, dt=dt, nsteps=1)
            L += float((wq[s + 1] * qq).sum() + (wv[s + 1] * vv).sum())
        return L
    # Atlas' light links amplify the rollout's rounding (the host integrator agrees with the CPU run to ~1e-11 only): at eps = 1e-5
    # that noise reaches 1e-6 of the Kp derivative, at 1e-4 the central differences agree to 3e-7
    eps = 1e-4 if which == "atlas" else EPS_FD
    for k, x in base.items():
        if x is None:
            continue
        dk = rng.standard_normal(np.shape(x))
        if k == "q0":
            dk = _tangent(mech, q, dk)
        xp, xm = dict(base), dict(base)
        xp[k], xm[k] = x + eps * dk, x - eps * dk
        fd = (loss(xp) - loss(xm)) / (2 * eps)
        ad = float((grads[k] * dk).sum())
        assert abs(fd - ad) <= TOL_FD * max(1.0, abs(fd)), (k, fd, ad)


@pytest.mark.parametrize("which", ["atlas", "randtree", "double_pendulum"])
def test_cpu_zero_gains_equal_open_loop_cpu_run(which):
    """PD mode with Kp = Kd = 0 and no bounds: the CPU backward pass equals rbd_integrate_vjp's CPU run
    (tests/hostsim/hostsim_integrate_vjp.cpp) to 1e-12."""
    mech = _cpu_model(which)
    d = mech.flatten()
    n, B = 4, 3
    q, v, tau, _, _ = rand_inputs(mech, B, 12)
    rng = np.random.default_rng(2)
    taus = rng.standard_normal((n, d.nv, B))
    ctrl = Ctrl(np.zeros(d.nv), np.zeros(d.nv), _controller(mech, q, rng).q_ref, rng.standard_normal((d.nv, B)))
    qt, vt = host_pd_traj(d, q, v, ctrl, taus, n)
    wq, wv = rng.standard_normal(qt.shape), rng.standard_normal(vt.shape)
    r = host_pd_vjp(d, qt, vt, ctrl, taus, wq, wv)
    o = host_ivjp(d, qt, vt, taus, n, wq, wv, dt=1e-3)
    for a, b in (("q0t", "q0t"), ("q0c", "q0c"), ("v0b", "v0b"), ("taub", "taub")):
        assert rel_err(r[a], o[b]) < 1e-12, a


# ------------------------------------------------------------------------------------------------------------------
# CPU tier: C-ABI argument checks (host only, nothing launched)
# ------------------------------------------------------------------------------------------------------------------
def test_integrate_pd_vjp_argument_checks(built):
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

    def call(pd, dtype=F64, B=4, step=0, stage=0, dt=1e-3, n=1, handle=h, contact=None, tau=fake, tau_bar=None, bar=None,
             traj=(fake, fake), s_traj=None):
        return lib.rbd_integrate_pd_vjp(handle.ptr, dtype, B, *traj, s_traj, tau, step, stage, None if pd is None else ctypes.byref(pd),
                                        contact, dt, n, None, None, None, None, None, None, None, tau_bar,
                                        None if bar is None else ctypes.byref(bar), None)

    def status(rc, text=None, want=_cabi.RBD_EINVAL):
        assert rc == want, rc
        if text:
            assert text.encode() in lib.rbd_last_error(), lib.rbd_last_error()
    status(call(None), "pd must not be NULL")
    for k in ("kp", "kd", "q_ref"):
        status(call(desc(**{k: None})), "must not be NULL")
    status(call(desc(mode=2)), "unknown mode")
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
    status(call(desc(), n=-1))
    status(call(desc(), dt=0.0))
    status(call(desc(), tau=None, tau_bar=fake), "tau_bar needs tau")
    status(call(desc(), traj=(None, fake)), "must not be NULL")
    # adjoints of arrays the controller does not have
    status(call(desc(), bar=_PdBar(None, None, None, fake, None)), "pd_bar")
    status(call(desc(mode=1, v_ref=fake), bar=_PdBar(None, None, None, None, fake)), "pd_bar")
    status(call(desc(mode=1, v_ref=fake, vd_ref=fake), bar=_PdBar(fake, fake, fake, fake, fake), B=0), want=_cabi.RBD_OK)
    assert call(desc(), dtype=_cabi.RBD_DUAL64X6) == _cabi.RBD_EUNSUPPORTED
    assert call(desc(), B=0) == _cabi.RBD_OK                              # empty batch: nothing to do
    status(call(desc(gain_ld=4), dtype=F32, B=0), "gain_ld")              # the leading dimension is B
    # contact: descriptor checks, and s_traj with contact pairs
    am, cd = atlas_on_floor()
    ha = _cabi.ModelHandle(am.flatten())
    cst, keep = cd.c_struct()
    nolim = desc(effort_lo=None, effort_hi=None)
    status(call(nolim, handle=ha, contact=ctypes.byref(cst)), "s_traj must not be NULL")
    for x in (h, ha):
        x.close()


def test_python_refuses_loops():
    """autodiff.simulate with a controller refuses a mechanism with loops before anything reaches the library."""
    import torch
    from tests.loops_oracle import four_bar
    fb = four_bar()
    z = torch.zeros(1, 1, dtype=torch.float64)
    ctl = rbd.JointPD(z, z, z)
    with pytest.raises(_cabi.RbdError) as ei:
        rbd.autodiff.simulate(fb, z, z, dt=1e-3, nsteps=1, controller=ctl)
    assert ei.value.status == _cabi.RBD_ELOOP
    with pytest.raises(_cabi.RbdError) as ei:
        rbd.integrate_pd_vjp_(fb, z[None], z[None], controller=ctl, dt=1e-3)
    assert ei.value.status == _cabi.RBD_ELOOP


# ------------------------------------------------------------------------------------------------------------------
# GPU tier
# ------------------------------------------------------------------------------------------------------------------
def _torch_ctrl(ctrl, dtype, grad=False):
    import torch
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dtype).cuda().requires_grad_(grad)   # noqa: E731
    return rbd.JointPD(t(ctrl.kp), t(ctrl.kd), t(ctrl.q_ref), t(ctrl.v_ref), vd_ref=t(ctrl.vd_ref), computed_torque=ctrl.ct,
                       effort_bounds=ctrl.bounds)


def _tangent(mech, q, d):
    """d with every quaternion block made orthogonal to q's quaternion (a direction the configuration gradient sees)."""
    fl = mech.flatten()
    d = d.copy()
    for i, jt in enumerate(fl.jtype):
        if jt in (K_QFLOAT, K_QSPH):
            s = fl.qstart[i]
            qq = q[s:s + 4]
            d[s:s + 4] -= qq * (qq * d[s:s + 4]).sum(0) / (qq * qq).sum(0)
        elif jt == K_SINCOS:
            s = fl.qstart[i]
            qq = q[s:s + 2]
            d[s:s + 2] -= qq * (qq * d[s:s + 2]).sum(0) / (qq * qq).sum(0)
    return d


def _fd_case(mech, B, nsteps, mode, per_step, per_sample, clamp, tau_kind, seed, contact=None, s0=None, q=None, v=None, tau=None):
    """Inputs of one closed-loop rollout: (q, v, taus, ctrl) in numpy."""
    rng = np.random.default_rng(seed)
    if q is None:
        q, v, tau, _, _ = rand_inputs(mech, B, seed % 97)
        v *= 0.3
    ctrl = _controller(mech, q, rng, ct=mode == "ct", per_step=per_step, per_sample=per_sample, clamp=clamp)
    taus = {"none": None, "const": tau, "step": tau[None] * rng.uniform(0.5, 1.5, (nsteps, 1, 1)),
            "stage": tau[None, None] * rng.uniform(0.5, 1.5, (nsteps, 4, 1, 1))}[tau_kind]
    return q, v, taus, ctrl, rng


def _check_fd(mech, q, v, taus, ctrl, rng, nsteps, dt=1e-3, contact=None, s0=None, eps=1e-5, tol=1e-6):
    """autodiff.simulate(_contact) with the controller: autograd gradients against central differences of the fp64 GPU rollout
    along random directions of every input."""
    import torch
    f64 = torch.float64
    T = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(f64).cuda()      # noqa: E731
    names = ["q0", "v0", "tau", "kp", "kd", "q_ref", "v_ref", "vd_ref"] + (["s0"] if contact is not None else [])
    base = dict(q0=q, v0=v, tau=taus, kp=ctrl.kp, kd=ctrl.kd, q_ref=ctrl.q_ref, v_ref=ctrl.v_ref, vd_ref=ctrl.vd_ref, s0=s0)
    nq, nv = q.shape[0], v.shape[0]
    wq, wv = rng.standard_normal((nq, q.shape[1])), rng.standard_normal((nv, q.shape[1]))
    ws = None if contact is None else rng.standard_normal(s0.shape)

    def run(x, grad=False):
        t = {k: (None if x[k] is None else T(x[k]).requires_grad_(grad)) for k in names}
        ctl = rbd.JointPD(t["kp"], t["kd"], t["q_ref"], t["v_ref"], vd_ref=t["vd_ref"], computed_torque=ctrl.ct,
                          effort_bounds=ctrl.bounds)
        if contact is None:
            out = rbd.autodiff.simulate(mech, t["q0"], t["v0"], t["tau"], dt=dt, nsteps=nsteps, trajectory=False, controller=ctl)
        else:
            out = rbd.autodiff.simulate_contact(mech, t["q0"], t["v0"], t["s0"], t["tau"], contact=contact, dt=dt, nsteps=nsteps,
                                                trajectory=False, controller=ctl)
        L = (out[0] * T(wq)).sum() + (out[1] * T(wv)).sum() + (0 if contact is None else (out[2] * T(ws)).sum())
        if grad:
            L.backward()
            return {k: (None if t[k] is None else t[k].grad.cpu().numpy()) for k in names}
        return float(L)
    g = run(base, grad=True)
    for k in names:
        if base[k] is None:
            continue
        d = rng.standard_normal(np.shape(base[k]))
        if k == "q0":
            d = _tangent(mech, q, d)
        xp, xm = dict(base), dict(base)
        xp[k] = base[k] + eps * d
        xm[k] = base[k] - eps * d
        fd = (run(xp) - run(xm)) / (2 * eps)
        ad = float((g[k] * d).sum())
        print(f"{k}: fd {fd:.10e} ad {ad:.10e}")
        assert abs(fd - ad) <= tol * max(1.0, abs(fd)), (k, fd, ad)


@pytest.mark.gpu
@pytest.mark.parametrize("which,mode,per_step,per_sample,clamp,tau_kind,nsteps", [
    ("atlas", "pd", 0, False, True, "const", 5), ("atlas", "ct", 5, True, False, "step", 5), ("atlas", "pd", 1, True, True, "none", 1),
    ("randmech1", "pd", 5, True, True, "stage", 5), ("randmech2", "ct", 0, False, True, "const", 5),
    ("double_pendulum", "pd", 0, True, False, "step", 5), ("double_pendulum", "ct", 1, False, True, "none", 1)])
def test_gpu_gradients_match_central_differences(built, which, mode, per_step, per_sample, clamp, tau_kind, nsteps):
    mech = _model(which)
    q, v, taus, ctrl, rng = _fd_case(mech, 7, nsteps, mode, per_step, per_sample, clamp, tau_kind,
                                     zlib.crc32(f"{which}{mode}{per_step}".encode()))
    _check_fd(mech, q, v, taus, ctrl, rng, nsteps)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["pd", "ct"])
def test_gpu_contact_gradients_match_central_differences(built, mode):
    """Atlas on the floor holding its posture under PD / computed-torque control (targets = the initial configuration)."""
    from tests.test_loops_rollout import atlas_on_floor, atlas_states
    mech, cd = atlas_on_floor()
    B = 5
    q, v, tau = atlas_states(mech, B, 44)
    rng = np.random.default_rng(9)
    ctrl = _controller(mech, q, rng, ct=mode == "ct", per_sample=mode == "pd", clamp=False, vref=False)
    ctrl.q_ref = q.copy()
    s0 = rng.standard_normal((cd.nstates, B)) * 1e-3
    # the stiff contacts make the gradients large (|q0 gradient| ~ 1e10 here): a smaller step keeps the truncation error down
    _check_fd(mech, q, v, tau, ctrl, rng, 3, contact=cd, s0=s0, eps=1e-7, tol=1e-5)


def _direct(mech, qt, vt, taus, ctl, dt, gq, gv, B, nv, contact=None, st=None, gs=None):
    """integrate_pd_vjp_ with every output: (q0_bar_cfg, v0_bar, s0_bar, tau_bar, kp_bar, kd_bar, q_ref_bar, v_ref_bar, vd_ref_bar)."""
    import torch
    n = qt.shape[0] - 1
    qtb, vtb = torch.zeros_like(qt), torch.zeros_like(vt)
    qtb[-1] = gq; vtb[-1] = gv
    stb = None
    if contact is not None:
        stb = torch.zeros_like(st)
        stb[-1] = gs
    z = lambda t: None if t is None else torch.zeros_like(t)      # noqa: E731
    out = dict(q0_bar_cfg=torch.empty_like(qt[0]), v0_bar=torch.empty_like(vt[0]),
               s0_bar=None if contact is None else torch.empty_like(st[0]), tau_bar=z(taus),
               kp_bar=torch.zeros_like(vt[0]), kd_bar=torch.zeros_like(vt[0]), q_ref_bar=z(ctl.q_ref), v_ref_bar=z(ctl.v_ref),
               vd_ref_bar=z(ctl.vd_ref))
    rbd.integrate_pd_vjp_(mech, qt, vt, taus, controller=ctl, dt=dt, contact=contact, s_traj=st, q_traj_bar=qtb, v_traj_bar=vtb,
                          s_traj_bar=stb, **out)
    return out


def _record(mech, q, v, taus, ctl, dt, n, contact=None, s=None):
    import torch
    from rigidbodydynamics.jl_b200.autodiff import _model_handle, _pd_trajectory
    h = _model_handle(mech)
    B = q.shape[1]
    step, stage = (0, 0) if taus is None or taus.dim() == 2 else ((taus[0].numel(), 0) if taus.dim() == 3 else
                                                                  (taus[0].numel(), taus[0, 0].numel()))
    return _pd_trajectory(h, q, v, s, taus, 0, n, step, stage, ctl, contact, dt, "test")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
def test_gpu_zero_gains_bit_identical_to_open_loop_vjp(built, dtype_name):
    """PD mode, Kp = Kd = 0, no bounds: the gradients to q0, v0 and the torques are bit-identical to rbd_integrate_vjp's and, with
    contact, rbd_integrate_contact_vjp's; the gain gradients are not zero (the law is still differentiated)."""
    import torch
    from tests.test_loops_rollout import atlas_on_floor, atlas_states
    dtype = getattr(torch, dtype_name)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dtype).cuda()     # noqa: E731
    n, dt = 3, 1e-3
    for which in ("tree", "contact"):
        for B in (37, 2048):
            if which == "tree":
                mech = rbd.load_model("atlas", floating=True)
                q, v, tau, _, _ = rand_inputs(mech, B, 2)
                cd, s = None, None
            else:
                mech, cd = atlas_on_floor()
                q, v, tau = atlas_states(mech, B, 3)
                s = T(np.random.default_rng(1).standard_normal((cd.nstates, B)) * 1e-3)
            nv = mech.num_velocities()
            rng = np.random.default_rng(B)
            taus = T(tau[None, None] * rng.uniform(0.5, 1.5, (n, 4, 1, 1)))
            zero = torch.zeros(nv, dtype=dtype, device="cuda")
            ctl = rbd.JointPD(zero, zero, T(q) + 0.25, T(v) * 0 + 1)
            qt, vt, st = _record(mech, T(q), T(v), taus, ctl, dt, n, cd, s)
            gq, gv = T(rng.standard_normal(q.shape)), T(rng.standard_normal(v.shape))
            gs = None if cd is None else T(rng.standard_normal(s.shape))
            out = _direct(mech, qt, vt, taus, ctl, dt, gq, gv, B, nv, cd, st, gs)
            qtb, vtb = torch.zeros_like(qt), torch.zeros_like(vt)
            qtb[-1] = gq; vtb[-1] = gv
            qc, vb, tb = torch.empty_like(qt[0]), torch.empty_like(vt[0]), torch.zeros_like(taus)
            if cd is None:
                rbd.integrate_vjp_(mech, qt, vt, taus, dt=dt, q_traj_bar=qtb, v_traj_bar=vtb, q0_bar_cfg=qc, v0_bar=vb, tau_bar=tb)
            else:
                stb = torch.zeros_like(st)
                stb[-1] = gs
                sb = torch.empty_like(st[0])
                rbd.integrate_contact_vjp_(mech, qt, vt, st, taus, contact=cd, dt=dt, q_traj_bar=qtb, v_traj_bar=vtb, s_traj_bar=stb,
                                           q0_bar_cfg=qc, v0_bar=vb, s0_bar=sb, tau_bar=tb)
                assert torch.equal(sb, out["s0_bar"]), (which, B)
            assert torch.equal(qc, out["q0_bar_cfg"]) and torch.equal(vb, out["v0_bar"]) and torch.equal(tb, out["tau_bar"]), (which, B)
            assert bool(out["kp_bar"].abs().sum() > 0) and bool(out["v_ref_bar"].abs().sum() == 0)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,per_sample", [("pd", False), ("pd", True), ("ct", True)])
def test_gpu_vectorised_phase_kernel(built, mode, per_sample):
    """Atlas at B = 1024, fp64: the vectorised controller phase kernel against the per-(sample, joint) fallback, forced by a misaligned
    q_ref, to 1e-12; the launch counts show which path ran."""
    import torch
    mech = rbd.load_model("atlas", floating=True)
    n, dt, B = 2, 1e-3, 1024
    q, v, taus, ctrl, rng = _fd_case(mech, B, n, mode, n, per_sample, True, "step", 77 + per_sample)
    f64 = torch.float64
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(f64).cuda()     # noqa: E731
    gq, gv = T(rng.standard_normal(q.shape)), T(rng.standard_normal(v.shape))
    nv = v.shape[0]

    def run(misalign):
        ctl = _torch_ctrl(ctrl, f64)
        if misalign:
            buf = torch.empty(ctl.q_ref.numel() + 1, dtype=f64, device="cuda")
            qr = buf[1:].view(ctl.q_ref.shape)
            qr.copy_(ctl.q_ref)
            ctl.q_ref = qr
        qt, vt, _ = _record(mech, T(q), T(v), T(taus), ctl, dt, n)
        out = _direct(mech, qt, vt, T(taus), ctl, dt, gq, gv, B, nv)
        return out, rbd.launch_info().kernels_launched
    a, ka = run(False)
    b, kb = run(True)
    # per step: 4 vectorised stage kernels of the recompute and 5 vectorised phase kernels (Atlas' floating base always takes the
    # per-(sample, joint) kernels too)
    assert ka - kb == 9 * n, (ka, kb)
    for k in a:
        if a[k] is not None:
            x, y = a[k], b[k]
            assert float((x - y).abs().max()) <= 1e-12 * max(1.0, float(y.abs().max())), k


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["pd", "ct"])
def test_gpu_autograd_equals_direct_and_checkpoints(built, mode):
    """autodiff.simulate with the controller equals integrate_pd_vjp_ bit for bit, and checkpoint_every in {1, 3, nsteps} gives
    bit-identical gradients, gain and reference gradients included (per-step q_ref, shared gains summed over the batch)."""
    import torch
    mech = rbd.load_model("atlas", floating=True)
    n, dt, B = 6, 1e-3, 9
    q, v, taus, ctrl, rng = _fd_case(mech, B, n, mode, n, False, True, "stage", 5)
    f64 = torch.float64
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(f64).cuda()     # noqa: E731
    wq, wv = T(rng.standard_normal(q.shape)), T(rng.standard_normal(v.shape))
    names = ("kp", "kd", "q_ref", "v_ref", "vd_ref")

    def grads(every, trajectory=False):
        ctl = _torch_ctrl(ctrl, f64, grad=True)
        q0, v0, tt = T(q).requires_grad_(), T(v).requires_grad_(), T(taus).requires_grad_()
        out = rbd.autodiff.simulate(mech, q0, v0, tt, dt=dt, nsteps=n, trajectory=trajectory, checkpoint_every=every, controller=ctl)
        qn, vn = (out[0][-1], out[1][-1]) if trajectory else out
        ((qn * wq).sum() + (vn * wv).sum()).backward()
        return [q0.grad, v0.grad, tt.grad] + [None if getattr(ctl, k) is None else getattr(ctl, k).grad for k in names]
    ref = grads(None, trajectory=True)
    for every in (1, 3, n):
        g = grads(every)
        for a, b in zip(ref, g):
            assert (a is None) == (b is None)
            assert a is None or torch.equal(a, b), every
    ctl = _torch_ctrl(ctrl, f64)
    qt, vt, _ = _record(mech, T(q), T(v), T(taus), ctl, dt, n)
    out = _direct(mech, qt, vt, T(taus), ctl, dt, wq, wv, B, v.shape[0])
    assert torch.equal(out["q0_bar_cfg"], ref[0]) and torch.equal(out["v0_bar"], ref[1]) and torch.equal(out["tau_bar"], ref[2])
    assert torch.equal(out["kp_bar"].sum(1), ref[3]) and torch.equal(out["kd_bar"].sum(1), ref[4])
    for k, r in zip(("q_ref_bar", "v_ref_bar", "vd_ref_bar"), ref[5:]):
        assert (out[k] is None) == (r is None) and (r is None or torch.equal(out[k], r)), k


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["pd", "ct"])
def test_gpu_launch_counts(built, mode):
    """PD mode launches exactly the open-loop VJP's kernels plus the recompute's controller work; computed-torque mode adds per stage
    one inverse-dynamics VJP and, with bounds, one mask kernel."""
    import torch
    mech = rbd.load_model("iiwa14")
    n, dt, B = 2, 1e-3, 33
    f64 = torch.float64
    q, v, taus, ctrl, rng = _fd_case(mech, B, n, mode, 0, False, True, "const", 3)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(f64).cuda()     # noqa: E731
    ctl = _torch_ctrl(ctrl, f64)
    qt, vt, _ = _record(mech, T(q), T(v), T(taus), ctl, dt, n)
    gq, gv = T(rng.standard_normal(q.shape)), T(rng.standard_normal(v.shape))
    _direct(mech, qt, vt, T(taus), ctl, dt, gq, gv, B, v.shape[0])
    k_pd = rbd.launch_info().kernels_launched
    qtb, vtb = torch.zeros_like(qt), torch.zeros_like(vt)
    qtb[-1] = gq; vtb[-1] = gv
    rbd.integrate_vjp_(mech, qt, vt, T(taus), dt=dt, q_traj_bar=qtb, v_traj_bar=vtb, q0_bar_cfg=torch.empty_like(qt[0]),
                       v0_bar=torch.empty_like(vt[0]))
    k_open = rbd.launch_info().kernels_launched
    # computed torque, per stage: the recompute's inverse dynamics and pd_finish_kernel (as rbd_integrate_pd), then the mask kernel
    # and the inverse-dynamics VJP
    assert k_pd - k_open == (0 if mode == "pd" else 4 * 4 * n), (k_pd, k_open)


def _state(mech, q, v):
    import torch
    st = rbd.MechanismState(mech, q.shape[1], torch.float64)
    st.q.copy_(torch.from_numpy(np.ascontiguousarray(q)))
    st.v.copy_(torch.from_numpy(np.ascontiguousarray(v)))
    return st


@pytest.mark.gpu
def test_gpu_gradient_descent_on_target(built):
    """The double pendulum tracking a goal under PD control: a few gradient steps on the held q_ref lower the tracking loss
    |q(T) - q_goal|^2 monotonically."""
    import torch
    mech = rbd.load_model("double_pendulum")
    f64 = torch.float64
    B, n, dt = 4, 200, 2e-3
    q0 = torch.zeros(2, B, dtype=f64, device="cuda")
    v0 = torch.zeros_like(q0)
    goal = torch.tensor([[0.6], [-0.4]], dtype=f64, device="cuda").expand(2, B)
    kp, kd = torch.full((2,), 30.0, dtype=f64, device="cuda"), torch.full((2,), 6.0, dtype=f64, device="cuda")
    qref = goal.clone().contiguous().requires_grad_()
    losses = []
    for it in range(6):
        ctl = rbd.JointPD(kp, kd, qref)
        qn, vn = rbd.autodiff.simulate(mech, q0, v0, dt=dt, nsteps=n, trajectory=False, checkpoint_every=50, controller=ctl)
        loss = ((qn - goal) ** 2).sum()
        losses.append(float(loss))
        qref.grad = None
        loss.backward()
        with torch.no_grad():
            qref -= 0.5 * qref.grad
    print(losses)
    assert all(b < a for a, b in zip(losses, losses[1:])) and losses[-1] < 0.5 * losses[0]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["pd", "ct"])
def test_gpu_at_scale(built, mode):
    """Atlas fp32 at B = 2^20, 5 steps: finite gradients."""
    import torch
    mech = rbd.load_model("atlas", floating=True)
    B, n, dt = 1 << 20, 5, 1e-3
    f32 = torch.float32
    q, v, tau, _, _ = rand_inputs(mech, 1024, 5)
    rng = np.random.default_rng(1)
    ctrl = _controller(mech, q, rng, ct=mode == "ct", per_sample=False, clamp=True)
    rep = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(f32).cuda().repeat(1, B // 1024)   # noqa: E731
    kp, kd = (torch.from_numpy(a).to(f32).cuda() for a in (ctrl.kp, ctrl.kd))
    ctl = rbd.JointPD(kp, kd, rep(ctrl.q_ref), rep(ctrl.v_ref), vd_ref=rep(ctrl.vd_ref), computed_torque=ctrl.ct,
                      effort_bounds=ctrl.bounds)
    qt, vt, _ = _record(mech, rep(q), rep(v) * 0.3, rep(tau), ctl, dt, n)
    gq = torch.ones_like(qt[0])
    out = _direct(mech, qt, vt, rep(tau), ctl, dt, gq, torch.zeros_like(vt[0]), B, v.shape[0])
    for k, t in out.items():
        assert t is None or bool(torch.isfinite(t).all()), k


@pytest.mark.gpu
def test_gpu_python_argument_checks(built):
    """integrate_pd_vjp_ and controller= refuse inconsistent arguments before any call into the library."""
    import torch
    mech = rbd.load_model("iiwa14")
    nq, nv, B, n = 7, 7, 3, 2
    f64 = torch.float64
    z = lambda *s: torch.zeros(*s, dtype=f64, device="cuda")      # noqa: E731
    qt, vt = z(n + 1, nq, B), z(n + 1, nv, B)
    ctl = rbd.JointPD(z(nv), z(nv), z(nq, B))
    with pytest.raises(ValueError, match="v_ref_bar"):
        rbd.integrate_pd_vjp_(mech, qt, vt, controller=ctl, dt=1e-3, v_ref_bar=z(nv, B))
    with pytest.raises(ValueError, match="vd_ref_bar"):
        rbd.integrate_pd_vjp_(mech, qt, vt, controller=ctl, dt=1e-3, vd_ref_bar=z(nv, B))
    with pytest.raises(ValueError, match="need contact"):
        rbd.integrate_pd_vjp_(mech, qt, vt, controller=ctl, dt=1e-3, s_traj=z(n + 1, 0, B))
    for kw in (dict(kp_bar=z(nv)), dict(kd_bar=z(nv, B + 1)), dict(q_ref_bar=z(n, nq, B)), dict(q0_bar_cfg=z(nq + 1, B)),
               dict(tau_bar=z(nv, B))):
        with pytest.raises(rbd.DimensionMismatch):
            rbd.integrate_pd_vjp_(mech, qt, vt, controller=ctl, dt=1e-3, **kw)
    with pytest.raises(TypeError):
        rbd.integrate_pd_vjp_(mech, qt, vt, controller=object(), dt=1e-3)
    with pytest.raises(TypeError):
        rbd.autodiff.simulate(mech, qt[0], vt[0], dt=1e-3, nsteps=n, controller=object())
    with pytest.raises(rbd.DimensionMismatch):
        rbd.autodiff.simulate(mech, qt[0], vt[0], dt=1e-3, nsteps=n, controller=rbd.JointPD(z(nv + 1), z(nv + 1), z(nq, B)))
    with pytest.raises(TypeError):
        rbd.autodiff.simulate(mech, qt[0], vt[0], dt=1e-3, nsteps=n, controller=rbd.JointPD(z(nv).float(), z(nv).float(), z(nq, B)))


# fp32 GPU backward against the fp64 CPU run of the same trajectory (upcast), relative, worst over all gradients.  Measured on an
# H100 80GB HBM3: PD 1.2e-4 (Atlas), 3.8e-3 (random tree), 2.6e-7 (double pendulum); computed torque 1.6e-3 (random tree), 1.5e-2
# (Atlas, its q_ref gradient: the feedback through Atlas' light links amplifies fp32 rounding).  Each bound is about 5x the largest
# error of its mode.
TOL32 = {"pd": 2e-2, "ct": 8e-2}


@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
@pytest.mark.parametrize("which,mode,per_step,per_sample,clamp,tau_kind", [
    ("atlas", "pd", 0, True, True, "const"), ("atlas", "ct", 3, False, True, "step"), ("randtree", "pd", 3, True, True, "stage"),
    ("randtree", "ct", 0, True, False, "none"), ("double_pendulum", "pd", 0, False, True, "step")])
def test_gpu_matches_cpu_run(built, dtype_name, which, mode, per_step, per_sample, clamp, tau_kind):
    """rbd_integrate_pd_vjp on the GPU against the CPU run of the same code on the same recorded trajectory: fp64 to 1e-10, fp32
    against the fp64 CPU run to TOL32."""
    import torch
    dtype = getattr(torch, dtype_name)
    mech = _cpu_model(which)
    d = mech.flatten()
    n, B, dt = 3, 37, 1e-3
    q, v, taus, ctrl, rng = _fd_case(mech, B, n, mode, per_step, per_sample, clamp, tau_kind, zlib.crc32(f"{which}{mode}".encode()))
    r32 = lambda a: None if a is None else a.astype(np.float32).astype(np.float64)     # noqa: E731
    if dtype == torch.float32:                     # fp32-representable inputs for the fp64 CPU run
        q, v, taus = r32(q), r32(v), r32(taus)
        ctrl.kp, ctrl.kd, ctrl.q_ref, ctrl.v_ref, ctrl.vd_ref = (r32(a) for a in (ctrl.kp, ctrl.kd, ctrl.q_ref, ctrl.v_ref, ctrl.vd_ref))
    T = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dtype).cuda()     # noqa: E731
    ctl = _torch_ctrl(ctrl, dtype)
    qt, vt, _ = _record(mech, T(q), T(v), T(taus), ctl, dt, n)
    wq, wv = r32(rng.standard_normal(q.shape)), r32(rng.standard_normal(v.shape))
    out = _direct(mech, qt, vt, T(taus), ctl, dt, T(wq), T(wv), B, d.nv)
    qtn, vtn = qt.double().cpu().numpy(), vt.double().cpu().numpy()
    qtb, vtb = np.zeros_like(qtn), np.zeros_like(vtn)
    qtb[-1], vtb[-1] = wq, wv
    h = host_pd_vjp(d, qtn, vtn, ctrl, taus, qtb, vtb, dt)
    pairs = (("q0_bar_cfg", "q0c"), ("v0_bar", "v0b"), ("tau_bar", "taub"), ("kp_bar", "kp"), ("kd_bar", "kd"), ("q_ref_bar", "q_ref"),
             ("v_ref_bar", "v_ref"), ("vd_ref_bar", "vd_ref"))
    worst = 0.0
    for g, c in pairs:
        if out[g] is None:
            continue
        e = rel_err(out[g].double().cpu().numpy(), h[c])
        worst = max(worst, e)
        assert e < (TOL64 if dtype == torch.float64 else TOL32[mode]), (g, e)
    print(f"{dtype_name} {which} {mode}: worst rel_err {worst:.2e}")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["pd", "ct"])
def test_gpu_gradcheck(built, mode):
    """torch.autograd.gradcheck in fp64 on a small revolute / prismatic tree with respect to q0, v0, τ_ff and every controller
    tensor, with clamps active on some rows, held 0.5 away from the bounds."""
    import torch
    rng = np.random.default_rng(11)
    mech = rbd.rand_tree_mechanism(rng, [rbd.Revolute, rbd.Prismatic, rbd.Revolute, rbd.Prismatic])
    d = mech.flatten()
    B, n, dt = 3, 3, 1e-2
    q, v, tau, _, _ = rand_inputs(mech, B, 6)
    ctrl = _controller(mech, q, rng, ct=mode == "ct", per_sample=True)
    u = ctrl.torque(Oracle(d), 0, q, v, tau)
    ctrl.bounds = (np.full(d.nv, -1e6), np.full(d.nv, 1e6))
    ctrl.bounds[1][0] = float(u[0].min()) - 0.5 * float(np.ptp(u[0]) + 1)        # row 0 saturated on every sample, with a margin
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda().requires_grad_(True)     # noqa: E731
    args = [T(q), T(v), T(tau), T(ctrl.kp), T(ctrl.kd), T(ctrl.q_ref), T(ctrl.v_ref)] + ([T(ctrl.vd_ref)] if mode == "ct" else [])

    def f(q0, v0, t, kp, kd, qr, vr, vdr=None):
        c = rbd.JointPD(kp, kd, qr, vr, vd_ref=vdr, computed_torque=mode == "ct", effort_bounds=ctrl.bounds)
        return rbd.autodiff.simulate(mech, q0, v0, t, dt=dt, nsteps=n, controller=c)
    assert torch.autograd.gradcheck(f, args, eps=1e-6, atol=1e-6, rtol=1e-5)
