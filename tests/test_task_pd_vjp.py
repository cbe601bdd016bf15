"""Reverse-mode gradients through task-space closed-loop rollouts (rbd_integrate_task_pd_vjp, DESIGN 4.22).

CPU tier: the law's adjoint (csrc/rbd_task_pd_adjoint.cuh's task_pd_vjp_column, compiled for the host by
tests/hostsim/hostsim_task_pd_vjp.cpp) against central differences of the host law (hostsim_task_pd_law), the task velocity ξ = J w
against TaskOracle's explicit Jacobians, and the argument checks of the C entry point and of the Python layer.
GPU tier: autodiff.simulate / simulate_contact with a TaskPD against central differences of the fp64 rollout, autograd against
the direct call across checkpoints, bit-identity with the JointPD and open-loop VJPs at zero task gains, a gradient-descent use
case and Atlas fp32 at 2^20."""
import ctypes
import functools
import zlib

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from rigidbodydynamics.jl_b200 import _cabi
from rigidbodydynamics.jl_b200._cabi import RbdModelDesc, make_desc
from rigidbodydynamics.jl_b200.kinematics import TaskFrame
from rigidbodydynamics.jl_b200.pd import _RbdTaskPdDesc
from tests import hostsim
from tests.task_oracle import TaskOracle
from tests.test_pd_rollout import _controller, _model
from tests.test_pd_vjp import _tangent
from tests.test_task_pd import TaskCtrl, _cpu_models, _gains, _rows, _task_struct, hostsim_task_law, targets, task_mix
from tests.util import rand_inputs


@functools.cache
def _shim():
    """tests/hostsim/hostsim_task_pd_vjp.cpp, compiled and loaded by hostsim.shim."""
    lib = hostsim.shim("hostsim_task_pd_vjp")
    vp = ctypes.c_void_p
    lib.hostsim_task_pd_law_vjp.argtypes = [ctypes.POINTER(RbdModelDesc), ctypes.POINTER(_RbdTaskPdDesc), ctypes.c_int, ctypes.c_int64,
                                            vp, vp, vp, vp, vp, vp, vp]
    return lib


BARS = ("kp", "kd", "x_ref", "xd_ref", "jkp", "jkd", "jq_ref", "jv_ref", "jvd_ref")


def hostsim_task_law_vjp(mech, tasks, kinds, q, v, w, kp, kd, xref, xdref=None, joint=None, ct=False):
    """The law's adjoint on the CPU (fp64): dict with q_cfg [nq, B], q_tan [nv, B], v [nv, B] and the bars of BARS (per sample for
    the gains)."""
    dt = np.float64
    c = lambda a: None if a is None else np.ascontiguousarray(a, dt)      # noqa: E731
    B = q.shape[1]
    arrays = tuple(c(a) for a in (kp, kd, xref, xdref))
    ja = None if joint is None else tuple(c(a) for a in (joint.kp, joint.kd, joint.q_ref, joint.v_ref, joint.vd_ref))
    d, keep = _task_struct(mech, tasks, kinds, ct, arrays, ja, None, gain_ld=B)
    q, v, w = c(q), c(v), c(w)
    nq, nv = q.shape[0], v.shape[0]
    R = kp.shape[0]
    srcs = list(arrays) + (list(ja) if ja is not None else [None] * 5)
    bars = [None if a is None else np.zeros(((a.shape[0], B) if i in (0, 1, 4, 5) else a.shape), dt) for i, a in enumerate(srcs)]
    out = dict(q_cfg=np.zeros((nq, B)), q_tan=np.zeros((nv, B)), v=np.zeros((nv, B)))
    p = lambda a: None if a is None else a.ctypes.data                    # noqa: E731
    pb = (ctypes.c_void_p * 9)(*[p(b) for b in bars])
    md, keep2 = make_desc(mech.flatten())
    rc = _shim().hostsim_task_pd_law_vjp(ctypes.byref(md), ctypes.byref(d), 1, B, p(q), p(v), p(w), p(out["q_cfg"]), p(out["q_tan"]),
                                         p(out["v"]), pb)
    assert rc == 0, rc
    assert R == bars[0].shape[0]
    out.update({k: b for k, b in zip(BARS, bars)})
    return out


def _targets(mech, q, tasks, kinds, rng, mode):
    """test_task_pd.targets, with the "near_pi" pose errors at angles in [pi - 2e-2, pi - 1e-2]: far enough from pi that a central
    difference does not cross the branch cut of the rotation log."""
    if mode != "near_pi":
        return targets(mech, q, tasks, kinds, rng, mode)
    from scipy.spatial.transform import Rotation
    xr = targets(mech, q, tasks, kinds, rng, "zero")
    B, x0 = q.shape[1], 0
    for k in kinds:
        if k == "pose":
            ax = rng.standard_normal((3, B))
            ax /= np.linalg.norm(ax, axis=0)
            d = Rotation.from_rotvec((ax * (np.pi - 1e-2 * (1 + rng.random(B)))).T).as_matrix().transpose(1, 2, 0)
            Rx = xr[x0:x0 + 9].reshape(3, 3, B)
            xr[x0:x0 + 9] = np.einsum("ijb,jkb->ikb", Rx, d).reshape(9, B)
        x0 += _rows(k)[1]
    return xr


def _law_case(which, seed, mode, ct, with_joint, per_sample):
    mech = dict(_cpu_models())[which]
    rng = np.random.default_rng(seed)
    B = 5
    q, v, _, _, _ = rand_inputs(mech, B, seed % 1000)
    tasks, kinds = task_mix(mech, seed % 97)
    R = sum(_rows(k)[0] for k in kinds)
    xref = _targets(mech, q, tasks, kinds, rng, mode)
    xdref = rng.standard_normal((R, B))
    kp, kd = _gains(rng, kinds, B, per_sample=per_sample)
    joint = _controller(mech, q, rng, ct=ct, per_sample=per_sample) if with_joint else None
    return mech, rng, q, v, tasks, kinds, kp, kd, xref, xdref, joint


@pytest.mark.parametrize("mode", ["random", "near_pi", "zero"])
@pytest.mark.parametrize("ct,with_joint,per_sample", [(False, False, False), (False, True, True), (True, False, True), (True, True, False)])
@pytest.mark.parametrize("which", ["atlas", "valkyrie", "iiwa14", "double_pendulum", "randmech0", "randmech1", "randmech2", "randmech3"])
def test_law_adjoint_matches_central_differences(which, mode, ct, with_joint, per_sample):
    """w . law(q, v; ...) differentiated by task_pd_vjp_column against central differences of the host law along a tangent direction
    of q, unit directions of v, and random directions of every gain, reference and joint-term array."""
    seed = zlib.crc32(f"{which}{mode}{ct}{with_joint}".encode())
    mech, rng, q, v, tasks, kinds, kp, kd, xref, xdref, joint = _law_case(which, seed, mode, ct, with_joint, per_sample)
    nv, B = v.shape
    w = rng.standard_normal((nv, B))
    g = hostsim_task_law_vjp(mech, tasks, kinds, q, v, w, kp, kd, xref, xdref, joint, ct)
    base = dict(q=q, v=v, kp=kp, kd=kd, x_ref=xref, xd_ref=xdref)
    if joint is not None:
        base.update(jkp=joint.kp, jkd=joint.kd, jq_ref=joint.q_ref, jv_ref=joint.v_ref, jvd_ref=joint.vd_ref)

    def L(x):
        jt = None
        if joint is not None:
            jt = type(joint)(x["jkp"], x["jkd"], x["jq_ref"], x["jv_ref"], x["jvd_ref"], ct)
        u = hostsim_task_law(mech, tasks, kinds, x["q"], x["v"], x["kp"], x["kd"], x["x_ref"], x["xd_ref"], None, jt, ct)
        return float((w * u).sum())

    grads = dict(q=g["q_cfg"], v=g["v"], **{k: g[k] for k in BARS if k in base})
    eps = 1e-6
    dirs = []
    for k in base:
        if base[k] is None:
            continue
        if k == "v":
            for j in range(nv):
                d = np.zeros_like(v)
                d[j] = 1.0
                dirs.append((k, d))
            continue
        d = rng.standard_normal(np.shape(base[k]))
        if k == "q":
            d = _tangent(mech, q, d)
        if k == "jq_ref":
            d = _tangent(mech, joint.q_ref, d)
        dirs.append((k, d))
    for k, d in dirs:
        xp, xm = dict(base), dict(base)
        xp[k] = base[k] + eps * d
        xm[k] = base[k] - eps * d
        fd = (L(xp) - L(xm)) / (2 * eps)
        gk = grads[k]
        if gk.shape != d.shape:       # shared gains: per-sample bars summed over the batch
            gk = gk.sum(1)
        ad = float((gk * d).sum())
        assert abs(fd - ad) <= 1e-6 * max(1.0, abs(fd)), (k, fd, ad)
    assert np.isfinite(g["q_tan"]).all()


@pytest.mark.parametrize("which", ["atlas", "iiwa14", "randmech1", "randmech3"])
def test_task_velocity_is_jacobian_times_w(which):
    """With Kp = 0, Kd = 1 on one task and no references, K̄d = -ξ ė per row, so -K̄d / ė recovers ξ = J w; checked against the
    explicit point and geometric Jacobians of TaskOracle to 1e-12."""
    mech = dict(_cpu_models())[which]
    seed = zlib.crc32(which.encode())
    rng = np.random.default_rng(seed)
    B = 4
    q, v, _, _, _ = rand_inputs(mech, B, seed % 1000)
    tasks, kinds = task_mix(mech, seed % 97)
    nv = v.shape[0]
    w = rng.standard_normal((nv, B))
    to = TaskOracle(mech, q)
    for t, k in zip(tasks, kinds):
        R = _rows(k)[0]
        xref = targets(mech, q, [t], [k], rng)
        kp, kd = np.zeros((R, B)), np.ones((R, B))
        g = hostsim_task_law_vjp(mech, [t], [k], q, v, w, kp, kd, xref, None)
        frame = t.body if k == "pose" else t.frame
        out = to.task(TaskFrame(t.body, t.base, t.point, frame))
        if k == "point":
            J = out["point_jacobian"].reshape(nv, 3, B)
            xi = np.einsum("kcb,kb->cb", J, w)
        else:
            Jg = out["geometric_jacobian"].reshape(nv, 6, B)
            Jp = to.task(TaskFrame(t.body, t.base, t.point, t.body))["point_jacobian"].reshape(nv, 3, B)
            xi = np.concatenate([np.einsum("kcb,kb->cb", Jg[:, :3], w), np.einsum("kcb,kb->cb", Jp, w)])
        ed = _task_rate(mech, t, k, q, v)
        np.testing.assert_allclose(g["kd"], -xi * ed, rtol=0, atol=1e-12 * max(1.0, np.abs(xi * ed).max()))


def _task_rate(mech, t, k, q, v):
    """ė of one task with ẋ_ref = 0: point velocity in F (point task) or twist of C in C (pose task), from TaskOracle."""
    to = TaskOracle(mech, q, v)
    if k == "point":
        return to.task(TaskFrame(t.body, t.base, t.point, t.frame))["point_velocity"]
    tw = to.task(TaskFrame(t.body, t.base, t.point, t.body))
    return np.concatenate([tw["twist"][:3], tw["point_velocity"]])


# ------------------------------------------------------------------------------------------------------------------
# C-ABI and Python argument checks (host only, nothing launched)
# ------------------------------------------------------------------------------------------------------------------
def test_integrate_task_pd_vjp_argument_checks(built):
    from rigidbodydynamics.jl_b200.kinematics import task_desc
    from rigidbodydynamics.jl_b200.pd import _RbdPdBar, _RbdPdDesc, _RbdTaskPdBar
    from tests.test_loops_rollout import atlas_on_floor
    lib = rbd.load_library()
    mech = rbd.load_model("iiwa14")
    h = _cabi.ModelHandle(mech.flatten())
    fake = 64                                         # never dereferenced by the checks below
    nv = mech.num_velocities()
    hand = mech.joints[-1].successor
    td, keep_t = task_desc(mech, [TaskFrame(hand, None, None)])
    kind = np.zeros(1, np.int32)
    lo_ok, hi_ok = (np.ascontiguousarray(b) for b in rbd.effort_bounds(mech))
    dp = ctypes.POINTER(ctypes.c_double)

    def joint(**kw):
        f = dict(mode=0, kp=fake, kd=fake, gain_ld=0, q_ref=fake, v_ref=None, vd_ref=None, q_ref_step_stride=0, v_ref_step_stride=0,
                 effort_lo=None, effort_hi=None)
        f.update(kw)
        return _RbdPdDesc(**f)

    def desc(j=None, **kw):
        f = dict(mode=0, tasks=td, kind=kind.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), kp=fake, kd=fake, gain_ld=0, x_ref=fake,
                 x_ref_step_stride=0, xd_ref=None, xd_ref_step_stride=0, joint=None if j is None else ctypes.pointer(j),
                 effort_lo=lo_ok.ctypes.data_as(dp), effort_hi=hi_ok.ctypes.data_as(dp))
        f.update(kw)
        return _RbdTaskPdDesc(**f)

    def call(c, dtype=_cabi.RBD_F64, B=4, stage=0, dt=1e-3, n=1, handle=h, contact=None, tau=fake, tau_bar=None, bar=None,
             traj=(fake, fake)):
        return lib.rbd_integrate_task_pd_vjp(handle.ptr, dtype, B, *traj, None, tau, 0, stage, None if c is None else ctypes.byref(c),
                                             contact, dt, n, None, None, None, None, None, None, None, tau_bar,
                                             None if bar is None else ctypes.byref(bar), None)

    def status(rc, text=None, want=_cabi.RBD_EINVAL):
        assert rc == want, rc
        if text:
            assert text.encode() in lib.rbd_last_error(), lib.rbd_last_error()
    status(call(None), "ctrl must not be NULL")
    status(call(desc(mode=3)), "unknown mode")
    status(call(desc(kp=None)), "must not be NULL")
    status(call(desc(x_ref=None)), "must not be NULL")
    status(call(desc(gain_ld=3)), "gain_ld")
    status(call(desc(x_ref_step_stride=-1)), "strides")
    status(call(desc(effort_hi=None)), "both")
    bad_lo = lo_ok.copy()
    bad_lo[2] = 1e9
    status(call(desc(effort_lo=bad_lo.ctypes.data_as(dp))), "lo <= hi")
    status(call(desc(joint(kp=None))), "joint term")
    status(call(desc(joint(mode=1))), "mode")
    status(call(desc(joint(effort_lo=lo_ok.ctypes.data_as(dp), effort_hi=hi_ok.ctypes.data_as(dp)))), "effort bounds")
    status(call(desc(), n=-1))
    status(call(desc(), dt=0.0))
    status(call(desc(), stage=-1), "strides")
    status(call(desc(), tau=None, tau_bar=fake), "tau_bar needs tau")
    status(call(desc(), traj=(None, fake)), "must not be NULL")
    # adjoints of arrays the controller does not have
    status(call(desc(), bar=_RbdTaskPdBar(None, None, None, fake, None)), "xd_ref")
    jb = _RbdPdBar(None, None, None, fake, None)
    status(call(desc(), bar=_RbdTaskPdBar(None, None, None, None, ctypes.pointer(jb))), "joint")
    status(call(desc(joint()), bar=_RbdTaskPdBar(None, None, None, None, ctypes.pointer(jb))), "v_ref")
    assert call(desc(), dtype=_cabi.RBD_DUAL64X6) == _cabi.RBD_EUNSUPPORTED
    assert call(desc(), B=0) == _cabi.RBD_OK                              # empty batch: nothing to do
    # contact: s_traj with contact pairs
    am, cd = atlas_on_floor()
    ha = _cabi.ModelHandle(am.flatten())
    cst, keep = cd.c_struct()
    tda, keep_a = task_desc(am, [TaskFrame(am.joints[0].successor, None, None)])
    status(call(desc(tasks=tda, effort_lo=None, effort_hi=None), handle=ha, contact=ctypes.byref(cst)), "s_traj must not be NULL")
    for x in (h, ha):
        x.close()


def test_python_checks():
    """autodiff.simulate: a controller that is neither a JointPD nor a TaskPD is a TypeError; loops are refused with RBD_ELOOP;
    integrate_task_pd_vjp_ refuses anything but a TaskPD."""
    import torch
    from tests.loops_oracle import four_bar
    fb = four_bar()
    z = torch.zeros(1, 1, dtype=torch.float64)
    with pytest.raises(TypeError):
        rbd.autodiff.simulate(rbd.load_model("double_pendulum"), torch.zeros(2, 1, dtype=torch.float64),
                              torch.zeros(2, 1, dtype=torch.float64), dt=1e-3, nsteps=1, controller=object())
    ctl = rbd.TaskPD([TaskFrame(fb.joints[-1].successor, None, None)], ["point"], z, z, z)
    with pytest.raises(_cabi.RbdError) as ei:
        rbd.autodiff.simulate(fb, z, z, dt=1e-3, nsteps=1, controller=ctl)
    assert ei.value.status == _cabi.RBD_ELOOP
    with pytest.raises(_cabi.RbdError) as ei:
        rbd.autodiff.integrate_task_pd_vjp_(fb, z[None], z[None], controller=ctl, dt=1e-3)
    assert ei.value.status == _cabi.RBD_ELOOP
    m = rbd.load_model("double_pendulum")
    with pytest.raises(TypeError):
        rbd.autodiff.integrate_task_pd_vjp_(m, torch.zeros(2, 2, 1, dtype=torch.float64), torch.zeros(2, 2, 1, dtype=torch.float64),
                                            controller=rbd.JointPD(z, z, z), dt=1e-3)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def _torch(a, dtype, grad=False):
    import torch
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dtype).cuda().requires_grad_(grad)


def _rollout_case(which, B, nsteps, ct, with_joint, per_step, per_sample, clamp, seed):
    """Inputs of one task-space rollout in numpy: (mech, q, v, tau, tasks, kinds, arrays dict, bounds, rng)."""
    mech = _model(which)
    rng = np.random.default_rng(seed)
    q, v, tau, _, _ = rand_inputs(mech, B, seed % 97)
    v *= 0.3
    tasks, kinds = task_mix(mech, seed % 89, npoint=3)
    R = sum(_rows(k)[0] for k in kinds)
    xr = lambda: _targets(mech, q, tasks, kinds, rng, "random")          # noqa: E731
    x_ref = np.stack([xr() for _ in range(nsteps)]) if per_step else xr()
    xd_ref = rng.standard_normal((nsteps, R, B) if per_step else (R, B)) * 0.3
    kp, kd = _gains(rng, kinds, B, per_sample, scale=0.5)
    arrays = dict(kp=kp, kd=kd, x_ref=x_ref, xd_ref=xd_ref)
    if with_joint:
        j = _controller(mech, q, rng, ct=ct, per_step=nsteps if per_step else 0, per_sample=per_sample, scale=0.2)
        arrays.update(jkp=j.kp, jkd=j.kd, jq_ref=j.q_ref, jv_ref=j.v_ref, jvd_ref=j.vd_ref)
    bounds = None
    if clamp:
        lim = rng.uniform(20, 60, v.shape[0])
        bounds = (-lim, lim)
    return mech, q, v, tau, tasks, kinds, arrays, bounds, rng


def _task_pd(tasks, kinds, t, ct, bounds):
    j = None
    if "jkp" in t:
        j = rbd.JointPD(t["jkp"], t["jkd"], t["jq_ref"], t.get("jv_ref"), vd_ref=t.get("jvd_ref"), computed_torque=ct)
    return rbd.TaskPD(tasks, kinds, t["kp"], t["kd"], t["x_ref"], t.get("xd_ref"), joint=j, computed_torque=ct, effort_bounds=bounds)


def _check_fd(mech, q, v, tau, tasks, kinds, arrays, bounds, ct, rng, nsteps, dt=1e-3, contact=None, s0=None, eps=1e-5, tol=1e-6):
    """autodiff.simulate(_contact) with a TaskPD: autograd against central differences of the fp64 GPU rollout along random directions
    of every input."""
    import torch
    f64 = torch.float64
    base = dict(q0=q, v0=v, tau=tau, s0=s0, **arrays)
    names = [k for k in base if base[k] is not None]
    wq, wv = rng.standard_normal(q.shape), rng.standard_normal(v.shape)
    ws = None if contact is None else rng.standard_normal(s0.shape)

    def run(x, grad=False):
        t = {k: _torch(x[k], f64, grad) for k in names}
        ctl = _task_pd(tasks, kinds, t, ct, bounds)
        if contact is None:
            out = rbd.autodiff.simulate(mech, t["q0"], t["v0"], t.get("tau"), dt=dt, nsteps=nsteps, trajectory=False, controller=ctl)
        else:
            out = rbd.autodiff.simulate_contact(mech, t["q0"], t["v0"], t["s0"], t.get("tau"), contact=contact, dt=dt, nsteps=nsteps,
                                                trajectory=False, controller=ctl)
        L = (out[0] * _torch(wq, f64)).sum() + (out[1] * _torch(wv, f64)).sum() + (0 if contact is None else (out[2] * _torch(ws, f64)).sum())
        if grad:
            L.backward()
            return {k: t[k].grad.cpu().numpy() for k in names}
        return float(L)
    g = run(base, grad=True)
    for k in names:
        d = rng.standard_normal(np.shape(base[k]))
        if k == "q0":
            d = _tangent(mech, q, d)
        if k == "jq_ref":
            d = _tangent(mech, base[k], d) if base[k].ndim == 2 else np.stack([_tangent(mech, r, dd) for r, dd in zip(base[k], d)])
        xp, xm = dict(base), dict(base)
        xp[k] = base[k] + eps * d
        xm[k] = base[k] - eps * d
        fd = (run(xp) - run(xm)) / (2 * eps)
        ad = float((g[k] * d).sum())
        print(f"{k}: fd {fd:.10e} ad {ad:.10e}")
        assert abs(fd - ad) <= tol * max(1.0, abs(fd)), (k, fd, ad)


@pytest.mark.gpu
@pytest.mark.parametrize("which,ct,with_joint,per_step,per_sample,clamp,nsteps", [
    ("atlas", False, True, False, False, True, 5), ("atlas", True, True, True, True, False, 5), ("atlas", False, False, True, True, False, 1),
    ("iiwa14", True, False, False, False, True, 5), ("valkyrie", False, True, True, False, False, 5),
    ("randmech1", False, True, False, True, True, 3), ("randmech2", True, True, False, False, True, 3),
    ("double_pendulum", False, False, False, True, False, 5)])
def test_gpu_gradients_match_central_differences(built, which, ct, with_joint, per_step, per_sample, clamp, nsteps):
    seed = zlib.crc32(f"{which}{ct}{with_joint}{per_step}".encode())
    mech, q, v, tau, tasks, kinds, arrays, bounds, rng = _rollout_case(which, 5, nsteps, ct, with_joint, per_step, per_sample, clamp, seed)
    _check_fd(mech, q, v, tau, tasks, kinds, arrays, bounds, ct, rng, nsteps)


@pytest.mark.gpu
@pytest.mark.parametrize("ct", [False, True])
def test_gpu_contact_gradients_match_central_differences(built, ct):
    """Atlas standing on the floor with a pelvis pose task and a damping joint term."""
    from tests.test_loops_rollout import atlas_on_floor, atlas_states
    mech, cd = atlas_on_floor()
    B, n = 3, 4
    q, v, tau = atlas_states(mech, B, 3)
    rng = np.random.default_rng(7)
    pelvis = mech.joints[0].successor
    tasks, kinds = [TaskFrame(pelvis, None, None)], ["pose"]
    x_ref = _targets(mech, q, tasks, kinds, rng, "random")
    nv = v.shape[0]
    arrays = dict(kp=np.full(6, 40.0), kd=np.full(6, 5.0), x_ref=x_ref, xd_ref=None, jkp=np.zeros(nv), jkd=np.full(nv, 2.0),
                  jq_ref=q.copy(), jv_ref=None, jvd_ref=None)
    s0 = rng.standard_normal((cd.nstates, B)) * 1e-3
    _check_fd(mech, q, v, tau, tasks, kinds, arrays, None, ct, rng, n, contact=cd, s0=s0)


def _direct(mech, qt, vt, tau, ctl, dt, gq, gv, contact=None, st=None, gs=None):
    """integrate_task_pd_vjp_ on a recorded trajectory with cotangents on the final state: every output."""
    import torch
    qtb, vtb = torch.zeros_like(qt), torch.zeros_like(vt)
    qtb[-1] = gq; vtb[-1] = gv
    stb = None
    if st is not None:
        stb = torch.zeros_like(st)
        stb[-1] = gs
    B = qt.shape[2]
    R, _ = ctl.rows()
    z = lambda t: None if t is None else torch.zeros_like(t)     # noqa: E731
    out = dict(q0_bar_cfg=torch.empty_like(qt[0]), v0_bar=torch.empty_like(vt[0]), tau_bar=z(tau),
               kp_bar=qt.new_zeros((R, B)), kd_bar=qt.new_zeros((R, B)), x_ref_bar=z(ctl.x_ref), xd_ref_bar=z(ctl.xd_ref))
    if st is not None:
        out["s0_bar"] = torch.empty_like(st[0])
    j = ctl.joint
    jb = None if j is None else [qt.new_zeros(vt[0].shape), qt.new_zeros(vt[0].shape), z(j.q_ref), z(j.v_ref), z(j.vd_ref)]
    rbd.autodiff.integrate_task_pd_vjp_(mech, qt, vt, tau, controller=ctl, dt=dt, contact=contact, s_traj=st, q_traj_bar=qtb,
                                        v_traj_bar=vtb, s_traj_bar=stb, joint_bars=jb, **out)
    if jb is not None:
        out.update(jkp_bar=jb[0], jkd_bar=jb[1], jq_ref_bar=jb[2], jv_ref_bar=jb[3], jvd_ref_bar=jb[4])
    return out


def _record(mech, q, v, tau, ctl, dt, n, contact=None, s=None):
    if contact is None:
        qt, vt = rbd.simulate_trajectory_(rbd_state(mech, q, v), n, tau, dt, controller=ctl)
        return qt, vt, None
    return rbd.simulate_contact_trajectory_(rbd_state(mech, q, v), n, s, tau, dt, contact, controller=ctl)


def rbd_state(mech, q, v):
    st = rbd.MechanismState(mech, q.shape[1], q.dtype)
    st.q.copy_(q)
    st.v.copy_(v)
    return st


@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
def test_gpu_zero_task_gains_bit_identical(built, dtype_name):
    """Kp = Kd = 0 on every task, no bounds: with a joint term the state, torque and joint-term gradients are bit-identical to
    rbd_integrate_pd_vjp's with that JointPD; without one (torque mode) to rbd_integrate_vjp's / rbd_integrate_contact_vjp's."""
    import torch
    from tests.test_loops_rollout import atlas_on_floor, atlas_states
    from tests.test_pd_vjp import _direct as pd_direct
    dtype = getattr(torch, dtype_name)
    T = lambda a: _torch(a, dtype)     # noqa: E731
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
            tasks, kinds = task_mix(mech, 5, npoint=3)
            R = sum(_rows(k)[0] for k in kinds)
            taus = T(tau[None, None] * rng.uniform(0.5, 1.5, (n, 4, 1, 1)))
            x_ref = T(_targets(mech, q, tasks, kinds, rng, "random"))
            zR = torch.zeros(R, dtype=dtype, device="cuda")
            gq, gv = T(rng.standard_normal(q.shape)), T(rng.standard_normal(v.shape))
            gs = None if cd is None else T(rng.standard_normal(s.shape))
            for ct in ((False, True) if which == "tree" else (False,)):
                joint = rbd.JointPD(T(rng.uniform(5, 20, nv)), T(rng.uniform(0.5, 2, nv)), T(q) + 0.1, T(v) * 0 + 0.5,
                                    vd_ref=T(v) * 0 + 0.1 if ct else None, computed_torque=ct)
                for jt in (joint, None):
                    if jt is None and ct:
                        continue
                    ctl = rbd.TaskPD(tasks, kinds, zR, zR, x_ref, joint=jt, computed_torque=ct)
                    qt, vt, st = _record(mech, T(q), T(v), taus, ctl, dt, n, cd, s)
                    out = _direct(mech, qt, vt, taus, ctl, dt, gq, gv, cd, st, gs)
                    if jt is not None:
                        ref = pd_direct(mech, qt, vt, taus, jt, dt, gq, gv, B, nv, cd, st, gs)
                        for k in ("kp_bar", "kd_bar", "q_ref_bar", "v_ref_bar"):
                            assert torch.equal(out["j" + k], ref[k]), (which, B, ct, k)
                    else:
                        ref = {}
                        qtb, vtb = torch.zeros_like(qt), torch.zeros_like(vt)
                        qtb[-1] = gq; vtb[-1] = gv
                        ref = dict(q0_bar_cfg=torch.empty_like(qt[0]), v0_bar=torch.empty_like(vt[0]), tau_bar=torch.zeros_like(taus))
                        if cd is None:
                            rbd.integrate_vjp_(mech, qt, vt, taus, dt=dt, q_traj_bar=qtb, v_traj_bar=vtb, **ref)
                        else:
                            stb = torch.zeros_like(st)
                            stb[-1] = gs
                            ref["s0_bar"] = torch.empty_like(st[0])
                            rbd.integrate_contact_vjp_(mech, qt, vt, st, taus, contact=cd, dt=dt, q_traj_bar=qtb, v_traj_bar=vtb,
                                                       s_traj_bar=stb, **ref)
                    for k in ("q0_bar_cfg", "v0_bar", "tau_bar") + (("s0_bar",) if cd is not None else ()):
                        assert torch.equal(out[k], ref[k]), (which, B, ct, jt is None, k)
                    assert bool(out["kp_bar"].abs().sum() > 0)


@pytest.mark.gpu
@pytest.mark.parametrize("ct", [False, True])
def test_gpu_autograd_equals_direct_and_checkpoints(built, ct):
    """autodiff.simulate with a TaskPD: the gradients of trajectory=True, and of trajectory=False with checkpoint_every in {1, 3,
    nsteps}, are bit-identical to the direct call on the recorded trajectory."""
    import torch
    f64 = torch.float64
    n, dt = 7, 1e-3
    mech, q, v, tau, tasks, kinds, arrays, bounds, rng = _rollout_case("atlas", 64, n, ct, True, True, True, True, 11)
    gq, gv = _torch(rng.standard_normal(q.shape), f64), _torch(rng.standard_normal(v.shape), f64)
    t = {k: _torch(a, f64) for k, a in arrays.items()}
    ctl = _task_pd(tasks, kinds, t, ct, bounds)
    qt, vt, _ = _record(mech, _torch(q, f64), _torch(v, f64), _torch(tau, f64), ctl, dt, n)
    ref = _direct(mech, qt, vt, _torch(tau, f64), ctl, dt, gq, gv)
    names = ["q0", "v0", "tau"] + list(arrays)
    refk = dict(q0="q0_bar_cfg", v0="v0_bar", tau="tau_bar", kp="kp_bar", kd="kd_bar", x_ref="x_ref_bar", xd_ref="xd_ref_bar",
                jkp="jkp_bar", jkd="jkd_bar", jq_ref="jq_ref_bar", jv_ref="jv_ref_bar", jvd_ref="jvd_ref_bar")
    for every in (None, 1, 3, n):
        x = {k: _torch(a, f64, True) for k, a in dict(q0=q, v0=v, tau=tau, **arrays).items() if a is not None}
        c = _task_pd(tasks, kinds, x, ct, bounds)
        out = rbd.autodiff.simulate(mech, x["q0"], x["v0"], x["tau"], dt=dt, nsteps=n, trajectory=every is None,
                                    checkpoint_every=every, controller=c)
        qn, vn = (out[0][-1], out[1][-1]) if every is None else out
        ((qn * gq).sum() + (vn * gv).sum()).backward()
        for k in names:
            if k in x:
                assert torch.equal(x[k].grad, ref[refk[k]]), (every, k)


@pytest.mark.gpu
def test_gpu_gradient_descent_on_hand_target(built):
    """iiwa14 under a point task on its last link: a few gradient steps on x_ref bring the hand to a goal point at the end of the
    rollout -- the loss falls below a quarter of its start."""
    import torch
    mech = rbd.load_model("iiwa14")
    f64 = torch.float64
    B, n, dt = 4, 150, 2e-3
    nv = mech.num_velocities()
    q0 = torch.zeros(nv, B, dtype=f64, device="cuda")
    v0 = torch.zeros_like(q0)
    hand = mech.joints[-1].successor
    task = TaskFrame(hand, None, np.array([0.0, 0.0, 0.1]))
    to = TaskOracle(mech, q0.cpu().numpy())
    start = to.task(task)["point"]
    goal = torch.from_numpy(start + np.array([[0.1], [0.05], [-0.1]])).to(f64).cuda()
    xref = goal.clone().contiguous().requires_grad_()
    st = rbd.MechanismState(mech, B, f64)
    st.q.copy_(q0)
    M = rbd.mass_matrix(st).view(nv, nv, B)[:, :, 0]
    eff = 1.0 / torch.linalg.inv(M).diagonal()          # posture and damping at 5 rad/s on each joint's effective inertia
    joint = rbd.JointPD((25.0 * eff).contiguous(), (10.0 * eff).contiguous(), q0.clone())
    kp, kd = torch.full((3,), 300.0, dtype=f64, device="cuda"), torch.full((3,), 30.0, dtype=f64, device="cuda")
    losses = []
    for it in range(8):
        ctl = rbd.TaskPD([task], ["point"], kp, kd, xref, joint=joint)
        qn, vn = rbd.autodiff.simulate(mech, q0, v0, dt=dt, nsteps=n, trajectory=False, checkpoint_every=50, controller=ctl)
        hand_pt = rbd.autodiff.task_kinematics(mech, qn, tasks=[task], outputs=("point",))["point"]
        loss = ((hand_pt - goal) ** 2).sum()
        losses.append(float(loss))
        xref.grad = None
        loss.backward()
        with torch.no_grad():
            xref -= 0.5 * xref.grad
    print(losses)
    assert losses[-1] < 0.25 * losses[0]


@pytest.mark.gpu
@pytest.mark.parametrize("ct", [False, True])
def test_gpu_at_scale(built, ct):
    """Atlas fp32 at B = 2^20, 3 steps, both hands as point tasks and both feet as pose tasks with a damping joint term: finite
    gradients, and the workspace fits beside the trajectories."""
    import torch
    mech = rbd.load_model("atlas", floating=True)
    B, n, dt = 1 << 20, 3, 1e-3
    f32 = torch.float32
    q, v, tau, _, _ = rand_inputs(mech, 1024, 5)
    rep = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(f32).cuda().repeat(1, B // 1024)   # noqa: E731
    f = mech.findbody
    tasks = [TaskFrame(f("l_hand"), None, np.array([0.0, 0.1, 0.0])), TaskFrame(f("r_hand"), None, np.array([0.0, -0.1, 0.0])),
             TaskFrame(f("l_foot"), None, None), TaskFrame(f("r_foot"), None, None)]
    kinds = ["point", "point", "pose", "pose"]
    x_ref = targets(mech, q, tasks, kinds, np.random.default_rng(2))
    nv = v.shape[0]
    joint = rbd.JointPD(torch.zeros(nv, dtype=f32, device="cuda"), torch.full((nv,), 2.0, dtype=f32, device="cuda"), rep(q),
                        computed_torque=ct)
    kp, kd = torch.full((18,), 50.0, dtype=f32, device="cuda"), torch.full((18,), 5.0, dtype=f32, device="cuda")
    ctl = rbd.TaskPD(tasks, kinds, kp, kd, rep(x_ref), joint=joint, computed_torque=ct, effort_bounds=rbd.effort_bounds(mech))
    qt, vt, _ = _record(mech, rep(q), rep(v) * 0.3, rep(tau), ctl, dt, n)
    out = _direct(mech, qt, vt, rep(tau), ctl, dt, torch.ones_like(qt[0]), torch.zeros_like(vt[0]))
    for k, t in out.items():
        assert t is None or bool(torch.isfinite(t).all()), k


# ------------------------------------------------------------------------------------------------------------------
# the law at one state: rbd_task_pd_torques_vjp, autodiff.task_pd_torques
# ------------------------------------------------------------------------------------------------------------------
def test_law_adjoint_with_feedforward_and_active_clamps():
    """Torque mode with a joint term, τ_ff and effort bounds active on some rows (every torque held at least 1e-3 away from its
    bound): the masked cotangent m = w 1[lo < τ < hi] through the law's adjoint, and τ̄_ff = m, against central differences of the
    clamped host law along every input, τ_ff included."""
    mech, rng, q, v, tasks, kinds, kp, kd, xref, xdref, joint = _law_case("atlas", 5, "random", False, True, True)
    nv, B = v.shape
    tau = rng.standard_normal((nv, B)) * 5
    u = hostsim_task_law(mech, tasks, kinds, q, v, kp, kd, xref, xdref, tau, joint, False)
    lo, hi = -np.abs(u).mean(1) * 0.5, np.abs(u).mean(1) * 0.4
    gap = np.minimum(np.abs(u - lo[:, None]), np.abs(u - hi[:, None]))
    lo, hi = np.where(gap.min(1) < 1e-3, lo - 1e-2, lo), np.where(gap.min(1) < 1e-3, hi + 1e-2, hi)
    inside = (u > lo[:, None]) & (u < hi[:, None])
    assert inside.any() and (~inside).any()
    w = rng.standard_normal((nv, B))
    m = w * inside
    g = hostsim_task_law_vjp(mech, tasks, kinds, q, v, m, kp, kd, xref, xdref, joint, False)
    base = dict(q=q, v=v, tau=tau, kp=kp, kd=kd, x_ref=xref, xd_ref=xdref, jkp=joint.kp, jkd=joint.kd, jq_ref=joint.q_ref,
                jv_ref=joint.v_ref)
    grads = dict(q=g["q_cfg"], v=g["v"], tau=m, **{k: g[k] for k in BARS if k in base})

    def L(x):
        jt = type(joint)(x["jkp"], x["jkd"], x["jq_ref"], x["jv_ref"], None, False)
        uu = hostsim_task_law(mech, tasks, kinds, x["q"], x["v"], x["kp"], x["kd"], x["x_ref"], x["xd_ref"], x["tau"], jt, False,
                              (lo, hi))
        return float((w * uu).sum())
    eps = 1e-6
    for k in base:
        d = rng.standard_normal(np.shape(base[k]))
        if k in ("q", "jq_ref"):
            d = _tangent(mech, base[k], d)
        xp, xm = dict(base), dict(base)
        xp[k], xm[k] = base[k] + eps * d, base[k] - eps * d
        fd = (L(xp) - L(xm)) / (2 * eps)
        gk = grads[k] if grads[k].shape == d.shape else grads[k].sum(1)
        ad = float((gk * d).sum())
        assert abs(fd - ad) <= 1e-6 * max(1.0, abs(fd)), (k, fd, ad)


def test_task_pd_torques_vjp_argument_checks(built):
    from rigidbodydynamics.jl_b200.kinematics import task_desc
    from rigidbodydynamics.jl_b200.pd import _RbdPdBar, _RbdPdDesc, _RbdTaskPdBar
    lib = rbd.load_library()
    mech = rbd.load_model("iiwa14")
    h = _cabi.ModelHandle(mech.flatten())
    fake = 64
    td, keep_t = task_desc(mech, [TaskFrame(mech.joints[-1].successor, None, None)])
    kind = np.zeros(1, np.int32)

    def desc(j=None, **kw):
        f = dict(mode=0, tasks=td, kind=kind.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), kp=fake, kd=fake, gain_ld=0, x_ref=fake,
                 x_ref_step_stride=0, xd_ref=None, xd_ref_step_stride=0, joint=None if j is None else ctypes.pointer(j),
                 effort_lo=None, effort_hi=None)
        f.update(kw)
        return _RbdTaskPdDesc(**f)

    def call(c, dtype=_cabi.RBD_F64, B=4, step=0, tau=fake, tau_bar=None, taub_out=fake, bar=None, q=fake):
        return lib.rbd_task_pd_torques_vjp(h.ptr, dtype, B, q, fake, tau, None if c is None else ctypes.byref(c), step, taub_out,
                                           None, None, None, tau_bar, None if bar is None else ctypes.byref(bar), None)

    def status(rc, text=None, want=_cabi.RBD_EINVAL):
        assert rc == want, rc
        if text:
            assert text.encode() in lib.rbd_last_error(), lib.rbd_last_error()
    status(call(None), "ctrl must not be NULL")
    status(call(desc(mode=3)), "unknown mode")
    status(call(desc(x_ref=None)), "must not be NULL")
    status(call(desc(gain_ld=3)), "gain_ld")
    status(call(desc(), step=-1), "step")
    status(call(desc(), tau=None, tau_bar=fake), "tau_ff_bar needs tau_ff")
    status(call(desc(), taub_out=None), "must not be NULL")
    status(call(desc(), q=None), "must not be NULL")
    status(call(desc(), bar=_RbdTaskPdBar(None, None, None, fake, None)), "xd_ref")
    jb = _RbdPdBar(None, None, None, None, fake)
    status(call(desc(), bar=_RbdTaskPdBar(None, None, None, None, ctypes.pointer(jb))), "joint")
    j = _RbdPdDesc(0, fake, fake, 0, fake, None, None, 0, 0, None, None)
    status(call(desc(j), bar=_RbdTaskPdBar(None, None, None, None, ctypes.pointer(jb))), "vd_ref")
    status(call(desc(_RbdPdDesc(1, fake, fake, 0, fake, None, None, 0, 0, None, None))), "mode")
    assert call(desc(), dtype=_cabi.RBD_DUAL64X6) == _cabi.RBD_EUNSUPPORTED
    assert call(desc(), B=0) == _cabi.RBD_OK
    h.close()


@pytest.mark.gpu
def test_gpu_python_vjp_argument_checks(built):
    """integrate_task_pd_vjp_: bars of arrays the controller does not have, and s_* arguments without contact; task_pd_torques of a
    JointPD."""
    import torch
    mech = rbd.load_model("double_pendulum")
    f64 = torch.float64
    z = lambda *s: torch.zeros(*s, dtype=f64, device="cuda")      # noqa: E731
    body = mech.joints[-1].successor
    jt = rbd.JointPD(z(2), z(2), z(2, 1))
    ctl = rbd.TaskPD([TaskFrame(body, None, None)], ["point"], z(3), z(3), z(3, 1), joint=jt)
    qt, vt = z(2, 2, 1), z(2, 2, 1)
    f = rbd.autodiff.integrate_task_pd_vjp_
    with pytest.raises(ValueError, match="xd_ref_bar"):
        f(mech, qt, vt, controller=ctl, dt=1e-3, xd_ref_bar=z(3, 1))
    with pytest.raises(ValueError, match="joint_bars"):
        f(mech, qt, vt, controller=rbd.TaskPD([TaskFrame(body, None, None)], ["point"], z(3), z(3), z(3, 1)), dt=1e-3,
          joint_bars=(z(2, 1), None, None, None, None))
    with pytest.raises(ValueError, match="v_ref"):
        f(mech, qt, vt, controller=ctl, dt=1e-3, joint_bars=(None, None, None, z(2, 1), None))
    with pytest.raises(ValueError, match="need contact"):
        f(mech, qt, vt, controller=ctl, dt=1e-3, s_traj=z(2, 0, 1))
    with pytest.raises(TypeError):
        rbd.autodiff.task_pd_torques(rbd.MechanismState(mech, 1, f64), jt)
    with pytest.raises(TypeError):
        rbd.autodiff.task_pd_torques_vjp_(rbd.MechanismState(mech, 1, f64), jt, z(2, 1))


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["atlas", "iiwa14", "randmech1", "randmech3"])
def test_gpu_torques_vjp_matches_cpu_run(built, which):
    """rbd_task_pd_torques_vjp (torque mode, with and without a joint term) against task_pd_vjp_column run on the CPU: fp64 to
    1e-10, fp32 against the fp64 CPU run to TOL32 (about 5x the worst error measured on an H100, DESIGN 4.22)."""
    import torch
    seed = zlib.crc32(which.encode())
    for with_joint in (False, True):
        mech, rng, q, v, tasks, kinds, kp, kd, xref, xdref, joint = _law_case(which, seed, "random", False, with_joint, True)
        nv, B = v.shape
        w = rng.standard_normal((nv, B))
        ref = hostsim_task_law_vjp(mech, tasks, kinds, q, v, w, kp, kd, xref, xdref, joint, False)
        for dtype, tol in ((torch.float64, 1e-10), (torch.float32, TOL32)):
            r = lambda a: None if a is None else a.astype(np.float32 if dtype == torch.float32 else np.float64)    # noqa: E731
            st = rbd.MechanismState(mech, B, dtype)
            st.q.copy_(torch.from_numpy(r(q))); st.v.copy_(torch.from_numpy(r(v)))
            t = {k: _torch(a, dtype) for k, a in dict(kp=kp, kd=kd, x_ref=xref, xd_ref=xdref).items()}
            if joint is not None:
                t.update(jkp=_torch(joint.kp, dtype), jkd=_torch(joint.kd, dtype), jq_ref=_torch(joint.q_ref, dtype),
                         jv_ref=_torch(joint.v_ref, dtype))
            ctl = _task_pd(tasks, kinds, t, False, None)
            R = kp.shape[0]
            out = dict(q_tan=torch.empty_like(st.v), v=torch.empty_like(st.v), kp=st.q.new_zeros((R, B)), kd=st.q.new_zeros((R, B)),
                       x_ref=torch.zeros_like(t["x_ref"]), xd_ref=torch.zeros_like(t["xd_ref"]))
            jb = None if joint is None else [st.v.new_zeros(st.v.shape), st.v.new_zeros(st.v.shape), torch.zeros_like(t["jq_ref"]),
                                             torch.zeros_like(t["jv_ref"]), None]
            rbd.autodiff.task_pd_torques_vjp_(st, ctl, _torch(w, dtype), q_bar_tan=out["q_tan"], v_bar=out["v"], kp_bar=out["kp"],
                                              kd_bar=out["kd"], x_ref_bar=out["x_ref"], xd_ref_bar=out["xd_ref"], joint_bars=jb)
            if jb is not None:
                out.update(jkp=jb[0], jkd=jb[1], jq_ref=jb[2], jv_ref=jb[3])
            for k, got in out.items():
                e = np.abs(got.double().cpu().numpy() - ref[k]).max() / max(1.0, np.abs(ref[k]).max())
                print(f"{which} joint={with_joint} {dtype} {k}: {e:.3e}")
                assert e <= (TOL32_JQ_REF if (k == "jq_ref" and dtype == torch.float32) else tol), (which, with_joint, dtype, k, e)


# fp32 against the fp64 CPU run, relative to max(1, |reference|): about 5x the worst error measured on an NVIDIA H100 80GB HBM3
# (2.4e-6, randmech3 kp).  The joint term's q_ref adjoint (pd_adj_joint's Dual1 through joint_error, not new code here) measured
# 6.5e-4 on randmech1 and has its own bound.
TOL32 = 1.2e-5
TOL32_JQ_REF = 3e-3


def _law_torch(c, outs_v, aux_kinds, pls, B, dt, dev):
    """The law's f in torch from autodiff.task_kinematics outputs (transform, point, twist, point_velocity of the helper tasks of
    test_task_pd.composed_task_torques): (cotangent on point_velocity, cotangent on twist) rows per helper task."""
    import torch
    from tests.test_task_pd import _rotvec_torch
    K = len(aux_kinds)
    tr, pt, tw, pv = (outs_v[n].view(K, r, B) for n, r in (("transform", 12), ("point", 3), ("twist", 6), ("point_velocity", 3)))
    kp = c.kp if c.kp.dim() == 2 else c.kp[:, None]
    kd = c.kd if c.kd.dim() == 2 else c.kd[:, None]
    xdr = torch.zeros((c.rows()[0], B), dtype=dt, device=dev) if c.xd_ref is None else c.xd_ref
    fpv, ftw = [None] * K, [None] * K
    a = r = x = 0
    for k, pl in zip(c.kinds, pls):
        if k == "point":
            RbF = tr[a + 2, :9].view(3, 3, B)
            e = torch.einsum("jib,jb->ib", RbF, pt[a] - c.x_ref[x:x + 3])
            ed = pv[a + 1] - torch.einsum("jib,jb->ib", RbF, xdr[r:r + 3])
            fpv[a + 1] = -kp[r:r + 3] * e - kd[r:r + 3] * ed
            a, r, x = a + 3, r + 3, x + 3
        else:
            Rx = tr[a + 1, :9].view(3, 3, B)
            Rr, pr = c.x_ref[x:x + 9].view(3, 3, B), c.x_ref[x + 9:x + 12]
            Re = torch.einsum("jib,jkb->ikb", Rr, Rx)
            pe = torch.einsum("jib,jb->ib", Rr, pt[a] - pr)
            psi = _rotvec_torch(Re)
            w = tw[a + 1, :3]
            vC = tw[a + 1, 3:] + torch.cross(w, pl.expand(3, B), dim=0)
            ang = -kp[r:r + 3] * psi - kd[r:r + 3] * (w - xdr[r:r + 3])
            lin = -kp[r + 3:r + 6] * torch.einsum("jib,jb->ib", Re, pe) - kd[r + 3:r + 6] * (vC - xdr[r + 3:r + 6])
            ftw[a + 1] = torch.cat([ang + torch.cross(pl.expand(3, B), lin, dim=0), lin])
            a, r, x = a + 2, r + 6, x + 12
    return fpv, ftw


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["atlas", "iiwa14", "randmech2"])
def test_gpu_task_pd_torques_grad_matches_torch_composition(built, which):
    """autodiff.task_pd_torques (torque mode, no joint term, no bounds, τ_ff = 0) against torch autograd through the composition
    autodiff.task_kinematics -> the law in torch -> Σ Jᵀf, written as w . u = Σ_t f_t . (J_t w) with J_t w the twist / point
    velocity of the helper tasks at velocity w: gradients to q, v, kp, kd, x_ref and xd_ref to 1e-10 in fp64."""
    import torch
    f64 = torch.float64
    mech = _model(which)
    seed = zlib.crc32(which.encode()) % 1000
    rng = np.random.default_rng(seed)
    B = 6
    q, v, _, _, _ = rand_inputs(mech, B, seed)
    tasks, kinds = task_mix(mech, seed % 89, npoint=4)
    R = sum(_rows(k)[0] for k in kinds)
    xref = _targets(mech, q, tasks, kinds, rng, "random")
    kp, kd = _gains(rng, kinds, B, True)
    xdref = rng.standard_normal((R, B))
    w = _torch(rng.standard_normal(v.shape), f64)
    names = ("q", "v", "kp", "kd", "x_ref", "xd_ref")

    def inputs():
        return {k: _torch(a, f64, True) for k, a in zip(names, (q, v, kp, kd, xref, xdref))}
    t = inputs()
    st = rbd.MechanismState(mech, B, f64)
    st.q.copy_(t["q"].detach()); st.v.copy_(t["v"].detach())
    st.q.requires_grad_(); st.v.requires_grad_()
    ctl = rbd.TaskPD(tasks, kinds, t["kp"], t["kd"], t["x_ref"], t["xd_ref"])
    (rbd.autodiff.task_pd_torques(st, ctl) * w).sum().backward()
    got = dict(q=st.q.grad, v=st.v.grad, kp=t["kp"].grad, kd=t["kd"].grad, x_ref=t["x_ref"].grad, xd_ref=t["xd_ref"].grad)
    # the composition
    s = inputs()
    aux, pls = [], []
    for tk, k in zip(tasks, kinds):
        if k == "point":
            aux += [TaskFrame(tk.body, tk.base, tk.point, tk.base), TaskFrame(tk.body, tk.base, tk.point, tk.frame), TaskFrame(tk.frame, tk.base)]
        else:
            aux += [TaskFrame(tk.body, tk.base, tk.point, tk.base), TaskFrame(tk.body, tk.base, None, tk.body)]
        pls.append(_torch(np.zeros(3) if tk.point is None else np.asarray(tk.point, np.float64), f64)[:, None])
    outs_v = rbd.autodiff.task_kinematics(mech, s["q"], s["v"], tasks=aux, outputs=("transform", "point", "twist", "point_velocity"))
    outs_w = rbd.autodiff.task_kinematics(mech, s["q"], w, tasks=aux, outputs=("twist", "point_velocity"))
    c = rbd.TaskPD(tasks, kinds, s["kp"], s["kd"], s["x_ref"], s["xd_ref"])
    fpv, ftw = _law_torch(c, outs_v, aux, pls, B, f64, "cuda")
    K = len(aux)
    tw_w, pv_w = outs_w["twist"].view(K, 6, B), outs_w["point_velocity"].view(K, 3, B)
    L = sum((f * pv_w[i]).sum() for i, f in enumerate(fpv) if f is not None) + sum((f * tw_w[i]).sum() for i, f in enumerate(ftw)
                                                                                  if f is not None)
    L.backward()
    for k in names:
        ref = s[k].grad.cpu().numpy()
        e = np.abs(got[k].cpu().numpy() - ref).max() / max(1.0, np.abs(ref).max())
        assert e <= 1e-10, (which, k, e)


@pytest.mark.gpu
@pytest.mark.parametrize("ct", [False, True])
def test_gpu_gradcheck(built, ct):
    """torch.autograd.gradcheck in fp64 on a small revolute / prismatic tree: autodiff.simulate with a TaskPD (point and pose tasks,
    a joint term, clamps with row 0 saturated on every sample, held 0.5 away from the bound) and autodiff.task_pd_torques, with
    respect to q0, v0, τ_ff and every controller tensor."""
    import torch
    from oracle import Oracle
    rng = np.random.default_rng(11)
    mech = rbd.rand_tree_mechanism(rng, [rbd.Revolute, rbd.Prismatic, rbd.Revolute, rbd.Prismatic])
    d = mech.flatten()
    B, n, dt = 3, 3, 1e-2
    q, v, tau, _, _ = rand_inputs(mech, B, 6)
    bodies = [j.successor for j in mech.joints]
    tasks = [TaskFrame(bodies[-1], None, np.array([0.1, 0.0, 0.2])), TaskFrame(bodies[1], None, np.array([0.0, 0.1, 0.0]))]
    kinds = ["point", "pose"]
    R = 9
    xref = _targets(mech, q, tasks, kinds, rng, "random")
    kp, kd = rng.uniform(1, 5, (R, B)), rng.uniform(0.1, 1, (R, B))
    xdref = rng.standard_normal((R, B)) * 0.3
    j = _controller(mech, q, rng, ct=ct, per_sample=True, scale=0.3)
    bounds = None
    if not ct:
        u = TaskCtrl(mech, tasks, kinds, kp, kd, xref, xdref, j, ct).torque(Oracle(d), 0, q, v, tau)
        bounds = (np.full(d.nv, -1e6), np.full(d.nv, 1e6))
        bounds[1][0] = float(u[0].min()) - 0.5 * float(np.ptp(u[0]) + 1)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda().requires_grad_(True)     # noqa: E731
    arrays = [kp, kd, xref, xdref, j.kp, j.kd, j.q_ref, j.v_ref] + ([j.vd_ref] if ct else [])
    args = [T(q), T(v), T(tau)] + [T(a) for a in arrays]

    def ctl(kp_, kd_, xr, xdr, jkp, jkd, jqr, jvr, jvdr=None):
        jt = rbd.JointPD(jkp, jkd, jqr, jvr, vd_ref=jvdr, computed_torque=ct)
        return rbd.TaskPD(tasks, kinds, kp_, kd_, xr, xdr, joint=jt, computed_torque=ct, effort_bounds=bounds)

    def f(q0, v0, t, *a):
        return rbd.autodiff.simulate(mech, q0, v0, t, dt=dt, nsteps=n, controller=ctl(*a))
    assert torch.autograd.gradcheck(f, args, eps=1e-6, atol=1e-6, rtol=1e-5)

    def g(q0, v0, t, *a):
        st = rbd.MechanismState(mech, B, torch.float64)
        st.q = q0
        st.v = v0
        return rbd.autodiff.task_pd_torques(st, ctl(*a), t)
    assert torch.autograd.gradcheck(g, args, eps=1e-6, atol=1e-6, rtol=1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("ct,with_joint,clamp", [(False, False, False), (False, True, True), (True, True, True), (True, False, False)])
def test_gpu_launch_counts(built, ct, with_joint, clamp):
    """Per step, beyond rbd_integrate_pd_vjp's launches with the joint term (rbd_integrate_vjp's without one): the recompute's four
    task kernels, and per stage one task-adjoint kernel plus, in torque mode with bounds, one mask kernel."""
    import torch
    f64 = torch.float64
    n, dt = 2, 1e-3
    mech, q, v, tau, tasks, kinds, arrays, bounds, rng = _rollout_case("iiwa14", 33, n, ct, True, False, False, clamp, 3)
    t = {k: _torch(a, f64) for k, a in arrays.items()}
    if not with_joint:
        t = {k: a for k, a in t.items() if not k.startswith("j")}
    ctl = _task_pd(tasks, kinds, t, ct, bounds)
    gq, gv = _torch(rng.standard_normal(q.shape), f64), _torch(rng.standard_normal(v.shape), f64)
    qt, vt, _ = _record(mech, _torch(q, f64), _torch(v, f64), _torch(tau, f64), ctl, dt, n)
    _direct(mech, qt, vt, _torch(tau, f64), ctl, dt, gq, gv)
    k_task = rbd.launch_info().kernels_launched
    qtb, vtb = torch.zeros_like(qt), torch.zeros_like(vt)
    qtb[-1] = gq; vtb[-1] = gv
    out = dict(q0_bar_cfg=torch.empty_like(qt[0]), v0_bar=torch.empty_like(vt[0]))
    if with_joint:
        jt = ctl.joint
        j2 = rbd.JointPD(jt.kp, jt.kd, jt.q_ref, jt.v_ref, vd_ref=jt.vd_ref, computed_torque=ct, effort_bounds=bounds)
        rbd.integrate_pd_vjp_(mech, qt, vt, _torch(tau, f64), controller=j2, dt=dt, q_traj_bar=qtb, v_traj_bar=vtb, **out)
        base = rbd.launch_info().kernels_launched
    else:
        rbd.integrate_vjp_(mech, qt, vt, _torch(tau, f64), dt=dt, q_traj_bar=qtb, v_traj_bar=vtb, **out)
        base = rbd.launch_info().kernels_launched
        if ct:      # the recompute's inverse dynamics + pd_finish_kernel, the inverse-dynamics VJP, per stage
            base += 3 * 4 * n
    extra = 4 * n + 4 * n + (4 * n if clamp and not ct else 0)
    assert k_task - base == extra, (k_task, base, extra)
