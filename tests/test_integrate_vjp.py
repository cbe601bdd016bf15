"""Reverse mode through simulate: rbd_integrate_trajectory, rbd_integrate_vjp (csrc/rbd_integrate_adjoint.cuh,
csrc/rbd_integrate_vjp.cu) and rigidbodydynamics.jl_b200.autodiff.simulate.

The loss of every check is  L = sum_s q̄_s . q_s + v̄_s . v_s  over the recorded trajectory (q_0, v_0) ... (q_n, v_n).
CPU tier: the per-joint adjoints of the coordinate maps against central differences, and the whole backward pass, run on the CPU
(tests/hostsim/hostsim_integrate_vjp.cpp), against central differences of the oracle's fp64 `integrate` stepped one step at a time,
along q + eps q̇(e_k), v + eps e_k and tau + eps e_k.  GPU tier: the kernels against that CPU run, the trajectory against
rbd_integrate, and the torch.autograd function."""
import ctypes
import functools

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from oracle import Oracle
from rigidbodydynamics.jl_b200._cabi import RbdModelDesc, make_desc
from tests import hostsim
from tests.test_vjp import _qdot_dirs
from tests.util import double_pendulum, rand_inputs, randmech, rel_err

# central differences of the fp64 oracle at eps = 1e-5: the loss's rounding noise over eps dominates their error (Atlas, 5 steps:
# 1.3e-6 at eps = 1e-6, 1.4e-7 at 1e-5, 1.6e-8 at 1e-4)
TOL_FD = 1e-6
EPS_FD = 1e-5
TOL64 = 1e-10        # GPU kernels against the CPU run of the same code, fp64
# fp32 kernels against the fp64 CPU run: measured worst rel_err 2.9e-4 over the models and schedules of test_kernels_vs_hostsim
# (Atlas, B = 161, 3 steps); the bound is the derivative tests' 5e-3, as for the single-call VJPs (tests/test_vjp.py).
TOL32 = 5e-3
DT = 2e-3

K_REV, K_PRIS, K_FIXED, K_PLANAR, K_QFLOAT, K_SPQFLOAT, K_QSPH, K_SINCOS = range(8)
NQ, NV = (1, 1, 0, 3, 7, 6, 4, 2), (1, 1, 0, 3, 6, 6, 3, 1)


@functools.cache
def _shim():
    """tests/hostsim/hostsim_integrate_vjp.cpp, compiled and loaded by hostsim.shim."""
    lib = hostsim.shim("hostsim_integrate_vjp")
    vp, i64, c_int, c_double = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_double
    lib.hostsim_integrate_traj.argtypes = [ctypes.POINTER(RbdModelDesc), c_int, i64, vp, vp, vp, i64, i64, c_double, c_int]
    lib.hostsim_integrate_vjp.argtypes = [ctypes.POINTER(RbdModelDesc), c_int, i64, vp, vp, vp, i64, i64, c_double, c_int] + [vp] * 6
    lib.hostsim_joint_global.argtypes = [c_int] + [vp] * 3
    lib.hostsim_joint_rate.argtypes = [c_int] + [vp] * 4
    lib.hostsim_joint_g_adjoint.argtypes = [c_int] + [vp] * 5
    lib.hostsim_joint_l_adjoint.argtypes = [c_int] + [vp] * 7
    return lib


def _p(a):
    return None if a is None or a.size == 0 else a.ctypes.data


def _sched(tau, nv, B):
    """(contiguous array or None, step stride, stage stride) of a torque argument: None, [nv, B], [n, nv, B] or [n, 4, nv, B]."""
    if tau is None:
        return None, 0, 0
    blk = nv * B
    return np.ascontiguousarray(tau), {2: 0, 3: blk, 4: 4 * blk}[tau.ndim], blk if tau.ndim == 4 else 0


def host_traj(desc, q0, v0, tau, n, dt=DT):
    dt_ = q0.dtype
    B = q0.shape[1]
    qt = np.zeros((n + 1, desc.nq, B), dt_); vt = np.zeros((n + 1, desc.nv, B), dt_)
    qt[0], vt[0] = q0, v0
    t, step, stage = _sched(None if tau is None else tau.astype(dt_), desc.nv, B)
    d, keep = make_desc(desc)
    assert _shim().hostsim_integrate_traj(ctypes.byref(d), 0 if dt_ == np.float32 else 1, B, _p(qt), _p(vt), _p(t), step, stage, dt, n) == 0
    return qt, vt


def host_ivjp(desc, qt, vt, tau, n, qtb, vtb, dt=DT):
    """The CPU run of rbd_integrate_vjp: dict q0t [nv, B], q0c [nq, B], v0b [nv, B], taub (shape of tau)."""
    dt_ = qt.dtype
    B = qt.shape[2]
    c = lambda a: None if a is None else np.ascontiguousarray(a, dt_)
    t, step, stage = _sched(c(tau), desc.nv, B)
    out = {"q0t": np.full((desc.nv, B), np.nan, dt_), "q0c": np.full((desc.nq, B), np.nan, dt_), "v0b": np.full((desc.nv, B), np.nan, dt_),
           "taub": None if tau is None else np.zeros(tau.shape, dt_)}
    d, keep = make_desc(desc)
    assert _shim().hostsim_integrate_vjp(ctypes.byref(d), 0 if dt_ == np.float32 else 1, B, _p(c(qt)), _p(c(vt)), _p(t), step, stage, dt,
                                         n, _p(c(qtb)), _p(c(vtb)), _p(out["q0t"]), _p(out["q0c"]), _p(out["v0b"]), _p(out["taub"])) == 0
    return out


def _oracle_loss(o, q0, v0, taus, n, qtb, vtb, dt=DT):
    """sum_s q̄_s . q_s + v̄_s . v_s per sample, the oracle stepped one step at a time with the torques of each step."""
    q, v = q0, v0
    L = (qtb[0] * q).sum(0) + (vtb[0] * v).sum(0)
    for s in range(n):
        q, v = o.integrate(q, v, taus[s], dt=dt, nsteps=1)
        L = L + (qtb[s + 1] * q).sum(0) + (vtb[s + 1] * v).sum(0)
    return L


def _taus(tau, n):
    """per-step torques of a constant [nv, B] / per-step [n, nv, B] argument (the oracle has no per-stage schedule)"""
    if tau is None:
        return [None] * n
    return [tau] * n if tau.ndim == 2 else [tau[s] for s in range(n)]


def _models():
    return [("atlas", rbd.load_model("atlas", floating=True)), ("randmech0", randmech(0, shuffle=True)),
            ("double_pendulum", double_pendulum())]


# ----------------------------------------------------------------------------------------------------------------------
# CPU tier
# ----------------------------------------------------------------------------------------------------------------------
def _unit(rng, n):
    x = rng.standard_normal(n)
    return x / np.linalg.norm(x)


def _joint_point(kind, rng, scale):
    """(q0, phi, vs) of one joint: unit quaternions / (sin, cos) pairs, stage angles of size `scale`."""
    nq, nv = NQ[kind], NV[kind]
    q0 = rng.standard_normal(nq)
    if kind in (K_QFLOAT, K_QSPH):
        q0[:4] = _unit(rng, 4)
    elif kind == K_SINCOS:
        q0 = _unit(rng, 2)
    elif kind == K_SPQFLOAT:
        q0[:3] *= 0.3
    phi = rng.standard_normal(nv) * scale
    return q0, phi, rng.standard_normal(nv)


@pytest.mark.parametrize("kind", [k for k in range(8) if k != K_FIXED])
@pytest.mark.parametrize("scale", [1e-4, 0.7], ids=["taylor", "closed_form"])
def test_joint_adjoints_match_finite_differences(kind, scale):
    """G_q0^T, G_φ^T, L_q0^T, L_qs^T and L_vs^T of every joint type against central differences of the same fp64 maps, on the
    Taylor branch (stage angles 1e-4) and the closed forms (0.7)."""
    lib = _shim()
    rng = np.random.default_rng(kind + int(scale * 10))
    nq, nv = NQ[kind], NV[kind]
    eps = 1e-7
    for _ in range(3):
        q0, phi, vs = _joint_point(kind, rng, scale)
        G = lambda a, b: (lib.hostsim_joint_global(kind, _p(a), _p(b), _p(out := np.zeros(nq))), out)[1]
        qs = G(q0, phi)
        Lr = lambda a, b, c: (lib.hostsim_joint_rate(kind, _p(a), _p(b), _p(c), _p(out := np.zeros(nv))), out)[1]
        qsb, pdb = rng.standard_normal(nq), rng.standard_normal(nv)
        q0b, phib = np.zeros(nq), np.zeros(nv)
        lib.hostsim_joint_g_adjoint(kind, _p(q0), _p(phi), _p(qsb), _p(q0b), _p(phib))
        e = lambda n, k: np.eye(n)[k] * eps
        fd_q0 = [qsb @ (G(q0 + e(nq, k), phi) - G(q0 - e(nq, k), phi)) / (2 * eps) for k in range(nq)]
        fd_phi = [qsb @ (G(q0, phi + e(nv, k)) - G(q0, phi - e(nv, k))) / (2 * eps) for k in range(nv)]
        assert rel_err(q0b, fd_q0) < 1e-7 and rel_err(phib, fd_phi) < 1e-7, (q0b, fd_q0, phib, fd_phi)
        lq0b, lqsb, lvsb = np.zeros(nq), np.zeros(nq), np.zeros(nv)
        lib.hostsim_joint_l_adjoint(kind, _p(q0), _p(qs), _p(vs), _p(pdb), _p(lq0b), _p(lqsb), _p(lvsb))
        fd = lambda f: pdb @ f
        ref_q0 = [fd(Lr(q0 + e(nq, k), qs, vs) - Lr(q0 - e(nq, k), qs, vs)) / (2 * eps) for k in range(nq)]
        ref_qs = [fd(Lr(q0, qs + e(nq, k), vs) - Lr(q0, qs - e(nq, k), vs)) / (2 * eps) for k in range(nq)]
        ref_vs = [fd(Lr(q0, qs, vs + e(nv, k)) - Lr(q0, qs, vs - e(nv, k))) / (2 * eps) for k in range(nv)]
        for got, ref in ((lq0b, ref_q0), (lqsb, ref_qs), (lvsb, ref_vs)):
            assert rel_err(got, ref) < 1e-7, (got, ref)


def _fd_case(mech, n, tmode, B=2, seed=0):
    d = mech.flatten()
    q, v, tau, _, _ = rand_inputs(mech, B, seed)
    rng = np.random.default_rng(seed + 100)
    tau = {"none": None, "const": tau, "step": rng.standard_normal((n, d.nv, B))}[tmode]
    qtb, vtb = rng.standard_normal((n + 1, d.nq, B)), rng.standard_normal((n + 1, d.nv, B))
    return d, q, v, tau, qtb, vtb


@pytest.mark.parametrize("name,mech", _models(), ids=[n for n, _ in _models()])
@pytest.mark.parametrize("n", [1, 5])
@pytest.mark.parametrize("tmode", ["none", "const", "step"])
def test_rollout_vjp_hostsim_matches_oracle_finite_differences(name, mech, n, tmode):
    d, q, v, tau, qtb, vtb = _fd_case(mech, n, tmode)
    o = Oracle(d)
    B, eps = q.shape[1], EPS_FD
    qt, vt = host_traj(d, q, v, tau, n)
    oq, ov = o.integrate(q, v, _taus(tau, n)[0], dt=DT, nsteps=1) if n else (q, v)
    assert rel_err(qt[1], oq) < 1e-12 and rel_err(vt[1], ov) < 1e-12     # the CPU run steps like the oracle
    r = host_ivjp(d, qt, vt, tau, n, qtb, vtb)
    f = lambda q_=q, v_=v, t_=tau: _oracle_loss(o, q_, v_, _taus(t_, n), n, qtb, vtb)
    cd = lambda g: (g(eps) - g(-eps)) / (2 * eps)
    dirs_q = _qdot_dirs(o, q, d.nv, None)
    ref_q = np.stack([cd(lambda h: f(q_=q + h * dirs_q[k])) for k in range(d.nv)])
    eye = lambda k: np.repeat(np.eye(d.nv)[:, k:k + 1], B, 1)
    ref_v = np.stack([cd(lambda h: f(v_=v + h * eye(k))) for k in range(d.nv)])
    assert rel_err(r["q0t"], ref_q) < TOL_FD, rel_err(r["q0t"], ref_q)
    assert rel_err(r["v0b"], ref_v) < TOL_FD, rel_err(r["v0b"], ref_v)
    if tau is not None:
        blocks = [None] if tau.ndim == 2 else range(n)
        for s in blocks:
            def pert(h, k, s=s):
                t = tau.copy()
                if s is None:
                    t += h * eye(k)
                else:
                    t[s] += h * eye(k)
                return f(t_=t)
            ref_t = np.stack([cd(lambda h: pert(h, k)) for k in range(d.nv)])
            got = r["taub"] if s is None else r["taub"][s]
            assert rel_err(got, ref_t) < TOL_FD, (s, rel_err(got, ref_t))
    # the configuration form pairs with q̇ like the tangent form with v (configuration_derivative_to_velocity_adjoint!)
    u = np.random.default_rng(1).standard_normal((d.nv, B))
    qd = o.dynamics(q, u, None, want_qd=True)[1]
    assert np.abs((r["q0c"] * qd).sum(0) - (r["q0t"] * u).sum(0)).max() < 1e-10 * max(1.0, np.abs(r["q0t"]).max() * np.abs(u).max() * d.nv)


def test_rollout_vjp_hostsim_revolute_tree_cfg_is_plain_gradient():
    mech = rbd.rand_tree_mechanism(np.random.default_rng(3), [rbd.Revolute, rbd.Prismatic] * 4)
    d, q, v, tau, qtb, vtb = _fd_case(mech, 3, "const")
    qt, vt = host_traj(d, q, v, tau, 3)
    r = host_ivjp(d, qt, vt, tau, 3, qtb, vtb)
    assert np.array_equal(r["q0c"], r["q0t"])


def test_zero_steps_is_the_identity():
    mech = rbd.load_model("atlas", floating=True)
    d, q, v, tau, qtb, vtb = _fd_case(mech, 0, "const")
    r = host_ivjp(d, q[None], v[None], tau, 0, qtb, vtb)
    assert np.array_equal(r["v0b"], vtb[0])
    o = Oracle(d)
    dirs_q = _qdot_dirs(o, q, d.nv, None)
    assert rel_err(r["q0t"], np.einsum("kib,ib->kb", dirs_q, qtb[0])) < 1e-12


# ----------------------------------------------------------------------------------------------------------------------
# GPU tier
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch():
    import torch as t
    assert t.cuda.is_available()
    rbd.load_library()
    return t


def _gpu_traj(torch, mech, q, v, tau, n, dtype):
    st = rbd.MechanismState(mech, q.shape[1], dtype)
    st.q.copy_(torch.from_numpy(q)); st.v.copy_(torch.from_numpy(v))
    t = None if tau is None else torch.from_numpy(np.ascontiguousarray(tau)).to(dtype).cuda()
    qt, vt = rbd.simulate_trajectory_(st, n, t, dt=DT)
    return st, t, qt, vt


def _tau_shapes(rng, nv, B, n):
    return {"none": None, "const": rng.standard_normal((nv, B)), "step": rng.standard_normal((n, nv, B)),
            "stage": rng.standard_normal((n, 4, nv, B))}


@pytest.mark.gpu
@pytest.mark.parametrize("name,mech", _models(), ids=[n for n, _ in _models()])
@pytest.mark.parametrize("B", [1, 161])
def test_kernels_vs_hostsim(torch, name, mech, B):
    """rbd_integrate_vjp against the CPU run of the same code: fp64 and fp32, every torque shape, trajectory adjoints on every
    step and on the final state only."""
    d = mech.flatten()
    n = 3
    q, v, _, _, _ = rand_inputs(mech, B, 7)
    rng = np.random.default_rng(B)
    worst = 0.0
    for tmode, tau in _tau_shapes(rng, d.nv, B, n).items():
        for final_only in (False, True):
            qtb, vtb = rng.standard_normal((n + 1, d.nq, B)), rng.standard_normal((n + 1, d.nv, B))
            if final_only:
                qtb[:-1] = 0; vtb[:-1] = 0
            for dtype in (torch.float64, torch.float32):
                st, t, qt, vt = _gpu_traj(torch, mech, q, v, tau, n, dtype)
                T = lambda a: torch.from_numpy(a).to(dtype).cuda()
                e = lambda rows: torch.full((rows, B), float("nan"), dtype=dtype, device="cuda")
                out = {"q0t": e(d.nv), "q0c": e(d.nq), "v0b": e(d.nv), "taub": None if t is None else torch.zeros_like(t)}
                rbd.integrate_vjp_(mech, qt, vt, t, dt=DT, q_traj_bar=T(qtb), v_traj_bar=T(vtb), q0_bar_tan=out["q0t"],
                                   q0_bar_cfg=out["q0c"], v0_bar=out["v0b"], tau_bar=out["taub"])
                torch.cuda.synchronize()
                np64 = lambda x: x.double().cpu().numpy()
                ref = host_ivjp(d, np64(qt), np64(vt), None if tau is None else np64(t), n, qtb, vtb)
                tol = TOL64 if dtype == torch.float64 else TOL32
                for k in ("q0t", "q0c", "v0b", "taub"):
                    if out[k] is None:
                        continue
                    got = np64(out[k]).reshape(ref[k].shape[0], -1)
                    err = rel_err(got, ref[k].reshape(got.shape))
                    if dtype == torch.float32:
                        worst = max(worst, err)
                    assert err < tol, (tmode, final_only, dtype, k, err)
    print(f"{name} B={B}: worst fp32 rel_err {worst:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("name,mech", _models()[:2], ids=[n for n, _ in _models()[:2]])
def test_trajectory_blocks_bit_identical_to_rbd_integrate(torch, name, mech):
    d = mech.flatten()
    n = 4
    for B in (3, 1024):
        q, v, _, _, _ = rand_inputs(mech, B, 2)
        rng = np.random.default_rng(0)
        for tmode, tau in _tau_shapes(rng, d.nv, B, n).items():
            for dtype in (torch.float64, torch.float32):
                st, t, qt, vt = _gpu_traj(torch, mech, q, v, tau, n, dtype)
                for s in range(n + 1):
                    s2 = rbd.MechanismState(mech, B, dtype)
                    s2.q.copy_(torch.from_numpy(q)); s2.v.copy_(torch.from_numpy(v))
                    if s:
                        rbd.simulate_(s2, s * DT - DT / 2, t if t is None or t.dim() == 2 else t[:s].contiguous(), dt=DT)
                    assert torch.equal(qt[s], s2.q) and torch.equal(vt[s], s2.v), (tmode, dtype, s)
                assert torch.equal(st.q, qt[n]) and torch.equal(st.v, vt[n])


@pytest.mark.gpu
@pytest.mark.parametrize("trajectory", [True, False])
def test_simulate_gradcheck(torch, trajectory):
    from rigidbodydynamics.jl_b200 import autodiff
    rng = np.random.default_rng(8)
    mech = rbd.rand_tree_mechanism(rng, [rbd.Revolute, rbd.Prismatic, rbd.Revolute, rbd.Revolute, rbd.Prismatic])
    d = mech.flatten()
    B, n = 3, 3
    q, v, _, _, _ = rand_inputs(mech, B, 6)
    T = lambda a: torch.from_numpy(a).cuda().requires_grad_(True)
    for tau in _tau_shapes(rng, d.nv, B, n).values():
        args = (T(q), T(v)) + (() if tau is None else (T(tau),))
        f = lambda q_, v_, t_=None: autodiff.simulate(mech, q_, v_, t_, dt=0.01, nsteps=n, trajectory=trajectory)
        assert torch.autograd.gradcheck(f, args, eps=1e-6, atol=1e-6, rtol=1e-5)


@pytest.mark.gpu
def test_autograd_on_floating_atlas(torch):
    from rigidbodydynamics.jl_b200 import autodiff
    from tests.test_vjp import _qdot_dirs as qdot_dirs
    mech = rbd.load_model("atlas", floating=True)
    d = mech.flatten()
    B, n = 5, 6
    q, v, tau, _, _ = rand_inputs(mech, B, 9)
    rng = np.random.default_rng(4)
    tau = rng.standard_normal((n, d.nv, B))
    T = lambda a: torch.from_numpy(a).cuda().requires_grad_(True)
    tq, tv, tt = T(q), T(v), T(tau)
    qt, vt = autodiff.simulate(mech, tq, tv, tt, dt=DT, nsteps=n)
    qtb, vtb = torch.randn_like(qt), torch.randn_like(vt)
    ((qt * qtb).sum() + (vt * vtb).sum()).backward()
    outs = {"q": torch.empty_like(tq), "v": torch.empty_like(tv), "t": torch.zeros_like(tt)}
    rbd.integrate_vjp_(mech, qt.detach(), vt.detach(), tt.detach(), dt=DT, q_traj_bar=qtb, v_traj_bar=vtb, q0_bar_cfg=outs["q"],
                       v0_bar=outs["v"], tau_bar=outs["t"])
    torch.cuda.synchronize()
    for k, x in (("q", tq), ("v", tv), ("t", tt)):
        assert torch.equal(x.grad, outs[k]), k
    # the q0 gradient along tangent directions against fp64 central differences of the oracle
    o = Oracle(d)
    qtb_, vtb_ = qtb.cpu().numpy(), vtb.cpu().numpy()
    f = lambda q_: _oracle_loss(o, q_, v, list(tau), n, qtb_, vtb_)
    dirs = qdot_dirs(o, q, d.nv, None)
    ref = np.stack([(f(q + EPS_FD * dirs[k]) - f(q - EPS_FD * dirs[k])) / (2 * EPS_FD) for k in range(d.nv)])
    got = np.einsum("kib,ib->kb", dirs, tq.grad.cpu().numpy())
    assert rel_err(got, ref) < TOL_FD, rel_err(got, ref)
    # checkpointing does not change the gradients, bit for bit
    grads = []
    for k in (1, 3, n):
        tq.grad = tv.grad = tt.grad = None
        qf, vf = autodiff.simulate(mech, tq, tv, tt, dt=DT, nsteps=n, trajectory=False, checkpoint_every=k)
        ((qf * qtb[-1]).sum() + (vf * vtb[-1]).sum()).backward()
        grads.append((tq.grad.clone(), tv.grad.clone(), tt.grad.clone()))
    for g in grads[1:]:
        assert all(torch.equal(a, b) for a, b in zip(g, grads[0]))
    # a double backward raises
    tq.grad = None
    qf, _ = autodiff.simulate(mech, tq, tv, None, dt=DT, nsteps=2, trajectory=False)
    g, = torch.autograd.grad(qf.sum(), tq, create_graph=True)
    with pytest.raises(RuntimeError):
        g.sum().backward()


@pytest.mark.gpu
def test_refusals(torch):
    from rigidbodydynamics.jl_b200 import _cabi, autodiff
    from rigidbodydynamics.jl_b200.state import _DT, _model_handle
    mech = rbd.load_model("iiwa14", floating=False)
    d = mech.flatten()
    B, n = 8, 2
    q, v, tau, _, _ = rand_inputs(mech, B, 1)
    st, t, qt, vt = _gpu_traj(torch, mech, q, v, tau, n, torch.float64)
    lib = _cabi.load_library()
    h = _model_handle(mech)
    p = lambda x: None if x is None else x.data_ptr()
    out = torch.full((d.nv, B), 7.0, dtype=torch.float64, device="cuda")
    call = lambda dtype=_cabi.RBD_F64, qt_=qt, vt_=vt, t_=t, step=0, stage=0, dt=DT, n_=n, tb=None, o=out: lib.rbd_integrate_vjp(
        h.ptr, dtype, B, p(qt_), p(vt_), p(t_), step, stage, dt, n_, None, None, None, None, p(o), p(tb), None)
    assert call(dtype=_cabi.RBD_DUAL64X6) == _cabi.RBD_EUNSUPPORTED
    assert call(step=-1) == _cabi.RBD_EINVAL and call(stage=-5) == _cabi.RBD_EINVAL
    assert call(n_=-1) == _cabi.RBD_EINVAL and call(dt=0.0) == _cabi.RBD_EINVAL
    assert call(qt_=None) == _cabi.RBD_EINVAL and call(vt_=None) == _cabi.RBD_EINVAL
    assert call(t_=None, tb=torch.zeros_like(t)) == _cabi.RBD_EINVAL
    torch.cuda.synchronize()
    assert (out == 7.0).all()           # nothing written by a refused call
    # omitted outputs are left untouched; present ones equal an all-outputs call
    full = torch.empty_like(out)
    assert call(o=full) == _cabi.RBD_OK
    none = call(o=None)
    torch.cuda.synchronize()
    assert none == _cabi.RBD_OK and torch.isfinite(full).all()
    # B = 0 and nsteps = 0
    assert lib.rbd_integrate_vjp(h.ptr, _cabi.RBD_F64, 0, None, None, None, 0, 0, DT, n, None, None, None, None, None, None, None) == 0
    vtb = torch.randn_like(vt[:1])
    v0b = torch.empty_like(out)
    rbd.integrate_vjp_(mech, qt[:1].contiguous(), vt[:1].contiguous(), t, dt=DT, v_traj_bar=vtb, v0_bar=v0b)
    torch.cuda.synchronize()
    assert torch.equal(v0b, vtb[0])
    with pytest.raises(rbd.DimensionMismatch):
        autodiff.simulate(mech, st.q, st.v, t[:3], dt=DT, nsteps=n)
    from tests.loops_oracle import four_bar
    m4 = four_bar()
    s4 = rbd.MechanismState(m4, 2, torch.float64)
    with pytest.raises(_cabi.RbdError) as e:
        autodiff.simulate(m4, s4.q, s4.v, dt=DT, nsteps=1)
    assert e.value.status == _cabi.RBD_ELOOP
    with pytest.raises(_cabi.RbdError) as e:
        rbd.simulate_trajectory_(s4, 1)
    assert e.value.status == _cabi.RBD_ELOOP


@pytest.mark.gpu
def test_full_batch_atlas_fp32(torch):
    mech = rbd.load_model("atlas", floating=True)
    d = mech.flatten()
    B, n = 1 << 20, 3
    rng = np.random.default_rng(12)
    st = rbd.MechanismState(mech, B, torch.float32)
    rbd.rand_(st, rng)
    tau = torch.from_numpy(rng.standard_normal((d.nv, B))).float().cuda()
    qt, vt = rbd.simulate_trajectory_(st, n, tau, dt=DT)
    qtb, vtb = torch.zeros_like(qt), torch.zeros_like(vt)
    qtb[-1].normal_(); vtb[-1].normal_()
    e = lambda rows: torch.empty((rows, B), dtype=torch.float32, device="cuda")
    qc, vb, tb = e(d.nq), e(d.nv), torch.zeros_like(tau)
    rbd.integrate_vjp_(mech, qt, vt, tau, dt=DT, q_traj_bar=qtb, v_traj_bar=vtb, q0_bar_cfg=qc, v0_bar=vb, tau_bar=tb)
    torch.cuda.synchronize()
    assert torch.isfinite(qc).all() and torch.isfinite(vb).all() and torch.isfinite(tb).all()
    idx = torch.arange(7, B, B // 256, device="cuda")
    g = lambda x: x[..., idx].double().cpu().numpy()
    ref = host_ivjp(d, g(qt), g(vt), g(tau), n, g(qtb), g(vtb))
    for k, x in (("q0c", qc), ("v0b", vb), ("taub", tb)):
        assert rel_err(g(x), ref[k]) < TOL32, (k, rel_err(g(x), ref[k]))
