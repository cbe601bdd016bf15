"""Linearisation of recorded RK4 steps: rbd_integrate_derivatives (csrc/rbd_integrate_deriv.cuh, csrc/rbd_integrate_deriv.cu) and
rigidbodydynamics.jl_b200.autodiff.integrate_derivatives.

A_s = ∂x_{s+1}/∂x_s and B_s = ∂x_{s+1}/∂τ_s, x = (q, v), configuration columns along q̇ = N(q) e_j and rows through N⁺(q_{s+1}).
CPU tier: the per-joint maps against central differences, the whole step run on the CPU (tests/hostsim/hostsim_integrate_deriv.cpp)
against central differences of the oracle's fp64 `integrate`, the exact identity with the rollout VJP's CPU run, a closed form, and
the argument refusals.  GPU tier: the kernels against that CPU run, the identity with rbd_integrate_vjp, torch.autograd, and the
paths (chunks, generic solve, flattened batch)."""
import ctypes
import functools

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from oracle import Oracle
from rigidbodydynamics.jl_b200._cabi import RbdModelDesc, make_desc
from tests import hostsim
from tests.test_integrate_vjp import DT, NQ, NV, K_FIXED, _joint_point, host_ivjp, host_traj
from tests.test_integrate_vjp import _shim as vjp_shim
from tests.test_vjp import _qdot_dirs
from tests.util import double_pendulum, rand_inputs, randmech, rel_err

# central differences of the fp64 oracle at eps = 1e-5, as tests/test_integrate_vjp.py's (their error on Atlas is about 1e-7)
TOL_FD = 1e-6
EPS_FD = 1e-5
TOL64 = 1e-10        # kernels against the CPU run of the same code, fp64; the identity with the rollout VJP
# fp32 kernels against the fp64 CPU run at the fp32 trajectory: measured worst rel_err 3.8e-4 on the H100 (Atlas, B = 161, 5 steps,
# test_kernels_vs_hostsim); the bound is about 5x that
TOL32 = 2e-3


@functools.cache
def _shim():
    """tests/hostsim/hostsim_integrate_deriv.cpp, compiled and loaded by hostsim.shim."""
    lib = hostsim.shim("hostsim_integrate_deriv")
    vp, i64, c_int, c_double = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_double
    lib.hostsim_integrate_derivatives.argtypes = [ctypes.POINTER(RbdModelDesc), c_int, i64, vp, vp, vp, i64, c_double, c_int, vp, vp]
    lib.hostsim_joint_g_jvp.argtypes = [c_int] + [vp] * 6
    lib.hostsim_joint_l_jvp.argtypes = [c_int] + [vp] * 7
    lib.hostsim_joint_vel_to_cfg.argtypes = [c_int] + [vp] * 3
    lib.hostsim_joint_cfg_to_vel.argtypes = [c_int] + [vp] * 3
    return lib


def _p(a):
    """a pointer that keeps its array alive through the call (arguments here are often temporaries)"""
    return None if a is None or a.size == 0 else a.ctypes.data_as(ctypes.c_void_p)


def host_lin(desc, qt, vt, tau, n, dt=DT):
    """The CPU run of rbd_integrate_derivatives: (A [n, 2nv, 2nv, B], B [n, 2nv, nv, B]) indexed [s, i, j, b]."""
    dt_ = qt.dtype
    B, nv = qt.shape[2], desc.nv
    t = None if tau is None else np.ascontiguousarray(tau, dt_)
    step = 0 if tau is None or tau.ndim == 2 else nv * B
    A = np.full((n, 4 * nv * nv, B), np.nan, dt_)
    Bm = np.full((n, 2 * nv * nv, B), np.nan, dt_)
    d, keep = make_desc(desc)
    assert _shim().hostsim_integrate_derivatives(ctypes.byref(d), 0 if dt_ == np.float32 else 1, B, _p(np.ascontiguousarray(qt, dt_)),
                                                 _p(np.ascontiguousarray(vt, dt_)), _p(t), step, dt, n, _p(A), _p(Bm)) == 0
    return A.reshape(n, 2 * nv, 2 * nv, B).transpose(0, 2, 1, 3), Bm.reshape(n, nv, 2 * nv, B).transpose(0, 2, 1, 3)


def _kinds(d):
    return [int(d.jtype[i]) for i in range(d.nb)]


def cfg_to_vel(d, q, dq):
    """N⁺(q) dq per joint of the flattened model: [nq, B] -> [nv, B]"""
    lib = _shim()
    out = np.zeros((d.nv, q.shape[1]))
    qr = vr = 0
    for kind in _kinds(d):
        nq, nv = NQ[kind], NV[kind]
        for b in range(q.shape[1]):
            o = np.zeros(nv)
            if nv:
                lib.hostsim_joint_cfg_to_vel(kind, _p(np.ascontiguousarray(q[qr:qr + nq, b])), _p(np.ascontiguousarray(dq[qr:qr + nq, b])), _p(o))
            out[vr:vr + nv, b] = o
        qr += nq; vr += nv
    return out


def _models():
    return [("double_pendulum", double_pendulum()), ("iiwa14", rbd.load_model("iiwa14", floating=False)),
            ("atlas", rbd.load_model("atlas", floating=True)), ("randmech0", randmech(0, shuffle=True)),
            ("randmech1", randmech(1, shuffle=True))]


# ----------------------------------------------------------------------------------------------------------------------
# CPU tier
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", [k for k in range(8) if k != K_FIXED])
@pytest.mark.parametrize("scale", [1e-4, 0.7], ids=["taylor", "closed_form"])
def test_joint_maps_match_finite_differences(kind, scale):
    """The Jacobian blocks of G and L taken through their Dual1 JVPs (unit seeds) against central differences of the same fp64
    maps, on the Taylor branch and the closed forms; N⁺ N = I and N⁺ of a finite-difference q̇ along N e_k."""
    lib = _shim()
    rng = np.random.default_rng(kind + int(scale * 10))
    nq, nv = NQ[kind], NV[kind]
    eps = 1e-7
    e = lambda n, k: np.eye(n)[k]
    z = lambda n: np.zeros(n)
    for _ in range(3):
        q0, phi, vs = _joint_point(kind, rng, scale)

        def G(a, b):
            qs, dqs = np.zeros(nq), np.zeros(nq)
            lib.hostsim_joint_g_jvp(kind, _p(a), _p(z(nq)), _p(b), _p(z(nv)), _p(qs), _p(dqs))
            return qs

        Lr = lambda a, b, c: (vjp_shim().hostsim_joint_rate(kind, _p(a), _p(b), _p(c), _p(out := np.zeros(nv))), out)[1]
        qs = G(q0, phi)
        for k in range(nq + nv):
            dq0, dphi = (e(nq, k), z(nv)) if k < nq else (z(nq), e(nv, k - nq))
            got_qs, got = np.zeros(nq), np.zeros(nq)
            lib.hostsim_joint_g_jvp(kind, _p(q0), _p(dq0), _p(phi), _p(dphi), _p(got_qs), _p(got))
            ref = (G(q0 + eps * dq0, phi + eps * dphi) - G(q0 - eps * dq0, phi - eps * dphi)) / (2 * eps)
            assert rel_err(got, ref) < 1e-7, ("G", k, got, ref)
            assert np.array_equal(got_qs, qs)
        for k in range(2 * nq + nv):
            dq0 = e(nq, k) if k < nq else z(nq)
            dqs = e(nq, k - nq) if nq <= k < 2 * nq else z(nq)
            dvs = e(nv, k - 2 * nq) if k >= 2 * nq else z(nv)
            got = np.zeros(nv)
            lib.hostsim_joint_l_jvp(kind, _p(q0), _p(dq0), _p(qs), _p(dqs), _p(vs), _p(dvs), _p(got))
            ref = (Lr(q0 + eps * dq0, qs + eps * dqs, vs + eps * dvs) - Lr(q0 - eps * dq0, qs - eps * dqs, vs - eps * dvs)) / (2 * eps)
            assert rel_err(got, ref) < 1e-7, ("L", k, got, ref)
        # N⁺(q) N(q) = I at the unit configurations of _joint_point, and at the stage configuration
        for q in (q0, qs):
            for k in range(nv):
                qd, back = np.zeros(nq), np.zeros(nv)
                lib.hostsim_joint_vel_to_cfg(kind, _p(q), _p(e(nv, k)), _p(qd))
                lib.hostsim_joint_cfg_to_vel(kind, _p(q), _p(qd), _p(back))
                assert rel_err(back, e(nv, k)) < 1e-12, (k, back)


def test_vel_to_cfg_matches_the_oracle():
    """N(q) e_k of every joint against the oracle's velocity_to_configuration_derivative on a tree with every joint type."""
    mech = randmech(2, shuffle=True)
    d = mech.flatten()
    o = Oracle(d)
    q, _, _, _, _ = rand_inputs(mech, 2, 3)
    ref = _qdot_dirs(o, q, d.nv, None)
    lib = _shim()
    qr = vr = 0
    for kind in _kinds(d):
        nq, nv = NQ[kind], NV[kind]
        for k in range(nv):
            for b in range(2):
                qd = np.zeros(nq)
                lib.hostsim_joint_vel_to_cfg(kind, _p(np.ascontiguousarray(q[qr:qr + nq, b])), _p(np.eye(nv)[k]), _p(qd))
                assert np.abs(qd - ref[vr + k, qr:qr + nq, b]).max() < 1e-14
        qr += nq; vr += nv


def _fd_step(o, d, q, v, tau_s, eps=EPS_FD):
    """[A B] of one oracle step at (q, v) by central differences: [2nv, 3nv, B]"""
    B = q.shape[1]
    dirs_q = _qdot_dirs(o, q, d.nv, None)
    cols = []
    t0 = np.zeros((d.nv, B)) if tau_s is None else tau_s
    q1, _ = o.integrate(q, v, t0, dt=DT, nsteps=1)
    for k in range(3 * d.nv):
        def f(h):
            qq, vv, tt = q.copy(), v.copy(), t0.copy()
            if k < d.nv:
                qq = q + h * dirs_q[k]
            elif k < 2 * d.nv:
                vv[k - d.nv] += h
            else:
                tt[k - 2 * d.nv] += h
            return o.integrate(qq, vv, tt, dt=DT, nsteps=1)
        (qp, vp), (qm, vm) = f(eps), f(-eps)
        cols.append(np.concatenate([cfg_to_vel(d, q1, (qp - qm) / (2 * eps)), (vp - vm) / (2 * eps)]))
    return np.stack(cols, 1)


@pytest.mark.parametrize("name,mech", _models(), ids=[n for n, _ in _models()])
@pytest.mark.parametrize("tmode", ["none", "const", "step"])
def test_hostsim_matches_oracle_finite_differences(name, mech, tmode):
    d = mech.flatten()
    o = Oracle(d)
    n, B = 2, 2
    q, v, tau, _, _ = rand_inputs(mech, B, 5)
    rng = np.random.default_rng(6)
    tau = {"none": None, "const": tau, "step": rng.standard_normal((n, d.nv, B))}[tmode]
    qt, vt = host_traj(d, q, v, tau, n)
    A, Bm = host_lin(d, qt, vt, tau, n)
    for s in range(n):
        ts = None if tau is None else (tau if tau.ndim == 2 else tau[s])
        ref = _fd_step(o, d, qt[s], vt[s], ts)
        got = np.concatenate([A[s], Bm[s]], 1)
        assert np.isfinite(got).all()
        err = rel_err(got.reshape(-1, B), ref.reshape(-1, B))
        assert err < TOL_FD, (s, err)


def _vjp_identity(d, qt, vt, tau, A, Bm, rng):
    """ȳᵀ [A_0 B_0] against the rollout VJP's CPU run for one step seeded with q_traj_bar[1] = g, v_traj_bar[1] = ȳ_v, where
    ȳ_q = N(q1)ᵀ g; returns the largest relative error."""
    B = qt.shape[2]
    g, yv = rng.standard_normal((d.nq, B)), rng.standard_normal((d.nv, B))
    qtb, vtb = np.zeros((2, d.nq, B)), np.zeros((2, d.nv, B))
    qtb[1], vtb[1] = g, yv
    r = host_ivjp(d, qt[:2], vt[:2], None if tau is None else (tau if tau.ndim == 2 else tau[:1]), 1, qtb, vtb)
    # ȳ_q = N(q1)ᵀ g, the tangent form of g at q1: the zero-step VJP's q0_bar_tan
    yq = host_ivjp(d, qt[1:2], vt[1:2], None, 0, qtb[1:2], vtb[1:2])["q0t"]
    y = np.concatenate([yq, yv])
    lhs = np.einsum("ib,ijb->jb", y, np.concatenate([A[0], Bm[0]], 1))
    ref = np.concatenate([r["q0t"], r["v0b"], r["taub"] if tau is not None else np.zeros((d.nv, B))])
    return rel_err(lhs, ref)


@pytest.mark.parametrize("name,mech", _models(), ids=[n for n, _ in _models()])
def test_hostsim_vjp_identity(name, mech):
    """ȳᵀ [A B] equals rbd_integrate_vjp's (q0_bar_tan, v0_bar, tau_bar) of one step, to rounding."""
    d = mech.flatten()
    B = 3
    q, v, tau, _, _ = rand_inputs(mech, B, 9)
    qt, vt = host_traj(d, q, v, tau, 1)
    A, Bm = host_lin(d, qt, vt, tau, 1)
    assert _vjp_identity(d, qt, vt, tau, A, Bm, np.random.default_rng(1)) < TOL64


def test_closed_form_prismatic_under_gravity():
    """One prismatic joint of mass m along gravity: RK4 integrates the constant acceleration exactly, so
    A = [[1, dt], [0, 1]] and B = [dt²/2m; dt/m]."""
    m, g = 2.5, -9.81
    mech = rbd.Mechanism(rbd.RigidBody("world"), gravity=(0, 0, g))
    body = rbd.RigidBody("slider", rbd.SpatialInertia(0.1 * np.eye(3), None, m, com=[0, 0, 0]))
    mech.attach(mech.root_body, body, rbd.Joint("z", rbd.Prismatic(np.array([0.0, 0.0, 1.0]))))
    d = mech.flatten()
    B, n, dt = 3, 3, 0.01
    rng = np.random.default_rng(0)
    q, v, tau = rng.standard_normal((1, B)), rng.standard_normal((1, B)), rng.standard_normal((n, 1, B))
    qt, vt = host_traj(d, q, v, tau, n, dt=dt)
    A, Bm = host_lin(d, qt, vt, tau, n, dt=dt)
    refA = np.array([[1.0, dt], [0.0, 1.0]])[None, :, :, None]
    refB = np.array([[dt * dt / (2 * m)], [dt / m]])[None, :, :, None]
    assert np.abs(A - refA).max() < 1e-14 and np.abs(Bm - refB).max() < 1e-14, (A[..., 0], Bm[..., 0])


def test_refusals_before_any_cuda_call():
    """Every argument error returns its status from the checks, which run before any CUDA call (this test needs no GPU)."""
    from rigidbodydynamics.jl_b200 import _cabi
    try:
        from rigidbodydynamics.jl_b200.state import _model_handle
        lib = _cabi.load_library()
        h = _model_handle(rbd.load_model("iiwa14", floating=False))
    except Exception as e:          # the library is built by build(); without it there is nothing to check here
        pytest.skip(f"library not loadable: {e}")
    B, n = 4, 2
    x = ctypes.c_void_p(8)           # never dereferenced: every call below fails its checks first
    call = lambda dtype=_cabi.RBD_F64, qt=x, vt=x, step=0, stage=0, dt=DT, n_=n, A=x, Bm=x, B_=B: lib.rbd_integrate_derivatives(
        h.ptr, dtype, B_, qt, vt, None, step, stage, dt, n_, A, Bm, None)
    assert call(dtype=_cabi.RBD_DUAL64X6) == _cabi.RBD_EUNSUPPORTED
    assert call(stage=8) == _cabi.RBD_EINVAL
    assert call(step=-1) == _cabi.RBD_EINVAL
    assert call(n_=-1) == _cabi.RBD_EINVAL
    assert call(dt=0.0) == _cabi.RBD_EINVAL and call(dt=-1e-3) == _cabi.RBD_EINVAL
    assert call(A=None, Bm=None) == _cabi.RBD_EINVAL
    assert call(qt=None) == _cabi.RBD_EINVAL and call(vt=None) == _cabi.RBD_EINVAL
    assert call(B_=0) == _cabi.RBD_OK and call(n_=0) == _cabi.RBD_OK


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
    return t, qt, vt


np64 = lambda x: x.double().cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("name,mech", _models(), ids=[n for n, _ in _models()])
@pytest.mark.parametrize("B", [1, 161])
def test_kernels_vs_hostsim(torch, name, mech, B):
    """fp64 against the CPU run of the same code; fp32 against the fp64 CPU run at the fp32 trajectory."""
    d = mech.flatten()
    q, v, _, _, _ = rand_inputs(mech, B, 7)
    rng = np.random.default_rng(B)
    worst = 0.0
    for n in (1, 5):
        for tmode, tau in {"none": None, "const": rng.standard_normal((d.nv, B)), "step": rng.standard_normal((n, d.nv, B))}.items():
            for dtype in (torch.float64, torch.float32):
                t, qt, vt = _gpu_traj(torch, mech, q, v, tau, n, dtype)
                A, Bm = rbd.autodiff.integrate_derivatives(mech, qt, vt, t, dt=DT)
                torch.cuda.synchronize()
                refA, refB = host_lin(d, np64(qt), np64(vt), None if t is None else np64(t), n)
                for got, ref in ((A, refA), (Bm, refB)):
                    err = rel_err(np64(got).reshape(-1, B), ref.reshape(-1, B))
                    if dtype == torch.float32:
                        worst = max(worst, err)
                    assert err < (TOL64 if dtype == torch.float64 else TOL32), (n, tmode, dtype, err)
    print(f"{name} B={B}: worst fp32 rel_err {worst:.3g}")


@pytest.mark.gpu
def test_vjp_identity_on_gpu(torch):
    """Atlas fp64: ȳᵀ[A B] of one step equals rbd_integrate_vjp; and ȳᵀ A_{N-1} ... A_0 equals the VJP of the whole N-step
    trajectory with a cotangent on the final state only (N = 8)."""
    mech = rbd.load_model("atlas", floating=True)
    d = mech.flatten()
    B, N = 33, 8
    q, v, tau, _, _ = rand_inputs(mech, B, 4)
    rng = np.random.default_rng(2)
    t, qt, vt = _gpu_traj(torch, mech, q, v, rng.standard_normal((N, d.nv, B)), N, torch.float64)
    A, Bm = rbd.autodiff.integrate_derivatives(mech, qt, vt, t, dt=DT)
    g, yv = torch.randn(d.nq, B, dtype=torch.float64, device="cuda"), torch.randn(d.nv, B, dtype=torch.float64, device="cuda")
    yq = torch.empty(d.nv, B, dtype=torch.float64, device="cuda")
    qtb, vtb = torch.zeros_like(qt), torch.zeros_like(vt)
    qtb[-1], vtb[-1] = g, yv
    rbd.integrate_vjp_(mech, qt[-1:].contiguous(), vt[-1:].contiguous(), None, dt=DT, q_traj_bar=qtb[-1:].contiguous(), q0_bar_tan=yq)
    y = torch.cat([yq, yv])
    # one step: the last one, seeded on its end state
    q0t, v0b, tb = torch.empty_like(yq), torch.empty_like(yv), torch.zeros_like(t[N - 1:])
    rbd.integrate_vjp_(mech, qt[N - 1:].contiguous(), vt[N - 1:].contiguous(), t[N - 1:].contiguous(), dt=DT,
                       q_traj_bar=qtb[N - 1:].contiguous(), v_traj_bar=vtb[N - 1:].contiguous(), q0_bar_tan=q0t, v0_bar=v0b, tau_bar=tb)
    lhs = torch.einsum("ib,ijb->jb", y, torch.cat([A[N - 1], Bm[N - 1]], 1))
    assert rel_err(np64(lhs), np64(torch.cat([q0t, v0b, tb[0]]))) < TOL64
    # the chain
    z = y
    for s in reversed(range(N)):
        z = torch.einsum("ib,ijb->jb", z, A[s])
    rbd.integrate_vjp_(mech, qt, vt, t, dt=DT, q_traj_bar=qtb, v_traj_bar=vtb, q0_bar_tan=q0t, v0_bar=v0b)
    assert rel_err(np64(z), np64(torch.cat([q0t, v0b]))) < TOL64


@pytest.mark.gpu
def test_autograd_jacobian_of_one_step(torch):
    """torch.autograd.functional.jacobian of one step of autodiff.simulate on a revolute-only tree (configuration = tangent)."""
    from rigidbodydynamics.jl_b200 import autodiff
    mech = rbd.rand_tree_mechanism(np.random.default_rng(4), [rbd.Revolute] * 6)
    d = mech.flatten()
    B = 2
    q, v, tau, _, _ = rand_inputs(mech, B, 1)
    T = lambda a: torch.from_numpy(a).cuda()
    tq, tv, tt = T(q), T(v), T(tau)
    f = lambda a, b, c: torch.cat(autodiff.simulate(mech, a, b, c, dt=DT, nsteps=1, trajectory=False))
    J = torch.autograd.functional.jacobian(f, (tq, tv, tt))          # each [2nv, B, rows, B]
    _, qt, vt = _gpu_traj(torch, mech, q, v, None, 1, torch.float64)
    qt, vt = autodiff._trajectory(rbd.state._model_handle(mech), tq, tv, tt, 0, 1, 0, 0, DT)
    A, Bm = rbd.autodiff.integrate_derivatives(mech, qt, vt, tt, dt=DT)
    for b in range(B):
        ref = torch.cat([J[0][:, b, :, b], J[1][:, b, :, b], J[2][:, b, :, b]], 1)
        got = torch.cat([A[0, :, :, b], Bm[0, :, :, b]], 1)
        assert rel_err(np64(got), np64(ref)) < TOL64, b


def _lin(torch, mech, qt, vt, t):
    A, Bm = rbd.autodiff.integrate_derivatives(mech, qt, vt, t, dt=DT)
    torch.cuda.synchronize()
    return A.contiguous(), Bm.contiguous()


@pytest.mark.gpu
def test_chunks_and_flattened_batch_bitwise(torch, monkeypatch):
    """A tree with a fixed joint, the generic solve and fewer than 1024 pairs, so that the recompute takes rbd_integrate's
    per-sample stage kernels whatever the chunk (it vectorises the revolute rows of batches of 1024 and more): a small
    RBD_DERIV_SCRATCH_MB (many chunks) equals one chunk bit for bit, and so do per-step calls and the flattened batch."""
    monkeypatch.setenv("RBD_DERIV_JIT", "0")
    mech = randmech(0, shuffle=True)
    d = mech.flatten()
    B, n = 16, 63
    q, v, _, _, _ = rand_inputs(mech, B, 3)
    rng = np.random.default_rng(5)
    for dtype in (torch.float64, torch.float32):
        t, qt, vt = _gpu_traj(torch, mech, q, v, rng.standard_normal((n, d.nv, B)), n, dtype)
        one = _lin(torch, mech, qt, vt, t)
        monkeypatch.setenv("RBD_DERIV_SCRATCH_MB", "1")
        many = _lin(torch, mech, qt, vt, t)
        monkeypatch.delenv("RBD_DERIV_SCRATCH_MB")
        assert torch.equal(one[0], many[0]) and torch.equal(one[1], many[1])
        for s in (0, 1, 37, n - 1):
            A, Bm = _lin(torch, mech, qt[s:s + 2].contiguous(), vt[s:s + 2].contiguous(), t[s:s + 1].contiguous())
            assert torch.equal(A[0], one[0][s]) and torch.equal(Bm[0], one[1][s]), s


@pytest.mark.gpu
def test_mpc_shape_matches_per_step_calls(torch):
    """100 steps x 16 samples, run as one batch of 1600 pairs, against 100 calls of one step: equal to rounding (the recompute of
    the large batch takes the vectorised stage kernels of rbd_integrate, the per-step calls the per-sample ones)."""
    mech = rbd.load_model("atlas", floating=True)
    d = mech.flatten()
    B, n = 16, 100
    q, v, _, _, _ = rand_inputs(mech, B, 6)
    rng = np.random.default_rng(7)
    for dtype, tol in ((torch.float64, 1e-12), (torch.float32, 1e-4)):
        t, qt, vt = _gpu_traj(torch, mech, q, v, rng.standard_normal((n, d.nv, B)), n, dtype)
        one = _lin(torch, mech, qt, vt, t)
        worst = 0.0
        for s in range(n):
            A, Bm = _lin(torch, mech, qt[s:s + 2].contiguous(), vt[s:s + 2].contiguous(), t[s:s + 1].contiguous())
            for got, ref in ((A[0], one[0][s]), (Bm[0], one[1][s])):
                worst = max(worst, rel_err(np64(got).reshape(-1, B), np64(ref).reshape(-1, B)))
        print(f"{dtype}: flattened vs per-step calls, worst rel_err {worst:.3g}")
        assert worst < tol


@pytest.mark.gpu
def test_generic_solve_and_large_batch(torch, monkeypatch):
    """Atlas fp64, 2^13 samples x 2 steps (the specialised solve, and grids of several passes): the generic solve (RBD_DERIV_JIT=0)
    agrees with it, and sampled columns agree with the CPU run."""
    mech = rbd.load_model("atlas", floating=True)
    d = mech.flatten()
    B, n = 1 << 13, 2
    q, v, tau, _, _ = rand_inputs(mech, B, 8)
    t, qt, vt = _gpu_traj(torch, mech, q, v, tau, n, torch.float64)
    spec = _lin(torch, mech, qt, vt, t)
    monkeypatch.setenv("RBD_DERIV_JIT", "0")
    gen = _lin(torch, mech, qt, vt, t)
    for a, b in zip(spec, gen):
        assert rel_err(np64(a).reshape(-1, B), np64(b).reshape(-1, B)) < 1e-9
    cols = np.array([0, 1, 31, 32, 4095, 4096, B - 1])
    refA, refB = host_lin(d, np64(qt)[..., cols], np64(vt)[..., cols], np64(t)[..., cols], n)
    assert rel_err(np64(spec[0])[..., cols].reshape(-1, len(cols)), refA.reshape(-1, len(cols))) < TOL64
    assert rel_err(np64(spec[1])[..., cols].reshape(-1, len(cols)), refB.reshape(-1, len(cols))) < TOL64


@pytest.mark.gpu
def test_python_refusals(torch):
    mech = rbd.load_model("iiwa14", floating=False)
    d = mech.flatten()
    B, n = 4, 2
    q, v, _, _, _ = rand_inputs(mech, B, 1)
    _, qt, vt = _gpu_traj(torch, mech, q, v, None, n, torch.float64)
    stage = torch.zeros(n, 4, d.nv, B, dtype=torch.float64, device="cuda")
    with pytest.raises(ValueError):
        rbd.autodiff.integrate_derivatives_(mech, qt, vt, stage, dt=DT, A_out=torch.empty(n, 4 * d.nv ** 2, B, dtype=torch.float64,
                                                                                            device="cuda"))
    with pytest.raises(ValueError):
        rbd.autodiff.integrate_derivatives_(mech, qt, vt, None, dt=DT)
    with pytest.raises(rbd.DimensionMismatch):
        rbd.autodiff.integrate_derivatives_(mech, qt, vt, None, dt=DT, B_out=torch.empty(n, 3, B, dtype=torch.float64, device="cuda"))
    # B only: equals the B of a call with both
    Bm = torch.empty(n, 2 * d.nv ** 2, B, dtype=torch.float64, device="cuda")
    rbd.autodiff.integrate_derivatives_(mech, qt, vt, None, dt=DT, B_out=Bm)
    _, ref = _lin(torch, mech, qt, vt, None)
    assert torch.equal(Bm.view(n, d.nv, 2 * d.nv, B).transpose(1, 2), ref)
