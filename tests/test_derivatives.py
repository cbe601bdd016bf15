"""Analytic Jacobians of forward dynamics (SURVEY 8(f) rank 3, csrc/rbd_deriv.cuh, rbd_dynamics_derivatives).

Oracle: the reference's own route -- dual numbers pushed through its dynamics! (oracle/rbd_oracle.hpp DualN<6>, CRBA + RNEA +
Cholesky in the world frame), seeded along velocity_to_configuration_derivative(e_k) -- and, independently of any dual-number
code, central finite differences of the oracle's plain fp64 dynamics along the same tangent directions.
CPU tier: the per-sample device functions compiled for the host (tests/hostsim).  GPU tier: the kernels through the C ABI."""
import os

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from oracle import Oracle
from tests import hostsim
from tests.util import axis_aligned_tree, double_pendulum, oracle_dynamics_derivatives, rand_inputs, randmech, rel_err

TOL64 = 1e-8          # parity with the oracle's DualN run in fp64
# fp32: a 36 x 36 factorisation in single precision.  Worst rel_err of the fp32 kernels against the fp64 run of the same code at the
# fp32-rounded inputs, 512 columns, measured on an H100 80GB HBM3 (700 W): 7.3e-4 on Atlas at B = 2^17; up to 1.2e-3 on Atlas with
# fixed tool bodies attached (tests/test_deriv_paths.py)
TOL32 = 2e-3


def _models():
    return [("double_pendulum", double_pendulum()), ("iiwa14", rbd.load_model("iiwa14", floating=False)),
            ("atlas_fixed", rbd.load_model("atlas", floating=False)), ("atlas", rbd.load_model("atlas", floating=True)),
            ("valkyrie", rbd.load_model("valkyrie", floating=True)), ("randmech0", randmech(0, shuffle=True)),
            ("randmech1", randmech(1, shuffle=True)), ("axis_aligned", axis_aligned_tree(3))]


@pytest.mark.parametrize("name,mech", _models(), ids=[n for n, _ in _models()])
def test_derivatives_hostsim_vs_oracle_duals(name, mech):
    d = mech.flatten()
    o = Oracle(d)
    q, v, tau, _, _ = rand_inputs(mech, 3, 11)
    rq, rv = oracle_dynamics_derivatives(o, mech, q, v, tau)
    vd, gq, gv = hostsim.dynamics_derivatives(d, q, v, tau)
    assert rel_err(vd, o.dynamics(q, v, tau)) < 1e-10
    assert rel_err(gq, rq) < TOL64 and rel_err(gv, rv) < TOL64, (rel_err(gq, rq), rel_err(gv, rv))
    # zero torques (the ConstVector default)
    rq0, rv0 = oracle_dynamics_derivatives(o, mech, q, v, np.zeros_like(tau))
    _, gq0, gv0 = hostsim.dynamics_derivatives(d, q, v, None)
    assert rel_err(gq0, rq0) < TOL64 and rel_err(gv0, rv0) < TOL64


def test_derivatives_match_finite_differences_of_plain_dynamics():
    """No dual numbers anywhere: central differences of the oracle's fp64 dynamics! along q ⊕ eps e_k (one Munthe-Kaas step of the
    oracle's integrator maps would do the same; here q + eps * q̇(e_k), renormalised to first order by construction) and v + eps e_k."""
    mech = randmech(2, shuffle=True)
    d = mech.flatten()
    o = Oracle(d)
    q, v, tau, _, _ = rand_inputs(mech, 2, 5)
    nv, B = d.nv, q.shape[1]
    _, gq, gv = hostsim.dynamics_derivatives(d, q, v, tau)
    eps = 1e-6
    fq = np.zeros((nv, nv, B)); fv = np.zeros((nv, nv, B))
    for k in range(nv):
        e = np.zeros((nv, B)); e[k] = 1.0
        qd = o.dynamics(q, e, tau, want_qd=True)[1]
        fq[:, k] = (o.dynamics(q + eps * qd, v, tau) - o.dynamics(q - eps * qd, v, tau)) / (2 * eps)
        fv[:, k] = (o.dynamics(q, v + eps * e, tau) - o.dynamics(q, v - eps * e, tau)) / (2 * eps)
    fq = fq.transpose(1, 0, 2).reshape(nv * nv, B); fv = fv.transpose(1, 0, 2).reshape(nv * nv, B)
    assert rel_err(gq, fq) < 2e-6 and rel_err(gv, fv) < 2e-6, (rel_err(gq, fq), rel_err(gv, fv))


def test_derivatives_hostsim_fp32():
    mech = rbd.load_model("atlas", floating=True)
    d = mech.flatten()
    o = Oracle(d)
    q, v, tau, _, _ = rand_inputs(mech, 3, 4)
    rq, rv = oracle_dynamics_derivatives(o, mech, q, v, tau)
    _, gq, gv = hostsim.dynamics_derivatives(d, q.astype(np.float32), v.astype(np.float32), tau.astype(np.float32))
    assert rel_err(gq, rq) < TOL32 and rel_err(gv, rv) < TOL32, (rel_err(gq, rq), rel_err(gv, rv))


def test_specialised_solve_kernel_compiles_without_a_gpu(tmp_path, monkeypatch):
    """The generator of the model-specialised solve kernel (csrc/rbd_deriv_jit.cpp) on mechanisms of different shapes -- 51
    coordinates with every joint type (one fp64 column per thread), Valkyrie, a serial chain, 66 coordinates (the high word of the
    relation masks) -- through NVRTC (no GPU needed); the cubins land in the cache directory."""
    from rigidbodydynamics.jl_b200 import _cabi
    from tests.test_deriv_paths import legs_model
    monkeypatch.setenv("RBD_JIT_CACHE", str(tmp_path))
    rng = np.random.default_rng(0)
    for mech in (randmech(6, shuffle=True), rbd.load_model("valkyrie", floating=True), rbd.rand_chain_mechanism(rng, [rbd.Revolute] * 30),
                 legs_model()):
        h = _cabi.ModelHandle(mech.flatten())
        for code in (_cabi.RBD_F64, _cabi.RBD_F32):
            try:
                h.precompile_derivatives(code)
            except _cabi.RbdError as e:
                if "NVRTC" in str(e):
                    pytest.skip("NVRTC not available")
                raise
        h.close()
    assert len([f for f in os.listdir(tmp_path) if "deriv" in f]) == 8
    # a 40-joint serial chain has 820 stored mass-matrix entries: in fp64 that does not fit into shared memory next to nothing
    # else -> RBD_EUNSUPPORTED, and rbd_dynamics_derivatives serves the model with the table-driven kernels
    h = _cabi.ModelHandle(rbd.rand_chain_mechanism(rng, [rbd.Revolute] * 40).flatten())
    with pytest.raises(_cabi.RbdError) as e:
        h.precompile_derivatives(_cabi.RBD_F64)
    assert e.value.status == _cabi.RBD_EUNSUPPORTED
    h.precompile_derivatives(_cabi.RBD_F32)
    h.close()


# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def built():
    import torch
    assert torch.cuda.is_available()
    rbd.load_library()
    return torch


def _gpu_run(torch, mech, q, v, tau, dtype):
    B = q.shape[1]
    st = rbd.MechanismState(mech, B, dtype)
    st.q.copy_(torch.from_numpy(q).to(dtype)); st.v.copy_(torch.from_numpy(v).to(dtype))
    t = None if tau is None else torch.from_numpy(tau).to(dtype).cuda()
    res = rbd.DynamicsResult(mech, B, dtype)
    nv = st.nv
    dq = torch.full((nv * nv, B), float("nan"), dtype=dtype, device="cuda")
    dv = torch.full((nv * nv, B), float("nan"), dtype=dtype, device="cuda")
    rbd.dynamics_derivatives_(dq, dv, res, st, t)
    torch.cuda.synchronize()
    return res.vd.double().cpu().numpy(), dq.double().cpu().numpy(), dv.double().cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("name,mech", _models(), ids=[n for n, _ in _models()])
@pytest.mark.parametrize("B", [1, 161])
def test_derivatives_gpu_vs_oracle(built, name, mech, B):
    torch = built
    o = Oracle(mech.flatten())
    q, v, tau, _, _ = rand_inputs(mech, B, 21)
    vd, gq, gv = _gpu_run(torch, mech, q, v, tau, torch.float64)
    n = min(B, 5)
    idx = np.linspace(0, B - 1, n).astype(int)
    rq, rv = oracle_dynamics_derivatives(o, mech, q[:, idx], v[:, idx], tau[:, idx])
    assert rel_err(vd, o.dynamics(q, v, tau)) < 1e-9
    assert not np.isnan(gq).any() and not np.isnan(gv).any()     # every entry is written, also the structural zeros
    assert rel_err(gq[:, idx], rq) < TOL64 and rel_err(gv[:, idx], rv) < TOL64, (rel_err(gq[:, idx], rq), rel_err(gv[:, idx], rv))
    # the device path and the host run of the same per-sample code agree to rounding
    _, hq, hv = hostsim.dynamics_derivatives(mech.flatten(), q[:, idx], v[:, idx], tau[:, idx])
    assert rel_err(gq[:, idx], hq) < 1e-10 and rel_err(gv[:, idx], hv) < 1e-10


@pytest.mark.gpu
def test_derivatives_gpu_fp32_and_chunks(built, monkeypatch):
    """fp32 at a batch that spans several chunks of the scratch (RBD_DERIV_SCRATCH_MB=4), ragged size, zero torques."""
    torch = built
    mech = rbd.load_model("atlas", floating=True)
    o = Oracle(mech.flatten())
    B = 3001
    q, v, tau, _, _ = rand_inputs(mech, B, 8)
    monkeypatch.setenv("RBD_DERIV_SCRATCH_MB", "4")
    idx = np.array([0, 1, 127, 128, 1500, 2999, 3000])
    rq, rv = oracle_dynamics_derivatives(o, mech, q[:, idx], v[:, idx], np.zeros_like(tau[:, idx]))
    for dtype, tol in ((torch.float64, TOL64), (torch.float32, TOL32)):
        vd, gq, gv = _gpu_run(torch, mech, q, v, None, dtype)
        assert not np.isnan(gq).any() and not np.isnan(gv).any()
        assert rel_err(gq[:, idx], rq) < tol and rel_err(gv[:, idx], rv) < tol, (dtype, rel_err(gq[:, idx], rq), rel_err(gv[:, idx], rv))


@pytest.mark.gpu
def test_derivatives_gpu_factor_in_scratch_fallback(built, monkeypatch):
    """Models whose mass matrix does not fit into shared memory next to the right-hand sides factor it on the scratch instead
    (deriv_factor_kernel + deriv_solve_kernel<T, false>); forced here on a random tree with every joint type."""
    torch = built
    mech = randmech(4, shuffle=True)
    o = Oracle(mech.flatten())
    q, v, tau, _, _ = rand_inputs(mech, 70, 9)
    idx = np.array([0, 31, 32, 69])
    rq, rv = oracle_dynamics_derivatives(o, mech, q[:, idx], v[:, idx], tau[:, idx])
    monkeypatch.setenv("RBD_DERIV_GLOBAL_FACTOR", "1")
    _, gq, gv = _gpu_run(torch, mech, q, v, tau, torch.float64)
    assert rel_err(gq[:, idx], rq) < TOL64 and rel_err(gv[:, idx], rv) < TOL64


@pytest.mark.gpu
@pytest.mark.parametrize("jit", ["0", "1"])
def test_derivatives_gpu_specialised_and_generic_solve_kernels(built, monkeypatch, jit):
    """The triangular solves exist twice: the table-driven kernel and the model-specialised one (right-hand sides in registers,
    NVRTC).  Both against the oracle, fp64 and fp32, on Atlas and on a random tree with every joint type (51 coordinates)."""
    torch = built
    from rigidbodydynamics.jl_b200 import _cabi
    monkeypatch.setenv("RBD_DERIV_JIT", jit)
    for mech in (rbd.load_model("atlas", floating=True), randmech(5, shuffle=True)):
        o = Oracle(mech.flatten())
        q, v, tau, _, _ = rand_inputs(mech, 97, 13)
        idx = np.array([0, 31, 32, 96])
        rq, rv = oracle_dynamics_derivatives(o, mech, q[:, idx], v[:, idx], tau[:, idx])
        for dtype, code, tol in ((torch.float64, _cabi.RBD_F64, TOL64), (torch.float32, _cabi.RBD_F32, TOL32)):
            if jit == "1":
                st = rbd.MechanismState(mech, 1, dtype)
                st.handle.precompile_derivatives(code)          # cached cubin => used at any batch size
            _, gq, gv = _gpu_run(torch, mech, q, v, tau, dtype)
            assert not np.isnan(gq).any() and not np.isnan(gv).any()
            assert rel_err(gq[:, idx], rq) < tol and rel_err(gv[:, idx], rv) < tol, (jit, dtype, rel_err(gq[:, idx], rq), rel_err(gv[:, idx], rv))


@pytest.mark.gpu
def test_derivatives_gpu_consistent_with_dual_entry_point(built):
    """The analytic Jacobians contracted with six seed directions == the library's own Dual{Float64,6} sweep (config 4)."""
    torch = built
    from tests.util import make_duals
    mech = rbd.load_model("atlas", floating=False)     # 1-DoF joints only: raw-coordinate partials are tangent partials
    B = 64
    q, v, tau, _, _ = rand_inputs(mech, B, 2)
    Q, V, T = make_duals(mech, q, v, np.zeros_like(tau), 3)
    T[..., 1:] = 0.0
    st = rbd.MechanismState(mech, B, torch.float64)
    out = torch.empty((st.nv, B, 7), dtype=torch.float64, device="cuda")
    rbd.dynamics_dual_(out, st, torch.from_numpy(Q).cuda(), torch.from_numpy(V).cuda(), torch.from_numpy(T).cuda())
    torch.cuda.synchronize()
    _, gq, gv = _gpu_run(torch, mech, q, v, np.zeros_like(tau), torch.float64)
    nv = st.nv
    Jq = gq.reshape(nv, nv, B).transpose(1, 0, 2); Jv = gv.reshape(nv, nv, B).transpose(1, 0, 2)   # [i, j, b]
    want = np.einsum("ijb,jbk->ibk", Jq, Q[..., 1:]) + np.einsum("ijb,jbk->ibk", Jv, V[..., 1:])
    got = out.cpu().numpy()[..., 1:]
    assert np.abs(got - want).max() / max(1.0, np.abs(want).max()) < 1e-9
