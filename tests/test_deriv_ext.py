"""Analytic Jacobians with external wrenches, d v̇ / d tau, and the Jacobians of inverse dynamics (csrc/rbd_deriv.cuh,
rbd_dynamics_derivatives_ext, rbd_inverse_dynamics_derivatives).

Oracles, none of them dual numbers: central differences of the oracle's plain fp64 dynamics / inverse_dynamics along
q + eps q̇(e_k) and v + eps e_k, the oracle's mass matrix and its inverse, and the reverse modes (the host VJP of tests/test_vjp.py),
whose products with any cotangent the Jacobians must reproduce.
CPU tier: the per-sample device functions compiled for the host (tests/hostsim/hostsim_deriv_ext.cpp), the NVRTC generator and the
argument checks.  GPU tier: the kernels through the C ABI on every path, fp32, and the Python wrappers."""
import ctypes
import functools
import os

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from oracle import Oracle
from rigidbodydynamics.jl_b200 import _cabi
from rigidbodydynamics.jl_b200._cabi import RbdModelDesc, make_desc
from tests import hostsim
from tests.test_derivatives import TOL32, _models
from tests.test_deriv_paths import atlas, iiwa14, legs_model, tables, tooled
from tests.test_vjp import _contract, host_vjp
from tests.test_vjp_paths import _dev, cols, rand_q
from tests.util import axis_aligned_tree, rand_inputs, randmech, rel_err

TOL_FD = 2e-6         # central differences, eps = 1e-6
TOL_CPU = 1e-10       # GPU against the CPU run of the same per-sample code, fp64; also exact identities in fp64
# fp32 against the fp64 run of the same code at the fp32-rounded inputs, with external wrenches, 512 columns, measured on an H100 80GB
# HBM3 (700 W).  Atlas at 2^14: d v̇ / dq 5.8e-4, d v̇ / dv 7.3e-4, d v̇ / d tau 5.8e-4 (bound: the derivative tests' TOL32); the
# inverse-dynamics Jacobians, which involve no factorisation: d tau / dq 4.2e-7, d tau / dv 8.1e-7, tau 1.0e-6, M 2.7e-7 (bound 1e-5).
# Atlas with seven fixed tool bodies at 63437 samples: 2.1e-3 for the forward Jacobians (bound TOL32_TOOLS).
TOL32_ID = 1e-5
TOL32_TOOLS = 4e-3


@functools.cache
def _shim():
    """tests/hostsim/hostsim_deriv_ext.cpp, compiled and loaded by hostsim.shim."""
    lib = hostsim.shim("hostsim_deriv_ext")
    lib.hostsim_deriv_ext.argtypes = [ctypes.POINTER(RbdModelDesc), ctypes.c_int, ctypes.c_int, ctypes.c_int64] + [ctypes.c_void_p] * 9
    return lib


def _run(desc, inverse, q, v, vd, wext, want_extra):
    dt = q.dtype
    d, keep = make_desc(desc)
    c = lambda a: None if a is None else np.ascontiguousarray(a, dt)      # noqa: E731
    q, v, vd, wext = c(q), c(v), c(vd), c(wext)
    B, nv = q.shape[1], desc.nv
    full = lambda rows: np.full((rows, B), np.nan, dt)                    # noqa: E731
    dq, dv = full(nv * nv), full(nv * nv)
    dtau = full(nv * nv) if want_extra and not inverse else None
    tau = full(nv) if want_extra and inverse else None
    M = full(nv * nv) if want_extra and inverse else None
    p = lambda a: None if a is None or a.size == 0 else a.ctypes.data    # noqa: E731
    rc = _shim().hostsim_deriv_ext(ctypes.byref(d), int(inverse), 0 if dt == np.float32 else 1, B, p(q), p(v), p(vd), p(wext), p(dq),
                                   p(dv), p(dtau), p(tau), p(M))
    assert rc == 0, rc
    return dq, dv, dtau, tau, M


def host_fd(desc, q, v, tau=None, wext=None, dtau=True):
    """The forward path on the CPU: (vd, dvd_dq, dvd_dv, dvd_dtau or None), v̇ from the device ABA run on the host."""
    vd = hostsim.dynamics(desc, q, v, tau, wext)
    dq, dv, dt, _, _ = _run(desc, False, q, v, vd, wext, dtau)
    return vd, dq, dv, dt


def host_id(desc, q, v, vd, wext=None):
    """The inverse path on the CPU: (dtau_dq, dtau_dv, tau, M)."""
    dq, dv, _, tau, M = _run(desc, True, q, v, vd, wext, True)
    return dq, dv, tau, M


def _mat(J, nv):
    """[nv*nv, B] (entry (i, j) at row i + j*nv) -> [B, nv, nv]."""
    return J.reshape(nv, nv, -1).transpose(2, 1, 0)


def _flat(A):
    """[B, nv, nv] -> [nv*nv, B]."""
    return A.transpose(2, 1, 0).reshape(A.shape[1] * A.shape[2], A.shape[0])


def _fd_jacobians(o, f, q, v, nv):
    """Central differences of f(q, v) -> [nv, B] along q + eps q̇(e_k) and v + eps e_k, as [nv*nv, B] each."""
    B, eps = q.shape[1], 1e-6
    fq = np.zeros((nv, nv, B)); fv = np.zeros((nv, nv, B))
    for k in range(nv):
        e = np.zeros((nv, B)); e[k] = 1.0
        qd = o.dynamics(q, e, None, want_qd=True)[1]
        fq[:, k] = (f(q + eps * qd, v) - f(q - eps * qd, v)) / (2 * eps)
        fv[:, k] = (f(q, v + eps * e) - f(q, v - eps * e)) / (2 * eps)
    return fq.transpose(1, 0, 2).reshape(nv * nv, B), fv.transpose(1, 0, 2).reshape(nv * nv, B)


def _fd_models():
    return [("randmech2", randmech(2, shuffle=True)), ("randmech7", randmech(7, shuffle=True)), ("axis_aligned", axis_aligned_tree(3)),
            ("atlas", atlas())]


# ----------------------------------------------------------------------------------------------------------------------
# CPU tier
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,mech", _fd_models(), ids=[n for n, _ in _fd_models()])
def test_forward_jacobians_with_wrenches_match_finite_differences(name, mech):
    d = mech.flatten()
    o = Oracle(d)
    q, v, tau, _, w = rand_inputs(mech, 2, 5, wext=True)
    vd, gq, gv, _ = host_fd(d, q, v, tau, w)
    assert rel_err(vd, o.dynamics(q, v, tau, w)) < 1e-10
    fq, fv = _fd_jacobians(o, lambda q_, v_: o.dynamics(q_, v_, tau, w), q, v, d.nv)
    assert rel_err(gq, fq) < TOL_FD and rel_err(gv, fv) < TOL_FD, (rel_err(gq, fq), rel_err(gv, fv))
    # the wrench term matters: without it the Jacobian is that of another function
    _, gq0, _, _ = host_fd(d, q, v, tau, None)
    assert rel_err(gq0, fq) > 1e3 * TOL_FD


@pytest.mark.parametrize("name,mech", _fd_models(), ids=[n for n, _ in _fd_models()])
def test_inverse_jacobians_match_finite_differences(name, mech):
    d = mech.flatten()
    o = Oracle(d)
    q, v, _, vd, w = rand_inputs(mech, 2, 8, wext=True)
    for wx in (None, w):
        gq, gv, tau, M = host_id(d, q, v, vd, wx)
        fq, fv = _fd_jacobians(o, lambda q_, v_: o.inverse_dynamics(q_, v_, vd, wx), q, v, d.nv)
        assert rel_err(gq, fq) < TOL_FD and rel_err(gv, fv) < TOL_FD, (wx is None, rel_err(gq, fq), rel_err(gv, fv))
        assert rel_err(tau, o.inverse_dynamics(q, v, vd, wx)) < TOL_CPU
        assert rel_err(M, o.mass_matrix(q)) < TOL_CPU


@pytest.mark.parametrize("name,mech", _models(), ids=[n for n, _ in _models()])
def test_dvd_dtau_is_the_inverse_mass_matrix(name, mech):
    d = mech.flatten()
    o = Oracle(d)
    q, v, tau, _, w = rand_inputs(mech, 3, 11, wext=True)
    _, _, _, Mi = host_fd(d, q, v, tau, w)
    ref = _flat(np.linalg.inv(_mat(o.mass_matrix(q), d.nv)))
    assert rel_err(Mi, ref) < TOL_CPU, rel_err(Mi, ref)


@pytest.mark.parametrize("name,mech", _fd_models(), ids=[n for n, _ in _fd_models()])
def test_forward_and_inverse_jacobians_are_related_by_the_inverse_mass_matrix(name, mech):
    """d v̇ / du = -M^-1 d ID / du at v̇ = FD(q, v, tau, wext), with both sides from the device code."""
    d = mech.flatten()
    q, v, tau, _, w = rand_inputs(mech, 3, 12, wext=True)
    vd, gq, gv, Mi = host_fd(d, q, v, tau, w)
    iq, iv, tau_id, M = host_id(d, q, v, vd, w)
    nv = d.nv
    assert rel_err(tau_id, tau) < TOL_CPU                      # ID(FD(tau)) = tau
    for g, i in ((gq, iq), (gv, iv)):
        want = _flat(-np.einsum("bij,bjk->bik", _mat(Mi, nv), _mat(i, nv)))
        assert rel_err(g, want) < TOL_CPU, rel_err(g, want)
    eye = np.einsum("bij,bjk->bik", _mat(Mi, nv), _mat(M, nv))
    assert np.abs(eye - np.eye(nv)).max() < TOL_CPU


def test_contraction_with_the_reverse_modes():
    """The Jacobians contracted with a cotangent equal the VJP kernels' per-sample code (tests/test_vjp.py's host_vjp), wrenches
    included: ν̄^T dvd_dq = q_bar_tan, ν̄^T dvd_dv = v_bar, (dvd_dtau)^T ν̄ = tau_bar; τ̄^T dtau_dq = q_bar_tan, τ̄^T dtau_dv = v_bar,
    M τ̄ = vd_bar."""
    mech = randmech(3, shuffle=True)
    d = mech.flatten()
    nv, B = d.nv, 3
    q, v, tau, vd_in, w = rand_inputs(mech, B, 13, wext=True)
    bar = np.random.default_rng(14).standard_normal((nv, B))
    vd, gq, gv, Mi = host_fd(d, q, v, tau, w)
    r = host_vjp(d, True, q, v, vd, bar, w)
    assert rel_err(_contract(gq, bar, nv), r["qt"]) < TOL_CPU and rel_err(_contract(gv, bar, nv), r["vb"]) < TOL_CPU
    assert rel_err(_contract(Mi, bar, nv), r["taub"]) < TOL_CPU
    iq, iv, _, M = host_id(d, q, v, vd_in, w)
    r = host_vjp(d, False, q, v, vd_in, bar, w)
    assert rel_err(_contract(iq, bar, nv), r["qt"]) < TOL_CPU and rel_err(_contract(iv, bar, nv), r["vb"]) < TOL_CPU
    assert rel_err(_contract(M, bar, nv), r["vdb"]) < TOL_CPU


@pytest.mark.parametrize("name,mech", _models(), ids=[n for n, _ in _models()])
def test_without_the_new_arguments_the_forward_path_is_unchanged(name, mech):
    """wext = NULL and dvd_dtau = NULL: exactly hostsim.dynamics_derivatives.  Asking for dvd_dtau leaves dq / dv bit for bit, and
    zero wrenches give the same values."""
    d = mech.flatten()
    q, v, tau, _, w = rand_inputs(mech, 3, 15, wext=True)
    vd0, gq0, gv0 = hostsim.dynamics_derivatives(d, q, v, tau)
    vd, gq, gv, dt = host_fd(d, q, v, tau, None, dtau=False)
    assert dt is None and np.array_equal(vd, vd0) and np.array_equal(gq, gq0) and np.array_equal(gv, gv0)
    _, gq, gv, _ = host_fd(d, q, v, tau, None, dtau=True)
    assert np.array_equal(gq, gq0) and np.array_equal(gv, gv0)
    _, gq, gv, _ = host_fd(d, q, v, tau, np.zeros_like(w))
    assert np.array_equal(gq, gq0) and np.array_equal(gv, gv0)


def test_three_block_solve_compiles_without_a_gpu(tmp_path, monkeypatch):
    """The generator's third block through NVRTC: every joint type, iiwa14 (21 columns in groups of 4: the last holds one) and 66
    coordinates (the high word of the masks).  The two-block text does not change when the third block exists."""
    monkeypatch.setenv("RBD_JIT_CACHE", str(tmp_path))
    dump = tmp_path / "dump"
    monkeypatch.setenv("RBD_DERIV_DUMP", str(dump))
    for mech in (randmech(6, shuffle=True), iiwa14(), legs_model()):
        h = _cabi.ModelHandle(mech.flatten())
        for code in (_cabi.RBD_F64, _cabi.RBD_F32):
            try:
                h.precompile_derivatives(code, with_dtau=True)
            except _cabi.RbdError as e:
                if "NVRTC" in str(e):
                    pytest.skip("NVRTC not available")
                raise
        tau64 = open(str(dump) + "_tau_f64.cu").read()
        assert "T* dtau" in tau64 and "< 3 * NV" in tau64
        h.precompile_derivatives(_cabi.RBD_F64)
        two = open(str(dump) + "_f64.cu").read()
        assert "dtau" not in two and "< 3 * NV" not in two
        h.close()
    assert len([f for f in os.listdir(tmp_path) if "deriv_tau" in f]) == 6


def test_argument_checks_without_a_gpu(built):
    """Every refusal is decided on the host, before any CUDA call."""
    lib = _cabi.load_library()
    h = _cabi.ModelHandle(iiwa14().flatten())
    x = ctypes.c_void_p(16)                                 # never dereferenced: every call below returns before a launch
    ext = lambda *a: lib.rbd_dynamics_derivatives_ext(*a)            # noqa: E731
    inv = lambda *a: lib.rbd_inverse_dynamics_derivatives(*a)        # noqa: E731
    for fn in (ext, inv):
        assert fn(None, 1, 4, 4, x, x, x, x, x, x, x, x, None) == _cabi.RBD_EINVAL
        assert fn(h.ptr, _cabi.RBD_DUAL64X6, 4, 4, x, x, x, x, x, x, x, x, None) == _cabi.RBD_EUNSUPPORTED
        assert fn(h.ptr, 1, 8, 4, x, x, x, x, x, x, x, x, None) == _cabi.RBD_EDIM
        assert fn(h.ptr, 1, 0, 0, None, None, None, None, None, None, None, None, None) == _cabi.RBD_OK
    # forward: q, v, vd_out, dvd_dq_out, dvd_dv_out required (tau, wext, dvd_dtau_out optional)
    for k in (4, 5, 8, 9, 10):
        a = [h.ptr, 1, 4, 4, x, x, x, x, x, x, x, x, None]
        a[k] = None
        assert ext(*a) == _cabi.RBD_EINVAL, k
        assert "must not be NULL" in lib.rbd_last_error().decode()
    # inverse: q, v, vd, dtau_dq_out, dtau_dv_out required (wext, tau_out, M_out optional)
    for k in (4, 5, 6, 9, 10):
        a = [h.ptr, 1, 4, 4, x, x, x, x, x, x, x, x, None]
        a[k] = None
        assert inv(*a) == _cabi.RBD_EINVAL, k
    # the model limits, and a model without velocity coordinates
    from tests.test_deriv_paths import REFUSED_MODELS
    big = _cabi.ModelHandle(REFUSED_MODELS["star129"]().flatten())
    for fn in (ext, inv):
        assert fn(big.ptr, 1, 4, 4, x, x, x, x, x, x, x, x, None) == _cabi.RBD_EUNSUPPORTED
        assert "more than 128 velocity coordinates" in lib.rbd_last_error().decode()
    fixed = rbd.Mechanism(rbd.RigidBody("world"))
    fixed.attach(fixed.root_body, rbd.RigidBody("b", rbd.SpatialInertia.rand(np.random.default_rng(0))), rbd.Joint("j", rbd.Fixed()))
    hf = _cabi.ModelHandle(fixed.flatten())
    for fn in (ext, inv):
        assert fn(hf.ptr, 1, 4, 4, x, x, x, x, x, x, x, x, None) == _cabi.RBD_OK
    for hh in (h, big, hf):
        hh.close()


# ----------------------------------------------------------------------------------------------------------------------
# GPU tier
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch():
    import torch as t
    assert t.cuda.is_available()
    rbd.load_library()
    return t


def _inputs(mech, B, seed):
    rng = np.random.default_rng(seed)
    d = mech.flatten()
    return {"q": rand_q(mech, B, rng), "v": rng.standard_normal((d.nv, B)), "tau": rng.standard_normal((d.nv, B)),
            "vd": rng.standard_normal((d.nv, B)), "wext": rng.standard_normal((6 * d.nb, B))}


def call_fd(torch, mech, ins, B, ld, dtype, wext=True, dtau=True, legacy=False):
    """rbd_dynamics_derivatives_ext (or, legacy, rbd_dynamics_derivatives) on [rows, ld] tensors with NaN-filled outputs."""
    from rigidbodydynamics.jl_b200.state import _DT, _model_handle
    nv = mech.num_velocities()
    outs = {k: torch.full((r, ld), float("nan"), dtype=dtype, device="cuda") for k, r in (("vd", nv), ("dq", nv * nv), ("dv", nv * nv))}
    if dtau:
        outs["dtau"] = torch.full((nv * nv, ld), float("nan"), dtype=dtype, device="cuda")
    p = lambda t: None if t is None else t.data_ptr()       # noqa: E731
    lib = _cabi.load_library()
    h = _model_handle(mech).ptr
    if legacy:
        st = lib.rbd_dynamics_derivatives(h, _DT[dtype], B, ld, p(ins["q"]), p(ins["v"]), p(ins["tau"]), p(outs["vd"]), p(outs["dq"]),
                                          p(outs["dv"]), None)
    else:
        st = lib.rbd_dynamics_derivatives_ext(h, _DT[dtype], B, ld, p(ins["q"]), p(ins["v"]), p(ins["tau"]),
                                              p(ins["wext"]) if wext else None, p(outs["vd"]), p(outs["dq"]), p(outs["dv"]),
                                              p(outs.get("dtau")), None)
    torch.cuda.synchronize()
    assert st == 0, lib.rbd_last_error().decode()
    return outs, rbd.launch_info()


def call_id(torch, mech, ins, B, ld, dtype, wext=True, extra=True):
    from rigidbodydynamics.jl_b200.state import _DT, _model_handle
    nv = mech.num_velocities()
    rows = (("dq", nv * nv), ("dv", nv * nv)) + ((("tau", nv), ("M", nv * nv)) if extra else ())
    outs = {k: torch.full((r, ld), float("nan"), dtype=dtype, device="cuda") for k, r in rows}
    p = lambda t: None if t is None else t.data_ptr()       # noqa: E731
    lib = _cabi.load_library()
    st = lib.rbd_inverse_dynamics_derivatives(_model_handle(mech).ptr, _DT[dtype], B, ld, p(ins["q"]), p(ins["v"]), p(ins["vd"]),
                                              p(ins["wext"]) if wext else None, p(outs.get("tau")), p(outs["dq"]), p(outs["dv"]),
                                              p(outs.get("M")), None)
    torch.cuda.synchronize()
    assert st == 0, lib.rbd_last_error().decode()
    return outs, rbd.launch_info()


def to_dev(torch, x, dtype, ld):
    return {k: _dev(torch, a, dtype, ld) for k, a in x.items()}


def check_written(torch, outs, B):
    for k, t in outs.items():
        assert bool(torch.isfinite(t[:, :B]).all()), k
        assert bool(torch.isnan(t[:, B:]).all()), k


def host(t, idx):
    return t[:, idx].double().cpu().numpy()


def cpu_ref(mech, ins, idx, wext=True):
    """The fp64 CPU run of the same code at the (possibly rounded) device inputs: forward with the device's v̇ recomputed, inverse."""
    h = {k: host(t, idx) for k, t in ins.items()}
    d = mech.flatten()
    w = h["wext"] if wext else None
    vd, gq, gv, dt = host_fd(d, h["q"], h["v"], h["tau"], w)
    iq, iv, tau, M = host_id(d, h["q"], h["v"], h["vd"], w)
    return {"vd": vd, "dq": gq, "dv": gv, "dtau": dt}, {"dq": iq, "dv": iv, "tau": tau, "M": M}


def worst(outs, ref, idx):
    return max(rel_err(host(outs[k], idx), ref[k]) for k in outs)


def _gpu_models():
    return _models() + [("legs66", legs_model())]


@pytest.mark.gpu
@pytest.mark.parametrize("name,mech", _gpu_models(), ids=[n for n, _ in _gpu_models()])
def test_gpu_vs_hostsim(torch, name, mech):
    B = 161
    x = _inputs(mech, B, 21)
    ins = to_dev(torch, x, torch.float64, B + 3)
    fo, info = call_fd(torch, mech, ins, B, B + 3, torch.float64)
    io, info_id = call_id(torch, mech, ins, B, B + 3, torch.float64)
    check_written(torch, fo, B)
    check_written(torch, io, B)
    assert info_id.kernels_launched == 4                  # world, accum, pairs, expand: no forward dynamics, factor or solve
    idx = cols(B)
    rf, ri = cpu_ref(mech, ins, idx)
    assert worst(fo, rf, idx) < TOL_CPU and worst(io, ri, idx) < TOL_CPU, (worst(fo, rf, idx), worst(io, ri, idx))
    # tau_out against the library's own inverse dynamics
    nv = mech.num_velocities()
    tau = torch.empty((nv, B + 3), dtype=torch.float64, device="cuda")
    from rigidbodydynamics.jl_b200.state import _DT, _model_handle
    lib = _cabi.load_library()
    assert lib.rbd_inverse_dynamics(_model_handle(mech).ptr, _DT[torch.float64], B, B + 3, ins["q"].data_ptr(), ins["v"].data_ptr(),
                                    ins["vd"].data_ptr(), ins["wext"].data_ptr(), tau.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert rel_err(host(io["tau"], np.arange(B)), host(tau, np.arange(B))) < TOL_CPU


@pytest.mark.gpu
def test_gpu_legacy_entry_point_is_the_ext_call_without_new_arguments(torch):
    mech = atlas()
    B = 300
    ins = to_dev(torch, _inputs(mech, B, 22), torch.float64, B)
    a, ia = call_fd(torch, mech, ins, B, B, torch.float64, dtau=False, legacy=True)
    b, ib = call_fd(torch, mech, ins, B, B, torch.float64, wext=False, dtau=False)
    c, _ = call_fd(torch, mech, ins, B, B, torch.float64, wext=False, dtau=True)
    assert ia.kernels_launched == ib.kernels_launched
    for k in a:
        assert torch.equal(a[k], b[k]) and torch.equal(a[k], c[k]), k


def _paths_bitwise(torch, monkeypatch, tmp_path, mech, dtype, B, label):
    """Every solve path, the forward Jacobians with wrenches and M^-1, bit for bit, against the CPU run."""
    monkeypatch.setenv("RBD_JIT_CACHE", str(tmp_path))
    _, nv, nnz, _ = tables(mech)
    ins = to_dev(torch, _inputs(mech, B, 30 + nv), dtype, B + 1)
    runs = {}
    jit, info = call_fd(torch, mech, ins, B, B + 1, dtype)
    assert info.smem_bytes == nnz * 32 * dtype.itemsize, ("specialised solve", info.smem_bytes)
    assert 3 * info.grid * 32 <= B, ("three passes of the specialised grid", info.grid, B)
    assert any("deriv_tau" in f for f in os.listdir(tmp_path)), "the three-block kernel compiled inside the call"
    runs["specialised"] = jit
    monkeypatch.setenv("RBD_DERIV_JIT", "0")
    runs["generic"], info = call_fd(torch, mech, ins, B, B + 1, dtype)
    assert 3 * info.grid * 32 <= B, ("three passes of the generic grid", info.grid, B)
    monkeypatch.setenv("RBD_DERIV_GLOBAL_FACTOR", "1")
    runs["scratch factor"], _ = call_fd(torch, mech, ins, B, B + 1, dtype)
    check_written(torch, jit, B)
    for k, r in runs.items():
        for key in jit:
            if not torch.equal(r[key][:, :B], jit[key][:, :B]):
                pytest.fail(f"{label} {k} {key}: differs from the specialised solve by {(r[key] - jit[key]).abs().max().item():.3e}")
    idx = cols(B)
    rf, _ = cpu_ref(mech, ins, idx)
    e = {k: rel_err(host(jit[k], idx), rf[k]) for k in jit}
    print(f"{label}: worst rel_err vs the fp64 CPU run {e}")
    assert max(e.values()) < (TOL_CPU if dtype == torch.float64 else TOL32_TOOLS), e


def jit_plan3(nv, f64):
    """deriv_jit_plan with the third block: (cg, ngroups, warps)."""
    cg = min(4, (150 if f64 else 110) // (nv * (2 if f64 else 1)))
    ngroups = -(-3 * nv // cg)
    rounds = -(-ngroups // 12)
    return cg, ngroups, -(-ngroups // rounds)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
@pytest.mark.parametrize("name", ["atlas", "iiwa14"])
def test_gpu_solve_paths_bit_identical(torch, monkeypatch, tmp_path, name, dtype_name):
    """The specialised three-block solve (compiled inside the call, three passes of its grid; iiwa14's last column group of the
    3 nv = 21 columns is partly filled), the generic solve and the scratch factor, one chunk."""
    from tests.test_deriv_paths import max_grid, multi_pass_batch
    dtype = getattr(torch, dtype_name)
    size = 8 if dtype == torch.float64 else 4
    mech = tooled(atlas() if name == "atlas" else iiwa14(), 7)
    _, nv, nnz, rows = tables(mech)
    cg, ngroups, warps = jit_plan3(nv, size == 8)
    if name == "iiwa14":
        assert 3 * nv % cg, "partly filled last column group"
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = max(4097, multi_pass_batch(max(max_grid(torch, 32 * warps, nnz * 32 * size), 4 * sms)))
    monkeypatch.setenv("RBD_DERIV_SCRATCH_MB", str(-(-(rows + 6 * len(mech.joints)) * size * B // (1 << 20)) + 1))
    _paths_bitwise(torch, monkeypatch, tmp_path, mech, dtype, B, f"{name} {dtype_name} B={B} cg={cg} groups={ngroups}")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
def test_gpu_chunks_bitwise_equal_one_chunk(torch, monkeypatch, dtype_name):
    """RBD_DERIV_SCRATCH_MB=4 against one chunk, forward with wrenches and M^-1 and inverse: the wrench rows make the chunks
    smaller, and the same samples give the same bits."""
    dtype = getattr(torch, dtype_name)
    mech = tooled(atlas(), 8)
    B = 2500
    monkeypatch.setenv("RBD_DERIV_JIT", "0")
    ins = to_dev(torch, _inputs(mech, B, 40), dtype, B + 2)
    one, i1 = call_fd(torch, mech, ins, B, B + 2, dtype)
    one_id, j1 = call_id(torch, mech, ins, B, B + 2, dtype)
    monkeypatch.setenv("RBD_DERIV_SCRATCH_MB", "4")
    many, i2 = call_fd(torch, mech, ins, B, B + 2, dtype)
    many_id, j2 = call_id(torch, mech, ins, B, B + 2, dtype)
    _, nv, nnz, rows = tables(mech)
    rows += 6 * (len(mech.joints))
    C = max(128, (4 << 20) // (rows * dtype.itemsize) // 128 * 128)
    n = -(-B // C)
    assert n > 1 and i2.kernels_launched == n * i1.kernels_launched and j2.kernels_launched == 4 * n, (n, i1.kernels_launched,
                                                                                                        i2.kernels_launched)
    check_written(torch, many, B)
    check_written(torch, many_id, B)
    for a, b in ((one, many), (one_id, many_id)):
        for k in a:
            assert torch.equal(a[k][:, :B], b[k][:, :B]), k
    edges = np.unique(np.concatenate([cols(B), np.arange(C, B, C), np.arange(C, B, C) - 1]))
    rf, ri = cpu_ref(mech, ins, edges)
    tol = TOL_CPU if dtype == torch.float64 else TOL32_TOOLS
    assert worst(many, rf, edges) < tol and worst(many_id, ri, edges) < tol


@pytest.mark.gpu
def test_gpu_fp32_against_fp64_at_rounded_inputs(torch):
    mech = atlas()
    B = 1 << 14
    x = _inputs(mech, B, 50)
    ins32 = to_dev(torch, x, torch.float32, B)
    fo, _ = call_fd(torch, mech, ins32, B, B, torch.float32)
    io, _ = call_id(torch, mech, ins32, B, B, torch.float32)
    ins64 = {k: t.double() for k, t in ins32.items()}        # the fp32-rounded inputs
    f64, _ = call_fd(torch, mech, ins64, B, B, torch.float64)
    i64, _ = call_id(torch, mech, ins64, B, B, torch.float64)
    idx = cols(B)
    ef = {k: rel_err(host(fo[k], idx), host(f64[k], idx)) for k in fo}
    ei = {k: rel_err(host(io[k], idx), host(i64[k], idx)) for k in io}
    print(f"atlas fp32 B={B}: forward {ef}, inverse {ei}")
    assert max(ef.values()) < TOL32 and max(ei.values()) < TOL32_ID, (ef, ei)


@pytest.mark.gpu
def test_gpu_contraction_with_the_vjp_kernels(torch):
    """ν̄^T dvd_dq, ν̄^T dvd_dv, (dvd_dtau)^T ν̄ against rbd_dynamics_vjp and τ̄^T dtau_dq, τ̄^T dtau_dv against
    rbd_inverse_dynamics_vjp, with external wrenches, on the GPU."""
    from rigidbodydynamics.jl_b200.state import _DT, _model_handle
    mech = randmech(5, shuffle=True)
    nv, B = mech.num_velocities(), 257
    x = _inputs(mech, B, 60)
    ins = to_dev(torch, x, torch.float64, B)
    bar = torch.from_numpy(np.random.default_rng(61).standard_normal((nv, B))).cuda()
    fo, _ = call_fd(torch, mech, ins, B, B, torch.float64)
    io, _ = call_id(torch, mech, ins, B, B, torch.float64)
    lib = _cabi.load_library()
    h = _model_handle(mech).ptr
    out = {k: torch.empty((nv, B), dtype=torch.float64, device="cuda") for k in ("qt", "vb", "tb")}
    p = lambda t: t.data_ptr()          # noqa: E731
    assert lib.rbd_dynamics_vjp(h, _DT[torch.float64], B, B, p(ins["q"]), p(ins["v"]), p(ins["tau"]), p(ins["wext"]), p(fo["vd"]),
                                p(bar), p(out["qt"]), None, p(out["vb"]), p(out["tb"]), None, None) == 0
    torch.cuda.synchronize()
    c = lambda J: _contract(J.cpu().numpy(), bar.cpu().numpy(), nv)      # noqa: E731
    assert rel_err(c(fo["dq"]), out["qt"].cpu().numpy()) < TOL_CPU
    assert rel_err(c(fo["dv"]), out["vb"].cpu().numpy()) < TOL_CPU
    assert rel_err(c(fo["dtau"]), out["tb"].cpu().numpy()) < TOL_CPU
    assert lib.rbd_inverse_dynamics_vjp(h, _DT[torch.float64], B, B, p(ins["q"]), p(ins["v"]), p(ins["vd"]), p(ins["wext"]), p(bar),
                                        p(out["qt"]), None, p(out["vb"]), None, None, None) == 0
    torch.cuda.synchronize()
    assert rel_err(c(io["dq"]), out["qt"].cpu().numpy()) < TOL_CPU
    assert rel_err(c(io["dv"]), out["vb"].cpu().numpy()) < TOL_CPU


@pytest.mark.gpu
def test_gpu_python_wrappers(torch):
    from tests.loops_oracle import four_bar
    mech = iiwa14()
    B = 33
    dtype = torch.float64
    st = rbd.MechanismState(mech, B, dtype)
    rbd.rand_(st, np.random.default_rng(70))
    nv, nb = st.nv, len(mech.joints)
    res = rbd.DynamicsResult(mech, B, dtype)
    new = lambda rows, dt=dtype: torch.empty((rows, B), dtype=dt, device="cuda")      # noqa: E731
    w = torch.randn((6 * nb, B), dtype=dtype, device="cuda")
    dq, dv, dt = new(nv * nv), new(nv * nv), new(nv * nv)
    rbd.dynamics_derivatives_(dq, dv, res, st, None, w, dt)
    vd = res.vd.clone()
    iq, iv = rbd.inverse_dynamics_derivatives(st, vd, w)
    tau, M = new(nv), new(nv * nv)
    rbd.inverse_dynamics_derivatives_(new(nv * nv), new(nv * nv), st, vd, w, torques=tau, massmatrix=M)
    torch.cuda.synchronize()
    assert tau.abs().max().item() < 1e-9                     # ID(FD(tau = 0)) = 0
    Mi = dt.cpu().numpy()
    eye = np.einsum("bij,bjk->bik", _mat(Mi, nv), _mat(M.cpu().numpy(), nv))
    assert np.abs(eye - np.eye(nv)).max() < 1e-9
    want = _flat(-np.einsum("bij,bjk->bik", _mat(Mi, nv), _mat(iq.cpu().numpy(), nv)))
    assert rel_err(dq.cpu().numpy(), want) < 1e-9
    # refusals: sizes, dtypes, loops
    with pytest.raises(rbd.DimensionMismatch):
        rbd.dynamics_derivatives_(dq, dv, res, st, None, new(6 * nb - 1))
    with pytest.raises(rbd.DimensionMismatch):
        rbd.dynamics_derivatives_(dq, dv, res, st, None, None, new(nv * nv - 1))
    with pytest.raises(TypeError):
        rbd.dynamics_derivatives_(dq, dv, res, st, None, None, new(nv * nv, torch.float32))
    with pytest.raises(rbd.DimensionMismatch):
        rbd.inverse_dynamics_derivatives_(new(nv * nv), new(nv), st, vd)
    with pytest.raises(rbd.DimensionMismatch):
        rbd.inverse_dynamics_derivatives_(new(nv * nv), new(nv * nv), st, vd, massmatrix=new(nv))
    with pytest.raises(TypeError):
        rbd.inverse_dynamics_derivatives(st, vd.float())
    lm = four_bar()
    ls = rbd.MechanismState(lm, 2, dtype)
    with pytest.raises(rbd.RbdError) as e:
        rbd.inverse_dynamics_derivatives(ls, torch.zeros((ls.nv, 2), dtype=dtype, device="cuda"))
    assert e.value.status == _cabi.RBD_ELOOP
