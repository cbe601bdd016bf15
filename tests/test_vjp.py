"""Reverse mode: vector-Jacobian products of dynamics! / inverse_dynamics! (csrc/rbd_adjoint.cuh, rbd_dynamics_vjp,
rbd_inverse_dynamics_vjp, rigidbodydynamics.jl_b200.autodiff).

Oracles: the oracle's dual-number Jacobians of dynamics! (tests.util.oracle_dynamics_derivatives) contracted with the adjoint, and --
with no dual numbers anywhere -- central finite differences of the oracle's plain fp64 dynamics / inverse_dynamics along the
tangent directions q + eps q̇(e_k), v + eps e_k, tau + eps e_k, w + eps e_r.
CPU tier: the per-sample device functions compiled for the host (tests/hostsim/hostsim_adjoint.cpp).  GPU tier: the kernels through
the C ABI and the torch.autograd functions."""
import ctypes
import functools

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from oracle import Oracle
from rigidbodydynamics.jl_b200._cabi import RbdModelDesc, make_desc
from tests import hostsim
from tests.test_derivatives import _models
from tests.util import axis_aligned_tree, oracle_dynamics_derivatives, rand_inputs, randmech, rel_err

TOL64 = 1e-8          # parity with the oracle's DualN Jacobians in fp64
TOL_FD = 2e-6         # central finite differences, eps = 1e-6
# fp32 Atlas against the fp64 oracle, measured: rel_err 1.8e-4 (q̄_tan), 4.5e-5 (v̄), 7.8e-8 (τ̄) on test_dynamics_vjp_hostsim_fp32's
# three samples; 1.05e-3 (q̄_tan), 2.1e-4 (v̄), 1.5e-6 (τ̄) as the worst of 512 strided samples of a 2^20 batch (tools/time_vjp.py).
# The bound is the derivative tests' 5e-3.
TOL32 = 5e-3


@functools.cache
def _shim():
    """tests/hostsim/hostsim_adjoint.cpp, compiled and loaded by hostsim.shim."""
    lib = hostsim.shim("hostsim_adjoint")
    lib.hostsim_vjp.argtypes = [ctypes.POINTER(RbdModelDesc), ctypes.c_int, ctypes.c_int, ctypes.c_int64] + [ctypes.c_void_p] * 11
    return lib


def host_vjp(desc, fd, q, v, vd, wbar, wext=None):
    """adjoint_sample (fd=False) / dynamics_vjp_sample (fd=True) on the CPU: dict of every output."""
    dt = q.dtype
    d, keep = make_desc(desc)
    c = lambda a: None if a is None else np.ascontiguousarray(a, dt)
    q, v, vd, wbar, wext = c(q), c(v), c(vd), c(wbar), c(wext)
    B = q.shape[1]
    out = {k: np.full((r, B), np.nan, dt) for k, r in (("qt", desc.nv), ("qc", desc.nq), ("vb", desc.nv), ("wb", 6 * desc.nb))}
    out["taub" if fd else "vdb"] = np.full((desc.nv, B), np.nan, dt)
    p = lambda a: None if a is None or a.size == 0 else a.ctypes.data
    rc = _shim().hostsim_vjp(ctypes.byref(d), int(fd), 0 if dt == np.float32 else 1, B, p(q), p(v), p(vd), p(wext), p(wbar), p(out["qt"]),
                             p(out["qc"]), p(out["vb"]), p(out.get("vdb")), p(out.get("taub")), p(out["wb"]))
    assert rc == 0, rc
    return out


def _contract(J, bar, nv):
    """bar^T J for J [nv*nv, B] with entry (i, j) at row i + j*nv: row j = sum_i bar_i J[i + j*nv]."""
    B = J.shape[1]
    return np.einsum("ijb,ib->jb", J.reshape(nv, nv, B).transpose(1, 0, 2), bar)


def _qdot_dirs(o, q, nv, tau):
    """q̇(e_k) = velocity_to_configuration_derivative(e_k) per sample, [nv, nq, B]."""
    B = q.shape[1]
    out = []
    for k in range(nv):
        e = np.zeros((nv, B)); e[k] = 1.0
        out.append(o.dynamics(q, e, tau, want_qd=True)[1])
    return np.stack(out)


# ----------------------------------------------------------------------------------------------------------------------
# CPU tier
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,mech", _models(), ids=[n for n, _ in _models()])
def test_dynamics_vjp_hostsim_vs_oracle_duals(name, mech):
    d = mech.flatten()
    o = Oracle(d)
    q, v, tau, _, _ = rand_inputs(mech, 3, 11)
    nu = np.random.default_rng(5).standard_normal((d.nv, 3))
    for t in (tau, np.zeros_like(tau)):
        vd = o.dynamics(q, v, t)
        rq, rv = oracle_dynamics_derivatives(o, mech, q, v, t)
        r = host_vjp(d, True, q, v, vd, nu)
        assert rel_err(r["qt"], _contract(rq, nu, d.nv)) < TOL64, rel_err(r["qt"], _contract(rq, nu, d.nv))
        assert rel_err(r["vb"], _contract(rv, nu, d.nv)) < TOL64
        M = o.mass_matrix(q).reshape(d.nv, d.nv, -1)
        mu = np.stack([np.linalg.solve(M[:, :, b].T, nu[:, b]) for b in range(3)], 1)
        assert rel_err(r["taub"], mu) < 1e-10


def test_dynamics_vjp_hostsim_fp32():
    mech = rbd.load_model("atlas", floating=True)
    d = mech.flatten()
    o = Oracle(d)
    q, v, tau, _, _ = rand_inputs(mech, 3, 4)
    nu = np.random.default_rng(6).standard_normal((d.nv, 3))
    vd = o.dynamics(q, v, tau)
    rq, rv = oracle_dynamics_derivatives(o, mech, q, v, tau)
    f = lambda a: a.astype(np.float32)
    r = host_vjp(d, True, f(q), f(v), f(vd), f(nu))
    eq, ev = rel_err(r["qt"], _contract(rq, nu, d.nv)), rel_err(r["vb"], _contract(rv, nu, d.nv))
    assert eq < TOL32 and ev < TOL32, (eq, ev)


def _fd_central(f, x, dirs, eps=1e-6):
    return np.stack([(f(x + eps * dk) - f(x - eps * dk)) / (2 * eps) for dk in dirs])     # [n_dirs, rows, B]


def test_dynamics_vjp_with_external_wrenches_matches_finite_differences():
    """No dual numbers: every output of the forward VJP, external wrenches included (the root-frame wrench term of q̄ that the
    closed forms of rbd_dynamics_derivatives leave out), against central differences of the oracle's fp64 dynamics."""
    mech = randmech(2, shuffle=True)
    d = mech.flatten()
    o = Oracle(d)
    B = 2
    q, v, tau, _, w = rand_inputs(mech, B, 5, wext=True)
    nu = np.random.default_rng(7).standard_normal((d.nv, B))
    vd = o.dynamics(q, v, tau, w)
    r = host_vjp(d, True, q, v, vd, nu, w)
    nv, nr = d.nv, 6 * d.nb
    dirs_q = _qdot_dirs(o, q, nv, tau)
    eye = lambda n, k: np.repeat(np.eye(n)[:, k:k + 1], B, 1)
    Jq = _fd_central(lambda x: o.dynamics(x, v, tau, w), q, dirs_q)
    Jv = _fd_central(lambda x: o.dynamics(q, x, tau, w), v, [eye(nv, k) for k in range(nv)])
    Jt = _fd_central(lambda x: o.dynamics(q, v, x, w), tau, [eye(nv, k) for k in range(nv)])
    Jw = _fd_central(lambda x: o.dynamics(q, v, tau, x), w, [eye(nr, k) for k in range(nr)])
    vjp = lambda J: np.einsum("kib,ib->kb", J, nu)
    for key, J in (("qt", Jq), ("vb", Jv), ("taub", Jt), ("wb", Jw)):
        assert rel_err(r[key], vjp(J)) < TOL_FD, (key, rel_err(r[key], vjp(J)))


def test_inverse_dynamics_vjp_matches_finite_differences():
    mech = randmech(3, shuffle=True)
    d = mech.flatten()
    o = Oracle(d)
    B = 2
    q, v, _, vd, w = rand_inputs(mech, B, 8, wext=True)
    tb = np.random.default_rng(9).standard_normal((d.nv, B))
    nv, nr = d.nv, 6 * d.nb
    eye = lambda n, k: np.repeat(np.eye(n)[:, k:k + 1], B, 1)
    dirs_q = _qdot_dirs(o, q, nv, None)
    for wx in (w, None):
        r = host_vjp(d, False, q, v, vd, tb, wx)
        ID = lambda q_=q, v_=v, vd_=vd, w_=wx: o.inverse_dynamics(q_, v_, vd_, w_)
        vjp = lambda J: np.einsum("kib,ib->kb", J, tb)
        assert rel_err(r["qt"], vjp(_fd_central(lambda x: ID(q_=x), q, dirs_q))) < TOL_FD
        assert rel_err(r["vb"], vjp(_fd_central(lambda x: ID(v_=x), v, [eye(nv, k) for k in range(nv)]))) < TOL_FD
        if wx is not None:
            assert rel_err(r["wb"], vjp(_fd_central(lambda x: ID(w_=x), w, [eye(nr, k) for k in range(nr)]))) < TOL_FD
        M = o.mass_matrix(q).reshape(nv, nv, B)
        assert rel_err(r["vdb"], np.einsum("ijb,jb->ib", M.transpose(1, 0, 2), tb)) < 1e-10


def test_q_bar_cfg_is_the_reference_adjoint_map():
    """configuration_derivative_to_velocity_adjoint!'s identity (test_mechanism_algorithms.jl:845-856):
    q̄_cfg . configuration_derivative(q, u) == q̄_tan . u for random u, at NON-unit random configurations."""
    for seed in (0, 1):
        mech = randmech(seed, shuffle=True)
        d = mech.flatten()
        rng = np.random.default_rng(45 + seed)
        B = 3
        q = rng.random((d.nq, B))                     # does not satisfy the state constraints, like the reference's test
        v, vd, tb = rng.random((d.nv, B)), rng.random((d.nv, B)), rng.standard_normal((d.nv, B))
        r = host_vjp(d, False, q, v, vd, tb)
        for _ in range(3):
            u = rng.standard_normal((d.nv, B))
            qd = hostsim.dynamics(d, q, u, want_qd=True)[1]     # configuration_derivative (the oracle's solve refuses a non-unit q)
            lhs, rhs = (r["qc"] * qd).sum(0), (r["qt"] * u).sum(0)
            assert np.abs(lhs - rhs).max() <= 1e-10 * max(1.0, np.abs(rhs).max()), (lhs, rhs)


def test_q_bar_cfg_equals_q_bar_tan_for_revolute_and_prismatic_trees():
    rng = np.random.default_rng(3)
    for mech in (rbd.rand_tree_mechanism(rng, [rbd.Revolute, rbd.Prismatic] * 5), rbd.load_model("iiwa14", floating=False)):
        d = mech.flatten()
        q, v, _, vd, _ = rand_inputs(mech, 4, 2)
        r = host_vjp(d, False, q, v, vd, rng.standard_normal((d.nv, 4)))
        assert np.array_equal(r["qc"], r["qt"])


# ----------------------------------------------------------------------------------------------------------------------
# GPU tier
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch():
    import torch as t
    assert t.cuda.is_available()
    rbd.load_library()
    return t


def _cuda(torch, a, dtype, ld=None):
    """[rows, B] numpy -> CUDA tensor; with ld > B the tensor is a [rows, ld] buffer (the extra columns NaN) and the caller passes ld."""
    if a is None:
        return None
    rows, B = a.shape
    t = torch.full((rows, ld or B), float("nan"), dtype=dtype, device="cuda")
    t[:, :B] = torch.from_numpy(np.ascontiguousarray(a)).to(dtype)
    return t


def _abi_vjp(torch, mech, fd, q, v, vd, bar, tau=None, w=None, dtype=None, ld=None, want=("qt", "qc", "vb", "xb", "wb")):
    """One call of rbd_dynamics_vjp (fd) / rbd_inverse_dynamics_vjp through the C ABI; NaN-filled output buffers, None for the
    outputs not in ``want``.  Returns (status, {key: numpy [rows, B]})."""
    from rigidbodydynamics.jl_b200 import _cabi
    from rigidbodydynamics.jl_b200.state import _DT, _model_handle
    dtype = dtype or torch.float64
    d = mech.flatten()
    B = q.shape[1]
    ld = ld or B
    h = _model_handle(mech)
    ins = [_cuda(torch, a, dtype, ld) for a in (q, v, tau, w, vd, bar)]
    rows = {"qt": d.nv, "qc": d.nq, "vb": d.nv, "xb": d.nv, "wb": 6 * d.nb}
    outs = {k: torch.full((rows[k], ld), float("nan"), dtype=dtype, device="cuda") if k in want else None for k in rows}
    p = lambda t: None if t is None else t.data_ptr()
    lib = _cabi.load_library()
    if fd:
        st = lib.rbd_dynamics_vjp(h.ptr, _DT[dtype], B, ld, p(ins[0]), p(ins[1]), p(ins[2]), p(ins[3]), p(ins[4]), p(ins[5]),
                                  p(outs["qt"]), p(outs["qc"]), p(outs["vb"]), p(outs["xb"]), p(outs["wb"]), None)
    else:
        st = lib.rbd_inverse_dynamics_vjp(h.ptr, _DT[dtype], B, ld, p(ins[0]), p(ins[1]), p(ins[4]), p(ins[3]), p(ins[5]),
                                          p(outs["qt"]), p(outs["qc"]), p(outs["vb"]), p(outs["xb"]), p(outs["wb"]), None)
    torch.cuda.synchronize()
    res = {k: (None if t is None else t.double().cpu().numpy()) for k, t in outs.items()}
    if ld > B:   # the padding columns are never written
        for t in res.values():
            if t is not None:
                assert np.isnan(t[:, B:]).all()
    return st, {k: (None if t is None else t[:, :B]) for k, t in res.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("name,mech", _models(), ids=[n for n, _ in _models()])
@pytest.mark.parametrize("B", [1, 161])
def test_vjp_gpu_vs_oracle(torch, name, mech, B):
    d = mech.flatten()
    o = Oracle(d)
    q, v, tau, _, w = rand_inputs(mech, B, 21, wext=True)
    nu = np.random.default_rng(B).standard_normal((d.nv, B))
    n = min(B, 4)
    idx = np.linspace(0, B - 1, n).astype(int)
    for t, wx in ((tau, None), (None, None), (tau, w)):
        vd = o.dynamics(q, v, t, wx)
        for dtype, ld in ((torch.float64, B), (torch.float64, B + 7), (torch.float32, B)):
            st, r = _abi_vjp(torch, mech, True, q, v, vd, nu, t, wx, dtype, ld)
            assert st == 0
            ref = host_vjp(d, True, q[:, idx], v[:, idx], vd[:, idx], nu[:, idx], None if wx is None else wx[:, idx])
            tol = 1e-10 if dtype == torch.float64 else TOL32
            for k, hk in (("qt", "qt"), ("qc", "qc"), ("vb", "vb"), ("xb", "taub"), ("wb", "wb")):
                assert not np.isnan(r[k]).any(), k
                assert rel_err(r[k][:, idx], ref[hk]) < tol, (k, dtype, rel_err(r[k][:, idx], ref[hk]))
            if wx is None and dtype == torch.float64:      # against the oracle's dual-number Jacobians
                rq, rv = oracle_dynamics_derivatives(o, mech, q[:, idx], v[:, idx], (t if t is not None else np.zeros_like(tau))[:, idx])
                assert rel_err(r["qt"][:, idx], _contract(rq, nu[:, idx], d.nv)) < TOL64
                assert rel_err(r["vb"][:, idx], _contract(rv, nu[:, idx], d.nv)) < TOL64
        st, r = _abi_vjp(torch, mech, False, q, v, vd, nu, None, wx)
        assert st == 0
        ref = host_vjp(d, False, q[:, idx], v[:, idx], vd[:, idx], nu[:, idx], None if wx is None else wx[:, idx])
        for k, hk in (("qt", "qt"), ("qc", "qc"), ("vb", "vb"), ("xb", "vdb"), ("wb", "wb")):
            assert rel_err(r[k][:, idx], ref[hk]) < 1e-10, k
        M = o.mass_matrix(q[:, idx]).reshape(d.nv, d.nv, n)
        assert rel_err(r["xb"][:, idx], np.einsum("ijb,jb->ib", M.transpose(1, 0, 2), nu[:, idx])) < 1e-10


@pytest.mark.gpu
def test_vjp_gpu_consistent_with_dynamics_derivatives(torch):
    for mech in (rbd.load_model("atlas", floating=True), randmech(1, shuffle=True)):
        d = mech.flatten()
        B = 64
        q, v, tau, _, _ = rand_inputs(mech, B, 3)
        st = rbd.MechanismState(mech, B, torch.float64)
        st.q.copy_(torch.from_numpy(q)); st.v.copy_(torch.from_numpy(v))
        res = rbd.DynamicsResult(mech, B, torch.float64)
        dq = torch.empty((d.nv * d.nv, B), dtype=torch.float64, device="cuda")
        dv = torch.empty_like(dq)
        rbd.dynamics_derivatives_(dq, dv, res, st, torch.from_numpy(tau).cuda())
        torch.cuda.synchronize()
        nu = np.random.default_rng(1).standard_normal((d.nv, B))
        _, r = _abi_vjp(torch, mech, True, q, v, res.vd.cpu().numpy(), nu, tau)
        nv = d.nv
        assert rel_err(r["qt"], _contract(dq.cpu().numpy(), nu, nv)) < 1e-10
        assert rel_err(r["vb"], _contract(dv.cpu().numpy(), nu, nv)) < 1e-10


@pytest.mark.gpu
def test_vjp_gpu_null_outputs_untouched_and_bit_identical(torch):
    mech = randmech(0, shuffle=True)
    d = mech.flatten()
    o = Oracle(d)
    B = 97
    q, v, tau, vd0, w = rand_inputs(mech, B, 4, wext=True)
    nu = np.random.default_rng(2).standard_normal((d.nv, B))
    vd = o.dynamics(q, v, tau, w)
    for fd, xv in ((True, vd), (False, vd0)):
        _, full = _abi_vjp(torch, mech, fd, q, v, xv, nu, tau, w)
        for want in (("qt",), ("qc",), ("vb", "wb"), ("xb",), ()):
            st, r = _abi_vjp(torch, mech, fd, q, v, xv, nu, tau, w, want=want)
            assert st == 0
            for k in want:
                assert np.array_equal(r[k], full[k]), (fd, want, k)


@pytest.mark.gpu
def test_vjp_gpu_full_batch_atlas_fp32(torch):
    mech = rbd.load_model("atlas", floating=True)
    d = mech.flatten()
    o = Oracle(d)
    B = 1 << 20
    rng = np.random.default_rng(12)
    q, v, tau, _, _ = rand_inputs(mech, 1, 1)
    q = np.repeat(q, B, 1) + 0.0
    q[:, :] = np.stack([mech.rand_configuration(rng) for _ in range(256)], 1)[:, np.arange(B) % 256]
    v = rng.random((d.nv, B)); tau = rng.random((d.nv, B)); nu = rng.standard_normal((d.nv, B))
    idx = np.arange(0, B, B // 512) + 7
    vd = o.dynamics(q[:, idx], v[:, idx], tau[:, idx])
    vd_all = np.zeros((d.nv, B)); vd_all[:, idx] = vd
    st, r = _abi_vjp(torch, mech, True, q, v, vd_all, nu, tau, dtype=torch.float32, want=("qt", "vb", "xb"))
    assert st == 0
    ref = host_vjp(d, True, q[:, idx], v[:, idx], vd, nu[:, idx])
    for k, hk in (("qt", "qt"), ("vb", "vb"), ("xb", "taub")):
        assert rel_err(r[k][:, idx], ref[hk]) < TOL32, (k, rel_err(r[k][:, idx], ref[hk]))


@pytest.mark.gpu
def test_vjp_gpu_refusals(torch):
    from rigidbodydynamics.jl_b200 import _cabi, autodiff
    from rigidbodydynamics.jl_b200.state import _model_handle
    mech = rbd.load_model("iiwa14", floating=False)
    d = mech.flatten()
    q, v, tau, vd, _ = rand_inputs(mech, 8, 1)
    lib = _cabi.load_library()
    h = _model_handle(mech)
    T = lambda a: torch.from_numpy(a).cuda()
    tq, tv, tvd = T(q), T(v), T(vd)
    out = torch.empty_like(tv)
    p = lambda t: t.data_ptr()
    assert lib.rbd_dynamics_vjp(h.ptr, _cabi.RBD_DUAL64X6, 8, 8, p(tq), p(tv), None, None, p(tvd), p(tvd), p(out), None, None, None, None,
                                None) == _cabi.RBD_EUNSUPPORTED
    assert lib.rbd_dynamics_vjp(h.ptr, _cabi.RBD_F64, 8, 8, p(tq), p(tv), None, None, p(tvd), None, p(out), None, None, None, None,
                                None) == _cabi.RBD_EINVAL
    assert lib.rbd_inverse_dynamics_vjp(h.ptr, _cabi.RBD_F64, 8, 8, p(tq), None, p(tvd), None, p(tvd), p(out), None, None, None, None,
                                        None) == _cabi.RBD_EINVAL
    assert lib.rbd_inverse_dynamics_vjp(h.ptr, _cabi.RBD_F64, 0, 0, None, None, None, None, None, None, None, None, None, None,
                                        None) == _cabi.RBD_OK
    st = rbd.MechanismState(mech, 8, torch.float64)
    st.q.copy_(tq); st.v.copy_(tv)
    with pytest.raises(rbd.DimensionMismatch):
        rbd.dynamics_vjp_(st, tvd, tvd[:3], v_bar=out)
    with pytest.raises(rbd.DimensionMismatch):
        rbd.inverse_dynamics_vjp_(st, tvd, tvd, v_bar=out[:, :4])
    # B = 0 through Python: nothing launched, nothing raised
    st0 = rbd.MechanismState(mech, 0, torch.float64)
    e0 = torch.empty((d.nv, 0), dtype=torch.float64, device="cuda")
    rbd.inverse_dynamics_vjp_(st0, e0, e0, v_bar=e0)
    # loops are refused before anything is launched
    from tests.loops_oracle import four_bar
    m4 = four_bar()
    s4 = rbd.MechanismState(m4, 2, torch.float64)
    z = torch.zeros((s4.nv, 2), dtype=torch.float64, device="cuda")
    with pytest.raises(_cabi.RbdError) as e:
        rbd.dynamics_vjp_(s4, z, z, v_bar=z)
    assert e.value.status == _cabi.RBD_ELOOP
    with pytest.raises(_cabi.RbdError) as e:
        autodiff.inverse_dynamics(m4, s4.q, s4.v, z)
    assert e.value.status == _cabi.RBD_ELOOP


@pytest.mark.gpu
def test_autograd_gradcheck(torch):
    from rigidbodydynamics.jl_b200 import autodiff
    rng = np.random.default_rng(8)
    mech = rbd.rand_tree_mechanism(rng, [rbd.Revolute, rbd.Prismatic, rbd.Revolute, rbd.Revolute, rbd.Prismatic])
    d = mech.flatten()
    B = 3
    q, v, tau, vd, w = rand_inputs(mech, B, 6, wext=True)
    T = lambda a: torch.from_numpy(a).cuda().requires_grad_(True)
    args = (T(q), T(v), T(tau), T(w))
    assert torch.autograd.gradcheck(lambda q_, v_, t_, w_: autodiff.dynamics(mech, q_, v_, t_, w_), args, eps=1e-6, atol=1e-6, rtol=1e-5)
    args = (T(q), T(v), T(vd), T(w))
    assert torch.autograd.gradcheck(lambda q_, v_, a_, w_: autodiff.inverse_dynamics(mech, q_, v_, a_, w_), args, eps=1e-6, atol=1e-6,
                                    rtol=1e-5)
    assert d.nv == 5


@pytest.mark.gpu
def test_autograd_backward_matches_vjp_on_floating_atlas(torch):
    from rigidbodydynamics.jl_b200 import autodiff
    mech = rbd.load_model("atlas", floating=True)
    d = mech.flatten()
    B = 33
    q, v, tau, _, w = rand_inputs(mech, B, 9, wext=True)
    nu = torch.from_numpy(np.random.default_rng(4).standard_normal((d.nv, B))).cuda()
    T = lambda a: torch.from_numpy(a).cuda().requires_grad_(True)
    tq, tv, tt, tw = T(q), T(v), T(tau), T(w)
    vd = autodiff.dynamics(mech, tq, tv, tt, tw)
    (vd * nu).sum().backward()
    st = rbd.MechanismState(mech, B, torch.float64)
    st.q.copy_(tq.detach()); st.v.copy_(tv.detach())
    outs = {k: torch.empty_like(x) for k, x in (("q", tq), ("v", tv), ("t", tt), ("w", tw))}
    rbd.dynamics_vjp_(st, vd.detach(), nu, tt.detach(), tw.detach(), q_bar_cfg=outs["q"], v_bar=outs["v"], tau_bar=outs["t"],
                      wext_bar=outs["w"])
    torch.cuda.synchronize()
    for k, x in (("q", tq), ("v", tv), ("t", tt), ("w", tw)):
        assert torch.equal(x.grad, outs[k]), k
    # inverse dynamics, and a double backward raises
    a = T(rand_inputs(mech, B, 10)[3])
    tq.grad = None
    tau_out = autodiff.inverse_dynamics(mech, tq, tv, a, tw)
    g, = torch.autograd.grad((tau_out * nu).sum(), a, create_graph=True)
    with pytest.raises(RuntimeError):
        g.sum().backward()
