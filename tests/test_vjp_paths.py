"""Every path the reverse-mode kernels take only at large batches, forced on purpose and checked column by column against the CPU run
of the same per-sample code (host_vjp / host_ivjp / host_cvjp / host_pd_vjp and the task VJP's host_vjp) and, on a handful of
columns, against central differences of the fp64 oracle.

Paths (csrc/rbd_adjoint.cu, csrc/rbd_integrate_vjp.cu):
1. Multi-pass persistent grids: dynamics_vjp_kernel, inverse_dynamics_vjp_kernel, task_vjp_kernel and contact_vjp_kernel give every
   resident thread one workspace column and reuse it for every group of 32 samples the thread takes; plan_persistent trims the grid
   to keep the workspace within 512 MiB, so at tens of thousands of samples a thread takes three groups or more.
2. Workspace reuse across calls: the stream-ordered pool hands the next call the workspace the last one freed.  A call after an
   all-NaN call must equal the same call after a finite one bit for bit, and a NaN sample column must stay in its column.
3. The vectorised phase kernels of the rollout adjoints (integrate_adjoint_linear_kernel, integrate_adjoint_pd_linear_kernel: B a
   multiple of the vector width, B >= 1024, aligned arrays) against the per-(sample, joint) kernels they replace.
4. fp32 at 2^20 on Atlas, checked for accuracy: the contact VJP on distinct, partly touching states, the PD VJP in both modes and the
   task VJP with all eight cotangents.
5. The recompute through the model-specialised fp32 programs (B >= RBD_JIT_MIN_BATCH), with one sample beyond the fast sin / cos
   range so that the gated generic fallback runs inside it.
6. 64-bit element offsets in the task VJP's cotangent rows (2.16e9 elements).

Every GPU call fills its outputs with NaN first (the accumulated tau / controller gradients with zeros) and checks that every column
in [0, B) was written and, where the entry point takes a leading dimension, that the padding beyond B was not.  Every input column
is distinct.  The compared columns are 511 at an odd stride plus B - 1: every lane position, the first, middle and last persistent
pass, and the ragged last group."""
import ctypes
import types

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from oracle import Oracle
from rigidbodydynamics.jl_b200 import _cabi
from rigidbodydynamics.jl_b200.kinematics import TaskFrame, task_desc
from tests.task_oracle import OUTPUTS
from tests.test_contact_rollout import _atlas_on_floor, _atlas_states
from tests.test_contact_vjp import TOL32 as TOL32_CONTACT
from tests.test_contact_vjp import _loss as contact_loss
from tests.test_contact_vjp import host_cvjp
from tests.test_integrate_vjp import TOL32 as TOL32_ROLLOUT
from tests.test_integrate_vjp import _oracle_loss, host_ivjp
from tests.test_pd_rollout import Ctrl, _controller, integrate_pd
from tests.test_pd_vjp import TOL32 as TOL32_PD
from tests.test_pd_vjp import _record, host_pd_vjp
from tests.test_task_kinematics import _rows, task_set
from tests.test_task_vjp import END_EFFECTORS, GRADS, fd_jacobians, fd_vjp
from tests.test_task_vjp import TOL32 as TOL32_TASK
from tests.test_task_vjp import host_vjp as host_task_vjp
from tests.test_vjp import TOL32 as TOL32_VJP
from tests.test_vjp import _fd_central, _qdot_dirs, host_vjp
from tests.util import randmech, rel_err

TOL64 = 1e-10          # GPU against the CPU run of the same code, fp64
TOL_VEC = 1e-12        # vectorised phase kernels against the per-(sample, joint) kernels, fp64
TOL_FD = 2e-6          # the fp64 kernels against central differences of the oracle (eps = 1e-6 single calls, 1e-5 rollouts)
DT = 1e-3
NCOLS = 512
# fp32 contact adjoint on Atlas against the fp64 CPU run: worst rel_err measured on an H100 80GB HBM3 (700 W) 2.8e-4 (B = 208397,
# v̄0) and 1.8e-4 (B = 2^20, q̄0) over 512 columns of distinct, partly touching states; the bound is about 7x that, tighter than the
# contact file's TOL32 (2e-2), which also covers the random tree with six contact points per body
TOL32_CONTACT_ATLAS = 2e-3

# The workspace of the persistent adjoint kernels (rbd_adjoint.cu, rbd_integrate_vjp.cu): one column of rows per resident thread,
# blocks of one warp, the grid trimmed to max(1, CAP // (row bytes x 32)) blocks.  Rows per thread, from the kernels' headers:
CAP = 512 << 20                 # kWorkspaceCap, and the contact stage adjoint's cap
ADJ_BODY_ROWS = 54              # kAdjBodyRows (rbd_adjoint.cuh): adjoint_rows = 54 nb + nv
TASK_ROWS = 42                  # kTaskAdjRows = kTaskAdjSlotRows (rbd_task_adjoint.cuh): 42 nb + 42 nnamed


def adjoint_rows(nb, nv):
    return ADJ_BODY_ROWS * nb + nv


def contact_vjp_rows(nb, nv):
    return adjoint_rows(nb, nv) + 6 * nb + nv


def cap_threads(rows, itemsize):
    """The most resident threads the 512 MiB cap allows: an upper bound on the grid, whatever the residency."""
    return max(1, CAP // (rows * itemsize * 32)) * 32


def multi_pass_batch(rows, itemsize):
    """A ragged batch that gives every thread at least three groups whatever the residency: three times the cap's threads, plus
    a part group."""
    return 3 * cap_threads(rows, itemsize) + 77


# ------------------------------------------------------------------------------------------------------------------
# models and inputs
# ------------------------------------------------------------------------------------------------------------------
MODELS = {
    "atlas": lambda: rbd.load_model("atlas", floating=True),          # floating root, revolute limbs: both phase kernels
    "iiwa14": lambda: rbd.load_model("iiwa14", floating=False),       # revolute only: the linear phase kernel alone
    "randmech": lambda: randmech(3, shuffle=True),                    # every joint type, shuffled: the general path
    "atlas_contact": lambda: _atlas_on_floor()[0],                    # Atlas with four points under each foot
}


def cols(B, n=NCOLS):
    """n - 1 columns at an odd stride (not a multiple of 32: every lane position) spread over [0, B), and B - 1."""
    if B <= n:
        return np.arange(B)
    s = max(1, (B - 1) // (n - 1))
    s -= 1 - s % 2
    return np.unique(np.append(np.arange(n - 1) * s, B - 1))


def fd_cols(B):
    return np.array([0, B // 2 + 3, B - 1])


def rand_q(mech, B, rng):
    """rand_configuration! for a batch, vectorised on the host (distinct columns, fp64)."""
    import torch
    nq = mech.num_positions()
    st = types.SimpleNamespace(mechanism=mech, batch=B, nq=nq, dtype=torch.float64, q=torch.empty((nq, B), dtype=torch.float64))
    rbd.state.rand_configuration_(st, rng)
    return st.q.numpy()


def r32(a):
    return None if a is None else np.asarray(a, np.float32).astype(np.float64)


def _passes(idx, grid):
    return set(((idx // 32) // grid).tolist())


# ------------------------------------------------------------------------------------------------------------------
# CPU tier
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(MODELS))
def test_model_set_covers_its_purpose(name):
    """Each model still exercises what it is here for."""
    mech = MODELS[name]()
    d = mech.flatten()
    kinds = {type(j.joint_type) for j in mech.joints}
    linear = {rbd.Revolute, rbd.Prismatic, rbd.Fixed}
    if name == "atlas":
        assert type(mech.joints[0].joint_type) is rbd.QuaternionFloating and not kinds <= linear and rbd.Revolute in kinds
        assert (d.nb, d.nv) == (31, 36)
    elif name == "iiwa14":
        assert kinds == {rbd.Revolute}                                     # has_other is false: no per-(sample, joint) kernel
    elif name == "randmech":
        assert kinds == {rbd.QuaternionFloating, rbd.Revolute, rbd.Fixed, rbd.Prismatic, rbd.Planar, rbd.SPQuatFloating,
                         rbd.SinCosRevolute, rbd.QuaternionSpherical}
        assert type(mech.joints[0].joint_type) is not rbd.QuaternionFloating   # shuffled: the multi-DoF joints below the root
    else:
        cd = rbd.contact_desc(mech)
        assert len(cd.body) == 8 and len(set(cd.body.tolist())) == 2 and len(cd.halfspace) == 1 and cd.nstates == 24


def test_column_choice_covers_lanes_and_passes():
    for B in (4095, 4096, 1 << 15, 117773, 1 << 20):
        idx = cols(B)
        assert len(idx) == NCOLS and idx[0] == 0 and idx[-1] == B - 1
        assert set((idx % 32).tolist()) == set(range(32))
        s = idx[1] - idx[0]
        assert s % 2 == 1 and s % 32
        grid = (B // 32) // 3 or 1                       # three passes
        assert _passes(idx, grid) >= {0, 1, 2}


def test_pass_count_arithmetic():
    """Atlas in fp64: the cap alone limits the dynamics VJP to about 39 k resident threads and the contact stage adjoint to about 35 k,
    so only batches in the tens of thousands take a second group; the batches of the multi-pass tests take at least three."""
    d = MODELS["atlas"]().flatten()
    assert adjoint_rows(d.nb, d.nv) == 1710 and contact_vjp_rows(d.nb, d.nv) == 1932
    assert cap_threads(adjoint_rows(d.nb, d.nv), 8) == 39232 and cap_threads(contact_vjp_rows(d.nb, d.nv), 8) == 34720
    for rows in (adjoint_rows(d.nb, d.nv), contact_vjp_rows(d.nb, d.nv), TASK_ROWS * (d.nb + 4)):
        for size in (4, 8):
            B = multi_pass_batch(rows, size)
            groups = (B + 31) // 32
            assert B % 32 and groups >= 3 * (cap_threads(rows, size) // 32) + 1
    # the 64-bit offset case: the cotangent's last rows start beyond 2^31 elements
    assert 6 * d.nv * 2 == 432 and 431 * 5_000_000 > 2 ** 31


# ------------------------------------------------------------------------------------------------------------------
# GPU tier: helpers
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch():
    import torch as t
    assert t.cuda.is_available()
    rbd.load_library()
    return t


def _dev(torch, a, dtype, ld=None):
    """[rows, B] numpy -> [rows, ld] CUDA tensor, the padding NaN."""
    rows, B = a.shape
    t = torch.full((rows, ld or B), float("nan"), dtype=dtype, device="cuda")
    t[:, :B] = torch.from_numpy(np.ascontiguousarray(a)).to(dtype)
    return t


def _host(t, idx):
    return t[..., idx].double().cpu().numpy()


def _check_written(torch, outs, B, ld=None):
    """Every column in [0, B) written (finite), the padding untouched (NaN)."""
    for k, t in outs.items():
        if t is None:
            continue
        assert bool(torch.isfinite(t[..., :B]).all()), k
        if ld and ld > B:
            assert bool(torch.isnan(t[..., B:]).all()), k


def _dyn_call(torch, mech, fd, ins, B, ld, dtype, outs=None):
    """rbd_dynamics_vjp (fd) / rbd_inverse_dynamics_vjp on [rows, ld] tensors ins = {q, v, vd, w, bar}; NaN-filled outputs
    {qt, qc, vb, xb, wb} (xb: τ̄ / v̇̄)."""
    from rigidbodydynamics.jl_b200.state import _DT, _model_handle
    d = mech.flatten()
    rows = {"qt": d.nv, "qc": d.nq, "vb": d.nv, "xb": d.nv, "wb": 6 * d.nb}
    if outs is None:
        outs = {k: torch.full((r, ld), float("nan"), dtype=dtype, device="cuda") for k, r in rows.items()}
    p = lambda t: None if t is None else t.data_ptr()      # noqa: E731
    lib = _cabi.load_library()
    h = _model_handle(mech)
    o = [p(outs[k]) for k in ("qt", "qc", "vb", "xb", "wb")]
    if fd:
        st = lib.rbd_dynamics_vjp(h.ptr, _DT[dtype], B, ld, p(ins["q"]), p(ins["v"]), None, p(ins.get("w")), p(ins["vd"]), p(ins["bar"]),
                                  *o, None)
    else:
        st = lib.rbd_inverse_dynamics_vjp(h.ptr, _DT[dtype], B, ld, p(ins["q"]), p(ins["v"]), p(ins["vd"]), p(ins.get("w")),
                                          p(ins["bar"]), *o, None)
    torch.cuda.synchronize()
    assert st == 0, st
    return outs, rbd.launch_info()


def _task_call(torch, mech, tasks, ins, bars, B, ld, dtype, want=GRADS):
    """rbd_task_kinematics_vjp on [rows, ld] tensors; NaN-filled outputs {qt, qc, vb, vdb} for the keys in `want`."""
    from rigidbodydynamics.jl_b200.state import _DT, _model_handle
    d = mech.flatten()
    outs = {k: torch.full((d.nq if k == "qc" else d.nv, ld), float("nan"), dtype=dtype, device="cuda") if k in want else None
            for k in GRADS}
    to = _cabi.RbdTaskOut()
    for k, t in bars.items():
        setattr(to, k, t.data_ptr())
    td, keep = task_desc(mech, tasks)
    p = lambda t: None if t is None else t.data_ptr()      # noqa: E731
    h = _model_handle(mech)
    _cabi.check(_cabi.load_library().rbd_task_kinematics_vjp(h.ptr, _DT[dtype], B, ld, p(ins["q"]), p(ins.get("v")), p(ins.get("vd")),
                                                             ctypes.byref(td), ctypes.byref(to), *[p(outs[k]) for k in GRADS], None))
    torch.cuda.synchronize()
    return outs, rbd.launch_info()


def _dyn_inputs(mech, B, seed, wext):
    rng = np.random.default_rng(seed)
    d = mech.flatten()
    x = {"q": rand_q(mech, B, rng), "v": rng.standard_normal((d.nv, B)), "tau": rng.standard_normal((d.nv, B)),
         "vd": rng.standard_normal((d.nv, B)), "bar": rng.standard_normal((d.nv, B))}
    if wext:
        x["w"] = rng.standard_normal((6 * d.nb, B))
    return x


def _dyn_fd_check(mech, fd, x, got, tol):
    """The VJP at the columns of x (fp64 numpy, vd = the oracle's v̇ for fd) against central differences of the oracle."""
    d = mech.flatten()
    o = Oracle(d)
    q, v, w, bar = x["q"], x["v"], x.get("w"), x["bar"]
    B = q.shape[1]
    f = (lambda q_, v_, a_, w_: o.dynamics(q_, v_, a_, w_)) if fd else (lambda q_, v_, a_, w_: o.inverse_dynamics(q_, v_, a_, w_))
    a = x["tau"] if fd else x["vd"]
    eye = lambda n, k: np.repeat(np.eye(n)[:, k:k + 1], B, 1)      # noqa: E731
    vjp = lambda J: np.einsum("kib,ib->kb", J, bar)                 # noqa: E731
    refs = {"qt": vjp(_fd_central(lambda y: f(y, v, a, w), q, _qdot_dirs(o, q, d.nv, None))),
            "vb": vjp(_fd_central(lambda y: f(q, y, a, w), v, [eye(d.nv, k) for k in range(d.nv)])),
            "xb": vjp(_fd_central(lambda y: f(q, v, y, w), a, [eye(d.nv, k) for k in range(d.nv)]))}
    if w is not None:
        refs["wb"] = vjp(_fd_central(lambda y: f(q, v, a, y), w, [eye(6 * d.nb, k) for k in range(6 * d.nb)]))
    for k, ref in refs.items():
        assert rel_err(got[k], ref) < tol, (k, rel_err(got[k], ref))


# ------------------------------------------------------------------------------------------------------------------
# GPU tier 1 and 2: multi-pass persistent grids, workspace reuse
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
@pytest.mark.parametrize("kind", ["dynamics", "dynamics_wext", "inverse"])
@pytest.mark.parametrize("name", ["atlas", "randmech"])
def test_dynamics_vjp_multi_pass(torch, name, kind, dtype_name):
    dtype = getattr(torch, dtype_name)
    mech = MODELS[name]()
    d = mech.flatten()
    fd, wext = kind != "inverse", kind != "dynamics"
    size = 8 if dtype == torch.float64 else 4
    B = multi_pass_batch(adjoint_rows(d.nb, d.nv), size)
    ld = B + 5
    x = _dyn_inputs(mech, B, 11 + size, wext)
    fc = fd_cols(B)
    if fd:       # v̇ of the forward dynamics on the columns checked against the oracle (any v̇ serves the CPU comparison)
        x["vd"][:, fc] = Oracle(d).dynamics(x["q"][:, fc], x["v"][:, fc], x["tau"][:, fc], None if not wext else x["w"][:, fc])
    ins = {k: _dev(torch, a, dtype, ld) for k, a in x.items() if k != "tau"}
    outs, info = _dyn_call(torch, mech, fd, ins, B, ld, dtype)
    assert info.kernels_launched == 1 and info.block == 32
    assert info.grid * info.block * 3 <= B, (info.grid, B)
    idx = cols(B)
    assert _passes(idx, info.grid) >= {0, 1, (B - 1) // 32 // info.grid}
    _check_written(torch, outs, B, ld)
    if not wext:
        outs["wb"] = None
    hx = {k: _host(t, idx) for k, t in ins.items()}
    ref = host_vjp(d, fd, hx["q"], hx["v"], hx["vd"], hx["bar"], hx.get("w"))
    tol = TOL64 if dtype == torch.float64 else TOL32_VJP
    worst = 0.0
    for k, hk in (("qt", "qt"), ("qc", "qc"), ("vb", "vb"), ("xb", "taub" if fd else "vdb"), ("wb", "wb")):
        if outs[k] is None:
            continue
        e = rel_err(_host(outs[k], idx), ref[hk])
        worst = max(worst, e)
        assert e < tol, (k, e)
    print(f"{name} {kind} {dtype_name} B={B} grid={info.grid}: worst rel_err vs CPU run {worst:.2e}")
    hx = {k: _host(ins[k], fc) for k in ins}
    hx["tau"] = x["tau"][:, fc]
    _dyn_fd_check(mech, fd, hx, {k: _host(t, fc) for k, t in outs.items() if t is not None},
                  TOL_FD if dtype == torch.float64 else TOL32_VJP)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["dynamics", "inverse"])
def test_dynamics_vjp_workspace_reuse_and_nan_isolation(torch, kind):
    """Atlas fp64, multi-pass: a call after an all-NaN call equals the same call after a finite call bit for bit; a NaN sample column
    leaves every other column bit-identical."""
    mech = MODELS["atlas"]()
    d = mech.flatten()
    fd = kind == "dynamics"
    B = multi_pass_batch(adjoint_rows(d.nb, d.nv), 8)
    x = _dyn_inputs(mech, B, 5, True)
    ins = {k: _dev(torch, a, torch.float64) for k, a in x.items() if k != "tau"}
    nan = {k: torch.full_like(t, float("nan")) for k, t in ins.items()}
    run = lambda i: _dyn_call(torch, mech, fd, i, B, B, torch.float64)[0]      # noqa: E731
    run(nan)
    after_nan = run(ins)
    run({k: t * 0.5 for k, t in ins.items()})
    after_finite = run(ins)
    _check_written(torch, after_finite, B)
    for k in after_nan:
        assert torch.equal(after_nan[k], after_finite[k]), k
    j = 5                                      # block 0, lane 5: the same thread then takes groups grid, 2 grid, ...
    bad = {k: t.clone() for k, t in ins.items()}
    for t in bad.values():
        t[:, j] = float("nan")
    got = run(bad)
    for k, t in got.items():
        assert torch.equal(t[:, :j], after_finite[k][:, :j]) and torch.equal(t[:, j + 1:], after_finite[k][:, j + 1:]), k
        assert not bool(torch.isfinite(t[:, j]).all()), k


def _task_inputs(torch, mech, tasks, B, ld, dtype, seed, want=OUTPUTS):
    rng = np.random.default_rng(seed)
    d = mech.flatten()
    ins = {"q": _dev(torch, rand_q(mech, B, rng), dtype, ld), "v": _dev(torch, rng.standard_normal((d.nv, B)), dtype, ld),
           "vd": _dev(torch, rng.standard_normal((d.nv, B)), dtype, ld)}
    gen = torch.Generator(device="cuda").manual_seed(seed)
    bars = {}
    for k in want:
        t = torch.randn((_rows(k, d.nv) * len(tasks), ld), generator=gen, dtype=dtype, device="cuda")
        t[:, B:] = float("nan")
        bars[k] = t
    return ins, bars


def _task_check(torch, mech, tasks, ins, bars, outs, idx, dtype, label):
    """outs at the columns idx against the fp64 CPU run on the same (fp32-rounded) inputs; the worst error is printed."""
    h = {k: _host(t, idx) for k, t in ins.items()}
    ref = host_task_vjp(mech, tasks, h["q"], h.get("v"), h.get("vd"), {k: _host(t, idx) for k, t in bars.items()})
    errs = {k: rel_err(_host(outs[k], idx), ref[k]) for k in GRADS if outs[k] is not None}
    print(f"{label}: " + ", ".join(f"{k} {e:.2e}" for k, e in errs.items()))
    tol = TOL64 if dtype == torch.float64 else TOL32_TASK
    assert max(errs.values()) < tol, errs


def _task_fd_check(torch, mech, tasks, ins, bars, outs, fc, tol):
    h = {k: _host(t, fc) for k, t in ins.items()}
    J = fd_jacobians(mech, tasks, h["q"], h["v"], h["vd"])
    ref = fd_vjp(J, {k: _host(t, fc) for k, t in bars.items()})
    for k in ("qt", "vb", "vdb"):
        assert rel_err(_host(outs[k], fc), ref[k]) < tol, (k, rel_err(_host(outs[k], fc), ref[k]))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
@pytest.mark.parametrize("name", ["atlas", "randmech"])
def test_task_vjp_multi_pass(torch, name, dtype_name):
    dtype = getattr(torch, dtype_name)
    mech = MODELS[name]()
    d = mech.flatten()
    tasks = task_set(mech, 7)
    size = 8 if dtype == torch.float64 else 4
    B = multi_pass_batch(TASK_ROWS * (d.nb + len(tasks)), size)       # the grid itself is read from the launch record
    ld = B + 3
    want = ("point", "twist", "point_jacobian", "acceleration", "point_acceleration")
    ins, bars = _task_inputs(torch, mech, tasks, B, ld, dtype, 3, want)
    outs, info = _task_call(torch, mech, tasks, ins, bars, B, ld, dtype)
    assert info.kernels_launched == 1 and info.grid * info.block * 3 <= B, (info.grid, B)
    idx = cols(B)
    assert _passes(idx, info.grid) >= {0, 1, (B - 1) // 32 // info.grid}
    _check_written(torch, outs, B, ld)
    _task_check(torch, mech, tasks, ins, bars, outs, idx, dtype, f"task {name} {dtype_name} B={B} grid={info.grid}")
    _task_fd_check(torch, mech, tasks, ins, bars, outs, fd_cols(B)[1:], TOL_FD if dtype == torch.float64 else 1e-5)


@pytest.mark.gpu
def test_task_vjp_workspace_reuse_and_nan_isolation(torch):
    mech = MODELS["atlas"]()
    d = mech.flatten()
    tasks = task_set(mech, 8)
    B = multi_pass_batch(TASK_ROWS * (d.nb + len(tasks)), 8)
    ins, bars = _task_inputs(torch, mech, tasks, B, B, torch.float64, 4, ("point", "twist", "point_jacobian", "acceleration"))
    nan = lambda m: {k: torch.full_like(t, float("nan")) for k, t in m.items()}      # noqa: E731
    run = lambda i, b: _task_call(torch, mech, tasks, i, b, B, B, torch.float64)[0]   # noqa: E731
    run(nan(ins), nan(bars))
    after_nan = run(ins, bars)
    run({k: t * 0.5 for k, t in ins.items()}, bars)
    after_finite = run(ins, bars)
    _check_written(torch, after_finite, B)
    for k in GRADS:
        assert torch.equal(after_nan[k], after_finite[k]), k
    j = 9
    bi, bb = {k: t.clone() for k, t in ins.items()}, {k: t.clone() for k, t in bars.items()}
    for t in list(bi.values()) + list(bb.values()):
        t[:, j] = float("nan")
    got = run(bi, bb)
    for k in GRADS:
        t, r = got[k], after_finite[k]
        assert torch.equal(t[:, :j], r[:, :j]) and torch.equal(t[:, j + 1:], r[:, j + 1:]), k
        assert not bool(torch.isfinite(t[:, j]).all()), k


# ------------------------------------------------------------------------------------------------------------------
# the contact rollout adjoint
# ------------------------------------------------------------------------------------------------------------------
def _contact_case(torch, B, dtype, seed, n=2):
    """Atlas on the floor, distinct states, partly in contact; the recorded trajectory and random trajectory cotangents."""
    mech, cd = _atlas_on_floor()
    q, v, tau = _atlas_states(mech, B, seed, vectorised=True)
    s = np.random.default_rng(seed + 1).standard_normal((cd.nstates, B)) * 1e-4
    st = rbd.MechanismState(mech, B, dtype)
    st.q.copy_(torch.from_numpy(q)); st.v.copy_(torch.from_numpy(v))
    sc = torch.from_numpy(s).to(dtype).cuda()
    t = torch.from_numpy(tau).to(dtype).cuda()
    qt, vt, stj = rbd.simulate_contact_trajectory_(st, n, sc, t, dt=DT, contact=cd)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    bars = [torch.randn(x.shape, generator=gen, dtype=dtype, device="cuda") for x in (qt, vt, stj)]
    return mech, cd, t, qt, vt, stj, bars


def _contact_call(torch, mech, cd, t, qt, vt, stj, bars):
    d = mech.flatten()
    B = qt.shape[2]
    e = lambda rows: torch.full((rows, B), float("nan"), dtype=qt.dtype, device="cuda")      # noqa: E731
    out = {"q0t": e(d.nv), "q0c": e(d.nq), "v0b": e(d.nv), "s0b": e(cd.nstates), "taub": torch.zeros_like(t)}
    rbd.integrate_contact_vjp_(mech, qt, vt, stj, t, contact=cd, dt=DT, q_traj_bar=bars[0], v_traj_bar=bars[1], s_traj_bar=bars[2],
                               q0_bar_tan=out["q0t"], q0_bar_cfg=out["q0c"], v0_bar=out["v0b"], s0_bar=out["s0b"], tau_bar=out["taub"])
    torch.cuda.synchronize()
    return out


def _contact_check(torch, mech, cd, t, qt, vt, stj, bars, out, idx, tol, label):
    d = mech.flatten()
    n = qt.shape[0] - 1
    g = lambda x: _host(x, idx)      # noqa: E731
    ref = host_cvjp(d, cd, g(qt), g(vt), g(stj), g(t), n, g(bars[0]), g(bars[1]), g(bars[2]), dt=DT)
    errs = {k: rel_err(g(out[k]), ref[k]) for k in ("q0t", "q0c", "v0b", "s0b", "taub")}
    print(f"{label}: " + ", ".join(f"{k} {e:.2e}" for k, e in errs.items()))
    assert max(errs.values()) < tol, errs
    return errs


def _contact_fd_check(torch, mech, cd, t, qt, vt, stj, bars, out, fc, tol, eps=1e-5):
    """Directional derivatives along v0 and the torques against central differences of the fp64 oracle integrator."""
    d = mech.flatten()
    n = qt.shape[0] - 1
    orc = Oracle(d)
    g = lambda x: _host(x, fc)      # noqa: E731
    q, v, s, tau = g(qt[0]), g(vt[0]), g(stj[0]), g(t)
    qtb, vtb, stb = (g(b) for b in bars)
    f = lambda v_=v, t_=tau: contact_loss(orc, cd, q, v_, s, t_, n, qtb, vtb, stb, dt=DT)      # noqa: E731
    rng = np.random.default_rng(1)
    for key, dx, fun in (("v0b", rng.standard_normal(v.shape), lambda h, dx: f(v_=v + h * dx)),
                         ("taub", rng.standard_normal(tau.shape), lambda h, dx: f(t_=tau + h * dx))):
        ref = (fun(eps, dx) - fun(-eps, dx)) / (2 * eps)
        got = (g(out[key]) * dx).sum(0)
        assert rel_err(got, ref) < tol, (key, got, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
def test_contact_vjp_multi_pass(torch, dtype_name):
    """The contact stage adjoint (contact_vjp_kernel, the last launch of each stage) over at least three persistent passes: its grid is
    at most cap_threads(contact_vjp_rows) threads, and B is three times that plus a part group."""
    dtype = getattr(torch, dtype_name)
    size = 8 if dtype == torch.float64 else 4
    d = MODELS["atlas_contact"]().flatten()
    B = multi_pass_batch(contact_vjp_rows(d.nb, d.nv), size)
    assert (B + 31) // 32 >= 3 * cap_threads(contact_vjp_rows(d.nb, d.nv), size) // 32 + 1
    mech, cd, t, qt, vt, stj, bars = _contact_case(torch, B, dtype, 21)
    touching = (stj[-1] != stj[0]).any(0)
    assert 0.1 < float(touching.double().mean()) < 0.9                # partly in contact
    out = _contact_call(torch, mech, cd, t, qt, vt, stj, bars)
    _check_written(torch, out, B)
    tol = TOL64 if dtype == torch.float64 else TOL32_CONTACT_ATLAS
    _contact_check(torch, mech, cd, t, qt, vt, stj, bars, out, cols(B), tol, f"contact {dtype_name} B={B}")
    _contact_fd_check(torch, mech, cd, t, qt, vt, stj, bars, out, fd_cols(B)[1:], 1e-6 if dtype == torch.float64 else TOL32_CONTACT)


@pytest.mark.gpu
def test_contact_vjp_workspace_reuse_and_nan_isolation(torch):
    d = MODELS["atlas_contact"]().flatten()
    B = multi_pass_batch(contact_vjp_rows(d.nb, d.nv), 8)
    mech, cd, t, qt, vt, stj, bars = _contact_case(torch, B, torch.float64, 31)
    nan = lambda x: torch.full_like(x, float("nan"))      # noqa: E731
    run = lambda a, b, c, e, f: _contact_call(torch, mech, cd, a, b, c, e, f)      # noqa: E731
    run(nan(t), nan(qt), nan(vt), nan(stj), [nan(x) for x in bars])
    after_nan = run(t, qt, vt, stj, bars)
    run(t * 0.5, qt, vt * 0.5, stj, bars)
    after_finite = run(t, qt, vt, stj, bars)
    _check_written(torch, after_finite, B)
    for k in after_nan:
        assert torch.equal(after_nan[k], after_finite[k]), k
    j = 3
    bad = [x.clone() for x in (t, qt, vt, stj)]
    for x in bad:
        x[..., j] = float("nan")
    got = run(*bad, bars)
    for k in got:
        a, r = got[k], after_finite[k]
        assert torch.equal(a[..., :j], r[..., :j]) and torch.equal(a[..., j + 1:], r[..., j + 1:]), k
    # a NaN state touches nothing, so s̄0 of that column may be finite (the cotangents passed through); v̄0 is NaN
    assert not bool(torch.isfinite(got["v0b"][:, j]).all())


# ------------------------------------------------------------------------------------------------------------------
# GPU tier 3: vectorised and per-(sample, joint) adjoint phases
# ------------------------------------------------------------------------------------------------------------------
PHASE = {"open": ("integrate_adjoint_linear_kernel<", "integrate_adjoint_kernel<"),
         "contact": ("integrate_adjoint_linear_kernel<", "integrate_adjoint_kernel<"),
         "pd": ("integrate_adjoint_pd_linear_kernel<", "integrate_adjoint_pd_kernel<")}


def _kernel_counts(torch, fn):
    """(result of fn(), launch record's kernel count, {kernel-name substring: launches}) of one call, from the CUDA activity trace."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    # every call runs 5 nsteps phase kernels on one path or the other: a trace without any of them is incomplete and is taken again
    # (the call is deterministic)
    for _ in range(2):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            res = fn()
            torch.cuda.synchronize()
        k = rbd.launch_info().kernels_launched
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        count = {s: sum(s in nm for nm in names) for pair in PHASE.values() for s in pair}
        if any(count.values()):
            break
    return res, k, count


def _offset(torch, x):
    """x as a contiguous view one element into a fresh buffer: not vector-aligned."""
    buf = torch.empty(x.numel() + 1, dtype=x.dtype, device="cuda")
    y = buf[1:].view(x.shape)
    y.copy_(x)
    return y


def _phase_case(torch, which, name, B, n, seed):
    """One rollout's recorded trajectory, cotangents and the call of its adjoint, in fp64: returns (call(qt, B'), host(idx) -> CPU run,
    fd(out, fc))."""
    f64 = torch.float64
    rng = np.random.default_rng(seed)
    mech = MODELS["atlas_contact" if which == "contact" else name]()
    d = mech.flatten()
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(f64).cuda()      # noqa: E731
    if which == "contact":
        mech, cd, t, qt, vt, stj, bars = _contact_case(torch, B, f64, seed, n)
    else:
        q, v, tau = rand_q(mech, B, rng), rng.standard_normal((d.nv, B)) * 0.3, rng.standard_normal((n, d.nv, B))
        ctrl = _controller(mech, q, rng, ct=False, per_sample=True, clamp=True) if which == "pd" else None
        t = T(tau)
        if which == "pd":
            qt, vt, _ = _record(mech, T(q), T(v), t, ctrl.torch(f64), DT, n)
        else:
            st = rbd.MechanismState(mech, B, f64)
            st.q.copy_(T(q)); st.v.copy_(T(v))
            qt, vt = rbd.simulate_trajectory_(st, n, t, dt=DT)
        gen = torch.Generator(device="cuda").manual_seed(seed)
        bars = [torch.randn(x.shape, generator=gen, dtype=f64, device="cuda") for x in (qt, vt)]

    def call(qt_, m):
        sl = lambda x: x[..., :m].contiguous()       # noqa: E731
        q_, v_, t_, b_ = (qt_ if m == B else sl(qt_)), sl(vt), sl(t), [sl(x) for x in bars]
        e = lambda rows: torch.full((rows, m), float("nan"), dtype=f64, device="cuda")      # noqa: E731
        out = {"q0t": e(d.nv), "q0c": e(d.nq), "v0b": e(d.nv), "taub": torch.zeros_like(t_)}
        if which == "contact":
            out["s0b"] = e(cd.nstates)
            rbd.integrate_contact_vjp_(mech, q_, v_, sl(stj), t_, contact=cd, dt=DT, q_traj_bar=b_[0], v_traj_bar=b_[1], s_traj_bar=b_[2],
                                       q0_bar_tan=out["q0t"], q0_bar_cfg=out["q0c"], v0_bar=out["v0b"], s0_bar=out["s0b"], tau_bar=out["taub"])
        elif which == "pd":
            ctl = _ctrl_cols(ctrl, slice(0, m)).torch(f64)
            out.update(kp_bar=torch.zeros((d.nv, m), dtype=f64, device="cuda"), kd_bar=torch.zeros((d.nv, m), dtype=f64, device="cuda"),
                       q_ref_bar=torch.zeros_like(ctl.q_ref), v_ref_bar=torch.zeros_like(ctl.v_ref))
            rbd.integrate_pd_vjp_(mech, q_, v_, t_, controller=ctl, dt=DT, q_traj_bar=b_[0], v_traj_bar=b_[1], q0_bar_tan=out["q0t"],
                                  q0_bar_cfg=out["q0c"], v0_bar=out["v0b"], tau_bar=out["taub"], kp_bar=out["kp_bar"], kd_bar=out["kd_bar"],
                                  q_ref_bar=out["q_ref_bar"], v_ref_bar=out["v_ref_bar"])
        else:
            rbd.integrate_vjp_(mech, q_, v_, t_, dt=DT, q_traj_bar=b_[0], v_traj_bar=b_[1], q0_bar_tan=out["q0t"], q0_bar_cfg=out["q0c"],
                               v0_bar=out["v0b"], tau_bar=out["taub"])
        return out

    def host(out, idx, tol):
        g = lambda x: _host(x, idx)      # noqa: E731
        if which == "contact":
            _contact_check(torch, mech, cd, t, qt, vt, stj, bars, out, idx, tol, f"contact {B}")
            return
        if which == "pd":
            ref = host_pd_vjp(d, g(qt), g(vt), _ctrl_cols(ctrl, idx), g(t), g(bars[0]), g(bars[1]), DT)
            pairs = (("q0c", "q0c"), ("v0b", "v0b"), ("taub", "taub"), ("kp_bar", "kp"), ("kd_bar", "kd"), ("q_ref_bar", "q_ref"),
                     ("v_ref_bar", "v_ref"))
        else:
            ref = host_ivjp(d, g(qt), g(vt), g(t), n, g(bars[0]), g(bars[1]), dt=DT)
            pairs = (("q0t", "q0t"), ("q0c", "q0c"), ("v0b", "v0b"), ("taub", "taub"))
        for k, hk in pairs:
            e = rel_err(g(out[k]).reshape(ref[hk].shape), ref[hk])
            assert e < tol, (which, name, k, e)

    def fd(out, fc, tol):
        if which == "contact":
            _contact_fd_check(torch, mech, cd, t, qt, vt, stj, bars, out, fc, tol)
            return
        g = lambda x: _host(x, fc)      # noqa: E731
        q0, v0, tau0, qtb, vtb = g(qt[0]), g(vt[0]), g(t), g(bars[0]), g(bars[1])
        o = Oracle(d)
        if which == "pd":
            c = _ctrl_cols(ctrl, fc)
            f = lambda v_, t_: _pd_loss(o, q0, v_, c, t_, n, qtb, vtb)      # noqa: E731
        else:
            f = lambda v_, t_: _oracle_loss(o, q0, v_, list(t_), n, qtb, vtb, dt=DT)      # noqa: E731
        _dir_fd(f, v0, tau0, g(out["v0b"]), g(out["taub"]), tol)

    return call, qt, host, fd


def _dir_fd(f, v0, tau0, v0b, taub, tol, eps=1e-5):
    rng = np.random.default_rng(2)
    dv, dt_ = rng.standard_normal(v0.shape), rng.standard_normal(tau0.shape)
    ref_v = (f(v0 + eps * dv, tau0) - f(v0 - eps * dv, tau0)) / (2 * eps)
    ref_t = (f(v0, tau0 + eps * dt_) - f(v0, tau0 - eps * dt_)) / (2 * eps)
    assert rel_err((v0b * dv).sum(0), ref_v) < tol, ((v0b * dv).sum(0), ref_v)
    assert rel_err((taub * dt_).sum(tuple(range(taub.ndim - 1))), ref_t) < tol


def _ctrl_cols(ctrl, idx):
    """The controller of the sample columns idx (per-sample arrays sliced, shared gains kept)."""
    c = lambda a, per: None if a is None else (a[..., idx] if per else a)      # noqa: E731
    per_gain = np.ndim(ctrl.kp) == 2
    return Ctrl(c(ctrl.kp, per_gain), c(ctrl.kd, per_gain), c(ctrl.q_ref, True), c(ctrl.v_ref, True), c(ctrl.vd_ref, True), ctrl.ct,
                ctrl.bounds)


def _pd_loss(o, q0, v0, ctrl, tau, n, qtb, vtb):
    """Σ_s q̄_s . q_s + v̄_s . v_s of the oracle's closed-loop rollout, one step at a time."""
    q, v = q0, v0
    L = (qtb[0] * q).sum(0) + (vtb[0] * v).sum(0)
    for s in range(n):
        c = Ctrl(ctrl.kp, ctrl.kd, ctrl.at(ctrl.q_ref, s), ctrl.at(ctrl.v_ref, s), ctrl.at(ctrl.vd_ref, s), ctrl.ct, ctrl.bounds)
        q, v, _ = integrate_pd(o, q, v, c, tau[s], dt=DT, nsteps=1)
        L = L + (qtb[s + 1] * q).sum(0) + (vtb[s + 1] * v).sum(0)
    return L


PHASE_CASES = [("open", "iiwa14"), ("open", "atlas"), ("pd", "iiwa14"), ("pd", "atlas"), ("contact", "atlas")]


@pytest.mark.gpu
@pytest.mark.parametrize("which,name", PHASE_CASES, ids=[f"{w}-{m}" for w, m in PHASE_CASES])
def test_vectorised_and_per_joint_phases(torch, which, name):
    """B = 4096 with aligned arrays runs the vectorised phase kernel; B = 4095 and a q_traj one element into its buffer run the
    per-(sample, joint) kernel on every row.  fp64: the three agree to 1e-12 and with the CPU run to 1e-10."""
    n, B = 2, 4096
    call, qt, host, fd = _phase_case(torch, which, name, B, n, 40 + len(name))
    lin, per = PHASE[which]
    other = name == "atlas"                # a floating base: the per-(sample, joint) kernel runs beside the vectorised one
    a, ka, ca = _kernel_counts(torch, lambda: call(qt, B))
    assert ca[lin] == 5 * n and ca[per] == (5 * n if other else 0), ca
    b, kb, cb = _kernel_counts(torch, lambda: call(_offset(torch, qt), B))
    assert cb[lin] == 0 and cb[per] == 5 * n, cb
    # the recompute is the same for both (it depends on B only): the launch-count difference is the vectorised phase kernels
    assert ka - kb == (5 * n if other else 0), (ka, kb)
    c, kc, cc = _kernel_counts(torch, lambda: call(qt, B - 1))
    assert cc[lin] == 0 and cc[per] == 5 * n, cc
    for k in a:
        x, y, z = a[k], b[k], c[k]
        scale = max(1.0, float(x.abs().max()))
        assert float((x - y).abs().max()) <= TOL_VEC * scale, k
        assert float((x[..., :B - 1] - z).abs().max()) <= TOL_VEC * scale, k
    _check_written(torch, a, B)
    idx = cols(B)
    host(a, idx, TOL64)
    host(c, idx[:-1].tolist() + [B - 2], TOL64)
    fd(a, fd_cols(B)[1:], 1e-6)


# ------------------------------------------------------------------------------------------------------------------
# GPU tier 4: fp32 at 2^20 on Atlas
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_fp32_at_scale_contact(torch):
    B = 1 << 20
    mech, cd, t, qt, vt, stj, bars = _contact_case(torch, B, torch.float32, 51)
    touching = (stj[-1] != stj[0]).any(0)
    assert 0.1 < float(touching.double().mean()) < 0.9
    out = _contact_call(torch, mech, cd, t, qt, vt, stj, bars)
    _check_written(torch, out, B)
    idx = cols(B)
    _contact_check(torch, mech, cd, t, qt, vt, stj, bars, out, idx, TOL32_CONTACT_ATLAS, "fp32 2^20 contact, worst rel_err")
    _contact_fd_check(torch, mech, cd, t, qt, vt, stj, bars, out, fd_cols(B)[1:], TOL32_CONTACT)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["pd", "ct"])
def test_fp32_at_scale_pd(torch, mode):
    B, n = 1 << 20, 2
    f32 = torch.float32
    mech = MODELS["atlas"]()
    d = mech.flatten()
    rng = np.random.default_rng(61)
    q, v = r32(rand_q(mech, B, rng)), r32(rng.standard_normal((d.nv, B)) * 0.3)
    tau = r32(rng.standard_normal((n, d.nv, B)))
    ctrl = _controller(mech, q, rng, ct=mode == "ct", per_sample=True, clamp=True)
    ctrl.kp, ctrl.kd, ctrl.q_ref, ctrl.v_ref, ctrl.vd_ref = (r32(a) for a in (ctrl.kp, ctrl.kd, ctrl.q_ref, ctrl.v_ref, ctrl.vd_ref))
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(f32).cuda()      # noqa: E731
    ctl = ctrl.torch(f32)
    t = T(tau)
    qt, vt, _ = _record(mech, T(q), T(v), t, ctl, DT, n)
    gen = torch.Generator(device="cuda").manual_seed(3)
    qtb, vtb = (torch.randn(x.shape, generator=gen, dtype=f32, device="cuda") for x in (qt, vt))
    e = lambda rows: torch.full((rows, B), float("nan"), dtype=f32, device="cuda")      # noqa: E731
    z = lambda x: None if x is None else torch.zeros_like(x)      # noqa: E731
    out = dict(q0_bar_cfg=e(d.nq), v0_bar=e(d.nv), tau_bar=z(t), kp_bar=z(ctl.kp), kd_bar=z(ctl.kd), q_ref_bar=z(ctl.q_ref),
               v_ref_bar=z(ctl.v_ref), vd_ref_bar=z(ctl.vd_ref))
    rbd.integrate_pd_vjp_(mech, qt, vt, t, controller=ctl, dt=DT, q_traj_bar=qtb, v_traj_bar=vtb, **out)
    torch.cuda.synchronize()
    _check_written(torch, out, B)
    idx = cols(B)
    g = lambda x: _host(x, idx)      # noqa: E731
    ref = host_pd_vjp(d, g(qt), g(vt), _ctrl_cols(ctrl, idx), tau[..., idx], g(qtb), g(vtb), DT)
    pairs = (("q0_bar_cfg", "q0c"), ("v0_bar", "v0b"), ("tau_bar", "taub"), ("kp_bar", "kp"), ("kd_bar", "kd"), ("q_ref_bar", "q_ref"),
             ("v_ref_bar", "v_ref"), ("vd_ref_bar", "vd_ref"))
    errs = {k: rel_err(g(out[k]), ref[hk]) for k, hk in pairs if out[k] is not None}
    print(f"fp32 2^20 PD {mode}, worst rel_err: " + ", ".join(f"{k} {x:.2e}" for k, x in errs.items()))
    assert max(errs.values()) < TOL32_PD[mode], errs
    fc = fd_cols(B)[1:]
    h = lambda x: _host(x, fc)      # noqa: E731
    c = _ctrl_cols(ctrl, fc)
    _dir_fd(lambda v_, t_: _pd_loss(Oracle(d), h(qt[0]), v_, c, t_, n, h(qtb), h(vtb)), h(vt[0]), tau[..., fc], h(out["v0_bar"]),
            h(out["tau_bar"]), TOL32_PD[mode])


@pytest.mark.gpu
def test_fp32_at_scale_task_all_outputs(torch):
    B = 1 << 20
    mech = MODELS["atlas"]()
    tasks = [TaskFrame(mech.findbody(nm), None, p, None) for nm, p in END_EFFECTORS]
    ins, bars = _task_inputs(torch, mech, tasks, B, B, torch.float32, 71)
    outs, info = _task_call(torch, mech, tasks, ins, bars, B, B, torch.float32)
    assert info.kernels_launched == 1 and info.grid * info.block * 3 <= B
    _check_written(torch, outs, B)
    _task_check(torch, mech, tasks, ins, bars, outs, cols(B), torch.float32, "fp32 2^20 task, all eight cotangents, worst rel_err")
    _task_fd_check(torch, mech, tasks, ins, bars, outs, fd_cols(B)[1:], 1e-5)


# ------------------------------------------------------------------------------------------------------------------
# GPU tier 5: the recompute through the model-specialised fp32 programs, the gated fallback inside it
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("which", ["open", "pd"])
def test_recompute_through_specialised_programs(torch, which):
    """Atlas fp32 at B = 2^15 (RBD_JIT_MIN_BATCH): the recorded trajectory and every step's recompute run the specialised programs; one
    sample's revolute angle is 2e4 rad, beyond their fast sin / cos range, so the gated generic fallback recomputes it."""
    B, n = 1 << 15, 2
    f32 = torch.float32
    mech = MODELS["atlas"]()
    d = mech.flatten()
    rng = np.random.default_rng(81)
    q, v = rand_q(mech, B, rng), rng.standard_normal((d.nv, B)) * 0.3
    j = B // 2 + 11
    assert type(mech.joints[1].joint_type) is rbd.Revolute and d.qstart[1] == 7
    q[7, j] = 2e4
    q, v, tau = r32(q), r32(v), r32(rng.standard_normal((n, d.nv, B)))
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(f32).cuda()      # noqa: E731
    t = T(tau)
    gen = torch.Generator(device="cuda").manual_seed(5)
    e = lambda rows: torch.full((rows, B), float("nan"), dtype=f32, device="cuda")      # noqa: E731
    out = {"q0_bar_cfg": e(d.nq), "v0_bar": e(d.nv), "tau_bar": torch.zeros_like(t)}
    if which == "pd":
        ctrl = _controller(mech, q, rng, per_sample=True, clamp=True)
        ctrl.kp, ctrl.kd, ctrl.q_ref, ctrl.v_ref = (r32(a) for a in (ctrl.kp, ctrl.kd, ctrl.q_ref, ctrl.v_ref))
        ctl = ctrl.torch(f32)
        qt, vt, _ = _record(mech, T(q), T(v), t, ctl, DT, n)
        qtb, vtb = (torch.randn(x.shape, generator=gen, dtype=f32, device="cuda") for x in (qt, vt))
        rbd.integrate_pd_vjp_(mech, qt, vt, t, controller=ctl, dt=DT, q_traj_bar=qtb, v_traj_bar=vtb, **out)
    else:
        st = rbd.MechanismState(mech, B, f32)
        st.q.copy_(T(q)); st.v.copy_(T(v))
        qt, vt = rbd.simulate_trajectory_(st, n, t, dt=DT)
        qtb, vtb = (torch.randn(x.shape, generator=gen, dtype=f32, device="cuda") for x in (qt, vt))
        rbd.integrate_vjp_(mech, qt, vt, t, dt=DT, q_traj_bar=qtb, v_traj_bar=vtb, q0_bar_cfg=out["q0_bar_cfg"], v0_bar=out["v0_bar"],
                           tau_bar=out["tau_bar"])
    torch.cuda.synchronize()
    assert rbd.launch_info().specialised == 1
    assert abs(float(qt[-1, 7, j])) > 1e4
    _check_written(torch, out, B)
    idx = np.unique(np.append(cols(B), j))
    g = lambda x: _host(x, idx)      # noqa: E731
    if which == "pd":
        ref = host_pd_vjp(d, g(qt), g(vt), _ctrl_cols(ctrl, idx), tau[..., idx], g(qtb), g(vtb), DT)
        tol = TOL32_PD["pd"]
    else:
        ref = host_ivjp(d, g(qt), g(vt), tau[..., idx], n, g(qtb), g(vtb), dt=DT)
        tol = TOL32_ROLLOUT
    for k, hk in (("q0_bar_cfg", "q0c"), ("v0_bar", "v0b"), ("tau_bar", "taub")):
        got = g(out[k])
        assert rel_err(got, ref[hk]) < tol, (k, rel_err(got, ref[hk]))
        jj = int(np.searchsorted(idx, j))
        assert rel_err(got[..., jj:jj + 1], ref[hk][..., jj:jj + 1]) < tol, k


# ------------------------------------------------------------------------------------------------------------------
# GPU tier 6: 64-bit element offsets
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_task_vjp_64bit_offsets(torch):
    """Atlas fp32, the geometric Jacobian of two tasks as the only cotangent: 432 rows x (5e6 + 3) columns, 2.16e9 elements (8.6 GB).
    Rows 430 and 431 start beyond 2^31 elements."""
    f32 = torch.float32
    mech = MODELS["atlas"]()
    d = mech.flatten()
    tasks = [TaskFrame(mech.findbody(nm), None, p, None) for nm, p in END_EFFECTORS[:2]]
    B, rows = 5_000_000, 6 * d.nv * 2
    ld = B + 3
    need = (rows + d.nq + d.nv) * ld * 4 + CAP + (256 << 20)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")
    gen = torch.Generator(device="cuda").manual_seed(9)
    q = torch.full((d.nq, ld), float("nan"), dtype=f32, device="cuda")        # Atlas: a unit quaternion, a position, revolute angles
    quat = torch.randn((4, B), generator=gen, dtype=f32, device="cuda")
    q[:4, :B] = quat / quat.norm(dim=0)
    q[4:7, :B] = torch.rand((3, B), generator=gen, dtype=f32, device="cuda") - 0.5
    q[7:, :B] = torch.randn((d.nq - 7, B), generator=gen, dtype=f32, device="cuda")
    del quat
    J = torch.randn((rows, ld), generator=gen, dtype=f32, device="cuda")
    J[:, B:] = float("nan")
    outs, info = _task_call(torch, mech, tasks, {"q": q}, {"geometric_jacobian": J}, B, ld, f32, want=("qt",))
    assert info.kernels_launched == 1
    _check_written(torch, {"qt": outs["qt"]}, B, ld)
    idx = np.concatenate([np.arange(64), np.arange(B // 2 - 17, B // 2 + 16), np.arange(B - 64, B)])
    ref = host_task_vjp(mech, tasks, _host(q, idx), None, None, {"geometric_jacobian": _host(J, idx)})
    e = rel_err(_host(outs["qt"], idx), ref["qt"])
    print(f"64-bit offsets: rel_err {e:.2e}")
    assert e < TOL32_TASK, e
    del q, J, outs
    torch.cuda.empty_cache()
