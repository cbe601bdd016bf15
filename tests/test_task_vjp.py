"""Reverse mode of task-space kinematics (DESIGN 4.20): rbd_task_kinematics_vjp, autodiff.task_kinematics_vjp_ and
autodiff.task_kinematics.

CPU tier (the device code compiled for the host: tests/hostsim/hostsim_task_vjp.cpp)
1. task_vjp_sample against central differences of the fp64 oracle (tests/task_oracle.py) along the tangent directions of q and the
   unit directions of v and v̇: Atlas, Valkyrie, iiwa14, the double pendulum and every-joint-type trees; tasks with body == base,
   base = root, body = root and F in {root, body, base, a third body}, points on and off the origin; vd given and None; each
   output's cotangent alone and all eight together.
2. Exact identities against the forward kernel's own Jacobians: twist -> v̄ = Jᵀ t̄, point_velocity -> v̄ = J_pᵀ ū, acceleration
   -> v̇̄ = Jᵀ ā, point_acceleration -> v̇̄ = J_pᵀ ū, and point -> q̄_tan = J_pᵀ p̄ for base = root and F = root.
3. q̄_cfg . (N(q) u) == q̄_tan . u, and no radial quaternion component.
4. Linearity over the outputs; cotangent rows of off-path Jacobian columns are not read.
5. The argument checks of rbd_task_kinematics_vjp, on the host.
GPU tier: the kernel against the CPU run of the same code, strides and tiles, the launch count, gradcheck, composition with
autodiff.simulate, batched gradient-descent IK, and Atlas fp32 at 2^20.
"""
import ctypes
import functools

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from oracle import Oracle
from rigidbodydynamics.jl_b200 import _cabi
from rigidbodydynamics.jl_b200._cabi import RbdModelDesc, RbdTaskDesc, make_desc
from rigidbodydynamics.jl_b200.kinematics import TaskFrame, task_desc
from tests import hostsim
from tests.task_oracle import OUTPUTS, TaskOracle
from tests.test_task_kinematics import VEL_OUTPUTS, _rows, hostsim_tasks, task_set
from tests.util import rand_inputs, randmech, rel_err


TOL_FD = 2e-6         # central finite differences, eps = 1e-6 (test_vjp.py)
GRADS = ("qt", "qc", "vb", "vdb")
K_QFLOAT, K_QSPH = 4, 6


@functools.cache
def _shim():
    """tests/hostsim/hostsim_task_vjp.cpp, compiled and loaded by hostsim.shim."""
    lib = hostsim.shim("hostsim_task_vjp")
    lib.hostsim_task_kinematics_vjp.argtypes = [ctypes.POINTER(RbdModelDesc), ctypes.POINTER(RbdTaskDesc), ctypes.c_int, ctypes.c_int64,
                                                ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def host_vjp(mech, tasks, q, v, vd, bars):
    """task_vjp_sample on the CPU for the cotangents ``bars`` ({output: [rows * K, B]}); returns {qt, qc, vb, vdb}."""
    desc = mech.flatten()
    dt = q.dtype
    d, keep = make_desc(desc)
    td, keep2 = task_desc(mech, tasks)
    c = lambda a: None if a is None else np.ascontiguousarray(a, dt)     # noqa: E731
    q, v, vd = c(q), c(v), c(vd)
    bars = {k: c(b) for k, b in bars.items()}
    B = q.shape[1]
    out = {k: np.full((desc.nq if k == "qc" else desc.nv, B), np.nan, dt) for k in GRADS}
    p = lambda a: None if a is None or a.size == 0 else a.ctypes.data      # noqa: E731
    bp = (ctypes.c_void_p * 8)(*[p(bars.get(k)) for k in OUTPUTS])
    op = (ctypes.c_void_p * 4)(*[p(out[k]) for k in GRADS])
    rc = _shim().hostsim_task_kinematics_vjp(ctypes.byref(d), ctypes.byref(td), 0 if dt == np.float32 else 1, B, p(q), p(v), p(vd),
                                             bp, op)
    assert rc == 0, rc
    return out


def rand_bars(mech, K, B, seed, want=OUTPUTS):
    rng = np.random.default_rng(seed)
    nv = mech.num_velocities()
    return {k: rng.standard_normal((_rows(k, nv) * K, B)) for k in want}


def qdot_dirs(mech, q):
    """velocity_to_configuration_derivative(e_k) per sample, [nv, nq, B]: the tangent directions of q."""
    d = mech.flatten()
    o = Oracle(d)
    B = q.shape[1]
    out = []
    for k in range(d.nv):
        e = np.zeros((d.nv, B)); e[k] = 1.0
        out.append(o.dynamics(q, e, None, want_qd=True)[1])
    return np.stack(out)


def fd_jacobians(mech, tasks, q, v, vd, eps=1e-6):
    """Central differences of every output of the oracle along the tangent directions of q and the unit directions of v and v̇:
    {var: {output: [n_dirs, rows, B]}}."""
    nv, B = mech.num_velocities(), q.shape[1]
    vd0 = np.zeros((nv, B)) if vd is None else vd
    f = lambda q_, v_, vd_: TaskOracle(mech, q_, v_, vd_).tasks(tasks)     # noqa: E731
    eye = [np.repeat(np.eye(nv)[:, k:k + 1], B, 1) for k in range(nv)]
    out = {}
    for var, x, dirs in (("q", q, qdot_dirs(mech, q)), ("v", v, eye), ("vd", vd0, eye)):
        per = []
        for dk in dirs:
            args_p, args_m = [q, v, vd0], [q, v, vd0]
            i = ("q", "v", "vd").index(var)
            args_p[i], args_m[i] = x + eps * dk, x - eps * dk
            yp, ym = f(*args_p), f(*args_m)
            per.append({k: (yp[k] - ym[k]) / (2 * eps) for k in OUTPUTS})
        out[var] = {k: np.stack([p[k] for p in per]) for k in OUTPUTS}
    return out


def fd_vjp(J, bars):
    """Σ_outputs ȳ . ∂y/∂x from the finite-difference Jacobians: {qt, vb, vdb}."""
    res = {}
    for var, key in (("q", "qt"), ("v", "vb"), ("vd", "vdb")):
        res[key] = sum(np.einsum("kib,ib->kb", J[var][k], b) for k, b in bars.items())
    return res


# ------------------------------------------------------------------------------------------------------------------
# CPU tier 1: central differences of the oracle
# ------------------------------------------------------------------------------------------------------------------
FD_MODELS = [("atlas", True), ("valkyrie", False), ("iiwa14", False), ("double_pendulum", False), ("randmech", 17),
             ("randmech", 18)]


def _model(name, arg):
    if name == "randmech":
        return randmech(arg, shuffle=arg % 2 == 1)
    return rbd.load_model(name, floating=arg)


@pytest.mark.parametrize("name,arg", FD_MODELS, ids=[f"{n}-{a}" for n, a in FD_MODELS])
def test_vjp_matches_central_differences(name, arg):
    mech = _model(name, arg)
    seed = 3 if name != "randmech" else arg
    q, v, _, vd, _ = rand_inputs(mech, 2, seed)
    if name == "randmech" and arg % 2 == 0:
        vd = None
    tasks = task_set(mech, seed)
    J = fd_jacobians(mech, tasks, q, v, vd)
    allbars = rand_bars(mech, len(tasks), 2, seed + 100)
    for want in [(k,) for k in OUTPUTS] + [OUTPUTS]:
        bars = {k: allbars[k] for k in want}
        got = host_vjp(mech, tasks, q, v if set(want) & set(VEL_OUTPUTS) else None, vd, bars)
        ref = fd_vjp(J, bars)
        for key in ("qt", "vb", "vdb"):
            assert rel_err(got[key], ref[key]) < TOL_FD, (want, key, rel_err(got[key], ref[key]))


# ------------------------------------------------------------------------------------------------------------------
# CPU tier 2: exact identities against the forward kernel's Jacobians
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,arg", [("atlas", True), ("randmech", 19), ("randmech", 20)])
def test_vjp_identities_with_forward_jacobians(name, arg):
    mech = _model(name, arg)
    nv = mech.num_velocities()
    q, v, _, vd, _ = rand_inputs(mech, 3, 7)
    tasks = task_set(mech, 7)
    K = len(tasks)
    fw = hostsim_tasks(mech, tasks, q, v, vd, want=("geometric_jacobian", "point_jacobian"))
    Jg = fw["geometric_jacobian"].reshape(K, nv, 6, -1)
    Jp = fw["point_jacobian"].reshape(K, nv, 3, -1)
    bars = rand_bars(mech, K, 3, 8, want=("twist", "point_velocity", "acceleration", "point_acceleration", "point"))
    JT = lambda Jm, b, r: np.einsum("tkcb,tcb->kb", Jm, b.reshape(K, r, -1))     # noqa: E731
    for out, key, Jm, r in (("twist", "vb", Jg, 6), ("point_velocity", "vb", Jp, 3), ("acceleration", "vdb", Jg, 6),
                            ("point_acceleration", "vdb", Jp, 3)):
        got = host_vjp(mech, tasks, q, v, vd, {out: bars[out]})[key]
        ref = JT(Jm, bars[out], r)
        assert rel_err(got, ref) < 1e-12, (out, rel_err(got, ref))
    # point, base = root, F = root: the point in the root frame moves with every joint on its path
    root_tasks = [TaskFrame(t.body, None, t.point, None) for t in tasks]
    fw = hostsim_tasks(mech, root_tasks, q, v, vd, want=("point_jacobian",))
    Jp = fw["point_jacobian"].reshape(K, nv, 3, -1)
    got = host_vjp(mech, root_tasks, q, None, None, {"point": bars["point"]})["qt"]
    assert rel_err(got, JT(Jp, bars["point"], 3)) < 1e-12


# ------------------------------------------------------------------------------------------------------------------
# CPU tier 3 and 4: configuration covector, linearity, off-path rows
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [21, 22])
def test_q_bar_cfg_and_linearity(seed):
    mech = randmech(seed, shuffle=True)
    desc = mech.flatten()
    nv = desc.nv
    B = 3
    q, v, _, vd, _ = rand_inputs(mech, B, seed)
    tasks = task_set(mech, seed)
    K = len(tasks)
    bars = rand_bars(mech, K, B, seed + 1)
    full = host_vjp(mech, tasks, q, v, vd, bars)
    rng = np.random.default_rng(seed)
    for _ in range(3):
        u = rng.standard_normal((nv, B))
        qd = hostsim.dynamics(desc, q, u, want_qd=True)[1]            # N(q) u
        lhs, rhs = (full["qc"] * qd).sum(0), (full["qt"] * u).sum(0)
        assert np.abs(lhs - rhs).max() <= 1e-12 * max(1.0, np.abs(rhs).max())
    for i, jt in enumerate(desc.jtype):                             # no radial quaternion component
        if jt in (K_QFLOAT, K_QSPH):
            s = desc.qstart[i]
            assert np.abs((full["qc"][s:s + 4] * q[s:s + 4]).sum(0)).max() < 1e-12
    parts = [host_vjp(mech, tasks, q, v, vd, {k: bars[k]}) for k in OUTPUTS]
    for key in GRADS:
        assert rel_err(sum(p[key] for p in parts), full[key]) < 1e-12, key
    # off-path Jacobian columns: their cotangent rows are not read (NaN there changes nothing)
    Jg = hostsim_tasks(mech, tasks, q, v, vd, want=("geometric_jacobian",))["geometric_jacobian"].reshape(K, nv, 6, B)
    sign = np.abs(Jg).sum((2, 3)) == 0
    nb = dict(bars)
    nb["geometric_jacobian"] = bars["geometric_jacobian"].reshape(K, nv, 6, B).copy()
    nb["geometric_jacobian"][sign] = np.nan
    nb["point_jacobian"] = bars["point_jacobian"].reshape(K, nv, 3, B).copy()
    nb["point_jacobian"][sign] = np.nan
    nb = {k: b.reshape(-1, B) for k, b in nb.items()}
    masked = host_vjp(mech, tasks, q, v, vd, nb)
    assert sign.any()
    for key in GRADS:
        assert np.isfinite(masked[key]).all(), key
        assert rel_err(masked[key], full[key]) < 1e-12, key


# ------------------------------------------------------------------------------------------------------------------
# CPU tier 5: argument checks (decided on the host before any CUDA call)
# ------------------------------------------------------------------------------------------------------------------
def test_argument_checks(built):
    lib = rbd.load_library()
    mech = rbd.load_model("iiwa14")
    h = _cabi.ModelHandle(mech.flatten())
    nb = len(mech.joints)
    good = [TaskFrame(mech.joints[-1].successor, None, [0.1, 0, 0], mech.joints[2].successor)]
    d, keep = task_desc(mech, good)
    buf = np.zeros(64)
    q = buf.ctypes.data_as(ctypes.c_void_p)
    bar = _cabi.RbdTaskOut()
    bar.point = buf.ctypes.data

    def call(model=h.ptr, dtype=_cabi.RBD_F64, B=1, ld=1, q=q, v=None, vd=None, tasks=ctypes.byref(d), out=ctypes.byref(bar)):
        return lib.rbd_task_kinematics_vjp(model, dtype, B, ld, q, v, vd, tasks, out, None, None, None, None, None)

    def edited(**kw):
        dd = _cabi.RbdTaskDesc()
        for f, _ in _cabi.RbdTaskDesc._fields_:
            setattr(dd, f, kw.get(f, getattr(d, f)))
        return ctypes.byref(dd)

    bad = lambda val: np.array([val], np.int32).ctypes.data_as(ctypes.POINTER(ctypes.c_int32))   # noqa: E731
    arrs = []
    for f in ("body", "base", "frame"):
        for val in (nb, -2):
            arrs.append(bad(val))
            assert call(tasks=edited(**{f: arrs[-1]})) == _cabi.RBD_EINVAL, (f, val)
    assert call(model=None) == _cabi.RBD_EINVAL
    assert call(q=None) == _cabi.RBD_EINVAL
    assert call(tasks=None) == _cabi.RBD_EINVAL
    assert call(out=None) == _cabi.RBD_EINVAL
    assert call(tasks=edited(ntasks=-1)) == _cabi.RBD_EINVAL
    assert call(tasks=edited(ntasks=_cabi.RBD_MAX_TASKS + 1)) == _cabi.RBD_EUNSUPPORTED
    assert call(tasks=edited(body=None)) == _cabi.RBD_EINVAL
    assert call(dtype=_cabi.RBD_DUAL64X6) == _cabi.RBD_EUNSUPPORTED
    assert call(dtype=7) == _cabi.RBD_EUNSUPPORTED
    assert call(B=4, ld=3) == _cabi.RBD_EDIM
    assert call(B=-1, ld=0) == _cabi.RBD_EDIM
    for name in VEL_OUTPUTS:                             # v NULL with a velocity-dependent cotangent
        o2 = _cabi.RbdTaskOut()
        setattr(o2, name, buf.ctypes.data)
        assert call(out=ctypes.byref(o2)) == _cabi.RBD_EINVAL, name
    assert call(B=0, ld=0) == _cabi.RBD_OK               # empty batch: nothing read or written, no device touched
    h.close()


# ------------------------------------------------------------------------------------------------------------------
# GPU tier
# ------------------------------------------------------------------------------------------------------------------
# fp32 kernel against the fp64 CPU run, rel_err over all four gradients: worst measured on an H100 80GB HBM3 1.6e-6 (Atlas, q̄_cfg;
# the other models 1.04e-6 and below, DESIGN 4.20); the bound is about 5x that
TOL32 = 8e-6
END_EFFECTORS = (("l_hand", [0.0, 0.1, 0.0]), ("r_hand", [0.0, -0.1, 0.0]), ("l_foot", [0.05, 0.0, -0.05]),
                 ("r_foot", [0.05, 0.0, -0.05]))        # tools/time_task.py


def _cuda(a, dtype, ld=None, fill=float("nan")):
    """[rows, B] numpy -> CUDA tensor [rows, ld] (columns B.. filled with `fill`); returns (tensor, data pointer)."""
    import torch
    B = a.shape[1]
    t = torch.full((a.shape[0], ld or B), fill, dtype=dtype, device="cuda")
    t[:, :B] = torch.from_numpy(np.ascontiguousarray(a)).to(dtype)
    return t


def _abi_vjp(mech, tasks, q, v, vd, bars, dtype, ld=None):
    """rbd_task_kinematics_vjp on the GPU with leading dimension ld (NaN padding); returns {qt, qc, vb, vdb} as [rows, ld] tensors."""
    import torch
    desc = mech.flatten()
    h = _cabi.ModelHandle(desc)
    B = q.shape[1]
    ld = ld or B
    ins = {k: _cuda(a, dtype, ld) for k, a in (("q", q), ("v", v), ("vd", vd)) if a is not None}
    bt = {k: _cuda(b, dtype, ld) for k, b in bars.items()}
    to = _cabi.RbdTaskOut()
    for k, t in bt.items():
        setattr(to, k, t.data_ptr())
    out = {k: torch.full((desc.nq if k == "qc" else desc.nv, ld), float("nan"), dtype=dtype, device="cuda") for k in GRADS}
    d, keep = task_desc(mech, tasks)
    p = lambda k: ins[k].data_ptr() if k in ins else None      # noqa: E731
    _cabi.check(rbd.load_library().rbd_task_kinematics_vjp(h.ptr, _cabi.RBD_F64 if dtype == torch.float64 else _cabi.RBD_F32, B, ld,
                                                           p("q"), p("v"), p("vd"), ctypes.byref(d), ctypes.byref(to),
                                                           *[out[k].data_ptr() for k in GRADS], None))
    torch.cuda.synchronize()
    info = rbd.launch_info()
    h.close()
    return out, info


@pytest.mark.gpu
@pytest.mark.parametrize("name,arg", [("atlas", True), ("iiwa14", False), ("randmech", 18), ("randmech", 19)])
def test_gpu_matches_cpu_run(built, name, arg):
    import torch
    mech = _model(name, arg)
    q, v, _, vd, _ = rand_inputs(mech, 67, 5)
    tasks = task_set(mech, 5)
    bars = rand_bars(mech, len(tasks), 67, 6)
    ref = host_vjp(mech, tasks, q, v, vd, bars)
    got, info = _abi_vjp(mech, tasks, q, v, vd, bars, torch.float64)
    assert info.kernels_launched == 1
    for k in GRADS:
        assert rel_err(got[k].cpu().numpy(), ref[k]) < 1e-10, k
    got32, _ = _abi_vjp(mech, tasks, q, v, vd, bars, torch.float32)
    errs = {k: rel_err(got32[k].double().cpu().numpy(), ref[k]) for k in GRADS}
    print(f"fp32 vs fp64 CPU run, {name}: " + ", ".join(f"{k} {e:.2e}" for k, e in errs.items()))
    assert max(errs.values()) < TOL32, errs


@pytest.mark.gpu
def test_gpu_strides_ragged_batches_and_tiles(built):
    import torch
    mech = rbd.load_model("atlas", floating=True)
    q, v, _, vd, _ = rand_inputs(mech, 45, 8)
    tasks = task_set(mech, 8)
    bars = rand_bars(mech, len(tasks), 45, 9)
    dense, _ = _abi_vjp(mech, tasks, q, v, vd, bars, torch.float64)
    for B, ld in ((45, 53), (37, 37), (33, 40), (1, 7)):
        g, _ = _abi_vjp(mech, tasks, q[:, :B], v[:, :B], vd[:, :B], {k: b[:, :B] for k, b in bars.items()}, torch.float64, ld)
        for k in GRADS:
            assert torch.equal(g[k][:, :B], dense[k][:, :B]), (k, B, ld)
            assert torch.isnan(g[k][:, B:]).all(), (k, B, ld)
    # a batch of one repeated column spanning several persistent passes (the workspace cap trims the grid)
    B = 1 << 17
    rep = lambda a: np.repeat(a[:, :1], B, 1)          # noqa: E731
    big, info = _abi_vjp(mech, tasks, rep(q), rep(v), rep(vd), {k: rep(b) for k, b in bars.items()}, torch.float64)
    assert info.kernels_launched == 1 and info.grid * info.block < B
    for k in GRADS:
        assert torch.equal(big[k], big[k][:, :1].expand_as(big[k])), k
        assert torch.equal(big[k][:, :1], dense[k][:, :1]), k


@pytest.mark.gpu
def test_gpu_empty_task_set_writes_zeros(built):
    import torch
    mech = rbd.load_model("iiwa14")
    q, v, _, vd, _ = rand_inputs(mech, 5, 1)
    got, info = _abi_vjp(mech, [], q, v, vd, {}, torch.float64, ld=8)
    assert info.kernels_launched == 0
    for k in GRADS:
        assert (got[k][:, :5] == 0).all() and torch.isnan(got[k][:, 5:]).all(), k


@pytest.mark.gpu
def test_gpu_gradcheck_every_output(built):
    import torch
    rng = np.random.default_rng(4)
    # revolute / prismatic / planar joints: q̄_cfg is then the full gradient in q, which gradcheck compares against
    mech = rbd.rand_tree_mechanism(rng, [rbd.Revolute, rbd.Prismatic, rbd.Planar] * 2)
    q, v, _, vd, _ = rand_inputs(mech, 2, 4)
    bodies = [j.successor for j in mech.joints]
    tasks = (TaskFrame(bodies[-1], bodies[1], [0.1, -0.2, 0.3], bodies[2]), TaskFrame(bodies[3], None, [0.2, 0.0, 0.1], None))
    t = lambda a: torch.from_numpy(a).cuda().requires_grad_(True)      # noqa: E731
    qt, vt, vdt = t(q), t(v), t(vd)
    for out in OUTPUTS:
        f = lambda q_, v_, vd_: rbd.autodiff.task_kinematics(mech, q_, v_, vd_, tasks=tasks, outputs=(out,))[out]   # noqa: E731
        assert torch.autograd.gradcheck(f, (qt, vt, vdt), eps=1e-6, atol=1e-7, rtol=1e-5), out


@pytest.mark.gpu
@pytest.mark.parametrize("pd", [False, True])
def test_gpu_composition_with_simulate(built, pd):
    """autodiff.simulate -> autodiff.task_kinematics on the final state -> a hand position + point velocity loss: gradients to q0,
    v0 and the torques against central differences of the fp64 rollout plus forward task kinematics."""
    import torch
    mech = rbd.load_model("iiwa14")
    nv = mech.num_velocities()
    B, nsteps, dt = 3, 6, 2e-3
    q, v, tau, _, _ = rand_inputs(mech, B, 12)
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()     # noqa: E731
    hand = [TaskFrame(mech.joints[-1].successor, None, [0.0, 0.0, 0.1], None)]
    rng = np.random.default_rng(13)
    wp, wv = cuda(rng.standard_normal((3, B))), cuda(rng.standard_normal((3, B)))
    ctl = rbd.JointPD(cuda(np.full(nv, 20.0)), cuda(np.full(nv, 2.0)), cuda(q)) if pd else None

    def loss(q0, v0, tq):
        qf, vf = rbd.autodiff.simulate(mech, q0, v0, tq, dt=dt, nsteps=nsteps, trajectory=False, controller=ctl)
        o = rbd.autodiff.task_kinematics(mech, qf, vf, tasks=hand, outputs=("point", "point_velocity"))
        return (wp * o["point"]).sum() + (wv * o["point_velocity"]).sum()

    x = [cuda(q).requires_grad_(True), cuda(v).requires_grad_(True), cuda(tau).requires_grad_(True)]
    loss(*x).backward()
    grads = [t.grad for t in x]
    eps = 1e-6
    for trial in range(3):
        dirs = [cuda(rng.standard_normal(a.shape)) for a in (q, v, tau)]
        with torch.no_grad():
            base = [t.detach() for t in x]
            lp = loss(*[b + eps * d for b, d in zip(base, dirs)])
            lm = loss(*[b - eps * d for b, d in zip(base, dirs)])
        fd = float((lp - lm) / (2 * eps))
        an = float(sum((g * d).sum() for g, d in zip(grads, dirs)))
        assert abs(fd - an) <= 1e-6 * max(1.0, abs(fd)), (trial, fd, an)


@pytest.mark.gpu
def test_gpu_batched_ik_converges(built):
    import torch
    mech = rbd.load_model("iiwa14")
    B = 256
    rng = np.random.default_rng(21)
    q_star = np.stack([mech.rand_configuration(rng) for _ in range(B)], 1)
    task = [TaskFrame(mech.joints[-1].successor, None, [0.0, 0.0, 0.1], None)]
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()     # noqa: E731
    with torch.no_grad():
        target = rbd.autodiff.task_kinematics(mech, cuda(q_star), tasks=task)["point"]
    q = cuda(q_star + rng.uniform(-0.1, 0.1, q_star.shape))
    step = torch.zeros_like(q)
    lr, mu = 1.0, 0.95                    # gradient descent with Nesterov momentum on 0.5 |p(q) - target|^2
    for _ in range(6000):
        x = (q + mu * step).requires_grad_(True)
        e = rbd.autodiff.task_kinematics(mech, x, tasks=task)["point"] - target
        (g,) = torch.autograd.grad(0.5 * (e * e).sum(), x)
        step = mu * step - lr * g
        q = q + step
    with torch.no_grad():
        err = (rbd.autodiff.task_kinematics(mech, q, tasks=task)["point"] - target).norm(dim=0).max().item()
    assert err < 1e-4, err


@pytest.mark.gpu
def test_gpu_atlas_fp32_full_batch(built):
    import torch
    mech = rbd.load_model("atlas", floating=True)
    nv = mech.num_velocities()
    B = 1 << 20
    st = rbd.MechanismState(mech, B, torch.float32)
    rbd.rand_(st, np.random.default_rng(3))
    tasks = [TaskFrame(mech.findbody(n), None, p, None) for n, p in END_EFFECTORS]
    K = len(tasks)
    gen = torch.Generator(device="cuda").manual_seed(0)
    bars = {k: torch.randn((_rows(k, nv) * K, B), generator=gen, device="cuda") for k in OUTPUTS}
    vd = torch.rand((nv, B), generator=gen, device="cuda")
    outs = {k: torch.empty((st.nq if k == "q_bar_cfg" else nv, B), device="cuda") for k in ("q_bar_tan", "q_bar_cfg", "v_bar", "vd_bar")}
    rbd.autodiff.task_kinematics_vjp_(st, tasks, vd, bars=bars, **outs)
    torch.cuda.synchronize()
    assert rbd.launch_info().kernels_launched == 1
    for k, t in outs.items():
        assert torch.isfinite(t).all(), k
