"""Reverse mode of the whole-body kinematics (DESIGN 4.23): rbd_kinematics_vjp, autodiff.kinematics_vjp_ and autodiff.kinematics.

CPU tier (the device code compiled for the host: tests/hostsim/hostsim_kin_vjp.cpp)
1. kin_vjp_sample against central differences of the fp64 oracle's kinematics along the tangent directions of q and the unit
   directions of v: Atlas, Valkyrie, iiwa14, the double pendulum and every-joint-type trees; each output's cotangent alone and all
   eight together; geometric-Jacobian paths with an up segment, a down segment and the root as one end.
2. Exact identities against the forward code (kin_sample, mass_matrix, inverse dynamics on the CPU): momentum -> v̄ = Aᵀ h̄, kinetic
   energy -> v̄ = k̄ M v, centre of mass -> q̄_tan = (A_lin / m)ᵀ c̄, potential energy -> q̄_tan = ē g(q) (the gravity torque is ∂U/∂q),
   geometric Jacobian -> v̄ = 0.
3. q̄_cfg . (N(q) u) == q̄_tan . u, and no radial quaternion component.
4. Linearity over the outputs; cotangent rows of off-path Jacobian columns are not read.
5. The argument checks of rbd_kinematics_vjp, on the host.
GPU tier: the kernel against the CPU run of the same code, strides, ragged and multi-pass batches, the launch count, gradcheck,
composition with autodiff.simulate, and Atlas fp32 at 2^20.
"""
import ctypes
import functools

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from oracle import Oracle
from rigidbodydynamics.jl_b200 import _cabi
from rigidbodydynamics.jl_b200._cabi import RbdModelDesc, make_desc
from tests import hostsim
from tests.util import double_pendulum, rand_inputs, randmech, rel_err


TOL_FD = 2e-6         # central finite differences, eps = 1e-6 (test_vjp.py)
GRADS = ("qt", "qc", "vb")
OUTPUTS = ("transforms_to_root", "center_of_mass", "kinetic_energy", "gravitational_potential_energy", "momentum",
           "momentum_rate_bias", "momentum_matrix", "geometric_jacobian")       # rbd_kinematics_out order
ORACLE_KEY = dict(zip(OUTPUTS, ("transforms", "com", "ke", "pe", "momentum", "mrb", "A", "J")))
VEL_OUTPUTS = ("kinetic_energy", "momentum", "momentum_rate_bias")
K_QFLOAT, K_QSPH = 4, 6


def _rows(name, nb, nv):
    return {"transforms_to_root": 12 * nb, "center_of_mass": 3, "kinetic_energy": 1, "gravitational_potential_energy": 1,
            "momentum": 6, "momentum_rate_bias": 6, "momentum_matrix": 6 * nv, "geometric_jacobian": 6 * nv}[name]


@functools.cache
def _shim():
    """tests/hostsim/hostsim_kin_vjp.cpp, compiled and loaded by hostsim.shim."""
    lib = hostsim.shim("hostsim_kin_vjp")
    lib.hostsim_kinematics_vjp.argtypes = [ctypes.POINTER(RbdModelDesc), ctypes.c_void_p, ctypes.c_int, ctypes.c_int64,
                                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def host_vjp(mech, sign, q, v, bars):
    """kin_vjp_sample on the CPU for the cotangents ``bars`` ({output: [rows, B]}); returns {qt, qc, vb}."""
    desc = mech.flatten()
    dt = q.dtype
    d, keep = make_desc(desc)
    c = lambda a: None if a is None else np.ascontiguousarray(a, dt)     # noqa: E731
    q, v = c(q), c(v)
    bars = {k: c(b) for k, b in bars.items()}
    sg = None if sign is None else np.ascontiguousarray(sign, np.int8)
    B = q.shape[1]
    out = {k: np.full((desc.nq if k == "qc" else desc.nv, B), np.nan, dt) for k in GRADS}
    p = lambda a: None if a is None or a.size == 0 else a.ctypes.data      # noqa: E731
    bp = (ctypes.c_void_p * 8)(*[p(bars.get(k)) for k in OUTPUTS])
    op = (ctypes.c_void_p * 3)(*[p(out[k]) for k in GRADS])
    rc = _shim().hostsim_kinematics_vjp(ctypes.byref(d), None if sg is None else sg.ctypes.data, 0 if dt == np.float32 else 1, B,
                                        p(q), p(v), bp, op)
    assert rc == 0, rc
    return out


def rand_bars(mech, B, seed, want=OUTPUTS):
    rng = np.random.default_rng(seed)
    nb, nv = len(mech.joints), mech.num_velocities()
    return {k: rng.standard_normal((_rows(k, nb, nv), B)) for k in want}


def paths(mech, seed):
    """Geometric-Jacobian paths: between two bodies of different branches (an up and a down segment), from the root down to a
    body, and from a body up to the root."""
    rng = np.random.default_rng(seed)
    bodies = [j.successor for j in mech.joints]
    index = {id(b): i for i, b in enumerate(bodies)}

    def chain(b):
        out = []
        while b is not mech.root_body:
            out.append(index[id(b)])
            b = mech.joints[index[id(b)]].predecessor
        return out
    best = None
    for _ in range(64):
        a, b = (bodies[int(i)] for i in rng.integers(0, len(bodies), 2))
        s = rbd.path(mech, a, b).sign
        if (s < 0).any() and (s > 0).any():
            best = s
            break
    out = [] if best is None else [best]
    deep = max(bodies, key=lambda b: len(chain(b)))
    out.append(rbd.path(mech, mech.root_body, deep).sign)
    out.append(rbd.path(mech, bodies[int(rng.integers(len(bodies)))], mech.root_body).sign)
    return out


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


def fd_jacobians(mech, sign, q, v, eps=1e-6):
    """Central differences of every oracle output along the tangent directions of q and the unit directions of v:
    {var: {output: [n_dirs, rows, B]}}."""
    o = Oracle(mech.flatten())
    nv, B = mech.num_velocities(), q.shape[1]
    f = lambda q_, v_: {k: o.kinematics(q_, v_, sign)[ORACLE_KEY[k]] for k in OUTPUTS}     # noqa: E731
    eye = [np.repeat(np.eye(nv)[:, k:k + 1], B, 1) for k in range(nv)]
    out = {}
    for var, dirs in (("q", qdot_dirs(mech, q)), ("v", eye)):
        per = []
        for dk in dirs:
            if var == "q":
                yp, ym = f(q + eps * dk, v), f(q - eps * dk, v)
            else:
                yp, ym = f(q, v + eps * dk), f(q, v - eps * dk)
            per.append({k: (yp[k] - ym[k]) / (2 * eps) for k in OUTPUTS})
        out[var] = {k: np.stack([p[k] for p in per]) for k in OUTPUTS}
    return out


def fd_vjp(J, bars):
    """Σ_outputs ȳ . ∂y/∂x from the finite-difference Jacobians: {qt, vb}."""
    return {key: sum(np.einsum("kib,ib->kb", J[var][k], b) for k, b in bars.items()) for var, key in (("q", "qt"), ("v", "vb"))}


# ------------------------------------------------------------------------------------------------------------------
# CPU tier 1: central differences of the oracle
# ------------------------------------------------------------------------------------------------------------------
FD_MODELS = [("atlas", True), ("valkyrie", False), ("iiwa14", False), ("double_pendulum", None), ("randmech", 17),
             ("randmech", 18)]


def _model(name, arg):
    if name == "randmech":
        return randmech(arg, shuffle=arg % 2 == 1)
    if name == "double_pendulum":
        return double_pendulum()
    return rbd.load_model(name, floating=arg)


@pytest.mark.parametrize("name,arg", FD_MODELS, ids=[f"{n}-{a}" for n, a in FD_MODELS])
def test_vjp_matches_central_differences(name, arg):
    mech = _model(name, arg)
    seed = 3 if name != "randmech" else arg
    q, v, _, _, _ = rand_inputs(mech, 2, seed)
    allbars = rand_bars(mech, 2, seed + 100)
    for pi, sign in enumerate(paths(mech, seed)):
        J = fd_jacobians(mech, sign, q, v)
        wants = [(k,) for k in OUTPUTS] + [OUTPUTS] if pi == 0 else [("geometric_jacobian",)]
        for want in wants:
            bars = {k: allbars[k] for k in want}
            got = host_vjp(mech, sign if "geometric_jacobian" in want else None, q, v if set(want) & set(VEL_OUTPUTS) else None, bars)
            ref = fd_vjp(J, bars)
            for key in ("qt", "vb"):
                assert rel_err(got[key], ref[key]) < TOL_FD, (pi, want, key, rel_err(got[key], ref[key]))


# ------------------------------------------------------------------------------------------------------------------
# CPU tier 2: exact identities against the forward code
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,arg", [("atlas", True), ("randmech", 19), ("randmech", 20)])
def test_vjp_identities_with_forward_code(name, arg):
    mech = _model(name, arg)
    desc = mech.flatten()
    nv, B = desc.nv, 3
    q, v, _, _, _ = rand_inputs(mech, B, 7)
    bars = rand_bars(mech, B, 8)
    fw = hostsim.kinematics(desc, q, v, None, want=("A",))
    A = fw["A"].reshape(nv, 6, B)                                        # column k of the momentum matrix
    mass = sum(b.inertia.mass for b in mech.bodies if b.inertia is not None)
    h = bars["momentum"]
    got = host_vjp(mech, None, q, v, {"momentum": h})
    assert rel_err(got["vb"], np.einsum("kcb,cb->kb", A, h)) < 1e-12        # v̄ = Aᵀ h̄
    Mm = hostsim.mass_matrix(desc, q).reshape(nv, nv, B)                  # entry (i, j) at row i + j nv
    kb = bars["kinetic_energy"]
    got = host_vjp(mech, None, q, v, {"kinetic_energy": kb})
    assert rel_err(got["vb"], kb * np.einsum("jib,jb->ib", Mm, v)) < 1e-12  # v̄ = k̄ M v
    cb = bars["center_of_mass"]
    got = host_vjp(mech, None, q, None, {"center_of_mass": cb})
    assert rel_err(got["qt"], np.einsum("kcb,cb->kb", A[:, 3:], cb) / mass) < 1e-12   # ċom = A_lin v / m
    eb = bars["gravitational_potential_energy"]
    g = hostsim.inverse_dynamics(desc, q, np.zeros((nv, B)))             # gravity torque = ∂U/∂q
    got = host_vjp(mech, None, q, None, {"gravitational_potential_energy": eb})
    assert rel_err(got["qt"], eb * g) < 1e-12
    sign = paths(mech, 7)[0]
    got = host_vjp(mech, sign, q, v, {"geometric_jacobian": bars["geometric_jacobian"]})
    assert (got["vb"] == 0).all()


# ------------------------------------------------------------------------------------------------------------------
# CPU tier 3 and 4: configuration covector, linearity, off-path rows
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [21, 22])
def test_q_bar_cfg_and_linearity(seed):
    mech = randmech(seed, shuffle=True)
    desc = mech.flatten()
    nv, B = desc.nv, 3
    q, v, _, _, _ = rand_inputs(mech, B, seed)
    sign = paths(mech, seed)[0]
    bars = rand_bars(mech, B, seed + 1)
    full = host_vjp(mech, sign, q, v, bars)
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
    parts = [host_vjp(mech, sign if k == "geometric_jacobian" else None, q, v, {k: bars[k]}) for k in OUTPUTS]
    for key in GRADS:
        assert rel_err(sum(p[key] for p in parts), full[key]) < 1e-12, key
    # off-path Jacobian columns: their cotangent rows are not read (NaN there changes nothing)
    J = hostsim.kinematics(desc, q, None, sign, want=("J",))["J"].reshape(nv, 6, B)
    off = np.abs(J).sum((1, 2)) == 0
    assert off.any()
    nb_ = dict(bars)
    nb_["geometric_jacobian"] = bars["geometric_jacobian"].reshape(nv, 6, B).copy()
    nb_["geometric_jacobian"][off] = np.nan
    nb_["geometric_jacobian"] = nb_["geometric_jacobian"].reshape(-1, B)
    masked = host_vjp(mech, sign, q, v, nb_)
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
    buf = np.zeros(64)
    q = buf.ctypes.data_as(ctypes.c_void_p)
    sign = np.ones(nb, np.int8)

    def bar(**kw):
        o = _cabi.RbdKinematicsOut()
        for k in kw:
            setattr(o, k, buf.ctypes.data)
        return ctypes.byref(o)

    def call(model=h.ptr, dtype=_cabi.RBD_F64, B=1, ld=1, q=q, v=None, sign=None, out=None):
        out = bar(center_of_mass=1) if out is None else out
        return lib.rbd_kinematics_vjp(model, dtype, B, ld, q, v, sign, out, None, None, None, None)

    assert call(model=None) == _cabi.RBD_EINVAL
    assert call(dtype=_cabi.RBD_DUAL64X6) == _cabi.RBD_EUNSUPPORTED
    assert call(dtype=7) == _cabi.RBD_EINVAL                       # as rbd_kinematics: not a dtype at all
    assert call(B=4, ld=3) == _cabi.RBD_EDIM
    assert call(B=-1, ld=0) == _cabi.RBD_EDIM
    assert lib.rbd_kinematics_vjp(h.ptr, _cabi.RBD_F64, 1, 1, q, None, None, None, None, None, None, None) == _cabi.RBD_EINVAL
    assert call(q=None) == _cabi.RBD_EINVAL
    for name in VEL_OUTPUTS:                                       # v NULL with a velocity-dependent cotangent
        assert call(out=bar(**{name: 1})) == _cabi.RBD_EINVAL, name
    sp = sign.ctypes.data_as(ctypes.c_void_p)
    assert call(out=bar(geometric_jacobian=1)) == _cabi.RBD_EINVAL           # Jacobian cotangent without a path
    assert call(sign=sp) == _cabi.RBD_EINVAL                                 # a path without a Jacobian cotangent
    bad = sign.copy(); bad[2] = 2
    assert call(out=bar(geometric_jacobian=1), sign=bad.ctypes.data_as(ctypes.c_void_p)) == _cabi.RBD_EINVAL
    h.close()
    massless = rbd.rand_tree_mechanism(np.random.default_rng(0), [rbd.Revolute] * 2)
    for b in massless.bodies:
        if b.inertia is not None:
            b.inertia = rbd.SpatialInertia(np.zeros((3, 3)), None, 0.0)
    h0 = _cabi.ModelHandle(massless.flatten())
    assert lib.rbd_kinematics_vjp(h0.ptr, _cabi.RBD_F64, 1, 1, q, None, None, bar(center_of_mass=1), None, None, None, None) \
        == _cabi.RBD_EINVAL
    assert lib.rbd_kinematics_vjp(h0.ptr, _cabi.RBD_F64, 0, 0, None, None, None, bar(center_of_mass=1), None, None, None, None) \
        == _cabi.RBD_OK                                            # empty batch: nothing read or written, no device touched
    h0.close()


def test_autodiff_kinematics_argument_checks(built):
    import torch
    mech = rbd.load_model("iiwa14")
    q = torch.zeros((mech.num_positions(), 2), dtype=torch.float64)
    with pytest.raises(TypeError, match="unknown kinematics output"):
        rbd.autodiff.kinematics(mech, q, outputs=("com",))
    with pytest.raises(ValueError, match="distinct"):
        rbd.autodiff.kinematics(mech, q, outputs=("momentum", "momentum"))
    with pytest.raises(ValueError, match="geometric_jacobian needs a path"):
        rbd.autodiff.kinematics(mech, q, outputs=("geometric_jacobian",))
    with pytest.raises(rbd.DimensionMismatch, match="path does not belong"):
        other = double_pendulum()
        rbd.autodiff.kinematics(mech, q, outputs=("geometric_jacobian",), path=rbd.path(other, other.root_body, other.bodies[-1]))
    with pytest.raises(TypeError, match="CUDA tensor"):
        rbd.autodiff.kinematics(mech, q)                               # a CPU tensor: the checks of the other autodiff functions


# ------------------------------------------------------------------------------------------------------------------
# GPU tier
# ------------------------------------------------------------------------------------------------------------------
# fp32 kernel against the fp64 CPU run, rel_err over the three gradients: worst measured on an H100 80GB HBM3 1.48e-6 (iiwa14, q̄_tan of
# a momentum-matrix cotangent; Atlas 6.6e-7, DESIGN 4.23); the bound is about 5x that
TOL32 = 8e-6


def _cuda(a, dtype, ld=None, fill=float("nan")):
    """[rows, B] numpy -> CUDA tensor [rows, ld] (columns B.. filled with `fill`)."""
    import torch
    B = a.shape[1]
    t = torch.full((a.shape[0], ld or B), fill, dtype=dtype, device="cuda")
    t[:, :B] = torch.from_numpy(np.ascontiguousarray(a)).to(dtype)
    return t


def _abi_vjp(mech, sign, q, v, bars, dtype, ld=None):
    """rbd_kinematics_vjp on the GPU with leading dimension ld (NaN padding); returns ({qt, qc, vb} as [rows, ld] tensors, launch
    info)."""
    import torch
    desc = mech.flatten()
    h = _cabi.ModelHandle(desc)
    B = q.shape[1]
    ld = ld or B
    ins = {k: _cuda(a, dtype, ld) for k, a in (("q", q), ("v", v)) if a is not None}
    bt = {k: _cuda(b, dtype, ld) for k, b in bars.items()}
    ko = _cabi.RbdKinematicsOut()
    for k, t in bt.items():
        setattr(ko, k, t.data_ptr())
    out = {k: torch.full((desc.nq if k == "qc" else desc.nv, ld), float("nan"), dtype=dtype, device="cuda") for k in GRADS}
    sg = None if sign is None else np.ascontiguousarray(sign, np.int8)
    p = lambda k: ins[k].data_ptr() if k in ins else None      # noqa: E731
    _cabi.check(rbd.load_library().rbd_kinematics_vjp(h.ptr, _cabi.RBD_F64 if dtype == torch.float64 else _cabi.RBD_F32, B, ld,
                                                      p("q"), p("v"), None if sg is None else sg.ctypes.data_as(ctypes.c_void_p),
                                                      ctypes.byref(ko), *[out[k].data_ptr() for k in GRADS], None))
    torch.cuda.synchronize()
    info = rbd.launch_info()
    h.close()
    return out, info


GPU_MODELS = [("atlas", True), ("valkyrie", True), ("iiwa14", False), ("randmech", 18), ("randmech", 19)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,arg", GPU_MODELS, ids=[f"{n}-{a}" for n, a in GPU_MODELS])
def test_gpu_matches_cpu_run(built, name, arg):
    import torch
    mech = _model(name, arg)
    q, v, _, _, _ = rand_inputs(mech, 67, 5)
    sign = paths(mech, 5)[0]
    for want in (("center_of_mass", "momentum"), ("momentum_matrix",), OUTPUTS):
        bars = rand_bars(mech, 67, 6, want)
        sg = sign if "geometric_jacobian" in want else None
        ref = host_vjp(mech, sg, q, v, bars)
        got, info = _abi_vjp(mech, sg, q, v, bars, torch.float64)
        assert info.kernels_launched == 1
        for k in GRADS:
            assert rel_err(got[k].cpu().numpy(), ref[k]) < 1e-10, (want, k)
        got32, _ = _abi_vjp(mech, sg, q, v, bars, torch.float32)
        errs = {k: rel_err(got32[k].double().cpu().numpy(), ref[k]) for k in GRADS}
        print(f"fp32 vs fp64 CPU run, {name}, {'+'.join(want) if len(want) < 8 else 'all eight'}: "
              + ", ".join(f"{k} {e:.2e}" for k, e in errs.items()))
        assert max(errs.values()) < TOL32, (want, errs)


@pytest.mark.gpu
def test_gpu_strides_ragged_and_multipass_batches(built):
    import torch
    mech = rbd.load_model("atlas", floating=True)
    q, v, _, _, _ = rand_inputs(mech, 45, 8)
    sign = paths(mech, 8)[0]
    bars = rand_bars(mech, 45, 9)
    dense, _ = _abi_vjp(mech, sign, q, v, bars, torch.float64)
    for B, ld in ((45, 53), (37, 37), (33, 40), (1, 7)):
        g, _ = _abi_vjp(mech, sign, q[:, :B], v[:, :B], {k: b[:, :B] for k, b in bars.items()}, torch.float64, ld)
        for k in GRADS:
            assert torch.equal(g[k][:, :B], dense[k][:, :B]), (k, B, ld)
            assert torch.isnan(g[k][:, B:]).all(), (k, B, ld)
    # 2^17 samples: several persistent passes (the workspace cap trims the grid); every column a distinct sample
    B = 1 << 17
    qb, vb, _, _, _ = rand_inputs(mech, 64, 10)
    tile = lambda a: np.tile(a, (1, B // a.shape[1]))          # noqa: E731
    qb[:, :45], vb[:, :45] = q, v
    big_bars = {k: tile(np.concatenate([b, rand_bars(mech, 19, 11)[k]], 1)) for k, b in bars.items()}
    big, info = _abi_vjp(mech, sign, tile(qb), tile(vb), big_bars, torch.float64)
    assert info.kernels_launched == 1 and info.grid * info.block < B
    for k in GRADS:
        per = big[k].reshape(big[k].shape[0], B // 64, 64)
        assert torch.equal(per, per[:, :1].expand_as(per)), k
        assert torch.equal(big[k][:, :45], dense[k]), k


@pytest.mark.gpu
def test_gpu_launch_counts(built):
    import torch
    mech = rbd.load_model("iiwa14")
    q, v, _, _, _ = rand_inputs(mech, 5, 1)
    got, info = _abi_vjp(mech, None, q, v, {}, torch.float64, ld=8)
    assert info.kernels_launched == 0
    for k in GRADS:
        assert (got[k][:, :5] == 0).all() and torch.isnan(got[k][:, 5:]).all(), k
    _, info = _abi_vjp(mech, None, q, None, rand_bars(mech, 5, 2, ("center_of_mass",)), torch.float64)
    assert info.kernels_launched == 1


@pytest.mark.gpu
def test_gpu_gradcheck_every_output(built):
    import torch
    rng = np.random.default_rng(4)
    # revolute / prismatic / planar joints: q̄_cfg is then the full gradient in q, which gradcheck compares against
    mech = rbd.rand_tree_mechanism(rng, [rbd.Revolute, rbd.Prismatic, rbd.Planar] * 2)
    q, v, _, _, _ = rand_inputs(mech, 2, 4)
    path = rbd.path(mech, mech.joints[-1].successor, mech.joints[2].successor)
    t = lambda a: torch.from_numpy(a).cuda().requires_grad_(True)      # noqa: E731
    qt, vt = t(q), t(v)
    for out in OUTPUTS:
        f = lambda q_, v_: rbd.autodiff.kinematics(mech, q_, v_, outputs=(out,), path=path)[out]   # noqa: E731
        assert torch.autograd.gradcheck(f, (qt, vt), eps=1e-6, atol=1e-7, rtol=1e-5), out


@pytest.mark.gpu
@pytest.mark.parametrize("pd", [False, True])
def test_gpu_composition_with_simulate(built, pd):
    """autodiff.simulate -> autodiff.kinematics on the final state -> a centre-of-mass plus angular-momentum loss on Atlas: gradients
    to q0, v0 and the torques against central differences of the fp64 rollout plus forward kinematics."""
    import torch
    mech = rbd.load_model("atlas", floating=True)
    nv = mech.num_velocities()
    B, nsteps, dt = 2, 5, 1e-3
    q, v, tau, _, _ = rand_inputs(mech, B, 12)
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()     # noqa: E731
    rng = np.random.default_rng(13)
    wc, wh = cuda(rng.standard_normal((3, B))), cuda(rng.standard_normal((3, B)))
    ctl = rbd.JointPD(cuda(np.full(nv, 20.0)), cuda(np.full(nv, 2.0)), cuda(q)) if pd else None

    def loss(q0, v0, tq):
        qf, vf = rbd.autodiff.simulate(mech, q0, v0, tq, dt=dt, nsteps=nsteps, trajectory=False, controller=ctl)
        o = rbd.autodiff.kinematics(mech, qf, vf, outputs=("center_of_mass", "momentum"))
        return (wc * o["center_of_mass"]).sum() + (wh * o["momentum"][:3]).sum()

    x = [cuda(q).requires_grad_(True), cuda(v).requires_grad_(True), cuda(tau).requires_grad_(True)]
    loss(*x).backward()
    grads = [t.grad for t in x]
    eps = 1e-6
    for trial in range(3):
        dirs = [cuda(rng.standard_normal(a.shape)) for a in (q, v, tau)]
        dirs[0] = cuda(np.einsum("kqb,kb->qb", qdot_dirs(mech, q), rng.standard_normal((nv, B))))   # tangent to the quaternions
        with torch.no_grad():
            base = [t.detach() for t in x]
            lp = loss(*[b + eps * d for b, d in zip(base, dirs)])
            lm = loss(*[b - eps * d for b, d in zip(base, dirs)])
        fd = float((lp - lm) / (2 * eps))
        an = float(sum((g * d).sum() for g, d in zip(grads, dirs)))
        assert abs(fd - an) <= 1e-6 * max(1.0, abs(fd)), (trial, fd, an)


@pytest.mark.gpu
def test_gpu_atlas_fp32_full_batch(built):
    import torch
    mech = rbd.load_model("atlas", floating=True)
    nb, nv = len(mech.joints), mech.num_velocities()
    B = 1 << 20
    st = rbd.MechanismState(mech, B, torch.float32)
    rbd.rand_(st, np.random.default_rng(3))
    path = rbd.path(mech, mech.findbody("l_hand"), mech.findbody("r_foot"))
    gen = torch.Generator(device="cuda").manual_seed(0)
    bars = {k: torch.randn((_rows(k, nb, nv), B), generator=gen, device="cuda") for k in OUTPUTS}
    outs = {k: torch.empty((st.nq if k == "q_bar_cfg" else nv, B), device="cuda") for k in ("q_bar_tan", "q_bar_cfg", "v_bar")}
    rbd.autodiff.kinematics_vjp_(st, path, bars=bars, **outs)
    torch.cuda.synchronize()
    assert rbd.launch_info().kernels_launched == 1
    for k, t in outs.items():
        assert torch.isfinite(t).all(), k
