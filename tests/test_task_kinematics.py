"""Task-space kinematics (DESIGN 4.17): rbd_task_kinematics / task_kinematics_ and its conveniences.

CPU tier
1. Closed form on the double pendulum: the position, point Jacobian, velocity and acceleration of a point on link 2.
2. The reference's own identities, restated for the oracle (tests/task_oracle.py) on random mechanisms with every joint type:
     Twist(J, v) == relative_twist in the root, a body and the target frame     test/test_mechanism_algorithms.jl:310-344
     point_jacobian * v == point_velocity(twist, point)                        :346-392
     relative_twist(body, parent) == S_joint v_joint                           :492-504
     relative_acceleration == d/dt of the root-frame relative twist            :459-481 (central differences here)
     transform(-Ṫ_base + Ṫ_body) == Ṫ                                         :485-487
     point_velocity / point_acceleration == derivatives of the point's base-frame coordinates   test/test_spatial.jl:221-229
3. The device code (task_sample, compiled for the host: tests/hostsim/hostsim_task.cpp) against that oracle, and each output alone
   bit-identical to the all-outputs call.
4. The argument checks of rbd_task_kinematics, on the host.
GPU tier: the kernel against the oracle, bit identity across output subsets, strides, alignment and tiles, the Python conveniences.
"""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from rigidbodydynamics.jl_b200 import _cabi
from rigidbodydynamics.jl_b200._cabi import RbdModelDesc, RbdTaskDesc, make_desc
from rigidbodydynamics.jl_b200.kinematics import TaskFrame, task_desc
from tests.task_oracle import OUTPUTS, TaskOracle, cross
from tests.util import double_pendulum, rand_inputs, randmech

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "..", "rigidbodydynamics", "jl_b200", "csrc")
_lib = None

TOL = {np.float64: 1e-11, np.float32: 2e-5}        # relative to max(1, |ref|), the scales of test_kinematics.py
MODELS = [("atlas", True), ("valkyrie", False), ("iiwa14", False), ("double_pendulum", False)]
VEL_OUTPUTS = ("twist", "point_velocity", "acceleration", "point_acceleration")


def _shim():
    """tests/hostsim/hostsim_task.cpp, compiled on first use into a temporary directory."""
    global _lib
    if _lib is not None:
        return _lib
    srcs = [os.path.join(_HERE, "hostsim", "hostsim_task.cpp")] + sorted(
        os.path.join(_CSRC, f) for f in os.listdir(_CSRC) if f.endswith((".cuh", ".h")) or f == "rbd_model.cpp")
    srcs.append(os.path.join(_HERE, "..", "include", "rbd_b200.h"))
    h = hashlib.sha1(b"".join(open(s, "rb").read() for s in srcs)).hexdigest()[:16]
    d = os.path.join(tempfile.gettempdir(), f"rbd_hostsim_task_{os.getuid()}")
    os.makedirs(d, exist_ok=True)
    so = os.path.join(d, f"hostsim_task_{h}.so")
    if not os.path.exists(so):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so + f".{os.getpid()}",
                               srcs[0], os.path.join(_CSRC, "rbd_model.cpp")])
        os.replace(so + f".{os.getpid()}", so)
    lib = ctypes.CDLL(so)
    lib.hostsim_task_kinematics.argtypes = [ctypes.POINTER(RbdModelDesc), ctypes.POINTER(RbdTaskDesc), ctypes.c_int, ctypes.c_int64,
                                            ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    _lib = lib
    return lib


def _rows(name, nv):
    return {"transform": 12, "point": 3, "twist": 6, "point_velocity": 3, "geometric_jacobian": 6 * nv, "point_jacobian": 3 * nv,
            "acceleration": 6, "point_acceleration": 3}[name]


def hostsim_tasks(mech, tasks, q, v=None, vd=None, want=OUTPUTS):
    """task_sample on the CPU; returns {output: [rows * K, B]}."""
    desc = mech.flatten()
    dt = q.dtype
    d, keep = make_desc(desc)
    td, keep2 = task_desc(mech, tasks)
    q = np.ascontiguousarray(q)
    v = None if v is None else np.ascontiguousarray(v, dt)
    vd = None if vd is None else np.ascontiguousarray(vd, dt)
    B, K = q.shape[1], len(tasks)
    out = {k: np.full((_rows(k, desc.nv) * K, B), np.nan, dt) for k in want}
    ptrs = (ctypes.c_void_p * 8)(*[out[k].ctypes.data if k in out else None for k in OUTPUTS])
    p = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)     # noqa: E731
    rc = _shim().hostsim_task_kinematics(ctypes.byref(d), ctypes.byref(td), 0 if dt == np.float32 else 1, B, p(q), p(v), p(vd), ptrs)
    assert rc == 0, rc
    return out


def task_set(mech, seed):
    """Tasks covering body == base, base = root, body = root, frame in {root, body, base, an unrelated third body}, points at the
    origin and off it."""
    rng = np.random.default_rng(seed)
    bodies = [j.successor for j in mech.joints]
    root = mech.root_body
    pick = lambda: bodies[int(rng.integers(len(bodies)))]          # noqa: E731
    pt = lambda: rng.standard_normal(3)                             # noqa: E731
    b1, b2 = pick(), pick()
    others = [b for b in bodies if b is not b1 and b is not b2]
    b3 = others[int(rng.integers(len(others)))] if others else root
    return [TaskFrame(b1, None, pt(), None),          # base = root, root frame
            TaskFrame(b1, b2, pt(), b1),              # frame = body
            TaskFrame(b2, b1, None, b1),              # frame = base, point at the origin
            TaskFrame(b1, b2, pt(), b3),              # an unrelated third body
            TaskFrame(b2, b2, pt(), b3),              # body == base
            TaskFrame(root, b1, pt(), b2),            # body = root
            TaskFrame(b2, root, None, b2)]            # base = root, the target's own frame


def _err(got, ref):
    return np.abs(np.asarray(got, np.float64) - ref).max() / max(1.0, np.abs(ref).max())


# ------------------------------------------------------------------------------------------------------------------
# CPU tier 1: closed form
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("source", ["oracle", "device_code"])
def test_double_pendulum_point_closed_form(source):
    l1, l = -1.0, 0.7
    mech = double_pendulum(l1=l1)
    q = np.array([[0.3, -1.1], [0.4, 2.0]]); v = np.array([[1.0, -0.5], [2.0, 0.3]]); vd = np.array([[0.5, 1.5], [-0.7, 0.2]])
    task = [TaskFrame(mech.joints[1].successor, None, [0.0, 0.0, l], None)]
    if source == "oracle":
        o = TaskOracle(mech, q, v, vd).tasks(task)
    else:
        o = hostsim_tasks(mech, task, q, v, vd)
    q1, q12 = q[0], q[0] + q[1]
    w1, w12 = v[0], v[0] + v[1]
    a1, a12 = vd[0], vd[0] + vd[1]
    x = l1 * np.sin(q1) + l * np.sin(q12)
    z = l1 * np.cos(q1) + l * np.cos(q12)
    J = np.zeros((3, 2, 2))
    J[0, 0], J[0, 1] = l1 * np.cos(q1) + l * np.cos(q12), l * np.cos(q12)
    J[2, 0], J[2, 1] = -l1 * np.sin(q1) - l * np.sin(q12), -l * np.sin(q12)
    xdd = -l1 * np.sin(q1) * w1 ** 2 - l * np.sin(q12) * w12 ** 2 + l1 * np.cos(q1) * a1 + l * np.cos(q12) * a12
    zdd = -l1 * np.cos(q1) * w1 ** 2 - l * np.cos(q12) * w12 ** 2 - l1 * np.sin(q1) * a1 - l * np.sin(q12) * a12
    assert np.abs(o["point"] - np.stack([x, 0 * x, z])).max() < 1e-12
    assert np.abs(o["point_jacobian"].reshape(2, 3, 2).transpose(1, 0, 2) - J).max() < 1e-12
    assert np.abs(o["point_velocity"] - np.einsum("ikb,kb->ib", J, v)).max() < 1e-12
    assert np.abs(o["point_acceleration"] - np.stack([xdd, 0 * x, zdd])).max() < 1e-12


# ------------------------------------------------------------------------------------------------------------------
# CPU tier 2: the reference's identities, for the oracle
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [31, 32])
def test_oracle_jacobian_and_twist_identities(seed):
    mech = randmech(seed, shuffle=seed % 2 == 0)
    desc = mech.flatten()
    q, v, _, vd, _ = rand_inputs(mech, 3, seed)
    orc = TaskOracle(mech, q, v, vd)
    rng = np.random.default_rng(seed)
    bodies = [j.successor for j in mech.joints]
    for _ in range(8):
        body, base, other = (bodies[int(i)] for i in rng.integers(len(bodies), size=3))
        pt = rng.standard_normal(3)
        for frame in (None, other, body):                     # root frame, a body frame, the target's frame
            o = orc.task(TaskFrame(body, base, pt, frame))
            Jv = np.einsum("kcb,kb->cb", o["geometric_jacobian"].reshape(desc.nv, 6, -1), v)       # Twist(J, v)
            assert _err(Jv, o["twist"]) < 1e-12
            Jpv = np.einsum("kcb,kb->cb", o["point_jacobian"].reshape(desc.nv, 3, -1), v)
            assert _err(Jpv, o["point_velocity"]) < 1e-12
            assert _err(cross(o["twist"][:3], o["point"]) + o["twist"][3:], o["point_velocity"]) < 1e-12
    # relative_twist(body, parent) == S v_joint, in the body frame (the frame after the joint)
    vs = 0
    for i, j in enumerate(mech.joints):
        tw = orc.task(TaskFrame(j.successor, j.predecessor, None, j.successor))["twist"]
        vj = v[vs:vs + j.nv]
        jt = desc.jtype[i]
        if jt == _cabi_jtype("REVOLUTE"):
            S = np.concatenate([desc.jparam[i, :3], np.zeros(3)])[:, None] * vj
        elif jt == _cabi_jtype("PRISMATIC"):
            S = np.concatenate([np.zeros(3), desc.jparam[i, :3]])[:, None] * vj
        elif jt == _cabi_jtype("QUATERNION_FLOATING"):
            S = vj
        elif jt == _cabi_jtype("FIXED"):
            S = np.zeros((6, v.shape[1]))
        else:
            vs += j.nv
            continue
        assert _err(tw, S) < 1e-12, (i, jt)
        vs += j.nv


def _cabi_jtype(name):
    return {"REVOLUTE": 0, "PRISMATIC": 1, "FIXED": 2, "QUATERNION_FLOATING": 4}[name]


@pytest.mark.parametrize("seed", [29, 30])
def test_oracle_relative_acceleration_identities(seed):
    """relative_acceleration is the time derivative of the root-frame relative twist along (q + ε q̇, v + ε v̇), and the body and
    base accelerations w.r.t. the root, each transformed to the body's frame, difference back to it."""
    mech = randmech(seed)
    q, v, _, vd, _ = rand_inputs(mech, 2, seed)
    orc = TaskOracle(mech, q, v, vd)
    qd = orc.orc.dynamics(q, v, want_qd=True)[1]
    eps = 1e-6
    op, om = TaskOracle(mech, q + eps * qd, v + eps * vd), TaskOracle(mech, q - eps * qd, v - eps * vd)
    rng = np.random.default_rng(seed)
    bodies = [j.successor for j in mech.joints] + [mech.root_body]
    for _ in range(10):
        body, base = (bodies[int(i)] for i in rng.integers(len(bodies), size=2))
        t = TaskFrame(body, base)
        acc = orc.task(t)["acceleration"]
        fd = (op.task(t)["twist"] - om.task(t)["twist"]) / (2 * eps)
        assert _err(fd, acc) < 1e-6
        b, a = orc.idx(body), orc.idx(base)
        root = -1
        Tb = orc.accel_in(orc.acc[b] - orc.acc[root], b, b, root)
        Ta = orc.accel_in(orc.acc[a] - orc.acc[root], b, a, root)
        assert _err(orc.accel_to_root(Tb - Ta, b, b, a), acc) < 1e-12


def test_oracle_point_derivatives_in_the_base_frame():
    """frame = base: point_velocity and point_acceleration are the first and second time derivatives of the point's base-frame
    coordinates (test_spatial.jl:221-229).  Revolute and prismatic joints, so that q(t) = q + t v + t²/2 v̇ exactly."""
    rng = np.random.default_rng(41)
    mech = rbd.rand_tree_mechanism(rng, [rbd.Revolute] * 8 + [rbd.Prismatic] * 4)
    q, v, _, vd, _ = rand_inputs(mech, 2, 41)
    bodies = [j.successor for j in mech.joints]
    h = 1e-4
    for _ in range(6):
        body, base = (bodies[int(i)] for i in rng.integers(len(bodies), size=2))
        t = TaskFrame(body, base, rng.standard_normal(3), base)
        x = [TaskOracle(mech, q + s * v + 0.5 * s * s * vd).task(t)["point"] for s in (-h, 0.0, h)]
        o = TaskOracle(mech, q, v, vd).task(t)
        assert _err((x[2] - x[0]) / (2 * h), o["point_velocity"]) < 1e-7
        assert _err((x[2] - 2 * x[1] + x[0]) / h ** 2, o["point_acceleration"]) < 1e-5


# ------------------------------------------------------------------------------------------------------------------
# CPU tier 3: device code against the oracle
# ------------------------------------------------------------------------------------------------------------------
def _compare_hostsim(mech, seed, dt, with_vd=True):
    q, v, _, vd, _ = rand_inputs(mech, 3, seed)
    tasks = task_set(mech, seed)
    ref = TaskOracle(mech, q, v, vd if with_vd else None).tasks(tasks)
    got = hostsim_tasks(mech, tasks, q.astype(dt), v.astype(dt), vd.astype(dt) if with_vd else None)
    for k in OUTPUTS:
        assert _err(got[k], ref[k]) < TOL[dt], (k, _err(got[k], ref[k]))
    # each output alone, bit for bit; without v for the outputs that do not need it
    for k in OUTPUTS:
        one = hostsim_tasks(mech, tasks, q.astype(dt), None if k not in VEL_OUTPUTS else v.astype(dt),
                            vd.astype(dt) if with_vd else None, want=(k,))
        assert np.array_equal(one[k], got[k]), k


@pytest.mark.parametrize("name,floating", MODELS)
@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_device_code_matches_oracle_named_models(name, floating, dt):
    _compare_hostsim(rbd.load_model(name, floating=floating), 17, dt)


@pytest.mark.parametrize("seed", [17, 18, 19, 20])
def test_device_code_matches_oracle_all_joint_types(seed):
    mech = randmech(seed, shuffle=seed % 2 == 1)
    _compare_hostsim(mech, seed, np.float64, with_vd=seed % 2 == 0)
    _compare_hostsim(mech, seed, np.float32, with_vd=seed % 2 == 1)


# ------------------------------------------------------------------------------------------------------------------
# CPU tier 4: argument checks (decided on the host before any CUDA call)
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
    out = _cabi.RbdTaskOut()
    out.point = buf.ctypes.data

    def call(model=h.ptr, dtype=_cabi.RBD_F64, B=1, ld=1, q=q, v=None, vd=None, tasks=ctypes.byref(d), out=ctypes.byref(out)):
        return lib.rbd_task_kinematics(model, dtype, B, ld, q, v, vd, tasks, out, None)

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
    assert call(dtype=_cabi.RBD_DUAL64X6) == _cabi.RBD_EUNSUPPORTED
    assert call(dtype=7) == _cabi.RBD_EUNSUPPORTED
    assert call(B=4, ld=3) == _cabi.RBD_EDIM
    for name in VEL_OUTPUTS:                             # v NULL with a velocity-dependent output
        o2 = _cabi.RbdTaskOut()
        setattr(o2, name, buf.ctypes.data)
        assert call(out=ctypes.byref(o2)) == _cabi.RBD_EINVAL, name
    # nothing to do: no device touched
    assert call(B=0, ld=0) == _cabi.RBD_OK
    assert call(tasks=edited(ntasks=0)) == _cabi.RBD_OK
    h.close()


# ------------------------------------------------------------------------------------------------------------------
# GPU tier
# ------------------------------------------------------------------------------------------------------------------
def _gpu_state(mech, q, v, dtype):
    import torch
    st = rbd.MechanismState(mech, q.shape[1], dtype)
    st.q.copy_(torch.from_numpy(q))
    st.v.copy_(torch.from_numpy(v))
    return st


def _gpu_outputs(st, tasks, vd=None, want=OUTPUTS):
    import torch
    K = len(tasks)
    outs = {k: torch.full((_rows(k, st.nv) * K, st.batch), float("nan"), dtype=st.dtype, device="cuda") for k in want}
    rbd.task_kinematics_(st, tasks, vd, **outs)
    torch.cuda.synchronize()
    return outs


@pytest.mark.gpu
@pytest.mark.parametrize("name,floating", MODELS + [("randmech", 18), ("randmech", 19)])
@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_gpu_matches_oracle(built, name, floating, dt):
    import torch
    tdt = torch.float64 if dt == np.float64 else torch.float32
    mech = randmech(floating, shuffle=floating % 2 == 1) if name == "randmech" else rbd.load_model(name, floating=floating)
    q, v, _, vd, _ = rand_inputs(mech, 67, 5)
    tasks = task_set(mech, 5)
    st = _gpu_state(mech, q.astype(dt), v.astype(dt), tdt)
    for with_vd in (True, False):
        vdt = torch.from_numpy(vd.astype(dt)).cuda() if with_vd else None
        got = _gpu_outputs(st, tasks, vdt)
        info = rbd.launch_info()
        assert info.kernels_launched == 1
        ref = TaskOracle(mech, q, v, vd if with_vd else None).tasks(tasks)
        for k in OUTPUTS:
            assert _err(got[k].cpu().numpy(), ref[k]) < TOL[dt], (k, with_vd)
        for k in OUTPUTS:                                # each output alone, bit for bit
            one = _gpu_outputs(st, tasks, vdt, want=(k,))[k]
            assert torch.equal(one, got[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_gpu_strides_alignment_and_tiles(built, dt):
    """ld > B with NaN padding leaves the padding NaN; a base pointer that is not 16-byte aligned gives the same bits; every
    512-sample tile of a 2^17 batch of one repeated column equals the first."""
    import torch
    tdt = torch.float64 if dt == np.float64 else torch.float32
    mech = rbd.load_model("atlas", floating=True)
    desc = mech.flatten()
    lib = rbd.load_library()
    h = _cabi.ModelHandle(desc)
    q, v, _, vd, _ = rand_inputs(mech, 37, 8)
    tasks = task_set(mech, 8)
    K, nv = len(tasks), desc.nv
    d, keep = task_desc(mech, tasks)
    code = _cabi.RBD_F64 if dt == np.float64 else _cabi.RBD_F32

    def run(B, ld, off, qn, vn, vdn):
        def col(a):
            t = torch.full((a.shape[0] * ld + off,), float("nan"), dtype=tdt, device="cuda")
            t[off:].view(a.shape[0], ld)[:, :B] = torch.from_numpy(a.astype(dt)).cuda()
            return t
        qt, vt, vdt = col(qn), col(vn), col(vdn)
        outs = {k: torch.full((_rows(k, nv) * K * ld + off,), float("nan"), dtype=tdt, device="cuda") for k in OUTPUTS}
        o = _cabi.RbdTaskOut()
        for k, t in outs.items():
            setattr(o, k, t[off:].data_ptr())
        _cabi.check(lib.rbd_task_kinematics(h.ptr, code, B, ld, qt[off:].data_ptr(), vt[off:].data_ptr(), vdt[off:].data_ptr(),
                                            ctypes.byref(d), ctypes.byref(o), None))
        torch.cuda.synchronize()
        return {k: t[off:].view(-1, ld) for k, t in outs.items()}

    dense = run(37, 37, 0, q, v, vd)
    for ld, off in ((41, 0), (37, 1), (45, 3)):
        g = run(37, ld, off, q, v, vd)
        for k in OUTPUTS:
            assert torch.equal(g[k][:, :37], dense[k]), (k, ld, off)
            assert torch.isnan(g[k][:, 37:]).all(), (k, ld, off)
    B = 1 << 17
    rep = lambda a: np.repeat(a[:, :1], B, 1)           # noqa: E731
    big = run(B, B, 0, rep(q), rep(v), rep(vd))
    for k in OUTPUTS:
        tiles = big[k].view(big[k].shape[0], B // 512, 512)
        assert torch.equal(tiles, tiles[:, :1].expand_as(tiles)), k
        assert torch.equal(big[k][:, :1], dense[k][:, :1]), k
    h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_gpu_conveniences_agree_with_fused_call(built, dt):
    import torch
    tdt = torch.float64 if dt == np.float64 else torch.float32
    mech = rbd.load_model("atlas", floating=True)
    q, v, _, vd, _ = rand_inputs(mech, 33, 9)
    st = _gpu_state(mech, q.astype(dt), v.astype(dt), tdt)
    vdt = torch.from_numpy(vd.astype(dt)).cuda()
    hand, foot, pelvis = mech.findbody("l_hand"), mech.findbody("r_foot"), mech.findbody("pelvis")
    pt = [0.05, -0.1, 0.2]
    p = rbd.path(mech, foot, hand)
    fused = _gpu_outputs(st, [TaskFrame(hand, foot, pt, pelvis)], vdt)
    fused_root = _gpu_outputs(st, [TaskFrame(hand, foot, pt, None)], vdt)
    checks = [(rbd.relative_transform(st, hand, foot), fused["transform"]),
              (rbd.relative_twist(st, hand, foot, pelvis), fused["twist"]),
              (rbd.relative_acceleration(st, hand, foot, vdt, pelvis), fused["acceleration"]),
              (rbd.point_jacobian(st, p, pt, pelvis), fused["point_jacobian"]),
              (rbd.point_velocity(st, p, pt, pelvis), fused["point_velocity"]),
              (rbd.point_acceleration(st, p, pt, vdt, pelvis), fused["point_acceleration"]),
              (rbd.geometric_jacobian(st, p, frame=pelvis), fused["geometric_jacobian"]),
              (rbd.point_jacobian(st, p, pt), fused_root["point_jacobian"])]
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(checks):
        assert torch.equal(a, b), i
    out = torch.empty_like(fused["geometric_jacobian"])
    assert torch.equal(rbd.geometric_jacobian_(out, st, p, frame=pelvis), fused["geometric_jacobian"])
    # without frame: the rbd_kinematics path, exactly as before
    jk = torch.empty((6 * st.nv, st.batch), dtype=tdt, device="cuda")
    rbd.kinematics_(st, p, geometric_jacobian=jk)
    j0 = rbd.geometric_jacobian(st, p)
    torch.cuda.synchronize()
    assert torch.equal(j0, jk)
    # and the root-frame task Jacobian agrees with it to rounding
    assert _err(fused_root["geometric_jacobian"].cpu().numpy(), jk.double().cpu().numpy()) < TOL[dt]
