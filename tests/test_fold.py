"""Folding of mirror-image chains in the model-specialised forward-dynamics program (csrc/rbd_codegen.cpp).

The left / right legs and arms of a humanoid run the same code with different model constants; the generator emits each such
pair's steps once per ABA pass, as a two-iteration loop.  CPU tier: the folded program's CPU flavour is bit-identical to the
straight-line form of the same trace, the bundled humanoids actually fold, and a pair whose chains differ in a joint's fast
class stays straight-line."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from rigidbodydynamics.jl_b200._cabi import RbdModelDesc, make_desc
from tests.util import rand_inputs

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "..", "rigidbodydynamics", "jl_b200", "csrc")


@pytest.fixture(scope="module")
def shim():
    d = tempfile.mkdtemp(prefix="rbd_fold_")
    so = os.path.join(d, "libfold.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-I", _CSRC, "-o", so,
                           os.path.join(_HERE, "hostsim", "hostsim_fold.cpp"), os.path.join(_CSRC, "rbd_model.cpp"),
                           os.path.join(_CSRC, "rbd_codegen.cpp")])
    lib = ctypes.CDLL(so)
    lib.fold_spec_source.restype = ctypes.c_void_p
    lib.fold_spec_source.argtypes = [ctypes.POINTER(RbdModelDesc), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                     ctypes.c_void_p]
    lib.fold_free.argtypes = [ctypes.c_void_p]
    return lib, d


def _source(shim, desc, dtype, fold, has_in2=True, has_out1=False):
    lib, _ = shim
    d, keep = make_desc(desc)
    st = (ctypes.c_int * 4)()
    p = lib.fold_spec_source(ctypes.byref(d), 0 if dtype == np.float32 else 1, int(has_in2), int(has_out1), int(fold), st)
    assert p
    src = ctypes.string_at(p).decode()
    lib.fold_free(p)
    return src, dict(zip(("nodes_live", "fold_loops", "fold_bodies", "pairs"), st))


def _run(shim, src, desc, dtype, q, v, tau, has_out1=False):
    _, d = shim
    import hashlib
    tag = hashlib.sha1(src.encode()).hexdigest()[:16]
    so = os.path.join(d, f"spec_{tag}.so")
    if not os.path.exists(so):
        cpp = os.path.join(d, f"spec_{tag}.cpp")
        with open(cpp, "w") as f:
            f.write(src)
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-ffp-contract=off",
                               "-I", _CSRC, "-o", so, cpp])
    fn = ctypes.CDLL(so).rbd_spec_cpu
    fn.argtypes = [ctypes.c_void_p] * 5 + [ctypes.c_longlong, ctypes.c_void_p]
    q = np.ascontiguousarray(q, dtype); v = np.ascontiguousarray(v, dtype); tau = np.ascontiguousarray(tau, dtype)
    B = q.shape[1]
    vd = np.full((desc.nv, B), np.nan, dtype)
    qd = np.full((desc.nq, B), np.nan, dtype) if has_out1 else None
    sh = np.zeros(4096, dtype)
    es = np.dtype(dtype).itemsize
    for b in range(B):
        fn(q.ctypes.data + b * es, v.ctypes.data + b * es, tau.ctypes.data + b * es, vd.ctypes.data + b * es,
           None if qd is None else qd.ctypes.data + b * es, B, sh.ctypes.data)
    return vd, qd


def _check_bit_identical(shim, mech, dtype, expect_fold):
    desc = mech.flatten()
    q, v, tau, _, _ = rand_inputs(mech, 16, 3)
    for has_out1 in (False, True):
        src0, st0 = _source(shim, desc, dtype, False, has_out1=has_out1)
        src1, st1 = _source(shim, desc, dtype, True, has_out1=has_out1)
        assert st0["fold_loops"] == 0
        if expect_fold:
            assert st1["fold_loops"] > 0 and st1["fold_bodies"] > 0 and "rbd_it" in src1
        a, qa = _run(shim, src0, desc, dtype, q, v, tau, has_out1)
        b, qb = _run(shim, src1, desc, dtype, q, v, tau, has_out1)
        assert np.isfinite(a).all() and np.array_equal(a, b)
        if has_out1:
            assert np.array_equal(qa, qb)
    return st1


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("name", ["atlas", "valkyrie"])
def test_humanoid_program_folds_bit_identical(shim, name, dtype):
    st = _check_bit_identical(shim, rbd.load_model(name, floating=True), dtype, True)
    assert st["pairs"] == 2                       # legs and arms
    assert st["fold_loops"] >= 4 and st["fold_bodies"] >= 4 * 6


def _mirrored_tree(seed, spoil=False):
    """Floating base, a short random branch, and two revolute chains of 4 bodies hung from the base: the same axis-aligned
    joint axes and tree rotations, translations mirrored in y, independent random inertias.  `spoil`: one joint of the right
    chain gets an origin shift where its left twin has none (F_ZERO_R), so the two chains no longer run the same code."""
    rng = np.random.default_rng(seed)
    eye = np.eye(3)
    M = np.diag([1.0, -1.0, 1.0])
    mech = rbd.Mechanism(rbd.RigidBody("world"))
    base = rbd.RigidBody("base", rbd.SpatialInertia.rand(rng))
    mech.attach(mech.root_body, base, rbd.Joint("floating", rbd.QuaternionFloating()))
    spec = []
    for k in range(4):
        perm = rng.permutation(3)
        R = eye[:, perm] * rng.choice([-1.0, 1.0], 3)
        if np.linalg.det(R) < 0:
            R[:, 0] = -R[:, 0]
        axis = eye[int(rng.integers(3))] * rng.choice([-1.0, 1.0])
        trans = np.zeros(3) if k == 2 else rng.standard_normal(3)
        spec.append((R, axis, trans))
    for side in ("l", "r"):
        parent = base
        for k, (R, axis, trans) in enumerate(spec):
            if side == "r":
                trans = M @ trans
                if spoil and k == 2:
                    trans = np.array([0.0, 0.0, 0.1])
            body = rbd.RigidBody(f"{side}{k}", rbd.SpatialInertia.rand(rng))
            mech.attach(parent, body, rbd.Joint(f"{side}j{k}", rbd.Revolute(axis)), joint_pose=rbd.Transform3D(R, trans))
            parent = body
    body = rbd.RigidBody("torso", rbd.SpatialInertia.rand(rng))
    mech.attach(base, body, rbd.Joint("tj", rbd.Revolute(eye[2])), joint_pose=rbd.Transform3D(eye, rng.standard_normal(3)))
    mech.attach(body, rbd.RigidBody("head", rbd.SpatialInertia.rand(rng)), rbd.Joint("hj", rbd.Revolute(eye[0])),
                joint_pose=rbd.Transform3D(eye, rng.standard_normal(3)))
    return mech


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_mirrored_random_chains_fold_bit_identical(shim, dtype):
    for seed in (1, 2):
        st = _check_bit_identical(shim, _mirrored_tree(seed), dtype, True)
        assert st["pairs"] == 1 and st["fold_loops"] == 3 and st["fold_bodies"] == 3 * 4


def test_mismatched_fast_class_stays_straight_line(shim):
    mech = _mirrored_tree(1, spoil=True)
    desc = mech.flatten()
    src0, st0 = _source(shim, desc, np.float32, False)
    src1, st1 = _source(shim, desc, np.float32, True)
    assert st1["pairs"] == 0 and st1["fold_loops"] == 0
    assert src0 == src1 and "rbd_it" not in src1 and "rbd_par_tab" not in src1
