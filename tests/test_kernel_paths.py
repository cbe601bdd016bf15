"""Every kernel path the host code can pick for dynamics! / inverse_dynamics! / dynamics_bias! / mass_matrix! / rbd_kinematics, forced
on purpose and checked against the oracle on models beyond the bundled robots (csrc/rbd_b200.cu dynamics_t, inverse_dynamics_t,
mass_matrix_t, kinematics_t, dynamics_dual; csrc/rbd_spec.cpp spec_try_launch).

Paths: the generic shared-memory kernels (small batch, no cubin), the generic mixed CTA (large batch, RBD_JIT_VARIANT=2), the
model-specialised NVRTC programs in single-warp blocks (rbd_jit_smem) and in the mixed CTA (rbd_jit_mix), and the generic kernel
queued behind an fp32 program (gated on angles beyond the fast sin / cos range).  Every call asserts the launch record, so a case
that silently ran another path fails.

Beyond the oracle, the fp32 programs are held to their CPU flavour (tests/hostsim.SpecProgram) bit for bit: both are compiled
without contraction, with explicit fma, round-to-nearest reciprocals / divisions and the same sincos_fast, so any difference is an
error in the kernel shell (work queue, prefetch, inactive lanes, shared / L2 stash, row addressing) or in the prelude."""
import ctypes
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from oracle import Oracle
from rigidbodydynamics.jl_b200 import _cabi as C
from tests import hostsim
from tests.test_contact import _with_contacts
from tests.test_fold import _mirrored_tree
from tests.util import axis_aligned_tree, config_distance, make_duals, rand_inputs, randmech, rel_err

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _all_types_tree(seed):
    """randmech's joint mix at half size, order shuffled: all eight joint types, multi-DoF joints below the root (the traced GENERAL
    blocks), and a forward-dynamics stash within the 256 rows of the specialised kernels -- the 27-body randmech tree needs 414
    rows, so its forward dynamics always runs the generic kernels."""
    rng = np.random.default_rng(seed)
    jts = [rbd.QuaternionFloating, rbd.Revolute, rbd.Revolute, rbd.Revolute, rbd.Fixed, rbd.Prismatic, rbd.Prismatic, rbd.Planar,
           rbd.Planar, rbd.SPQuatFloating, rbd.SinCosRevolute, rbd.QuaternionSpherical]
    return rbd.rand_tree_mechanism(rng, [jts[i] for i in rng.permutation(len(jts))])


def _single(joint_type, seed):
    return rbd.rand_chain_mechanism(np.random.default_rng(seed), [joint_type])


# Fresh Mechanism objects on every call: the library handle is cached on the mechanism and the specialised-kernel entries
# (including a failed one) on the handle.
MODELS = {
    "all_types": lambda: _all_types_tree(4),
    "fast_classes": lambda: axis_aligned_tree(5),
    "folded": lambda: _mirrored_tree(3),
    "revolute20": lambda: rbd.rand_floating_tree_mechanism(np.random.default_rng(20), [rbd.Revolute] * 20),
    "chain64": lambda: rbd.rand_chain_mechanism(np.random.default_rng(64), [rbd.Revolute] * 64),
    "planar1": lambda: _single(rbd.Planar, 1),
    "spherical1": lambda: _single(rbd.QuaternionSpherical, 2),
}
RANDOM_TREES = ("all_types", "fast_classes", "folded", "revolute20")     # fp32 class of test_general_trees_all_joint_types
SPEC32 = ("all_types", "fast_classes", "folded")  # the full fp32 program matrix
SPEC64 = ("all_types", "folded")
ALL_BITS = (C.RBD_SPEC_DYNAMICS | C.RBD_SPEC_DYNAMICS_QDOT | C.RBD_SPEC_DYNAMICS_NOTAU | C.RBD_SPEC_INVERSE_DYNAMICS
            | C.RBD_SPEC_DYNAMICS_BIAS | C.RBD_SPEC_MASS_MATRIX | C.RBD_SPEC_MASS_MATRIX_LOWER)
BITS64 = C.RBD_SPEC_DYNAMICS | C.RBD_SPEC_INVERSE_DYNAMICS | C.RBD_SPEC_MASS_MATRIX
OPS32 = ("aba", "aba_qd", "aba_notau", "aba_notau_qd", "rnea", "bias", "crba", "crba_lower")
KR = hostsim.KIN_ROWS
KIN = {"kin_all": (KR, True), "kin_A": (("A",), False), "kin_J": (("transforms", "com", "pe", "J"), False)}   # outputs, reads v
# Which programs take the mixed CTA when RBD_JIT_VARIANT=2 forces it (rbd_spec.cpp: only where it puts >= 15 % more warps on an
# SM than the single-warp blocks do; the programs with small stashes already fill the SM with blocks).  Measured on the H100.
SPEC_MIX = {"all_types": {"aba", "aba_qd", "aba_notau", "aba_notau_qd", "kin_A"},
            "fast_classes": {"aba", "aba_qd", "aba_notau", "aba_notau_qd", "rnea", "bias", "kin_A"},
            "folded": {"aba", "aba_qd", "aba_notau", "aba_notau_qd"}}
# The same rule for the generic inverse dynamics with external wrenches (launch_mix): small trees stay in single-warp blocks.
GENERIC_MIX = {"all_types": False, "fast_classes": True, "folded": False, "revolute20": True, "planar1": False, "spherical1": False}
TILE = 512
MIX_B = 1 << 17
KIN_B = 1 << 15          # no precompile bit for kinematics: a batch at the compile threshold loads the program
# fp64 programs against their CPU flavour: device sincos against glibc sin / cos, so not bit-identical; forward dynamics carries
# those last-bit differences through the articulated-inertia solve.  Largest difference (rel_err) measured on an H100 80GB HBM3
# (700 W): forward dynamics 1.6e-14 (all_types) / 1.6e-15 (folded), inverse dynamics and mass matrix <= 8e-16.
FP64_CPU_TOL = 5e-14


def _tol(name, dtype):
    if dtype == np.float64:
        return 1e-9
    if name == "chain64":
        return 5e-3          # fp32 class of the 64-body chain in test_edge_cases_empty_padded_and_defaults
    return 1e-3 if name in RANDOM_TREES else 2e-5


@pytest.fixture(scope="session")
def _jit_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("rbd_jit_cache"))


@pytest.fixture
def jit_cache(_jit_dir, monkeypatch):
    """One cubin cache for the session, set per test: nothing bundled leaks in, programs compiled once are shared between these
    tests, and the other test modules keep the library's own cache."""
    monkeypatch.setenv("RBD_JIT_CACHE", _jit_dir)
    return _jit_dir


@pytest.fixture
def empty_cache(tmp_path, monkeypatch):
    """An empty cubin cache for the calls that must run the generic kernels."""
    monkeypatch.setenv("RBD_JIT_CACHE", str(tmp_path))
    return str(tmp_path)


@pytest.fixture
def variant(monkeypatch):
    def set_(v):
        monkeypatch.setenv("RBD_JIT_VARIANT", str(v))
    return set_


def _model(name):
    mech = MODELS[name]()
    desc = mech.flatten()
    return mech, desc, C.ModelHandle(desc)


def _sign(mech):
    return rbd.path(mech, mech.joints[-1].successor, mech.joints[len(mech.joints) // 2].successor).sign


def _angle_row(mech):
    """q row of the last revolute joint that does not hang from the world (the mass matrix does not depend on the angle of a
    joint at the root, and the generated programs drop what an output does not depend on)."""
    qs, row = 0, None
    for j in mech.joints:
        if type(j.joint_type) is rbd.Revolute and j.predecessor is not mech.root_body:     # (Prismatic derives from Revolute)
            row = qs
        qs += j.nq
    assert row is not None
    return row


def _inputs(mech, B, seed, npdt, wext=False):
    """Seeded inputs, rounded to what the kernels of that precision see, tiled from TILE samples when B > TILE."""
    q, v, tau, vd, w = rand_inputs(mech, min(B, TILE), seed, wext)
    x = {"q": q, "v": v, "tau": tau, "vd": vd}
    if wext:
        x["wext"] = w
    for k in x:
        x[k] = x[k].astype(npdt).astype(np.float64)
        if B > TILE:
            x[k] = np.tile(x[k], (1, -(-B // TILE)))[:, :B].copy()
    return x


# ------------------------------------------------------------------------------------------------------- device calls through the C ABI
def _torch():
    import torch
    return torch


def _buf(rows, B, dtype, ld=None, shift=0, data=None):
    """A [rows, B] device array with leading dimension ``ld`` (NaN padding), starting ``shift`` elements into its allocation
    (shift = 1: not 16-byte aligned).  Returns the [rows, ld] view; its data_ptr() is the array's base pointer."""
    torch = _torch()
    ld = B if ld is None else ld
    flat = torch.full((rows * ld + shift,), float("nan"), dtype=dtype, device="cuda")
    view = flat[shift:].view(rows, ld)
    if data is not None:
        view[:, :B] = torch.from_numpy(np.asarray(data)).to(dtype)
    return view


def _p(t):
    return None if t is None else t.data_ptr()


def _dt_code(dtype):
    return C.RBD_F32 if dtype == _torch().float32 else C.RBD_F64


def _launch(status):
    C.check(status)
    _torch().cuda.synchronize()
    return C.launch_info()


def _kin_rows(desc):
    return {"transforms": 12 * desc.nb, "com": 3, "ke": 1, "pe": 1, "momentum": 6, "mrb": 6, "A": 6 * desc.nv, "J": 6 * desc.nv}


def _eval(h, desc, op, dtype, x, sign=None, ld=None, shift=0):
    """Run one entry point; returns ({output: [rows, ld] device view}, launch record)."""
    lib = C.load_library()
    B = x["q"].shape[1]
    ld = B if ld is None else ld
    nq, nv = desc.nq, desc.nv
    dt = _dt_code(dtype)
    inp = lambda k: _buf(x[k].shape[0], B, dtype, ld, shift, x[k])
    out = lambda rows: _buf(rows, B, dtype, ld, shift)
    q = inp("q")
    if op.startswith("aba"):
        v, tau = inp("v"), (None if "notau" in op else inp("tau"))
        o = {"vd": out(nv)}
        if op.endswith("qd"):
            o["qd"] = out(nq)
        info = _launch(lib.rbd_dynamics(h.ptr, dt, B, ld, _p(q), _p(v), _p(tau), None, _p(o["vd"]), _p(o.get("qd")), None))
    elif op in ("rnea", "rnea_wext", "bias"):
        v = inp("v")
        w = inp("wext") if op == "rnea_wext" else None
        o = {"tau": out(nv)}
        if op == "bias":
            info = _launch(lib.rbd_dynamics_bias(h.ptr, dt, B, ld, _p(q), _p(v), None, _p(o["tau"]), None))
        else:
            info = _launch(lib.rbd_inverse_dynamics(h.ptr, dt, B, ld, _p(q), _p(v), _p(inp("vd")), _p(w), _p(o["tau"]), None))
    elif op.startswith("crba"):
        o = {"M": out(nv * nv)}
        info = _launch(lib.rbd_mass_matrix_uplo(h.ptr, dt, B, ld, _p(q), _p(o["M"]), 1 if op == "crba_lower" else 0, None))
    else:
        names, with_v = KIN[op]
        rows = _kin_rows(desc)
        o = {k: out(rows[k]) for k in names}
        ko = C.RbdKinematicsOut(*[_p(o.get(k)) for k in KR])
        sg = np.ascontiguousarray(sign, np.int8) if "J" in names else None
        info = _launch(lib.rbd_kinematics(h.ptr, dt, B, ld, _p(q), _p(inp("v")) if with_v else None,
                                          None if sg is None else sg.ctypes.data_as(ctypes.c_void_p), ctypes.byref(ko), None))
    return o, info


def _np(o, B=None):
    return {k: (t if B is None else t[:, :B]).cpu().numpy() for k, t in o.items()}


def _oracle(o, desc, op, x, sign=None):
    q, v = x["q"], x["v"]
    if op.startswith("aba"):
        vd, qd = o.dynamics(q, v, None if "notau" in op else x["tau"], want_qd=True)
        return {"vd": vd, "qd": qd} if op.endswith("qd") else {"vd": vd}
    if op == "rnea":
        return {"tau": o.inverse_dynamics(q, v, x["vd"])}
    if op == "rnea_wext":
        return {"tau": o.inverse_dynamics(q, v, x["vd"], x["wext"])}
    if op == "bias":
        return {"tau": o.dynamics_bias(q, v)}
    if op.startswith("crba"):
        return {"M": o.mass_matrix(q)}
    names, with_v = KIN[op]
    ref = o.kinematics(q, v if with_v else None, sign if "J" in names else None)
    return {k: ref[k] for k in names}


def _lower_mask(nv):
    """[nv * nv] rows with row >= column (entry (i, j) at row i + j * nv)."""
    i, j = np.meshgrid(np.arange(nv), np.arange(nv), indexing="ij")
    return (i >= j).T.reshape(-1)


def _check_oracle(got, ref, op, nv, tol, what):
    for k, r in ref.items():
        g = np.asarray(got[k], float)
        if op == "crba_lower":
            keep = _lower_mask(nv)
            assert np.isnan(g[~keep]).all(), (what, "upper triangle written")
            g, r = g[keep], r[keep]
        if k == "qd":
            assert np.abs(g - r).max() < (1e-12 if tol < 1e-6 else 1e-5), (what, k)
        else:
            err = rel_err(g, r)
            assert err < tol, (what, k, err)


def _cpu(desc, op, npdt, x, sign=None):
    """The same program compiled for the CPU (tests/hostsim.SpecProgram), on the first TILE samples."""
    q, v = x["q"][:, :TILE], x["v"][:, :TILE]
    nv = desc.nv
    if op.startswith("aba"):
        notau, qd = "notau" in op, op.endswith("qd")
        r = hostsim.SpecProgram(desc, "aba", npdt, not notau, qd).run(q, v, None if notau else x["tau"][:, :TILE])
        return {"vd": r[0], "qd": r[1]} if qd else {"vd": r}
    if op in ("rnea", "bias"):
        r = hostsim.SpecProgram(desc, "rnea", npdt, op == "rnea").run(q, v, x["vd"][:, :TILE] if op == "rnea" else None)
        return {"tau": r}
    if op.startswith("crba"):
        lower = op == "crba_lower"
        prog = hostsim.SpecProgram(desc, "crba", npdt, has_in2=2 * lower, has_out1=False)
        return {"M": prog.run(q, np.zeros((nv, TILE)), None, out0_rows=nv * nv)}
    names, with_v = KIN[op]
    full = _kin_rows(desc)
    rows = [full[k] if k in names else 0 for k in KR]
    hostsim.spec_kin(sum(1 << k for k, r in enumerate(rows) if r), sign if "J" in names else None, desc.nb)
    outs = hostsim.SpecProgram(desc, "kin", npdt, has_in2=1 if with_v else 0, has_out1=False).run_kin(q, v if with_v else None, rows)
    return {k: outs[i] for i, k in enumerate(KR) if k in names}


def _same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def _tiles_equal(t, B):
    """Every TILE-sample tile of a device output equals the first one, bit for bit (NaN where the first tile has NaN)."""
    torch = _torch()
    n = B // TILE
    body = t[:, :n * TILE].reshape(t.shape[0], n, TILE)
    first = t[:, None, :TILE].expand_as(body)
    return bool(((body == first) | (torch.isnan(body) & torch.isnan(first))).all())


def _dev_equal(a, b):
    torch = _torch()
    return bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all())


# ---------------------------------------------------------------------------------------------------------------------- CPU tier
@pytest.mark.parametrize("name", list(MODELS))
def test_model_set_covers_its_purpose(built, name):
    """Each model of the matrix still exercises what it is there for (guards against the generator or the flattener drifting)."""
    mech, desc, h = _model(name)
    kinds = {type(j.joint_type) for j in mech.joints}
    try:
        if name == "all_types":
            assert h.info.general_path == 1
            assert hostsim.spec_source(desc, "aba", np.float32, True, False, 1)[1]["stash_rows"] <= 256
            assert hostsim.spec_source(randmech(6, shuffle=True).flatten(), "aba", np.float32, True, False, 1)[1]["stash_rows"] > 256
            assert kinds == {rbd.QuaternionFloating, rbd.Revolute, rbd.Fixed, rbd.Prismatic, rbd.Planar, rbd.SPQuatFloating,
                             rbd.SinCosRevolute, rbd.QuaternionSpherical}
        elif name == "fast_classes":
            assert h.info.general_path == 0
            assert {rbd.Prismatic, rbd.Fixed, rbd.SinCosRevolute} <= kinds        # kAllKinds instantiations
        elif name == "folded":
            src, _ = hostsim.spec_source(desc, "aba", np.float32, True, False, 1)
            assert "rbd_it" in src and "rbd_r" in src                             # folded limb loops, register stash rows
        elif name == "revolute20":
            assert kinds == {rbd.QuaternionFloating, rbd.Revolute} and h.info.general_path == 0     # KINDS = 0
            assert desc.nb > 15        # fp64 ABA program above the size rule of spec_worthwhile: stays generic
        elif name == "chain64":
            for algo in ("aba", "rnea"):
                for dt in (np.float32, np.float64):
                    assert hostsim.spec_source(desc, algo, dt, True, False, 1)[1]["stash_rows"] > 256, (algo, dt)
        else:
            assert desc.nb == 1 and len(kinds) == 1 and desc.nv == 3
            info = hostsim.info(desc)
            assert info["order"] == [0]
    finally:
        h.close()


@pytest.mark.parametrize("name", SPEC32)
def test_cpu_programs_match_oracle_and_compile(built, jit_cache, name, tmp_path, monkeypatch):
    """CPU tier of the program matrix: every fp32 program the GPU tests below load, compiled as plain C++ and checked against the
    oracle, plus the NVRTC compilation of the same programs for sm_90a (no GPU needed)."""
    monkeypatch.setenv("RBD_JIT_CACHE", str(tmp_path))
    mech, desc, h = _model(name)
    x = _inputs(mech, 16, 3, np.float32)
    sign = _sign(mech)
    o = Oracle(desc)
    for op in OPS32 + tuple(KIN):
        got = _cpu(desc, op, np.float32, x, sign)
        _check_oracle(got, _oracle(o, desc, op, {k: a[:, :16] for k, a in x.items()}, sign), op, desc.nv, _tol(name, np.float32), op)
    try:
        h.precompile(C.RBD_F32, ALL_BITS, load=False)
    except C.RbdError as e:
        pytest.skip(f"NVRTC not available here: {e}")
    finally:
        h.close()
    files = os.listdir(tmp_path)
    assert len(files) == 8 and all(f.endswith(".cubin") for f in files)
    for f in files:             # the GPU tests of the same session load these instead of compiling them again
        shutil.copy(os.path.join(tmp_path, f), jit_cache)


# ---------------------------------------------------------------------------------------------------------------------- GPU tier
@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float32", "float64"])
@pytest.mark.parametrize("name", list(MODELS))
def test_generic_kernels_gpu(built, empty_cache, name, dtype_name):
    """Small ragged batch, no cubin: the generic shared-memory kernels (one launch, single-warp blocks) against the oracle."""
    torch = _torch()
    dtype, npdt = getattr(torch, dtype_name), np.dtype(dtype_name)
    mech, desc, h = _model(name)
    B = 517
    x = _inputs(mech, B, 11, npdt)
    sign = _sign(mech)
    o = Oracle(desc)
    for op in OPS32 + tuple(KIN):
        got, info = _eval(h, desc, op, dtype, x, sign)
        assert (info.specialised, info.block, info.kernels_launched) == (0, 32, 1), (op, info.block)
        _check_oracle(_np(got, B), _oracle(o, desc, op, x, sign), op, desc.nv, _tol(name, npdt), (name, op))
    h.close()


def _spec_ops(name, npdt):
    if npdt == np.float32:
        return OPS32
    return ("aba", "rnea", "crba")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name,name", [("float32", n) for n in SPEC32] + [("float64", n) for n in SPEC64])
def test_specialised_smem_gpu(built, jit_cache, name, dtype_name):
    """The precompiled programs at a small ragged batch (single-warp blocks): launch record, oracle, the CPU flavour of the same
    program (fp32: bit for bit), leading dimension > B with NaN padding and a base pointer that is not 16-byte aligned
    (bit-identical, padding untouched)."""
    torch = _torch()
    dtype, npdt = getattr(torch, dtype_name), np.dtype(dtype_name)
    mech, desc, h = _model(name)
    h.precompile(_dt_code(dtype), ALL_BITS if npdt == np.float32 else BITS64, load=True)
    B = 517
    x = _inputs(mech, B, 12, npdt)
    sign = _sign(mech)
    o = Oracle(desc)
    for op in _spec_ops(name, npdt):
        got, info = _eval(h, desc, op, dtype, x, sign)
        assert (info.specialised, info.block, info.kernels_launched) == (1, 32, 2 if npdt == np.float32 else 1), (op, info.block)
        g = _np(got, B)
        _check_oracle(g, _oracle(o, desc, op, x, sign), op, desc.nv, _tol(name, npdt), (name, op))
        cpu = _cpu(desc, op, npdt, x, sign)
        for k in cpu:
            if npdt == np.float32:
                assert _same(g[k][:, :TILE], cpu[k]), (name, op, k, np.nanmax(np.abs(g[k][:, :TILE] - cpu[k])))
            else:
                err = rel_err(np.nan_to_num(g[k][:, :TILE]), np.nan_to_num(cpu[k]))
                assert err < FP64_CPU_TOL, (name, op, k, err)
        # leading dimension > B with NaN padding, and a base pointer one element past an aligned allocation
        for ld, shift in ((B + 13, 0), (B, 1), (B + 13, 1)):
            got2, info2 = _eval(h, desc, op, dtype, x, sign, ld=ld, shift=shift)
            assert (info2.specialised, info2.block, info2.kernels_launched) == (1, 32, info.kernels_launched), (op, ld, shift)
            for k in got:
                assert _same(got2[k][:, :B].cpu().numpy(), g[k]), (name, op, k, ld, shift)
                assert bool(torch.isnan(got2[k][:, B:]).all()), (name, op, k, ld, shift, "padding written")
    h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", SPEC32)
def test_specialised_mixed_cta_gpu(built, jit_cache, variant, name):
    """Large batch: every fp32 program (and the three kinematics programs) in single-warp blocks and in the mixed CTA, bit-identical
    to each other, every tile bit-identical to the first, the first tile bit-identical to the CPU flavour, and ld > B."""
    torch = _torch()
    dtype, npdt = torch.float32, np.dtype(np.float32)
    mech, desc, h = _model(name)
    h.precompile(C.RBD_F32, ALL_BITS, load=True)
    x = _inputs(mech, MIX_B, 13, npdt)
    sign = _sign(mech)
    o = Oracle(desc)
    x1 = {k: a[:, :TILE] for k, a in x.items()}
    for op in OPS32 + tuple(KIN):
        res = {}
        for var in (1, 2):
            variant(var)
            got, info = _eval(h, desc, op, dtype, x, sign)
            assert info.specialised == 1 and info.kernels_launched == 2, (op, var)
            assert info.block == (512 if var == 2 and op in SPEC_MIX[name] else 32), (op, var, info.block)
            res[var] = got
        for k in res[1]:
            assert _dev_equal(res[1][k], res[2][k]), (name, op, k, "smem != mixed CTA")
            assert _tiles_equal(res[2][k], MIX_B), (name, op, k, "tiles differ")
        g = _np(res[2], TILE)
        _check_oracle(g, _oracle(o, desc, op, x1, sign), op, desc.nv, _tol(name, npdt), (name, op))
        cpu = _cpu(desc, op, npdt, x, sign)
        for k in cpu:
            assert _same(g[k], cpu[k]), (name, op, k, np.nanmax(np.abs(g[k] - cpu[k])))
        if op.startswith("kin"):        # the kinematics programs have no small-batch run above: leading dimension > B here
            variant(1)
            got2, info2 = _eval(h, desc, op, dtype, {k: a[:, :KIN_B] for k, a in x.items()}, sign, ld=KIN_B + 5)
            assert info2.specialised == 1 and info2.block == 32
            for k in got2:
                assert _dev_equal(got2[k][:, :KIN_B], res[1][k][:, :KIN_B]), (name, op, k)
                assert bool(torch.isnan(got2[k][:, KIN_B:]).all()), (name, op, k, "padding written")
        del res
    h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float32", "float64"])
@pytest.mark.parametrize("name", [n for n in MODELS if n != "chain64"])
def test_generic_mixed_cta_gpu(built, empty_cache, variant, name, dtype_name):
    """inverse_dynamics! with external wrenches is always generic: at a large batch the mixed CTA (rnea_kernel_mix<T, true>) against
    the shared-memory kernel bit for bit, every tile against the first, the first tile against the oracle (small trees, whose
    single-warp blocks already fill an SM, stay in those blocks).  On the all-revolute tree the same for fp64 forward dynamics
    (aba_kernel_mix<double, 0>): at this batch an fp64 program would be compiled if it were worth it, so this also shows the size
    rule of spec_worthwhile keeping it generic."""
    torch = _torch()
    dtype, npdt = getattr(torch, dtype_name), np.dtype(dtype_name)
    mech, desc, h = _model(name)
    x = _inputs(mech, MIX_B, 14, npdt, wext=True)
    x1 = {k: a[:, :TILE] for k, a in x.items()}
    o = Oracle(desc)
    ops = ["rnea_wext"] + (["aba"] if name == "revolute20" and npdt == np.float64 else [])
    for op in ops:
        res = {}
        for var in (1, 2):
            variant(var)
            got, info = _eval(h, desc, op, dtype, x)
            assert info.specialised == 0 and info.kernels_launched == 1, (op, var)
            mixed = var == 2 and (op == "aba" or GENERIC_MIX[name])
            assert info.block == ({torch.float32: 512, torch.float64: 256}[dtype] if mixed else 32), (name, op, var, info.block)
            res[var] = got
        for k in res[1]:
            assert _dev_equal(res[1][k], res[2][k]), (name, op, k, "smem != mixed CTA")
            assert _tiles_equal(res[2][k], MIX_B), (name, op, k)
        _check_oracle(_np(res[2], TILE), _oracle(o, desc, op, x1), op, desc.nv, _tol(name, npdt), (name, op))
    h.close()


_CHILD = r"""
import json, sys
import numpy as np, torch
sys.path.insert(0, sys.argv[1])
from tests import test_kernel_paths as t
mech, desc, h = t._model("revolute20")
x = t._inputs(mech, t.MIX_B, 15, np.float32)
import os
o = t.Oracle(desc)
x1 = {k: a[:, :t.TILE] for k, a in x.items()}
for op in ("aba", "rnea"):
    out = {}
    for var in (1, 2):
        os.environ["RBD_JIT_VARIANT"] = str(var)
        got, info = t._eval(h, desc, op, torch.float32, x)
        out[var] = next(iter(got.values()))
        print(json.dumps({"op": op, "variant": var, "specialised": info.specialised, "block": info.block,
                          "kernels": info.kernels_launched}))
    ref = next(iter(t._oracle(o, desc, op, x1).values()))
    print(json.dumps({"op": op, "identical": t._dev_equal(out[1], out[2]), "tiles": t._tiles_equal(out[2], t.MIX_B),
                      "err": t.rel_err(out[2][:, :t.TILE].cpu().numpy(), ref)}))
"""


@pytest.mark.gpu
def test_generic_fp32_mixed_cta_without_programs_gpu(built, tmp_path):
    """aba_kernel_mix<float, 0> and rnea_kernel_mix<float, false> run only when no fp32 program serves the call (RBD_JIT=0, read
    once per process; the models whose programs are too large are also too large for these kernels): a child process runs the
    all-revolute tree at a large batch in both shapes."""
    env = dict(os.environ, RBD_JIT="0", RBD_JIT_CACHE=str(tmp_path))
    r = subprocess.run([sys.executable, "-c", _CHILD, ROOT], env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    lines = [json.loads(s) for s in r.stdout.splitlines() if s.startswith("{")]
    assert len(lines) == 6
    for op, shapes, check in (("aba", lines[0:2], lines[2]), ("rnea", lines[3:5], lines[5])):
        assert [(d["op"], d["specialised"], d["block"], d["kernels"]) for d in shapes] == [(op, 0, 32, 1), (op, 0, 512, 1)]
        assert check["identical"] and check["tiles"] and check["err"] < 2e-5, check


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["all_types", "folded"])
def test_gated_fallback_gpu(built, jit_cache, monkeypatch, name):
    """One sample with a joint angle of 3e4 rad (beyond the fast sin / cos range): the fp32 program raises the flag and the gated
    generic kernel behind it redoes the batch -- bit-identical to the generic kernel alone, and the whole batch matches the oracle."""
    torch = _torch()
    mech, desc, h = _model(name)
    h.precompile(C.RBD_F32, C.RBD_SPEC_DYNAMICS | C.RBD_SPEC_INVERSE_DYNAMICS | C.RBD_SPEC_MASS_MATRIX, load=True)
    o = Oracle(desc)
    sign = _sign(mech)
    row = _angle_row(mech)
    tol = _tol(name, np.float32)
    for op, B in (("aba", 517), ("rnea", 517), ("crba", 517), ("kin_all", KIN_B)):
        x = _inputs(mech, B, 16, np.float32)
        x["q"][row, 77] = 3.0e4                     # exactly representable in fp32
        got, info = _eval(h, desc, op, torch.float32, x, sign)
        assert (info.specialised, info.block, info.kernels_launched) == (1, 32, 2), (op, info.block)
        n = min(B, TILE)
        g = _np(got, n)
        _check_oracle(g, _oracle(o, desc, op, {k: a[:, :n] for k, a in x.items()}, sign), op, desc.nv, tol, (name, op))
        with monkeypatch.context() as m:           # the generic kernel alone on the same samples
            m.setenv("RBD_JIT_CACHE", os.path.join(jit_cache, "none"))
            os.makedirs(os.path.join(jit_cache, "none"), exist_ok=True)
            _, _, h2 = _model(name)
            ref, info2 = _eval(h2, desc, op, torch.float32, {k: a[:, :n] for k, a in x.items()}, sign)
            assert info2.specialised == 0
            h2.close()
        for k in g:
            assert _same(g[k], ref[k].cpu().numpy()), (name, op, k)
    h.close()


def _isolation(h, desc, op, dtype, x, col, sign=None):
    """NaN velocities in one sample and, separately, a NaN joint angle: only that column may be non-finite; every other column is
    bit-identical to the clean run (no leak through a shared stash, the L2 scratch or a pending slot).  All of the sample's v is
    poisoned: the generated programs fold terms that are exactly zero, so a single velocity can drop out of an output that the
    library's IEEE arithmetic would turn into NaN."""
    clean, info0 = _eval(h, desc, op, dtype, x, sign)
    row = x["_angle_row"]
    for what in ("v", "angle"):
        if what == "v" and op.startswith("crba"):
            continue
        y = {k: a.copy() for k, a in x.items() if not k.startswith("_")}
        if what == "v":
            y["v"][:, col] = np.nan
        else:
            y["q"][row, col] = np.nan
        got, info = _eval(h, desc, op, dtype, y, sign)
        assert (info.specialised, info.block, info.kernels_launched) == (info0.specialised, info0.block, info0.kernels_launched)
        for k in got:
            a, b = got[k], clean[k]
            assert not bool(_torch().isfinite(a[:, col]).all()), (op, what, k, "the poisoned sample came out finite")
            mask = _torch().ones(a.shape[1], dtype=_torch().bool, device=a.device)
            mask[col] = False
            # for the NaN angle this also pins that the fp32 program does not raise the gate flag (fmaxf drops NaN): a gated
            # generic rerun would not reproduce the program's bits in the clean columns
            assert _dev_equal(a[:, mask], b[:, mask]), (op, what, k, "a clean column changed")
    return info0


@pytest.mark.gpu
def test_non_finite_isolation_gpu(built, jit_cache, empty_cache, variant, monkeypatch):
    """Non-finite inputs in one sample on the specialised single-warp blocks, the specialised mixed CTA and the generic mixed CTA."""
    torch = _torch()
    variant(2)
    # generic mixed CTA (no cubin in this cache)
    mech, desc, h = _model("fast_classes")
    x = _inputs(mech, MIX_B, 17, np.float32, wext=True)
    x["_angle_row"] = _angle_row(mech)
    for dtype in (torch.float32, torch.float64):
        info = _isolation(h, desc, "rnea_wext", dtype, x, 40001)
        assert info.specialised == 0 and info.block == (512 if dtype == torch.float32 else 256)
    h.close()
    # specialised programs: small batch (single-warp blocks) and large batch in the mixed CTA
    monkeypatch.setenv("RBD_JIT_CACHE", jit_cache)
    mech, desc, h = _model("all_types")
    x = _inputs(mech, MIX_B, 17, np.float32)
    x["_angle_row"] = _angle_row(mech)
    h.precompile(C.RBD_F32, C.RBD_SPEC_DYNAMICS | C.RBD_SPEC_INVERSE_DYNAMICS | C.RBD_SPEC_MASS_MATRIX, load=True)
    small = {k: (a[:, :517].copy() if k != "_angle_row" else a) for k, a in x.items()}
    for op in ("aba", "rnea", "crba"):
        info = _isolation(h, desc, op, torch.float32, small, 300)
        assert info.specialised == 1 and info.block == 32
        info = _isolation(h, desc, op, torch.float32, x, 70001)
        assert info.specialised == 1 and info.block == (512 if op in SPEC_MIX["all_types"] else 32), (op, info.block)
    h.close()


# ------------------------------------------------------------------------------------------------ strides and alignment, all entry points
def _strided(fn, B, ld, shift):
    """fn(ld, shift) -> {name: [rows, ld] view}; the layouts (ld, 0) / (ld, 1)  against the dense call, bit for bit, padding untouched."""
    torch = _torch()
    dense = {k: t.clone() for k, t in fn(B, 0).items()}
    for l2, s2 in ((ld, 0), (B, shift), (ld, shift)):
        got = fn(l2, s2)
        for k, t in got.items():
            assert _dev_equal(t[:, :B], dense[k]), (k, l2, s2)
            assert bool(torch.isnan(t[:, B:]).all()), (k, l2, s2, "padding written")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float32", "float64"])
def test_strides_and_alignment_gpu(built, empty_cache, dtype_name):
    """Leading dimension > B and a base pointer one element past an aligned buffer on every batched entry point (the Julia shim
    hands over views): bit-identical to the dense call, padding untouched."""
    torch = _torch()
    dtype, npdt = getattr(torch, dtype_name), np.dtype(dtype_name)
    lib = C.load_library()
    mech = MODELS["all_types"]()
    cd = _with_contacts(mech, 3)
    desc = mech.flatten()
    h = C.ModelHandle(desc)
    dt = _dt_code(dtype)
    B, LD = 517, 531
    x = _inputs(mech, B, 18, npdt, wext=True)
    rng = np.random.default_rng(4)
    x["bar"] = rng.standard_normal((desc.nv, B))
    x["s"] = rng.standard_normal((3 * cd.npoints * cd.nhalfspaces, B)) * 1e-3
    nq, nv, nb, ns = desc.nq, desc.nv, desc.nb, 3 * cd.npoints * cd.nhalfspaces
    sign = np.ascontiguousarray(_sign(mech), np.int8)
    cst, keep = cd.c_struct()

    def mk(ld, shift):
        i = {k: _buf(a.shape[0], B, dtype, ld, shift, a) for k, a in x.items()}
        return i, (lambda rows: _buf(rows, B, dtype, ld, shift))

    def call(name):
        def run(ld, shift):
            i, out = mk(ld, shift)
            P = {k: _p(t) for k, t in i.items()}
            if name == "inverse_dynamics":
                o = {"tau": out(nv), "tau_w": out(nv)}
                _launch(lib.rbd_inverse_dynamics(h.ptr, dt, B, ld, P["q"], P["v"], P["vd"], None, _p(o["tau"]), None))
                _launch(lib.rbd_inverse_dynamics(h.ptr, dt, B, ld, P["q"], P["v"], P["vd"], P["wext"], _p(o["tau_w"]), None))
            elif name == "dynamics_bias":
                o = {"c": out(nv), "c_w": out(nv)}
                _launch(lib.rbd_dynamics_bias(h.ptr, dt, B, ld, P["q"], P["v"], None, _p(o["c"]), None))
                _launch(lib.rbd_dynamics_bias(h.ptr, dt, B, ld, P["q"], P["v"], P["wext"], _p(o["c_w"]), None))
            elif name == "mass_matrix":
                o = {"M": out(nv * nv), "L": out(nv * nv)}
                _launch(lib.rbd_mass_matrix(h.ptr, dt, B, ld, P["q"], _p(o["M"]), None))
                _launch(lib.rbd_mass_matrix_uplo(h.ptr, dt, B, ld, P["q"], _p(o["L"]), 1, None))
            elif name == "kinematics":
                rows = _kin_rows(desc)
                o = {k: out(rows[k]) for k in KR}
                ko = C.RbdKinematicsOut(*[_p(o[k]) for k in KR])
                _launch(lib.rbd_kinematics(h.ptr, dt, B, ld, P["q"], P["v"], sign.ctypes.data_as(ctypes.c_void_p), ctypes.byref(ko), None))
            elif name == "dynamics_result":
                o = {"vd": out(nv), "qd": out(nq), "M": out(nv * nv), "c": out(nv), "acc": out(6 * nb), "jw": out(6 * nb)}
                _launch(lib.rbd_dynamics_result(h.ptr, dt, B, ld, P["q"], P["v"], P["tau"], P["wext"], *[_p(o[k]) for k in o], None))
            elif name == "inverse_dynamics_bodies":
                o = {"acc": out(6 * nb), "jw": out(6 * nb)}
                _launch(lib.rbd_inverse_dynamics_bodies(h.ptr, dt, B, ld, P["q"], P["v"], P["vd"], P["wext"], _p(o["acc"]), _p(o["jw"]), None))
            elif name == "contact_dynamics":
                o = {"s": i["s"], "sd": out(ns), "w": out(6 * nb)}
                _launch(lib.rbd_contact_dynamics(h.ptr, dt, B, ld, P["q"], P["v"], ctypes.byref(cst), P["s"], _p(o["sd"]), _p(o["w"]), None))
            elif name == "dynamics_derivatives":
                o = {"vd": out(nv), "dq": out(nv * nv), "dv": out(nv * nv)}
                _launch(lib.rbd_dynamics_derivatives(h.ptr, dt, B, ld, P["q"], P["v"], P["tau"], *[_p(o[k]) for k in o], None))
            elif name == "dynamics_vjp":
                o = {"qt": out(nv), "qc": out(nq), "vb": out(nv), "tb": out(nv), "wb": out(6 * nb)}
                _launch(lib.rbd_dynamics_vjp(h.ptr, dt, B, ld, P["q"], P["v"], P["tau"], P["wext"], P["vd"], P["bar"],
                                             *[_p(o[k]) for k in o], None))
            else:
                o = {"qt": out(nv), "qc": out(nq), "vb": out(nv), "vdb": out(nv), "wb": out(6 * nb)}
                _launch(lib.rbd_inverse_dynamics_vjp(h.ptr, dt, B, ld, P["q"], P["v"], P["vd"], P["wext"], P["bar"],
                                                     *[_p(o[k]) for k in o], None))
            return o
        return run

    for name in ("inverse_dynamics", "dynamics_bias", "mass_matrix", "kinematics", "dynamics_result", "inverse_dynamics_bodies",
                 "contact_dynamics", "dynamics_derivatives", "dynamics_vjp", "inverse_dynamics_vjp"):
        _strided(call(name), B, LD, 1)
    # the dense call itself against the oracle on two of them (the others have their own suites)
    o = Oracle(desc)
    i, out = mk(B, 0)
    t = out(nv)
    _launch(lib.rbd_inverse_dynamics(h.ptr, dt, B, B, _p(i["q"]), _p(i["v"]), _p(i["vd"]), _p(i["wext"]), _p(t), None))
    assert rel_err(t.cpu().numpy(), o.inverse_dynamics(x["q"], x["v"], x["vd"], x["wext"])) < _tol("all_types", npdt)
    h.close()


@pytest.mark.gpu
def test_integrate_strides_and_alignment_gpu(built, empty_cache):
    """rbd_integrate / _schedule / _trajectory at B = 4096 (fp64): an odd leading dimension or a misaligned q / v switches the
    finishing step from the vectorised kernel to the scalar one -- per step 4 x (2 coordinate-map kernels + 1 dynamics kernel) +
    2 finishing kernels (vectorised + multi-DoF joints) for the dense layout, + 1 otherwise; the trajectory writes its blocks with
    leading dimension B, so its count does not change.  Results agree with the dense call and with the oracle."""
    torch = _torch()
    lib = C.load_library()
    mech, desc, h = _model("all_types")
    B, LD, nsteps, dtv = 4096, 4097, 2, 1e-3
    x = _inputs(mech, B, 19, np.float64)
    nq, nv = desc.nq, desc.nv
    o = Oracle(desc)
    sub = np.arange(0, B, 97)
    ref_q, ref_v = o.integrate(x["q"][:, sub], x["v"][:, sub], x["tau"][:, sub], dt=dtv, nsteps=nsteps)
    tau_sched = np.concatenate([x["tau"]] * nsteps, 0)          # [nsteps * nv, B]: step s at rows s * nv

    def run(kind, ld, shift):
        q = _buf(nq, B, torch.float64, ld, shift, x["q"])
        v = _buf(nv, B, torch.float64, ld, shift, x["v"])
        if kind == "integrate":
            tau = _buf(nv, B, torch.float64, ld, shift, x["tau"])
            info = _launch(lib.rbd_integrate(h.ptr, 1, B, ld, _p(q), _p(v), _p(tau), dtv, nsteps, None))
        else:
            tau = _buf(nsteps * nv, B, torch.float64, ld, shift, tau_sched)
            if kind == "schedule":
                info = _launch(lib.rbd_integrate_schedule(h.ptr, 1, B, ld, _p(q), _p(v), _p(tau), nv * ld, 0, dtv, nsteps, None))
            else:
                tq = torch.empty(((nsteps + 1) * nq, B), dtype=torch.float64, device="cuda")
                tv = torch.empty(((nsteps + 1) * nv, B), dtype=torch.float64, device="cuda")
                info = _launch(lib.rbd_integrate_trajectory(h.ptr, 1, B, ld, _p(q), _p(v), _p(tau), nv * ld, 0, dtv, nsteps,
                                                            _p(tq), _p(tv), None))
        assert bool(torch.isnan(q[:, B:]).all()) and bool(torch.isnan(v[:, B:]).all())
        return q[:, :B].cpu().numpy(), v[:, :B].cpu().numpy(), info.kernels_launched

    for kind in ("integrate", "schedule", "trajectory"):
        qd_, vd_, n_dense = run(kind, B, 0)
        assert n_dense == nsteps * 14, (kind, n_dense)
        assert config_distance(mech, qd_[:, sub], ref_q) < 1e-9 and rel_err(vd_[:, sub], ref_v) < 1e-9, kind
        for ld, shift in ((LD, 0), (B, 1), (LD, 1)):
            qs, vs, n = run(kind, ld, shift)
            assert n == nsteps * (14 if kind == "trajectory" else 13), (kind, ld, shift, n)
            assert np.abs(qs - qd_).max() < 1e-12 and np.abs(vs - vd_).max() < 1e-12 * max(1.0, np.abs(vd_).max()), (kind, ld, shift)
    h.close()


# --------------------------------------------------------------------------------------------------------------- dual numbers
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["all_types", "fast_classes"])
def test_dual_number_dynamics_general_gpu(built, name):
    """dynamics! on Dual{Float64,6}: the GENERAL instantiation (multi-DoF joints below the root) and the fast joint classes, values
    and partials against the oracle's dual-number run, tolerances of test_dual_number_dynamics_gpu."""
    torch = _torch()
    mech = MODELS[name]()
    o = Oracle(mech.flatten())
    B = 1000
    q, v, tau, _, _ = rand_inputs(mech, B, 4)
    Q, V, T = make_duals(mech, q, v, tau, 5)
    st = rbd.MechanismState(mech, 1, torch.float64)
    assert st.handle.info.general_path == (name == "all_types")
    out = torch.full((st.nv, B, 7), float("nan"), dtype=torch.float64, device="cuda")
    rbd.dynamics_dual_(out, st, torch.from_numpy(Q).cuda(), torch.from_numpy(V).cuda(), torch.from_numpy(T).cuda())
    torch.cuda.synchronize()
    info = rbd.launch_info()
    assert (info.specialised, info.block, info.kernels_launched) == (0, 32, 1)
    got = out.cpu().numpy()
    assert not np.isnan(got).any()
    n = 96
    ref = o.dynamics_dual6(Q[:, :n], V[:, :n], T[:, :n])
    assert np.abs(got[:, :n, 0] - ref[..., 0]).max() / np.abs(ref[..., 0]).max() < 1e-10
    assert np.abs(got[:, :n, 1:] - ref[..., 1:]).max() / np.abs(ref[..., 1:]).max() < 1e-8
