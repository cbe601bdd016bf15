"""Model-specialised kernels (csrc/rbd_sym.h, rbd_codegen.cpp, rbd_jit.cpp, rbd_spec.cpp).

CPU tier: the straight-line program the generator emits for a mechanism, compiled as plain C++ (tests/hostsim.SpecProgram),
against the oracle -- the same program text NVRTC compiles for the GPU, so its arithmetic is checked before any GPU time is
spent -- plus the NVRTC step itself (compilation needs no GPU).
GPU tier: the loaded kernels through the C ABI against the oracle, including the cases the specialised path treats
specially (angles beyond the fast sin / cos range, ragged batches, zero-torque default, q̇ output)."""
import ctypes
import os

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from oracle import Oracle
from rigidbodydynamics.jl_b200 import _cabi
from tests import hostsim
from tests.util import axis_aligned_tree, rand_inputs, randmech, rel_err


@pytest.mark.parametrize("name,floating", [("atlas", True), ("atlas", False), ("iiwa14", False), ("double_pendulum", False)])
@pytest.mark.parametrize("dtype,tol", [(np.float64, 1e-11), (np.float32, 2e-5)])
def test_specialised_program_matches_oracle_cpu(built, name, floating, dtype, tol):
    mech = rbd.load_model(name, floating=floating)
    desc = mech.flatten()
    q, v, tau, vd, _ = rand_inputs(mech, 24, 5)
    o = Oracle(desc)
    ref, ref_qd = o.dynamics(q, v, tau, want_qd=True)
    got, got_qd = hostsim.SpecProgram(desc, "aba", dtype, True, True).run(q, v, tau)
    assert rel_err(got, ref) < tol and np.abs(got_qd - ref_qd).max() < max(tol, 1e-6 if dtype == np.float32 else 0)
    got0 = hostsim.SpecProgram(desc, "aba", dtype, False, False).run(q, v)          # zero-torque default
    assert rel_err(got0, o.dynamics(q, v, None)) < tol
    assert rel_err(hostsim.SpecProgram(desc, "rnea", dtype, True).run(q, v, vd), o.inverse_dynamics(q, v, vd)) < tol
    assert rel_err(hostsim.SpecProgram(desc, "rnea", dtype, False).run(q, v), o.dynamics_bias(q, v)) < tol


def _mm_err(got, ref, nv, lower):
    G = np.asarray(got, float).reshape(nv, nv, -1); R = np.asarray(ref, float).reshape(nv, nv, -1)     # [column, row, sample]
    if not lower:
        return np.abs(G - R).max() / max(1.0, np.abs(R).max())
    keep = np.tril(np.ones((nv, nv), bool)).T           # row >= column  <->  [c, r] with r >= c
    assert np.isnan(G[~keep]).all()                     # the strict upper triangle is left untouched (NaN-filled by the caller)
    return np.abs(G[keep] - R[keep]).max() / max(1.0, np.abs(R).max())


@pytest.mark.parametrize("dtype,tol", [(np.float64, 1e-11), (np.float32, 2e-5)])
def test_specialised_mass_matrix_program_cpu(built, dtype, tol):
    """mass_matrix! traced on the mechanism (both triangles / lower only, mechanism_algorithms.jl:248-272): Atlas, the 7-DoF arm and
    random trees with every joint type against the oracle's composite-rigid-body algorithm."""
    for mech in (rbd.load_model("atlas", floating=True), rbd.load_model("iiwa14"), randmech(3, shuffle=True), axis_aligned_tree(1)):
        desc = mech.flatten()
        q = rand_inputs(mech, 5, 6)[0]
        ref = Oracle(desc).mass_matrix(q)
        for lower in (0, 1):
            prog = hostsim.SpecProgram(desc, "crba", dtype, has_in2=2 * lower, has_out1=False)
            got = prog.run(q, np.zeros((desc.nv, 5)), None, out0_rows=desc.nv * desc.nv)
            assert _mm_err(got, ref, desc.nv, lower) < tol


@pytest.mark.parametrize("dtype,tol", [(np.float64, 1e-10), (np.float32, 3e-5)])
def test_specialised_kinematics_programs_cpu(built, dtype, tol):
    """rbd_kinematics traced per mechanism, output subset and jacobian path: all outputs at once, and the subsets bench.py times,
    against the oracle."""
    KR = hostsim.KIN_ROWS
    for mech in (rbd.load_model("atlas", floating=True), randmech(2, shuffle=True), axis_aligned_tree(4)):
        desc = mech.flatten()
        o = Oracle(desc)
        q, v, _, _, _ = rand_inputs(mech, 4, 9)
        sign = np.random.default_rng(1).integers(-1, 2, desc.nb).astype(np.int8)
        ref = o.kinematics(q, v, sign)
        full = {"transforms": 12 * desc.nb, "com": 3, "ke": 1, "pe": 1, "momentum": 6, "mrb": 6, "A": 6 * desc.nv, "J": 6 * desc.nv}
        for sub, with_v in ((tuple(KR), True), (("J",), False), (("com", "ke", "pe", "momentum", "mrb"), True),
                            (("transforms", "com", "pe"), False), (("A",), False)):
            rows = [full[k] if k in sub else 0 for k in KR]
            hostsim.spec_kin(sum(1 << k for k, r in enumerate(rows) if r), sign, desc.nb)
            outs = hostsim.SpecProgram(desc, "kin", dtype, has_in2=1 if with_v else 0, has_out1=False).run_kin(q, v if with_v else None, rows)
            for k, name in enumerate(KR):
                if rows[k]:
                    assert rel_err(outs[k], ref[name]) < tol, (name, sub)


@pytest.mark.parametrize("seed", range(3))
def test_specialised_program_all_joint_types_cpu(built, seed):
    """The tracer resolves every joint kind / flag at generation time: random trees with all eight joint types and the
    axis-aligned trees that exercise the fast joint classes."""
    for mech in (randmech(seed, shuffle=seed % 2 == 1), axis_aligned_tree(seed)):
        desc = mech.flatten()
        q, v, tau, vd, _ = rand_inputs(mech, 9, seed)
        o = Oracle(desc)
        assert rel_err(hostsim.SpecProgram(desc, "aba", np.float64, True, False).run(q, v, tau), o.dynamics(q, v, tau)) < 1e-9
        assert rel_err(hostsim.SpecProgram(desc, "rnea", np.float64, True).run(q, v, vd), o.inverse_dynamics(q, v, vd)) < 1e-9


def test_specialised_program_is_smaller_than_the_generic_walk(built):
    """Folding the model into the program must pay: Atlas forward dynamics in well under the ~27.5 k instructions per sample
    of the generic kernel (VERDICT r1 target: <= 18 k), with floating-point work dominating."""
    _, st = hostsim.spec_source(rbd.load_model("atlas", floating=True).flatten(), "aba", np.float32, True, False, 1)
    fp = st["add"] + st["mul"] + st["div"] + 25 * st["sincos"]
    mem = st["load"] + st["store"] + st["sld"] + st["sst"]
    assert st["nodes_live"] < 14000 and fp > 3 * mem
    assert st["stash_rows"] == 213


def test_nvrtc_compiles_without_a_gpu(built, tmp_path, monkeypatch):
    """rbd_model_precompile(load = 0): generate + NVRTC-compile for sm_90a without a GPU, cubin lands in the cache."""
    monkeypatch.setenv("RBD_JIT_CACHE", str(tmp_path))
    mech = rbd.load_model("double_pendulum")
    h = _cabi.ModelHandle(mech.flatten())
    try:
        h.precompile(_cabi.RBD_F32, _cabi.RBD_SPEC_DYNAMICS | _cabi.RBD_SPEC_INVERSE_DYNAMICS, load=False)
    except _cabi.RbdError as e:
        pytest.skip(f"NVRTC not available here: {e}")
    finally:
        h.close()
    files = sorted(os.listdir(tmp_path))
    assert len(files) == 2 and all(f.endswith(".cubin") for f in files)
    assert any("_aba_f32_" in f for f in files) and any("_rnea_f32_" in f for f in files)
    # it is a real sm_90a ELF holding the kernel (the low byte of e_flags is the SM version)
    blob = open(tmp_path / files[0], "rb").read()
    assert blob[:4] == b"\x7fELF" and b"rbd_jit_smem" in blob
    assert blob[48] == 90


# ---------------------------------------------------------------------------------------------------------------- GPU tier
# fp32 tolerance of the 512-sample checks below.  tests/test_gpu_parity.py holds fp32 to 2e-5 on its 193 samples; over 512 random
# Atlas / Valkyrie states the worst sample reaches 2.4e-5 -- on the specialised AND on the generic kernels alike (RBD_JIT=0: 2.42e-5)
# -- so this is the arithmetic's conditioning (light distal links), not the code path.
FP32_TOL = 1e-4
def _gpu_dyn(mech, q, v, tau, dtype, want_qd=False):
    import torch
    st = rbd.MechanismState(mech, q.shape[1], dtype)
    st.q.copy_(torch.from_numpy(q).to(dtype)); st.v.copy_(torch.from_numpy(v).to(dtype))
    t = None if tau is None else torch.from_numpy(tau).to(dtype).cuda()
    res = rbd.DynamicsResult(mech, q.shape[1], dtype)
    rbd.dynamics_(res, st, t, want_qd=want_qd)
    torch.cuda.synchronize()
    info = rbd.launch_info()
    return res.vd.double().cpu().numpy(), res.qd.double().cpu().numpy(), info


@pytest.mark.gpu
@pytest.mark.parametrize("name,floating,B", [("atlas", True, 1 << 16), ("atlas", True, 40001), ("iiwa14", False, 1 << 15),
                                             ("valkyrie", True, 33000)])
def test_specialised_kernels_match_oracle_gpu(built, name, floating, B):
    """Large enough batches run the NVRTC kernels (launch_info().specialised); a strided sub-sample against the oracle; every
    entry of the batch finite; with and without torques / q̇."""
    import torch
    mech = rbd.load_model(name, floating=floating)
    base = rand_inputs(mech, 512, 11)
    reps = -(-B // 512)
    q, v, tau, vd = (np.tile(a, (1, reps))[:, :B].copy() for a in base[:4])
    o = Oracle(mech.flatten())
    got, got_qd, info = _gpu_dyn(mech, q, v, tau, torch.float32, want_qd=True)
    assert info.specialised == 1
    ref, ref_qd = o.dynamics(q[:, :512], v[:, :512], tau[:, :512], want_qd=True)
    assert rel_err(got[:, :512], ref) < FP32_TOL and np.abs(got_qd[:, :512] - ref_qd).max() < 1e-5
    assert np.array_equal(got[:, :512 * (B // 512)].reshape(got.shape[0], -1, 512), np.broadcast_to(got[:, None, :512], (got.shape[0], B // 512, 512)))
    got0, _, info0 = _gpu_dyn(mech, q, v, None, torch.float32)
    assert info0.specialised == 1
    assert rel_err(got0[:, :512], o.dynamics(q[:, :512], v[:, :512], None)) < FP32_TOL
    st = rbd.MechanismState(mech, B, torch.float32)
    st.q.copy_(torch.from_numpy(q).float()); st.v.copy_(torch.from_numpy(v).float())
    out = torch.empty((st.nv, B), dtype=torch.float32, device="cuda")
    rbd.inverse_dynamics_(out, st, torch.from_numpy(vd).float().cuda())
    assert rbd.launch_info().specialised == 1
    assert rel_err(out[:, :512].double().cpu().numpy(), o.inverse_dynamics(q[:, :512], v[:, :512], vd[:, :512])) < FP32_TOL
    rbd.dynamics_bias_(out, st)
    assert rel_err(out[:, :512].double().cpu().numpy(), o.dynamics_bias(q[:, :512], v[:, :512])) < FP32_TOL


@pytest.mark.gpu
def test_mixed_cta_with_l2_stash_matches_shared_memory_blocks_gpu(built, monkeypatch):
    """Atlas at 2^19 samples is large enough for the mixed CTA (warps whose stash does not fit shared memory keep it in L2).
    Forced either way, forward and inverse dynamics must be bit-identical and match the oracle."""
    import torch
    mech = rbd.load_model("atlas", floating=True)
    B = 1 << 19
    base = rand_inputs(mech, 512, 13)
    q, v, tau, vd = (np.tile(a, (1, B // 512)) for a in base[:4])
    o = Oracle(mech.flatten())
    st = rbd.MechanismState(mech, B, torch.float32)
    st.q.copy_(torch.from_numpy(q).float()); st.v.copy_(torch.from_numpy(v).float())
    tau_d, vd_d = torch.from_numpy(tau).float().cuda(), torch.from_numpy(vd).float().cuda()
    outs = {}
    for variant in ("1", "2"):
        monkeypatch.setenv("RBD_JIT_VARIANT", variant)
        res = rbd.DynamicsResult(mech, B, torch.float32)
        rbd.dynamics_(res, st, tau_d, want_qd=False)
        info = rbd.launch_info()
        assert info.specialised == 1 and info.block == (32 if variant == "1" else 512), (variant, info.block)
        tau_out = torch.empty((st.nv, B), dtype=torch.float32, device="cuda")
        rbd.inverse_dynamics_(tau_out, st, vd_d)
        assert rbd.launch_info().block == (32 if variant == "1" else 512)
        torch.cuda.synchronize()
        outs[variant] = (res.vd.clone(), tau_out)
    assert torch.equal(outs["1"][0], outs["2"][0]) and torch.equal(outs["1"][1], outs["2"][1])
    got = outs["2"][0].double().cpu().numpy()
    assert rel_err(got[:, :512], o.dynamics(q[:, :512], v[:, :512], tau[:, :512])) < FP32_TOL
    assert np.array_equal(got.reshape(got.shape[0], -1, 512), np.broadcast_to(got[:, None, :512], (got.shape[0], B // 512, 512)))
    assert rel_err(outs["2"][1][:, :512].double().cpu().numpy(), o.inverse_dynamics(q[:, :512], v[:, :512], vd[:, :512])) < FP32_TOL


@pytest.mark.gpu
@pytest.mark.parametrize("name,floating,B", [("atlas", True, 40001), ("iiwa14", False, 1 << 15)])
def test_specialised_mass_matrix_gpu(built, name, floating, B):
    """mass_matrix! on the model-specialised kernel (batch above the compile threshold), both triangles and lower only, fp32 and
    fp64 (the fp64 Atlas program is above the size limit and runs the generic kernel: same check), plus an angle beyond the fast
    sin / cos range, which must come out of the gated generic kernel."""
    import torch
    mech = rbd.load_model(name, floating=floating)
    o = Oracle(mech.flatten())
    q = rand_inputs(mech, B, 3)[0]
    q[-1, 7] = 3.0e4                     # exactly representable in fp32
    idx = np.array([0, 7, 31, 32, B // 2, B - 1])
    ref = o.mass_matrix(q[:, idx])
    nv = mech.num_velocities()
    for dtype, tol in ((torch.float32, 2e-5), (torch.float64, 1e-11)):
        st = rbd.MechanismState(mech, B, dtype)
        st.q.copy_(torch.from_numpy(q).to(dtype))
        for uplo in ("F", "L"):
            M = torch.full((nv * nv, B), float("nan"), dtype=dtype, device="cuda")
            rbd.mass_matrix_(M, st, uplo="L" if uplo == "L" else "full")
            torch.cuda.synchronize()
            if dtype == torch.float32:
                assert rbd.launch_info().specialised == 1
            assert _mm_err(M[:, idx].double().cpu().numpy(), ref, nv, uplo == "L") < tol, (name, dtype, uplo)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [40001])
def test_specialised_kinematics_gpu(built, B):
    """rbd_kinematics on the model-specialised kernels (batch above the compile threshold): output subsets with and without a
    jacobian path, two different paths through the same handle, fp32 and fp64, one angle beyond the fast sin / cos range."""
    import torch
    mech = rbd.load_model("atlas", floating=True)
    o = Oracle(mech.flatten())
    q, v, _, _, _ = rand_inputs(mech, B, 6)
    q[-1, 11] = 2.0e4
    idx = np.array([0, 11, 31, 32, B // 3, B - 1])
    p1 = rbd.path(mech, mech.findbody("r_foot"), mech.findbody("l_hand"))
    p2 = rbd.path(mech, mech.findbody("l_foot"), mech.findbody("head"))
    nb, nv = len(mech.joints), mech.num_velocities()
    for dtype, tol in ((torch.float32, 3e-5), (torch.float64, 1e-9)):
        st = rbd.MechanismState(mech, B, dtype)
        st.q.copy_(torch.from_numpy(q).to(dtype)); st.v.copy_(torch.from_numpy(v).to(dtype))
        for pth, names in ((p1, ("geometric_jacobian",)), (p2, ("geometric_jacobian", "center_of_mass")),
                           (None, ("center_of_mass", "kinetic_energy", "gravitational_potential_energy", "momentum", "momentum_rate_bias")),
                           (p1, ("transforms_to_root", "geometric_jacobian", "momentum")), (None, ("momentum_matrix", "center_of_mass")),
                           (None, ("momentum_matrix",))):      # alone: the two-sweep body-frame program
            rows = {"transforms_to_root": 12 * nb, "center_of_mass": 3, "kinetic_energy": 1, "gravitational_potential_energy": 1,
                    "momentum": 6, "momentum_rate_bias": 6, "momentum_matrix": 6 * nv, "geometric_jacobian": 6 * nv}
            outs = {k: torch.full((rows[k], B), float("nan"), dtype=dtype, device="cuda") for k in names}
            rbd.kinematics_(st, pth, **outs)
            torch.cuda.synchronize()
            assert rbd.launch_info().specialised == 1, names
            sign = None if pth is None else pth.sign
            ref = o.kinematics(q[:, idx], v[:, idx], sign)
            short = {"transforms_to_root": "transforms", "center_of_mass": "com", "kinetic_energy": "ke", "gravitational_potential_energy": "pe",
                     "momentum": "momentum", "momentum_rate_bias": "mrb", "momentum_matrix": "A", "geometric_jacobian": "J"}
            for k in names:
                assert rel_err(outs[k][:, idx].double().cpu().numpy(), ref[short[k]]) < tol, (dtype, k, names)


@pytest.mark.gpu
def test_angles_beyond_the_fast_range_gpu(built):
    """The specialised fp32 program has no slow sin / cos path: a sample with |q| > 1e4 rad raises a device flag and the generic
    kernel queued behind redoes the batch with the library path.  Results must match the oracle either way."""
    import torch
    mech = rbd.load_model("atlas", floating=True)
    B = 1 << 16
    q, v, tau, _, _ = rand_inputs(mech, 256, 3)
    q, v, tau = (np.tile(a, (1, B // 256)) for a in (q, v, tau))
    o = Oracle(mech.flatten())
    got, _, info = _gpu_dyn(mech, q, v, tau, torch.float32)
    assert info.specialised == 1 and rel_err(got[:, :256], o.dynamics(q[:, :256], v[:, :256], tau[:, :256])) < 2e-5
    q2 = q.copy()
    q2[9, 77] = 31415.9265 * 2 + 0.25          # one joint angle of one sample far outside +-1e4
    q2[20, 40000] = -2.5e5
    q2 = q2.astype(np.float32).astype(np.float64)      # what the fp32 kernels see
    got2, _, _ = _gpu_dyn(mech, q2, v, tau, torch.float32)
    idx = [77, 40000, 5, 40001]
    ref2 = o.dynamics(q2[:, idx], v[:, idx], tau[:, idx])
    assert rel_err(got2[:, idx], ref2) < 5e-5          # sin / cos of a 2.5e5 rad fp32 angle: one ulp of the angle is 0.016 rad
    assert np.isfinite(got2).all()


@pytest.mark.gpu
def test_small_batches_use_cached_cubins_only_gpu(built, tmp_path, monkeypatch):
    """Below RBD_JIT_MIN_BATCH nothing is compiled on the fly: an unseen mechanism runs the generic kernels, the same mechanism
    after rbd_model_precompile runs the specialised ones, with equal results (same tolerance class)."""
    import torch
    monkeypatch.setenv("RBD_JIT_CACHE", str(tmp_path))
    mech = axis_aligned_tree(7, n=12)
    q, v, tau, _, _ = rand_inputs(mech, 300, 7)
    ref = Oracle(mech.flatten()).dynamics(q, v, tau)
    got, _, info = _gpu_dyn(mech, q, v, tau, torch.float64)
    assert info.specialised == 0 and rel_err(got, ref) < 1e-9
    rbd.MechanismState(mech, 1, torch.float64).handle.precompile(_cabi.RBD_F64, _cabi.RBD_SPEC_DYNAMICS, load=True)
    got2, _, info2 = _gpu_dyn(mech, q, v, tau, torch.float64)
    assert info2.specialised == 1 and rel_err(got2, ref) < 1e-9
