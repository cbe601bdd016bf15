"""Sums planned as FMA chains (csrc/rbd_codegen.cpp, Emitter::plan_chains) and the gated reciprocal of the fp32 programs.

CPU tier: the planned programs against the oracle, with and without a length cap; no add / sub of the Atlas program is left with
two single-use products; the folded and straight-line programs stay bit-identical and Atlas still folds; RBD_JIT_FMA_CHAIN=0 emits
exactly the text of the planning before the chains (pinned by hash), and the default plans chains for forward dynamics and
kinematics only.  GPU tier: the kernel equals its CPU flavour bit for bit in both kernel shapes, chains on and off; a NaN sample
stays in its own column; a sub-normal and a huge divisor raise the range gate, and the generic kernel's results come back (the
CPU tier checks that those models' divisors are what the tests say)."""
import hashlib
import re

import numpy as np
import pytest
import torch

import rigidbodydynamics.jl_b200 as rbd
from oracle import Oracle
from tests import hostsim
from tests.test_fold import _check_bit_identical, _source, shim  # noqa: F401  (shim: the fold shim fixture)
from tests.test_reg_stash import _models
from tests.util import axis_aligned_tree, rand_inputs, rel_err

MODELS = dict(_models())
MODELS["axis_aligned"] = axis_aligned_tree(3)
TOL = {np.float64: 1e-10, np.float32: 3e-5}


@pytest.mark.parametrize("cap", ["0", "4"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("name", sorted(MODELS))
def test_chains_match_oracle_cpu(built, monkeypatch, name, dtype, cap):
    monkeypatch.setenv("RBD_JIT_FMA_CHAIN", "1")                # every program, not only the default ones
    monkeypatch.setenv("RBD_JIT_FMA_CAP", cap)
    mech = MODELS[name]
    desc = mech.flatten()
    o = Oracle(desc)
    q, v, tau, vd, _ = rand_inputs(mech, 6, 11)
    tol = TOL[dtype]
    got, got_qd = hostsim.SpecProgram(desc, "aba", dtype, True, True).run(q, v, tau)
    ref, ref_qd = o.dynamics(q, v, tau, want_qd=True)
    assert rel_err(got, ref) < tol and np.abs(got_qd - ref_qd).max() < max(tol, 1e-6 if dtype == np.float32 else 0)
    assert rel_err(hostsim.SpecProgram(desc, "rnea", dtype, True).run(q, v, vd), o.inverse_dynamics(q, v, vd)) < tol
    M = hostsim.SpecProgram(desc, "crba", dtype, 0, False).run(q, np.zeros_like(v), None, out0_rows=desc.nv * desc.nv)
    assert rel_err(M.reshape(desc.nv * desc.nv, -1), np.asarray(o.mass_matrix(q)).reshape(desc.nv * desc.nv, -1)) < tol
    rows = [0, 3, 1, 1, 6, 6, 0, 0]                            # com, ke, pe, momentum, mrb
    hostsim.spec_kin(sum(1 << k for k, r in enumerate(rows) if r))
    outs = hostsim.SpecProgram(desc, "kin", dtype, has_in2=1, has_out1=False).run_kin(q, v, rows)
    ref_k = o.kinematics(q, v)
    for k, r in enumerate(rows):
        if r:
            assert rel_err(outs[k], ref_k[hostsim.KIN_ROWS[k]]) < tol, hostsim.KIN_ROWS[k]


def _atlas_src(monkeypatch, algo="aba", chain=None, fold_flavor=3):
    monkeypatch.delenv("RBD_JIT_REG_ROWS", raising=False)
    monkeypatch.delenv("RBD_JIT_FMA_CAP", raising=False)
    if chain is None:
        monkeypatch.delenv("RBD_JIT_FMA_CHAIN", raising=False)
    else:
        monkeypatch.setenv("RBD_JIT_FMA_CHAIN", chain)
    desc = rbd.load_model("atlas", floating=True).flatten()
    return hostsim.spec_source(desc, algo, np.float32, True, False, fold_flavor)[0]


def test_no_add_of_two_single_use_products_cpu(built, monkeypatch):
    """Every product used once by a sum is an FMA of its chain: no emitted add / sub has two such operands."""
    src = _atlas_src(monkeypatch)
    muls = {m.group(1) for m in re.finditer(r"const rbd_v (\w+) = RBD_MUL\(", src)}
    uses = {n: len(re.findall(rf"\b{n}\b", src)) - 1 for n in muls}
    single = {n for n, k in uses.items() if k == 1}
    for a, b in re.findall(r"RBD_(?:ADD|SUB)\((\w+), (\w+)\)", src):
        assert not (a in single and b in single), (a, b)
    assert "RBD_ADD(RBD_MUL(" not in src and "RBD_SUB(RBD_MUL(" not in src
    assert src.count("RBD_FMA(") > src.count("RBD_ADD(")


@pytest.mark.parametrize("cap", ["0", "4"])
@pytest.mark.parametrize("name", ["atlas", "valkyrie", "mirrored"])
def test_folded_equals_straight_line_cpu(shim, monkeypatch, name, cap):  # noqa: F811
    monkeypatch.delenv("RBD_JIT_FMA_CHAIN", raising=False)
    monkeypatch.setenv("RBD_JIT_FMA_CAP", cap)
    _check_bit_identical(shim, MODELS[name], np.float32, True)


@pytest.mark.parametrize("cap", ["0", "4"])
def test_atlas_still_folds_cpu(shim, monkeypatch, cap):  # noqa: F811
    monkeypatch.delenv("RBD_JIT_FMA_CHAIN", raising=False)
    monkeypatch.setenv("RBD_JIT_FMA_CAP", cap)
    _, st = _source(shim, rbd.load_model("atlas", floating=True).flatten(), np.float32, True)
    assert st["fold_loops"] == 6 and st["fold_bodies"] == 39


def test_switch_off_keeps_the_single_product_planning_cpu(built, monkeypatch):
    """RBD_JIT_FMA_CHAIN=0: one product contracted per add / sub, never a nested chain; chains take out statements."""
    off = _atlas_src(monkeypatch, chain="0")
    on = _atlas_src(monkeypatch)
    assert not re.search(r"RBD_F\w*\([^;]*RBD_F", off)
    assert re.search(r"RBD_FMA\([^;]*RBD_FMA\(", on)
    stmts = lambda s: len(re.findall(r"^const rbd_v ", s, re.M))
    assert stmts(on) < 0.8 * stmts(off)
    for algo in ("rnea", "crba"):
        assert stmts(_atlas_src(monkeypatch, algo, chain="1")) < stmts(_atlas_src(monkeypatch, algo, chain="0"))


# sha256 of the source text the generator emitted before sums were planned as chains (RBD_JIT_FMA_CHAIN=0 must reproduce it):
# (model, algorithm, dtype, flavour: 0 = CPU translation unit, 3 = NVRTC translation unit)
PLANNING_BEFORE_CHAINS = {
    ("atlas", "aba", np.float32, 3): "9531472fc11a002cbfcb504c5245f8cccbe68e2305107b2903d0f3375dfe41d8",
    ("atlas", "aba", np.float32, 0): "49053ec3c3cf3685bc25b20952e9f0c60504c31e90503a91539e5bfc854c9f05",
    ("atlas", "rnea", np.float32, 3): "a8fdf6c1b6098e5eeb7aa40e8d496bafd5ceb3dfb6979afa5c124bac84cf9894",
    ("atlas", "crba", np.float32, 3): "892add609b29c7fc650085518dd99bd0eddc74c828d457e25fd369d823ba107d",
    ("atlas", "aba", np.float64, 0): "6bc0f4e8eaecccabcf5fb47ba6c0919c9cc589c50b2f6b1860cb7a761d5a8707",
    ("iiwa14", "crba", np.float64, 0): "be65f55f5273a20db609f8d83b30510121923f05eea7f700a32584c4170319ba",
    ("iiwa14", "aba", np.float32, 3): "b474bce148df69a21fb570902d9bddcfbb0d982b9fcd5bec493f91dbe9f4d18a",
    ("valkyrie", "aba", np.float32, 3): "ebcf888ee9d90403583165418db529c793af1449176cabf805bea7901d91599f",
}


@pytest.mark.parametrize("case", list(PLANNING_BEFORE_CHAINS), ids=lambda c: f"{c[0]}-{c[1]}-{np.dtype(c[2]).name}-{c[3]}")
def test_switch_off_reproduces_the_text_before_chains_cpu(built, monkeypatch, case):
    name, algo, dtype, flavor = case
    for k in ("RBD_JIT_REG_ROWS", "RBD_JIT_FMA_CAP", "RBD_JIT_RCP", "RBD_JIT_TRIG", "RBD_JIT_SMEM_BLOCKS", "RBD_JIT_SPLIT"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("RBD_JIT_FMA_CHAIN", "0")
    desc = rbd.load_model(name, floating=name != "iiwa14").flatten()
    src = hostsim.spec_source(desc, algo, dtype, True, False, flavor)[0]
    assert hashlib.sha256(src.encode()).hexdigest() == PLANNING_BEFORE_CHAINS[case]


def test_default_chains_forward_dynamics_and_kinematics_only_cpu(built, monkeypatch):
    """Without RBD_JIT_FMA_CHAIN the chains are planned where they measured faster (forward dynamics, kinematics); inverse
    dynamics and the mass matrix keep the single-product planning unless RBD_JIT_FMA_CHAIN=1."""
    desc = rbd.load_model("atlas", floating=True).flatten()
    nested = lambda src: re.search(r"RBD_FMA\([^;]*RBD_FMA\(", src) is not None
    for k in ("RBD_JIT_FMA_CHAIN", "RBD_JIT_FMA_CAP", "RBD_JIT_REG_ROWS"):
        monkeypatch.delenv(k, raising=False)
    assert nested(hostsim.spec_source(desc, "aba", np.float32, True, False, 3)[0])
    hostsim.spec_kin(1 << 4)                                   # momentum
    assert nested(hostsim.spec_source(desc, "kin", np.float32, True, False, 3)[0])
    for algo in ("rnea", "crba"):
        assert not nested(hostsim.spec_source(desc, algo, np.float32, True, False, 3)[0])
    monkeypatch.setenv("RBD_JIT_FMA_CHAIN", "1")
    for algo in ("rnea", "crba"):
        assert nested(hostsim.spec_source(desc, algo, np.float32, True, False, 3)[0])


def test_reciprocal_switch_cpu(built, monkeypatch):
    """The fp32 translation unit keeps the library reciprocal only under RBD_JIT_RCP=0; fp64 never defines it."""
    assert "RBD_SPEC_RCP_LIB" not in _atlas_src(monkeypatch)
    monkeypatch.setenv("RBD_JIT_RCP", "0")
    assert "#define RBD_SPEC_RCP_LIB 1" in _atlas_src(monkeypatch)
    desc = rbd.load_model("atlas", floating=True).flatten()
    assert "RBD_SPEC_RCP_LIB" not in hostsim.spec_source(desc, "aba", np.float64, True, False, 3)[0]


# ---------------------------------------------------------------------------------------------------------------- GPU tier
def _dyn_gpu(chain, variant, q, v, tau, monkeypatch):
    monkeypatch.delenv("RBD_JIT_REG_ROWS", raising=False)
    monkeypatch.delenv("RBD_JIT_FMA_CAP", raising=False)
    monkeypatch.setenv("RBD_JIT_FMA_CHAIN", chain)
    monkeypatch.setenv("RBD_JIT_VARIANT", variant)
    mech = rbd.load_model("atlas", floating=True)          # a fresh handle: generated and loaded under this setting
    B = q.shape[1]
    st = rbd.MechanismState(mech, B, torch.float32)
    st.q.copy_(q)
    st.v.copy_(v)
    res = rbd.DynamicsResult(mech, B, torch.float32)
    rbd.dynamics_(res, st, tau, want_qd=True)
    torch.cuda.synchronize()
    return res.vd.clone(), res.qd.clone(), rbd.launch_info()


def _atlas_inputs(B):
    st = rbd.MechanismState(rbd.load_model("atlas", floating=True), B, torch.float32)
    rbd.rand_(st, np.random.default_rng(29))
    tau = torch.rand((st.nv, B), dtype=torch.float32, device="cuda", generator=torch.Generator(device="cuda").manual_seed(7))
    return st.q.clone(), st.v.clone(), tau


@pytest.mark.gpu
def test_kernel_equals_cpu_flavour_gpu(built, monkeypatch, tmp_path):
    """Atlas fp32 forward dynamics, chains on and off, shared-memory blocks and the mixed CTA: the first 64 samples equal the CPU
    flavour of the same program bit for bit (the gated reciprocal is the correctly rounded 1 / x)."""
    monkeypatch.setenv("RBD_JIT_CACHE", str(tmp_path))
    q, v, tau = _atlas_inputs(1 << 17)
    desc = rbd.load_model("atlas", floating=True).flatten()
    n = 64
    qc, vc, tc = (x[:, :n].double().cpu().numpy() for x in (q, v, tau))
    for chain in ("0", "1"):
        monkeypatch.setenv("RBD_JIT_FMA_CHAIN", chain)
        monkeypatch.delenv("RBD_JIT_FMA_CAP", raising=False)
        ref, ref_qd = hostsim.SpecProgram(desc, "aba", np.float32, True, True).run(qc, vc, tc)
        for variant in ("1", "2"):
            vd, qd, info = _dyn_gpu(chain, variant, q, v, tau, monkeypatch)
            assert info.specialised == 1, (chain, variant, info)
            assert (info.block == 32) == (variant == "1"), (chain, variant, info.block)     # variant 2: the mixed CTA
            assert np.array_equal(vd[:, :n].cpu().numpy(), ref), (chain, variant)
            assert np.array_equal(qd[:, :n].cpu().numpy(), ref_qd), (chain, variant)


@pytest.mark.gpu
def test_nan_sample_stays_in_its_column_gpu(built, monkeypatch, tmp_path):
    """A NaN velocity in one sample: that column is NaN, every other equals the clean run, and the launch shape is the clean
    run's (a NaN divisor or angle does not raise the range gate)."""
    monkeypatch.setenv("RBD_JIT_CACHE", str(tmp_path))
    q, v, tau = _atlas_inputs(1 << 16)
    vd0, _, info0 = _dyn_gpu("1", "1", q, v, tau, monkeypatch)
    v[:, 123] = float("nan")
    q[7, 124] = float("nan")
    vd1, _, info1 = _dyn_gpu("1", "1", q, v, tau, monkeypatch)
    assert (info0.specialised, info0.kernels_launched, info0.grid, info0.block) == \
        (info1.specialised, info1.kernels_launched, info1.grid, info1.block)
    assert torch.isnan(vd1[:, 123]).any() and torch.isnan(vd1[:, 124]).any()
    keep = torch.ones(vd0.shape[1], dtype=torch.bool, device=vd0.device)
    keep[123:125] = False
    assert torch.equal(vd1[:, keep], vd0[:, keep])


def _pendulum(I1, m2):
    """Two links on parallel y axes, no gravity: link 1 with moment I1 about its axis and no mass, link 2 a point mass m2 one unit
    below joint 2, which sits one unit below joint 1.  The divisor of joint 1 is D1 = I1 + m2 sin^2(q2); at q2 = 0 every term of m2
    cancels exactly (powers of two), so D1 = I1.  Joint 2's divisor m2 is a model constant and folds into the program."""
    y = np.array([0.0, 1.0, 0.0])
    mech = rbd.Mechanism(rbd.RigidBody("world"), gravity=(0, 0, 0))
    b1 = rbd.RigidBody("l1", rbd.SpatialInertia(I1 * np.outer(y, y), None, 0.0, com=[0, 0, 0]))
    mech.attach(mech.root_body, b1, rbd.Joint("j1", rbd.Revolute(y)))
    b2 = rbd.RigidBody("l2", rbd.SpatialInertia(None, None, m2, com=[0, 0, -1.0], moment_about_com=np.zeros((3, 3))))
    mech.attach(b1, b2, rbd.Joint("j2", rbd.Revolute(y)), joint_pose=rbd.Transform3D(None, [0, 0, -1.0]))
    return mech


def _pendulum_gpu(I1, m2, q, v, tau, cache):
    """(v̇, launch info) of fp32 forward dynamics on a fresh handle with cubin cache `cache`."""
    mech = _pendulum(I1, m2)
    B = q.shape[1]
    st = rbd.MechanismState(mech, B, torch.float32)
    st.q.copy_(q)
    st.v.copy_(v)
    res = rbd.DynamicsResult(mech, B, torch.float32)
    rbd.dynamics_(res, st, tau)
    torch.cuda.synchronize()
    return res.vd.clone(), rbd.launch_info()


def _gate_inputs(B, tau1, tau2_scale, dev):
    """q = 0 (every rotation the identity, so the m2 terms of D1 cancel exactly in any precision), v = 0, tau = (tau1,
    tau2_scale * U[0, 1))."""
    g = torch.Generator(device=dev).manual_seed(13)
    q = torch.zeros((2, B), dtype=torch.float32, device=dev)
    v = torch.zeros((2, B), dtype=torch.float32, device=dev)
    tau = torch.empty((2, B), dtype=torch.float32, device=dev)
    tau[0] = tau1
    tau[1] = torch.rand(B, generator=g, device=dev) * tau2_scale
    return q, v, tau


# (I1, m2, tau1, tau2 scale): D1 sub-normal (1.5 * 2^-127) with v̇1 = tau1 / D1 = 1/12; D1 = 2^127 with v̇1 = tau1 / D1 = 2^-128
GATE_CASES = {"subnormal": (1.5 * 2.0 ** -127, 2.0 ** -60, 2.0 ** -130, 0.0), "huge": (2.0 ** 127, 1.0, 0.5, 0.0)}


@pytest.mark.parametrize("case", sorted(GATE_CASES))
def test_gate_models_cpu(built, monkeypatch, case):
    """The programs of the gate tests: joint 1's divisor is q-dependent (a reciprocal of the program, not a literal), and with
    1 / x (the CPU flavour) v̇1 = tau1 / D1 exactly as intended, so D1 really is 1.5 * 2^-127 (resp. 2^127)."""
    monkeypatch.delenv("RBD_JIT_FMA_CHAIN", raising=False)
    I1, m2, tau1, scale = GATE_CASES[case]
    desc = _pendulum(I1, m2).flatten()
    assert "RBD_RCP(" in hostsim.spec_source(desc, "aba", np.float32, True, False, 3)[0]
    q, v, tau = (x.numpy() for x in _gate_inputs(64, tau1, scale, "cpu"))
    vd = hostsim.SpecProgram(desc, "aba", np.float32, True, False).run(q, v, tau)
    assert np.isfinite(vd).all()
    assert (vd[0] == np.float32(tau1 / I1)).all()


def _gate_case(monkeypatch, tmp_path, case):
    """The specialised program (a batch large enough to compile it) and the generic kernel alone (a batch below the compile
    threshold, empty cache) on the same samples, and the fp64 oracle."""
    for k in ("RBD_JIT_FMA_CHAIN", "RBD_JIT_FMA_CAP", "RBD_JIT_RCP", "RBD_JIT_REG_ROWS", "RBD_JIT_VARIANT"):
        monkeypatch.delenv(k, raising=False)
    I1, m2, tau1, scale = GATE_CASES[case]
    B, n = 1 << 16, 1000
    q, v, tau = _gate_inputs(B, tau1, scale, "cuda")
    monkeypatch.setenv("RBD_JIT_CACHE", str(tmp_path / "jit"))
    vd, info = _pendulum_gpu(I1, m2, q, v, tau, tmp_path / "jit")
    assert (info.specialised, info.kernels_launched) == (1, 2), info      # the program, and the generic kernel gated behind it
    (tmp_path / "none").mkdir()
    monkeypatch.setenv("RBD_JIT_CACHE", str(tmp_path / "none"))
    ref, info2 = _pendulum_gpu(I1, m2, q[:, :n].contiguous(), v[:, :n].contiguous(), tau[:, :n].contiguous(), tmp_path / "none")
    assert info2.specialised == 0
    # the oracle's ABA: its CRBA + Cholesky cannot factor this mass matrix (second pivot I1 / 4 against entries of 2^-60)
    ora = Oracle(_pendulum(I1, m2).flatten()).dynamics(*(x[:, :n].double().cpu().numpy() for x in (q, v, tau)), algo="aba")
    return vd[:, :n], ref, ora, tau1 / I1


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(GATE_CASES))
def test_divisor_out_of_range_raises_the_gate_gpu(built, monkeypatch, tmp_path, case):
    """A divisor outside the fast reciprocal's range raises the gate, and v̇ is the generic kernel's, bit for bit, finite and
    equal to the oracle's.  Without the gate the branch-free reciprocal would show: for the sub-normal D1 its approximation is
    infinite and v̇1 NaN; for D1 = 2^127 it flushes 1 / D1 = 2^-127 to zero and v̇1 = 0 instead of the sub-normal 2^-128."""
    vd, ref, ora, vd1 = _gate_case(monkeypatch, tmp_path, case)
    assert np.isfinite(ora).all() and torch.isfinite(vd).all()
    assert torch.equal(vd.view(torch.int32), ref.view(torch.int32))
    assert (vd[0] == np.float32(vd1)).all() and vd1 != 0
    assert rel_err(vd.double().cpu().numpy(), ora) < 1e-5
