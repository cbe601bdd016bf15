"""Trig cache of the model-specialised fp32 forward-dynamics program (csrc/rbd_codegen.cpp, spec_trig).

Pass 1 of the ABA keeps the (sin, cos) of every revolute joint, in registers (trunk) or in a shared-memory region of its own after
the stash (folded limbs, rows 2i and 2i + 1 of body i); passes 2 and 3 read them back instead of loading the angle again and
evaluating sin / cos.  The values are the same floats, so results are bit-identical with the cache on and off (RBD_JIT_TRIG=0).
CPU tier: the CPU flavour both ways, folded and straight-line, and the structure of the Atlas translation unit; GPU tier: both
kernel shapes both ways, the range gate for an angle in a folded limb, and the resident blocks."""
import re

import numpy as np
import pytest
import torch

import rigidbodydynamics.jl_b200 as rbd
from tests import hostsim
from tests.test_reg_stash import _models, _shared_rows_used
from tests.util import rand_inputs

ATLAS_TRIG_ROWS = 52                   # the 26 limb joints (legs of 6, arms of 7) x (sin, cos)


@pytest.mark.parametrize("fold", [True, False])
@pytest.mark.parametrize("name", ["atlas", "valkyrie", "iiwa14", "randmech1", "randmech2", "mirrored"])
def test_trig_cache_bit_identical_cpu(built, monkeypatch, name, fold):
    mech = dict(_models())[name]
    desc = mech.flatten()
    q, v, tau, _, _ = rand_inputs(mech, 8, 7)
    outs, srcs = {}, {}
    monkeypatch.delenv("RBD_JIT_REG_ROWS", raising=False)
    for trig in ("0", "1"):
        monkeypatch.setenv("RBD_JIT_TRIG", trig)
        prog = hostsim.SpecProgram(desc, "aba", np.float32, True, True, fold=fold)
        srcs[trig], outs[trig] = prog.src, prog.run(q, v, tau)
    used = lambda src: re.search(r"RBD_T(?:LD|ST)\([\d(]|\brbd_sc\d", src) is not None     # a cache row read or written
    assert not used(srcs["0"]) and used(srcs["1"])
    assert srcs["1"].count("RBD_SINCOS(") < srcs["0"].count("RBD_SINCOS(")
    (a, qa), (b, qb) = outs["0"], outs["1"]
    assert np.isfinite(a).all()
    assert np.array_equal(a, b) and np.array_equal(qa, qb)


def _tu(monkeypatch, trig):
    monkeypatch.delenv("RBD_JIT_REG_ROWS", raising=False)
    monkeypatch.setenv("RBD_JIT_TRIG", trig)
    desc = rbd.load_model("atlas", floating=True).flatten()
    src, _ = hostsim.spec_source(desc, "aba", np.float32, True, False, 3)
    define = lambda k: int(re.search(rf"#define {k} (\d+)", src).group(1))
    return src, define("RBD_SPEC_ROWS"), define("RBD_SPEC_TRIG_ROWS"), define("RBD_SPEC_SMEM_BLOCKS")


def _rows(src, acc):
    """Rows addressed by accessor `acc` (a regex up to the row): constant rows, and both iterations of `row + rbd_it * d` with
    its Δ."""
    rows, deltas = set(), []
    for m in re.finditer(rf"{acc}(\d+|\((\d+) \+ rbd_it \* (-?\d+)\))", src):
        if m.group(2) is None:
            rows.add(int(m.group(1)))
        else:
            r, d = int(m.group(2)), int(m.group(3))
            rows.update((r, r + d))
            deltas.append(d)
    return rows, deltas


def test_atlas_program_structure_cpu(built, monkeypatch):
    """Atlas: one sin / cos site per revolute joint of the folded image (4 trunk joints, one leg of 6, one arm of 7), the angles are
    loaded in pass 1 only, the limbs' trig rows are affine in the loop iteration and packed after the stash, and the cache costs
    no resident blocks."""
    src0, rows0, trig0, blocks0 = _tu(monkeypatch, "0")
    src, rows, trig, blocks = _tu(monkeypatch, "1")
    assert trig0 == 0 and src0.count("RBD_SINCOS(") == 50          # the program without the cache: every pass evaluates
    assert src.count("RBD_SINCOS(") <= 17
    # after pass 1 only the floating base's rows (0 .. 6) are read again, by the root's joint-space solve
    later = lambda src: _rows(src[src.index("// ABA pass 2"):], r"RBD_LDG\(q, ")[0]
    assert later(src) <= set(range(7)) and not later(src0) <= set(range(7))
    # the stash is unchanged; the trig rows are their own region 0 .. RBD_SPEC_TRIG_ROWS - 1, none missing
    assert rows == rows0 == 156 and _shared_rows_used(src) == set(range(rows))
    assert trig == ATLAS_TRIG_ROWS
    tld, dl = _rows(src, r"RBD_TLD\(")
    tst, ds = _rows(src, r"RBD_TST\(")
    assert tld == tst == set(range(trig))
    assert dl and ds and all(d != 0 for d in dl + ds)
    assert not re.search(r"RBD_T(?:LD|ST)\(\d+[,)]", src)                 # limb rows only: every one indexed by the loop
    assert not re.search(r"rbd_sc\d+[^;\n]*rbd_it \*", src) and not re.search(r"rbd_it \*[^;\n]*rbd_sc\d+", src)
    assert len(set(re.findall(r"\brbd_sc(\d+)\b", src))) == 2 * 4    # the trunk joints' (sin, cos) are registers
    # (156 + 52) x 128 B per warp: still 8 blocks on a 228 KB SM with 1 KB reserved per block
    assert blocks == blocks0 == 8 == min(8, 233472 // ((rows + trig) * 32 * 4 + 1024))


def test_cache_dropped_where_it_costs_blocks_cpu(built, monkeypatch):
    """Without register rows the Atlas stash alone allows 8 blocks; its trig rows would cost two, so the program keeps none.
    Inverse dynamics and fp64 programs never have the cache."""
    monkeypatch.setenv("RBD_JIT_REG_ROWS", "0")
    monkeypatch.delenv("RBD_JIT_TRIG", raising=False)
    desc = rbd.load_model("atlas", floating=True).flatten()
    src, _ = hostsim.spec_source(desc, "aba", np.float32, True, False, 3)
    assert int(re.search(r"#define RBD_SPEC_TRIG_ROWS (\d+)", src).group(1)) == 0 and "RBD_TLD" not in src
    monkeypatch.delenv("RBD_JIT_REG_ROWS")
    for algo, dtype in (("rnea", np.float32), ("aba", np.float64)):
        src, _ = hostsim.spec_source(desc, algo, dtype, True, False, 3)
        assert int(re.search(r"#define RBD_SPEC_TRIG_ROWS (\d+)", src).group(1)) == 0
        assert "RBD_TLD" not in src and "rbd_sc" not in src


# ---------------------------------------------------------------------------------------------------------------- GPU tier
def _dyn_gpu(trig, variant, q, v, tau, monkeypatch):
    monkeypatch.delenv("RBD_JIT_REG_ROWS", raising=False)
    monkeypatch.setenv("RBD_JIT_TRIG", trig)
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
    rbd.rand_(st, np.random.default_rng(23))
    tau = torch.rand((st.nv, B), dtype=torch.float32, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    return st.q.clone(), st.v.clone(), tau


@pytest.mark.gpu
def test_trig_cache_on_the_device_gpu(built, monkeypatch, tmp_path):
    """Atlas fp32 forward dynamics: shared-memory blocks and the mixed CTA, with and without the cache, give the same bits; the
    blocks with the cache take its rows' shared memory on top of the stash's and still reside 8 to an SM."""
    monkeypatch.setenv("RBD_JIT_CACHE", str(tmp_path))
    q, v, tau = _atlas_inputs(1 << 17)                     # enough groups of 32 for the mixed CTA's 16 warps on every SM
    runs = {(t, var): _dyn_gpu(t, var, q, v, tau, monkeypatch) for t in ("0", "1") for var in ("1", "2")}
    ref_vd, ref_qd, _ = runs[("0", "1")]
    assert torch.isfinite(ref_vd).all()
    for k, (vd, qd, info) in runs.items():
        assert info.specialised == 1, (k, info)
        assert torch.equal(vd, ref_vd) and torch.equal(qd, ref_qd), k
    info0, info1 = runs[("0", "1")][2], runs[("1", "1")][2]
    assert info0.block == info1.block == 32
    assert info1.smem_bytes == info0.smem_bytes + ATLAS_TRIG_ROWS * 32 * 4
    assert info1.blocks_per_sm == info0.blocks_per_sm == 8


@pytest.mark.gpu
def test_gate_in_a_folded_limb_gpu(built, monkeypatch, tmp_path):
    """An angle of 3e4 rad in a folded limb joint (beyond the fast sin / cos range): pass 1 still folds it into the gate, so the
    generic kernel queued behind the program redoes the batch -- bit-identical to the generic kernel alone."""
    monkeypatch.delenv("RBD_JIT_REG_ROWS", raising=False)
    monkeypatch.delenv("RBD_JIT_TRIG", raising=False)
    src, _ = hostsim.spec_source(rbd.load_model("atlas", floating=True).flatten(), "aba", np.float32, True, False, 3)
    m = re.search(r"RBD_LDG\(q, \((\d+) \+ rbd_it \* (\d+)\)\)", src)   # an angle of a folded limb: the mirror instance
    row = int(m.group(1)) + int(m.group(2))
    monkeypatch.setenv("RBD_JIT_CACHE", str(tmp_path / "jit"))
    B, n = 1 << 16, 517
    q, v, tau = _atlas_inputs(B)
    q[row, 77] = 3.0e4                                     # exactly representable in fp32
    vd, qd, info = _dyn_gpu("1", "1", q, v, tau, monkeypatch)
    assert (info.specialised, info.kernels_launched) == (1, 2), info
    # the generic kernel alone: a batch below the on-the-fly compile threshold and no cubin in the cache
    monkeypatch.setenv("RBD_JIT_CACHE", str(tmp_path / "none"))
    (tmp_path / "none").mkdir()
    ref_vd, ref_qd, info2 = _dyn_gpu("1", "1", q[:, :n].contiguous(), v[:, :n].contiguous(), tau[:, :n].contiguous(), monkeypatch)
    assert info2.specialised == 0
    assert torch.isfinite(vd[:, 77]).all()
    assert torch.equal(vd[:, :n], ref_vd) and torch.equal(qd[:, :n], ref_qd)
