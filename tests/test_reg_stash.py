"""Register-resident stash rows of the model-specialised forward-dynamics program (csrc/rbd_codegen.cpp).

Stash rows that no folded loop addresses with its iteration (the trunk bodies' rows, the pending slot) are plain variables
instead of shared memory, up to a budget (RBD_JIT_REG_ROWS, read at generation time); the other rows are renumbered compactly
and RBD_SPEC_ROWS is their count.  The statements do not change, so every budget gives bit-identical results.  CPU tier: the
CPU flavour with and without register rows, folded and straight-line, and the structure of the CUDA translation unit; GPU tier:
both kernel shapes and budgets on the device, and the smaller shared-memory footprint in the launch record."""
import os
import re

import numpy as np
import pytest
import torch

import rigidbodydynamics.jl_b200 as rbd
from tests import hostsim
from tests.test_fold import _mirrored_tree
from tests.util import rand_inputs, randmech

ATLAS_ROWS = 213                       # 31 bodies x 6 rows + the 27-row pending slot


def _models():
    return [("atlas", rbd.load_model("atlas", floating=True)), ("valkyrie", rbd.load_model("valkyrie", floating=True)),
            ("iiwa14", rbd.load_model("iiwa14")), ("randmech1", randmech(1)), ("randmech2", randmech(2, shuffle=True)),
            ("mirrored", _mirrored_tree(1))]


@pytest.mark.parametrize("fold", [True, False])
@pytest.mark.parametrize("name", ["atlas", "valkyrie", "iiwa14", "randmech1", "randmech2", "mirrored"])
def test_register_rows_bit_identical_cpu(built, monkeypatch, name, fold):
    mech = dict(_models())[name]
    desc = mech.flatten()
    q, v, tau, _, _ = rand_inputs(mech, 8, 5)
    outs, srcs = {}, {}
    for budget in ("0", "27", "-1"):
        monkeypatch.setenv("RBD_JIT_REG_ROWS", budget)
        prog = hostsim.SpecProgram(desc, "aba", np.float32, True, True, fold=fold)
        srcs[budget], outs[budget] = prog.src, prog.run(q, v, tau)
    assert "rbd_r" not in srcs["0"]
    assert "rbd_r" in srcs["-1"]
    a, qa = outs["0"]
    assert np.isfinite(a).all()
    for budget in ("27", "-1"):
        b, qb = outs[budget]
        assert np.array_equal(a, b) and np.array_equal(qa, qb), budget


def _tu(desc, budget, monkeypatch):
    monkeypatch.setenv("RBD_JIT_REG_ROWS", budget)
    src, st = hostsim.spec_source(desc, "aba", np.float32, True, False, 3)
    define = lambda k: int(re.search(rf"#define {k} (\d+)", src).group(1))
    return src, st, define("RBD_SPEC_ROWS"), define("RBD_SPEC_SMEM_BLOCKS")


def _shared_rows_used(src):
    """Every shared row the program addresses: constant rows and both iterations of `row + rbd_it * d`."""
    rows = set()
    for m in re.finditer(r"RBD_S(?:LD|ST)\((\d+|\((\d+) \+ rbd_it \* (-?\d+)\))", src):
        if m.group(2) is None:
            rows.add(int(m.group(1)))
        else:
            r, d = int(m.group(2)), int(m.group(3))
            rows.update((r, r + d))
    return rows


@pytest.mark.parametrize("budget", ["0", "27", "-1"])
def test_register_rows_structure_cpu(built, monkeypatch, budget):
    """Atlas: register rows are plain names never indexed by the loop iteration, the shared rows are 0 .. RBD_SPEC_ROWS - 1
    with none missing, and RBD_SPEC_SMEM_BLOCKS is what that stash allows on a 228 KB SM (1 KB reserved per block)."""
    desc = rbd.load_model("atlas", floating=True).flatten()
    src, st, rows, blocks = _tu(desc, budget, monkeypatch)
    assert st["stash_rows"] == ATLAS_ROWS
    regs = set(int(r) for r in re.findall(r"\brbd_r(\d+)\b", src))
    assert not re.search(r"rbd_r\d+[^;\n]*rbd_it \*", src) and not re.search(r"rbd_it \*[^;\n]*rbd_r\d+", src)
    assert not re.search(r"RBD_S(?:LD|ST)\([^)]*rbd_r", src)
    used = _shared_rows_used(src)
    assert used == set(range(rows))
    assert rows + len(regs) == ATLAS_ROWS
    expect = {"0": 0, "27": 27}.get(budget)
    if expect is not None:
        assert len(regs) == expect
    else:                                  # every eligible row: the trunk (pelvis, three back links, head) and the pending slot
        assert len(regs) >= 5 * 6 + 27 - 6
    # with register rows the kernel is compiled for at most 8 blocks (up to 255 registers), else for at most 16 (128)
    assert blocks == min(16 if budget == "0" else 8, 233472 // (rows * 32 * 4 + 1024))
    if budget == "-1":
        assert 233472 // (rows * 32 * 4 + 1024) > 8


def test_other_programs_keep_the_shared_stash_cpu(built, monkeypatch):
    """The register rows apply to fp32 forward dynamics only: inverse dynamics, the mass matrix and fp64 programs are unchanged."""
    monkeypatch.delenv("RBD_JIT_REG_ROWS", raising=False)
    desc = rbd.load_model("atlas", floating=True).flatten()
    for algo, dtype in (("rnea", np.float32), ("crba", np.float32), ("aba", np.float64)):
        src, st = hostsim.spec_source(desc, algo, dtype, True, False, 3)
        assert "rbd_r" not in src
        assert int(re.search(r"#define RBD_SPEC_ROWS (\d+)", src).group(1)) == max(1, st["stash_rows"])


# ---------------------------------------------------------------------------------------------------------------- GPU tier
def _dyn_gpu(budget, variant, B, q, v, tau, monkeypatch):
    if budget is None:
        monkeypatch.delenv("RBD_JIT_REG_ROWS", raising=False)
    else:
        monkeypatch.setenv("RBD_JIT_REG_ROWS", budget)
    monkeypatch.setenv("RBD_JIT_VARIANT", variant)
    mech = rbd.load_model("atlas", floating=True)         # a fresh handle: generated and loaded under this budget
    st = rbd.MechanismState(mech, B, torch.float32)
    st.q.copy_(q)
    st.v.copy_(v)
    res = rbd.DynamicsResult(mech, B, torch.float32)
    rbd.dynamics_(res, st, tau, want_qd=True)
    torch.cuda.synchronize()
    li = rbd.launch_info()
    return res.vd.clone(), res.qd.clone(), (li.specialised, li.block, li.smem_bytes, li.blocks_per_sm)


@pytest.mark.gpu
def test_register_rows_on_the_device_gpu(built, monkeypatch, tmp_path):
    """Atlas fp32 forward dynamics: shared-memory blocks and the mixed CTA, with the default register rows and with none, give
    the same bits; with register rows the blocks take less shared memory, and no fewer of them reside on an SM."""
    monkeypatch.setenv("RBD_JIT_CACHE", str(tmp_path))    # the budget-0 program is compiled here if it is not cached
    B = 1 << 17                                            # enough groups of 32 for the mixed CTA's 16 warps on every SM
    st = rbd.MechanismState(rbd.load_model("atlas", floating=True), B, torch.float32)
    rbd.rand_(st, np.random.default_rng(11))
    tau = torch.rand((st.nv, B), dtype=torch.float32, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    runs = {(b, var): _dyn_gpu(b, var, B, st.q, st.v, tau, monkeypatch) for b in (None, "0") for var in ("1", "2")}
    ref_vd, ref_qd, _ = runs[("0", "1")]
    assert torch.isfinite(ref_vd).all()
    for k, (vd, qd, info) in runs.items():
        assert info[0] == 1, (k, info)
        assert torch.equal(vd, ref_vd) and torch.equal(qd, ref_qd), k
    _, _, (_, blk_reg, smem_reg, bps_reg) = runs[(None, "1")]
    _, _, (_, blk_0, smem_0, bps_0) = runs[("0", "1")]
    assert blk_reg == blk_0 == 32
    assert smem_0 == ATLAS_ROWS * 32 * 4 and smem_reg < smem_0
    assert bps_reg >= bps_0 >= 1
