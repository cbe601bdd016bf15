"""Every path of rbd_dynamics_derivatives (csrc/rbd_deriv.cu, rbd_deriv.cuh, rbd_deriv_jit.cpp) that only large batches or large
models take, forced on purpose, proven by the launch record and checked column by column against the CPU run of the same per-sample
code (tests/hostsim) and, on a few columns, against the oracle's dual numbers.

Paths:
1. The model-specialised solve kernel (NVRTC), compiled on demand inside the call (B >= 4096, fresh cubin cache, tables no other test
   loads), over at least three passes of its persistent grid, with a partly filled last column group (iiwa14: 14 columns, 4 per
   group).  Atlas fp32 runs at 2^17 samples and prints the worst fp32 error.
2. The specialised and the table-driven solve with 1 to 4 columns per group, and the shared-memory factor against the one on the
   scratch: the same operations in the same order per entry and column, so the results are bit-identical.
3. Models at the size edges: 66 coordinates (the high word of the specialised kernel's relation masks), a single-warp shared-memory
   solve, factors too large for shared memory (the scratch factor without the override), nv = 128 accepted, nv = 129 and
   nnz = 8001 refused before any launch.
4. More than one pass of deriv_world_kernel (8 blocks per SM).
5. Chunks of the scratch: samples on both sides of every boundary, the launch count, and bitwise equality with one chunk.
6. The chunk cap that keeps deriv_pairs_kernel's grid.y within 65535 blocks.
7. A NaN sample inside a 32-sample CTA stays in its column on every solve path.
8. 64-bit offsets in the outputs (optional: needs 24 GB free).

Every GPU call fills its outputs with NaN and checks that every column in [0, B) was written, the structural zeros included, and
that the padding beyond B (ld > B) was not.  Every input column is distinct.  The compared columns are 511 at an odd stride plus
B - 1 (tests/test_vjp_paths.py: every lane, the first, middle and last pass, the ragged last group).

The process-wide module map of rbd_deriv.cu keys the specialised kernel on the model's index tables, not on RBD_DERIV_CG or the
cubin cache; a model that gains fixed bodies gets new tables but the same coordinates (and the same kernel text).  The tests that
need a kernel loaded afresh therefore use Atlas or iiwa14 with a chain of fixed "tool" bodies of a length no other test uses."""
import os

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from oracle import Oracle
from rigidbodydynamics.jl_b200 import _cabi
from tests import hostsim
from tests.test_derivatives import TOL32, TOL64
from tests.test_vjp_paths import _dev, _passes, cols, rand_q
from tests.util import double_pendulum, oracle_dynamics_derivatives, rel_err

TOL_CPU = 1e-10             # GPU against the CPU run of the same per-sample code, fp64

# rbd_deriv.cuh / rbd_deriv.cu / rbd_deriv_jit.cpp
DOF_ROWS, BODY_ROWS = 24, 52            # kDofRows, kBodyRows
MAX_DOFS, MAX_NNZ = 128, 4096           # kMaxDofs, kMaxNnz
KNT = 128                               # kNT: samples per block of the per-sample kernels
JIT_MIN_BATCH = 4096                    # RBD_JIT_MIN_BATCH of this entry point
JIT_SMEM_MAX = 200 * 1024               # the specialised kernel's factor must fit in this much shared memory
WORLD_BLOCKS_PER_SM = 8                 # deriv_world_kernel's grid: min(groups, 8 x SMs)
GRID_Y_MAX = 65535
# sm_90 shared memory: per block (opt-in) and per SM; the GPU tier reads them from the device
SM90_SMEM_OPTIN, SM90_SMEM_PER_SM = 232448, 233472


# ------------------------------------------------------------------------------------------------------------------
# the host-side arithmetic of rbd_deriv.cu, re-derived
# ------------------------------------------------------------------------------------------------------------------
def tables(mech):
    """(nb, nv, nnz, rows) of build_deriv_dev: coordinate p stores depth(p) + 1 entries of M, depth = coordinates above it."""
    d = mech.flatten()
    above = [0] * d.nb                  # coordinates at or above body i
    nnz = 0
    for i, j in enumerate(mech.joints):
        base = above[d.parent[i]] if d.parent[i] >= 0 else 0
        for k in range(j.nv):
            nnz += base + k + 1
        above[i] = base + j.nv
    return d.nb, d.nv, nnz, DOF_ROWS * d.nv + BODY_ROWS * d.nb + nnz


def jit_plan(nv, f64):
    """deriv_jit_plan: (cg, ngroups, warps), or None when not even one right-hand side fits into the register budget."""
    cg = min(4, (150 if f64 else 110) // (nv * (2 if f64 else 1)))
    if cg < 1:
        return None
    ngroups = -(-2 * nv // cg)
    rounds = -(-ngroups // 12)
    return cg, ngroups, -(-ngroups // rounds)


def solve_geometry(nv, nnz, size, optin=SM90_SMEM_OPTIN, per_sm=SM90_SMEM_PER_SM):
    """The generic solve's (factor in shared memory, warps W, blocks per SM) and the bytes of its factor and right-hand sides."""
    hbytes, xbytes = nnz * 32 * size, nv * 32 * size
    best_w = best_nb = 0
    for nb in range(1, 5):
        avail = min(optin, per_sm // nb - 1024) - hbytes
        if avail < xbytes:
            continue
        w = min(16, 2 * nv, avail // xbytes)
        if w * nb > best_w * best_nb:
            best_w, best_nb = w, nb
    if best_w == 0:
        return False, min(8, 2 * nv, optin // xbytes), 1, hbytes, xbytes
    return True, best_w, best_nb, hbytes, xbytes


def jit_eligible(nv, nnz, size, **kw):
    return solve_geometry(nv, nnz, size, **kw)[0] and nnz * 32 * size <= JIT_SMEM_MAX and jit_plan(nv, size == 8) is not None


def chunk(rows, size, B, mb=2048):
    """Samples per chunk: the scratch budget, at least one block, at most GRID_Y_MAX blocks of deriv_pairs_kernel."""
    c = min(B, max(KNT, (mb << 20) // (rows * size) // KNT * KNT))
    return min(c, GRID_Y_MAX * KNT)


# ------------------------------------------------------------------------------------------------------------------
# models
# ------------------------------------------------------------------------------------------------------------------
def legs_model(nlegs=20, seed=0):
    """A floating base with `nlegs` three-link revolute legs: 6 + 3 nlegs coordinates (66 for 20 legs, nnz = 501)."""
    rng = np.random.default_rng(seed)
    mech = rbd.Mechanism(rbd.RigidBody("world"))
    base = rbd.RigidBody("base", rbd.SpatialInertia.rand(rng))
    mech.attach(mech.root_body, base, rbd.Joint("base", rbd.QuaternionFloating()))
    for leg in range(nlegs):
        parent = base
        for k in range(3):
            body = rbd.RigidBody(f"leg{leg}_{k}", rbd.SpatialInertia.rand(rng))
            mech.attach(parent, body, rbd.Joint(f"leg{leg}_{k}", rbd.Revolute.rand(rng)), joint_pose=rbd.Transform3D.rand(rng))
            parent = body
    return mech


def star_model(nfloat=21, nlinks=2, seed=1):
    """`nfloat` floating bodies under the world and a chain of `nlinks` revolute links below the last one."""
    rng = np.random.default_rng(seed)
    mech = rbd.Mechanism(rbd.RigidBody("world"))
    for k in range(nfloat):
        mech.attach(mech.root_body, rbd.RigidBody(f"float{k}", rbd.SpatialInertia.rand(rng)), rbd.Joint(f"float{k}", rbd.QuaternionFloating()),
                    joint_pose=rbd.Transform3D.rand(rng))
    for k in range(nlinks):
        body = rbd.RigidBody(f"link{k}", rbd.SpatialInertia.rand(rng))
        mech.attach(mech.bodies[-1], body, rbd.Joint(f"link{k}", rbd.Revolute.rand(rng)), joint_pose=rbd.Transform3D.rand(rng))
    return mech


def chain_model(n, joint_type=None, seed=2):
    return rbd.rand_chain_mechanism(np.random.default_rng(seed), [joint_type or rbd.Revolute] * n)


def tooled(mech, ntools, seed=3):
    """`mech` with a chain of `ntools` fixed bodies under its last body: the same coordinates, new index tables."""
    rng = np.random.default_rng(seed)
    parent = mech.bodies[-1]
    for k in range(ntools):
        body = rbd.RigidBody(f"tool{k}", rbd.SpatialInertia.rand(rng))
        mech.attach(parent, body, rbd.Joint(f"tool{k}", rbd.Fixed()), joint_pose=rbd.Transform3D.rand(rng))
        parent = body
    return mech


def atlas():
    return rbd.load_model("atlas", floating=True)


def iiwa14():
    return rbd.load_model("iiwa14", floating=False)


# fixed-tool chain lengths, one per test that needs its own entry in the module map
TOOLS_ON_DEMAND = 1
TOOLS_CG = {1: 2, 2: 3, 3: 4, 4: 5}
TOOLS_CHUNKS = 6

EDGE_MODELS = {
    "legs66": legs_model,
    "chain41": lambda: chain_model(41),
    "chain45": lambda: chain_model(45),
    "chain63": lambda: chain_model(63),
    "star128": star_model,
}
REFUSED_MODELS = {
    "star129": lambda: star_model(nlinks=3),
    "float_chain21": lambda: chain_model(21, rbd.QuaternionFloating),
}


# ------------------------------------------------------------------------------------------------------------------
# CPU tier
# ------------------------------------------------------------------------------------------------------------------
def test_models_hit_their_paths():
    """Each model still takes the path it is here for, on sm_90's shared memory."""
    # iiwa14: the specialised kernel with a partly filled last column group in both precisions
    _, nv, nnz, _ = tables(iiwa14())
    for f64 in (True, False):
        cg, ngroups, _ = jit_plan(nv, f64)
        assert (cg, ngroups) == (4, 4) and 2 * nv % cg, "partly filled last column group"
        assert jit_eligible(nv, nnz, 8 if f64 else 4), "specialised solve"
    # Atlas: specialised kernel, groups filled evenly
    nb, nv, nnz, rows = tables(atlas())
    assert (nb, nv, nnz) == (31, 36, 351), (nb, nv, nnz)
    assert jit_plan(36, True)[:2] == (2, 36) and jit_plan(36, False)[:2] == (3, 24)
    assert jit_eligible(nv, nnz, 8) and jit_eligible(nv, nnz, 4)
    # tools change the tables, not the coordinates
    assert tables(tooled(atlas(), 3))[1:3] == (nv, nnz) and tables(tooled(atlas(), 3))[0] == nb + 3
    # 66 coordinates: the high word of kRel, one column per group, specialised in both precisions
    nb, nv, nnz, _ = tables(legs_model())
    assert (nb, nv, nnz) == (61, 66, 501) and nv > 64, "kRel high word"
    for size in (8, 4):
        assert jit_plan(nv, size == 8) == (1, 132, 12) and jit_eligible(nv, nnz, size), "specialised solve, nv > 64"
    # a 41-joint chain in fp64: the factor fits next to exactly one warp's right-hand sides
    _, nv, nnz, _ = tables(chain_model(41))
    hs, w, nbk, hbytes, _ = solve_geometry(nv, nnz, 8)
    assert hs and (w, nbk) == (1, 1) and hbytes > JIT_SMEM_MAX, "single-warp shared-memory solve, not specialised"
    assert solve_geometry(*tables(chain_model(40))[1:3], 8)[1] == 2          # one joint fewer: two warps
    # 45 and 63 joints: the factor does not fit into shared memory (fp64; 63 also in fp32): factored on the scratch
    for n, sizes in ((45, (8,)), (63, (8, 4))):
        _, nv, nnz, _ = tables(chain_model(n))
        for size in sizes:
            assert not solve_geometry(nv, nnz, size)[0], ("scratch factor", n, size)
    assert solve_geometry(*tables(chain_model(45))[1:3], 4)[0]               # fp32 45-chain fits
    # nv = 128: accepted, no specialised plan in either precision (the generic shared-memory solve serves it)
    _, nv, nnz, _ = tables(star_model())
    assert nv == MAX_DOFS and nnz <= MAX_NNZ and jit_plan(nv, True) is None and jit_plan(nv, False) is None
    assert solve_geometry(nv, nnz, 8)[0]
    # the limits
    assert tables(star_model(nlinks=3))[1] == MAX_DOFS + 1
    _, nv, nnz, _ = tables(chain_model(21, rbd.QuaternionFloating))
    assert (nv, nnz) == (126, 8001) and nnz > MAX_NNZ


def test_chunk_arithmetic():
    """The scratch budget and the grid.y cap of deriv_pairs_kernel."""
    _, _, _, rows = tables(chain_model(1))
    assert rows == 77
    # a one-revolute model in fp32 with a 4096 MiB budget: the budget alone would allow more samples than grid.y can hold
    assert (4096 << 20) // (rows * 4) // KNT * KNT > GRID_Y_MAX * KNT
    B = (1 << 23) + 4096
    C = chunk(rows, 4, B, 4096)
    assert C == GRID_Y_MAX * KNT and -(-B // C) == 2
    # at the default budget no model reaches the cap
    assert chunk(rows, 4, 1 << 30) < GRID_Y_MAX * KNT
    # Atlas fp64: about 93 k samples per chunk by default, 128 (one block) with a 4 MiB budget
    _, _, _, rows = tables(atlas())
    assert 90_000 < chunk(rows, 8, 1 << 30) < 96_000 and chunk(rows, 8, 1 << 30, 4) == KNT


def test_column_choice_covers_chunk_edges():
    C = 3 * KNT
    B = 7 * C + 77
    idx = edge_cols(B, C)
    assert idx[-1] == B - 1 and set((idx % 32).tolist()) == set(range(32))
    for k in range(1, -(-B // C)):
        assert {k * C - 1, k * C} <= set(idx.tolist())


@pytest.mark.parametrize("name", list(REFUSED_MODELS))
def test_model_limits_refused_without_a_gpu(name):
    """The limits are checked on the host: the ahead-of-time compile refuses them too."""
    h = _cabi.ModelHandle(REFUSED_MODELS[name]().flatten())
    try:
        with pytest.raises(_cabi.RbdError) as e:
            h.precompile_derivatives(_cabi.RBD_F64)
        assert e.value.status == _cabi.RBD_EUNSUPPORTED and "too large" in str(e.value)
    finally:
        h.close()


# ------------------------------------------------------------------------------------------------------------------
# GPU tier: helpers
# ------------------------------------------------------------------------------------------------------------------
def edge_cols(B, C=None):
    """cols(B) plus both sides of every chunk boundary."""
    idx = cols(B)
    if C and C < B:
        b = np.arange(C, B, C)
        idx = np.unique(np.concatenate([idx, b - 1, b]))
    return idx


@pytest.fixture(scope="module")
def torch():
    import torch as t
    assert t.cuda.is_available()
    rbd.load_library()
    return t


def device(torch):
    p = torch.cuda.get_device_properties(torch.cuda.current_device())
    return p.multi_processor_count, p.shared_memory_per_block_optin, p.shared_memory_per_multiprocessor


def max_grid(torch, block, smem):
    """An upper bound on a persistent grid: the blocks that fit on an SM by shared memory and threads, times the SMs."""
    sms, _, per_sm = device(torch)
    return sms * max(1, min(per_sm // (smem + 1024), 2048 // block, 32))


def multi_pass_batch(grid):
    """Three passes of `grid` blocks of 32 samples, and a ragged part group."""
    return 3 * grid * 32 + 77


def inputs(mech, B, seed):
    rng = np.random.default_rng(seed)
    d = mech.flatten()
    return {"q": rand_q(mech, B, rng), "v": rng.standard_normal((d.nv, B)), "tau": rng.standard_normal((d.nv, B))}


def call(torch, mech, x, B, ld, dtype, ins=None):
    """rbd_dynamics_derivatives on [rows, ld] tensors; NaN-filled outputs.  Returns (status, message, ins, outs, launch record)."""
    from rigidbodydynamics.jl_b200.state import _DT, _model_handle
    nv = mech.num_velocities()
    if ins is None:
        ins = {k: _dev(torch, a, dtype, ld) for k, a in x.items()}
    outs = {k: torch.full((r, ld), float("nan"), dtype=dtype, device="cuda") for k, r in (("vd", nv), ("dq", nv * nv), ("dv", nv * nv))}
    p = lambda t: None if t is None else t.data_ptr()      # noqa: E731
    lib = _cabi.load_library()
    st = lib.rbd_dynamics_derivatives(_model_handle(mech).ptr, _DT[dtype], B, ld, p(ins["q"]), p(ins["v"]), p(ins.get("tau")),
                                      p(outs["vd"]), p(outs["dq"]), p(outs["dv"]), None)
    torch.cuda.synchronize()
    msg = lib.rbd_last_error().decode() if st else ""
    return st, msg, ins, outs, rbd.launch_info()


def check_written(torch, outs, B):
    for k, t in outs.items():
        assert bool(torch.isfinite(t[:, :B]).all()), k
        assert bool(torch.isnan(t[:, B:]).all()), k


def host(t, idx):
    return t[:, idx].double().cpu().numpy()


def check_cpu(torch, mech, ins, outs, idx, dtype, label):
    """outs at the columns idx against the fp64 CPU run of the same code on the same (rounded) inputs; returns the worst error."""
    h = {k: host(t, idx) for k, t in ins.items()}
    _, rq, rv = hostsim.dynamics_derivatives(mech.flatten(), h["q"], h["v"], h.get("tau"))
    e = max(rel_err(host(outs["dq"], idx), rq), rel_err(host(outs["dv"], idx), rv))
    print(f"{label}: worst rel_err vs the fp64 CPU run over {len(idx)} columns {e:.2e}")
    assert e < (TOL_CPU if dtype == torch.float64 else TOL32), (label, e)
    return e


def check_oracle(torch, mech, x, outs, fc, dtype):
    """A few columns against the oracle's dual numbers at the original fp64 inputs."""
    o = Oracle(mech.flatten())
    rq, rv = oracle_dynamics_derivatives(o, mech, x["q"][:, fc], x["v"][:, fc], x["tau"][:, fc])
    tol = TOL64 if dtype == torch.float64 else TOL32
    assert rel_err(host(outs["dq"], fc), rq) < tol and rel_err(host(outs["dv"], fc), rv) < tol, \
        (rel_err(host(outs["dq"], fc), rq), rel_err(host(outs["dv"], fc), rv))


def assert_jit(info, nv, nnz, dtype_size):
    _, _, warps = jit_plan(nv, dtype_size == 8)
    assert info.smem_bytes == nnz * 32 * dtype_size and info.block == 32 * warps, \
        ("specialised solve", info.smem_bytes, info.block)


def assert_generic(torch, info, nv, nnz, size, scratch_factor=False):
    _, optin, per_sm = device(torch)
    hs, w, _, hbytes, xbytes = solve_geometry(nv, nnz, size, optin, per_sm)
    if scratch_factor:
        w = min(8, 2 * nv, optin // xbytes)
        assert info.smem_bytes == w * xbytes and info.block == 32 * w, ("scratch factor", info.smem_bytes, info.block)
    else:
        assert hs and info.smem_bytes == hbytes + w * xbytes and info.block == 32 * w, ("shared-memory solve", info.smem_bytes, info.block)


# ------------------------------------------------------------------------------------------------------------------
# 1. the specialised solve, compiled inside the call, multi-pass
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
@pytest.mark.parametrize("name", ["atlas", "iiwa14"])
def test_jit_solve_compiled_on_demand_multi_pass(torch, tmp_path, monkeypatch, name, dtype_name):
    monkeypatch.setenv("RBD_JIT_CACHE", str(tmp_path))
    dtype = getattr(torch, dtype_name)
    size = 8 if dtype == torch.float64 else 4
    mech = tooled(atlas() if name == "atlas" else iiwa14(), TOOLS_ON_DEMAND)
    _, nv, nnz, rows = tables(mech)
    cg, ngroups, warps = jit_plan(nv, size == 8)
    B = max(JIT_MIN_BATCH + 1, multi_pass_batch(max_grid(torch, 32 * warps, nnz * 32 * size)))
    if name == "atlas" and size == 4:
        B = max(B, (1 << 17) + 77)         # the fp32 accuracy measurement
    assert chunk(rows, size, B) == B
    ld = B + 3
    x = inputs(mech, B, 31 + size)
    st, msg, ins, outs, info = call(torch, mech, x, B, ld, dtype)
    assert st == 0, msg
    assert_jit(info, nv, nnz, size)
    assert info.grid == min((B + 31) // 32, info.blocks_per_sm * device(torch)[0])
    assert 3 * info.grid * 32 <= B, (info.grid, B)
    assert any("_deriv_" in f for f in os.listdir(tmp_path)), "compiled inside the call"
    idx = cols(B)
    assert _passes(idx, info.grid) >= {0, 1, (B - 1) // 32 // info.grid}
    check_written(torch, outs, B)
    check_cpu(torch, mech, ins, outs, idx, dtype, f"{name} {dtype_name} B={B} grid={info.grid} cg={cg} groups={ngroups}")
    check_oracle(torch, mech, x, outs, np.array([0, B // 2 + 3, B - 1]), dtype)


# ------------------------------------------------------------------------------------------------------------------
# 2. solve paths against each other, bit for bit
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
@pytest.mark.parametrize("cg", [1, 2, 3, 4])
def test_jit_and_generic_solve_bit_identical(torch, monkeypatch, cg, dtype_name):
    """The generator writes out deriv_solve_column's arithmetic in its order per column (the rows outside a column's subtree and
    ancestors only ever add products with zero), so the specialised kernel with any number of columns per group equals the
    table-driven kernel bit for bit (signed zeros aside).  cg is clamped to the plan's (Atlas: 2 in fp64, 3 in fp32)."""
    dtype = getattr(torch, dtype_name)
    size = 8 if dtype == torch.float64 else 4
    mech = tooled(atlas(), TOOLS_CG[cg])
    _, nv, nnz, _ = tables(mech)
    _, optin, per_sm = device(torch)
    _, _, nbk, _, _ = solve_geometry(nv, nnz, size, optin, per_sm)
    B = max(JIT_MIN_BATCH + 1, multi_pass_batch(nbk * device(torch)[0]))       # the generic kernel's grid: three passes
    x = inputs(mech, B, 40 + cg)
    monkeypatch.setenv("RBD_DERIV_CG", str(cg))
    st, msg, ins, jit, info = call(torch, mech, x, B, B, dtype)
    assert st == 0, msg
    assert_jit(info, nv, nnz, size)
    monkeypatch.setenv("RBD_DERIV_JIT", "0")
    st, msg, _, gen, info = call(torch, mech, x, B, B, dtype, ins)
    assert st == 0, msg
    assert_generic(torch, info, nv, nnz, size)
    assert 3 * info.grid * 32 <= B
    check_written(torch, jit, B)
    for k in jit:
        if not torch.equal(jit[k], gen[k]):
            diff = (jit[k] - gen[k]).abs().max().item()
            pytest.fail(f"{k}: specialised and generic solve differ by up to {diff:.3e}")
    check_cpu(torch, mech, ins, jit, cols(B), dtype, f"atlas cg={cg} {dtype_name}")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
def test_shared_and_scratch_factor_bit_identical(torch, monkeypatch, dtype_name):
    """deriv_factor (one thread per sample, on the scratch) and the cooperative factor in shared memory update every entry with the
    same operations in the same order, and both feed deriv_solve_column: bit-identical, each over three passes of its grid."""
    dtype = getattr(torch, dtype_name)
    size = 8 if dtype == torch.float64 else 4
    mech = atlas()
    _, nv, nnz, _ = tables(mech)
    sms, optin, per_sm = device(torch)
    _, _, nbk, _, _ = solve_geometry(nv, nnz, size, optin, per_sm)
    B = multi_pass_batch(nbk * sms)
    x = inputs(mech, B, 50 + size)
    monkeypatch.setenv("RBD_DERIV_JIT", "0")
    st, msg, ins, shared, info = call(torch, mech, x, B, B + 1, dtype)
    assert st == 0, msg
    assert_generic(torch, info, nv, nnz, size)
    assert 3 * info.grid * 32 <= B
    n_shared = info.kernels_launched
    monkeypatch.setenv("RBD_DERIV_GLOBAL_FACTOR", "1")
    st, msg, _, glob, info = call(torch, mech, x, B, B + 1, dtype, ins)
    assert st == 0, msg
    assert_generic(torch, info, nv, nnz, size, scratch_factor=True)
    assert info.kernels_launched == n_shared + 1 and 3 * info.grid * 32 <= B
    check_written(torch, glob, B)
    for k in shared:
        if not torch.equal(shared[k][:, :B], glob[k][:, :B]):
            diff = (shared[k][:, :B] - glob[k][:, :B]).abs().max().item()
            pytest.fail(f"{k}: shared-memory and scratch factor differ by up to {diff:.3e}")
    check_cpu(torch, mech, ins, glob, cols(B), dtype, f"atlas scratch factor {dtype_name}")


# ------------------------------------------------------------------------------------------------------------------
# 3. models at the size edges
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,dtype_name", [("legs66", "float64"), ("legs66", "float32")] + [(n, "float64") for n in EDGE_MODELS if n != "legs66"])
def test_size_edge_models(torch, name, dtype_name):
    dtype = getattr(torch, dtype_name)
    size = 8 if dtype == torch.float64 else 4
    mech = EDGE_MODELS[name]()
    _, nv, nnz, rows = tables(mech)
    sms, optin, per_sm = device(torch)
    hs, w, nbk, hbytes, xbytes = solve_geometry(nv, nnz, size, optin, per_sm)
    jit = jit_eligible(nv, nnz, size, optin=optin, per_sm=per_sm)
    grid = max_grid(torch, 32 * jit_plan(nv, size == 8)[2], hbytes) if jit else nbk * sms
    B = max(JIT_MIN_BATCH + 1, multi_pass_batch(grid))
    assert chunk(rows, size, B) == B
    x = inputs(mech, B, 60 + nv)
    st, msg, ins, outs, info = call(torch, mech, x, B, B + 2, dtype)
    assert st == 0, msg
    if name == "legs66":
        assert jit, "specialised solve with the kRel high word"
        assert_jit(info, nv, nnz, size)
    else:
        assert not jit
        assert_generic(torch, info, nv, nnz, size, scratch_factor=not hs)
        assert (name in ("chain45", "chain63")) == (not hs), "scratch factor without the override"
        if name == "chain41":
            assert w == 1 and info.block == 32, "single-warp shared-memory solve"
    assert 3 * info.grid * 32 <= B, (info.grid, B)
    check_written(torch, outs, B)
    check_cpu(torch, mech, ins, outs, cols(B), dtype, f"{name} {dtype_name} nv={nv} nnz={nnz} B={B} grid={info.grid}")
    check_oracle(torch, mech, x, outs, np.array([0, B - 1]), dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(REFUSED_MODELS))
def test_model_limits_refused_before_any_launch(torch, name):
    mech = REFUSED_MODELS[name]()
    x = inputs(mech, 64, 7)
    st, msg, _, outs, info = call(torch, mech, x, 64, 64, torch.float64)
    assert st == _cabi.RBD_EUNSUPPORTED, st
    assert "more than 128 velocity coordinates or 4096 mass-matrix entries" in msg, msg
    assert info.kernels_launched == 0
    assert all(bool(torch.isnan(t).all()) for t in outs.values())


# ------------------------------------------------------------------------------------------------------------------
# 4. deriv_world_kernel over several passes
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["iiwa14", "double_pendulum"])
def test_world_kernel_multi_pass(torch, monkeypatch, name):
    mech = iiwa14() if name == "iiwa14" else double_pendulum()
    _, nv, nnz, rows = tables(mech)
    sms = device(torch)[0]
    B = 3 * WORLD_BLOCKS_PER_SM * sms * KNT + 77
    mb = -(-rows * 8 * B // (1 << 20)) + 1
    monkeypatch.setenv("RBD_DERIV_SCRATCH_MB", str(mb))          # one chunk: every block of the world kernel takes three passes
    assert chunk(rows, 8, B, mb) == B
    x = inputs(mech, B, 70)
    st, msg, ins, outs, info = call(torch, mech, x, B, B + 5, torch.float64)
    assert st == 0, msg
    check_written(torch, outs, B)
    idx = cols(B)
    assert _passes(idx // 4, WORLD_BLOCKS_PER_SM * sms) >= {0, 1, 2}     # groups of 128 samples = 4 groups of 32
    check_cpu(torch, mech, ins, outs, idx, torch.float64, f"{name} world kernel B={B}")
    check_oracle(torch, mech, x, outs, np.array([0, B // 2 + 3, B - 1]), torch.float64)


# ------------------------------------------------------------------------------------------------------------------
# 5. chunks
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
def test_chunks_bitwise_equal_one_chunk(torch, monkeypatch, dtype_name):
    """RBD_DERIV_SCRATCH_MB=4 against the default budget, with torques.  The model has a fixed joint and B < 2^15, so the forward
    dynamics takes the same generic kernel whatever batch size a chunk hands it; a sample's arithmetic does not depend on its
    chunk, so the outputs are bitwise equal."""
    dtype = getattr(torch, dtype_name)
    size = 8 if dtype == torch.float64 else 4
    mech = tooled(atlas(), TOOLS_CHUNKS)
    _, nv, nnz, rows = tables(mech)
    C = chunk(rows, size, 1 << 30, 4)
    B = 7 * C + 77
    assert B < JIT_MIN_BATCH
    monkeypatch.setenv("RBD_DERIV_JIT", "0")
    x = inputs(mech, B, 80 + size)
    st, msg, ins, one, info = call(torch, mech, x, B, B + 7, dtype)
    assert st == 0, msg
    assert info.grid == min((B + 31) // 32, solve_geometry(nv, nnz, size, *device(torch)[1:])[2] * device(torch)[0])
    n1 = info.kernels_launched
    monkeypatch.setenv("RBD_DERIV_SCRATCH_MB", "4")
    st, msg, _, many, info = call(torch, mech, x, B, B + 7, dtype, ins)
    assert st == 0, msg
    assert info.kernels_launched == -(-B // C) * n1, (info.kernels_launched, n1, C)
    check_written(torch, many, B)
    edges = np.array([C - 1, C, 2 * C - 1, 2 * C, B - 1])
    check_cpu(torch, mech, ins, many, edge_cols(B, C), dtype, f"atlas chunks of {C} {dtype_name}")
    check_oracle(torch, mech, x, many, edges, dtype)
    for k in one:
        assert torch.equal(one[k][:, :B], many[k][:, :B]), k


@pytest.mark.gpu
def test_chunk_cap_keeps_pairs_grid_in_range(torch, monkeypatch):
    """A one-revolute model in fp32 with a 4096 MiB budget: without the cap a chunk would hold 2^23 + 4096 samples, 65568 blocks
    of deriv_pairs_kernel in grid.y."""
    if torch.cuda.mem_get_info()[0] < (6 << 30):
        pytest.skip("needs 6 GB of free device memory")
    mech = chain_model(1)
    _, nv, nnz, rows = tables(mech)
    monkeypatch.setenv("RBD_DERIV_SCRATCH_MB", "4096")
    x = inputs(mech, 1 << 16, 90)          # one chunk, and the forward-dynamics kernel of the large chunks (B >= 2^15)
    st, msg, _, _, info = call(torch, mech, x, 1 << 16, 1 << 16, torch.float32)
    assert st == 0, msg
    n1 = info.kernels_launched
    B = (1 << 23) + 4096
    C = chunk(rows, 4, B, 4096)
    rng = np.random.default_rng(91)
    x = {"q": rng.uniform(-np.pi, np.pi, (1, B)), "v": rng.standard_normal((1, B)), "tau": rng.standard_normal((1, B))}
    st, msg, ins, outs, info = call(torch, mech, x, B, B, torch.float32)
    assert st == 0, msg
    assert info.kernels_launched == 2 * n1 and -(-B // C) == 2
    check_written(torch, outs, B)
    idx = edge_cols(B, C)
    check_cpu(torch, mech, ins, outs, idx, torch.float32, f"one revolute, chunks of {C}")


# ------------------------------------------------------------------------------------------------------------------
# 6. a NaN sample stays in its column
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("path", ["specialised", "shared", "scratch"])
def test_nan_sample_stays_in_its_column(torch, monkeypatch, path):
    mech = atlas()
    _, nv, nnz, _ = tables(mech)
    B = JIT_MIN_BATCH + 77
    if path != "specialised":
        monkeypatch.setenv("RBD_DERIV_JIT", "0")
    if path == "scratch":
        monkeypatch.setenv("RBD_DERIV_GLOBAL_FACTOR", "1")
    x = inputs(mech, B, 100)
    st, msg, ins, clean, info = call(torch, mech, x, B, B, torch.float64)
    assert st == 0, msg
    if path == "specialised":
        assert_jit(info, nv, nnz, 8)
    else:
        assert_generic(torch, info, nv, nnz, 8, scratch_factor=path == "scratch")
    j = 32 * 50 + 16                       # the middle of a 32-sample group
    bad = {k: t.clone() for k, t in ins.items()}
    bad["q"][:, j] = float("nan")
    st, msg, _, got, _ = call(torch, mech, None, B, B, torch.float64, bad)
    assert st == 0, msg
    for k in got:
        assert torch.equal(got[k][:, :j], clean[k][:, :j]) and torch.equal(got[k][:, j + 1:], clean[k][:, j + 1:]), k
        assert bool(torch.isnan(got[k][:, j]).any()), k


# ------------------------------------------------------------------------------------------------------------------
# 7. 64-bit offsets in the outputs
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_outputs_beyond_2_pow_31_elements(torch):
    """Atlas fp32 with nv^2 B > 2^31: the last rows of dq / dv lie beyond 32-bit element offsets."""
    mech = atlas()
    _, nv, _, _ = tables(mech)
    B = (1 << 31) // (nv * nv) + 4096
    if torch.cuda.mem_get_info()[0] < (24 << 30):
        pytest.skip("needs 24 GB of free device memory")
    x = inputs(mech, B, 110)
    st, msg, ins, outs, _ = call(torch, mech, x, B, B, torch.float32)
    assert st == 0, msg
    idx = np.array([0, B // 2, B - 2, B - 1])
    check_cpu(torch, mech, ins, outs, idx, torch.float32, f"atlas fp32 B={B}")
    assert bool(torch.isfinite(outs["dq"][-nv:]).all()) and bool(torch.isfinite(outs["dv"][-nv:]).all())
