"""GPU tier: the CUDA path, called through the C ABI, against the CPU oracle on identical seeded inputs.

Tolerances (stated per SURVEY 8(d) 'Accuracy', metric = max_b |x_gpu - x_oracle64|_inf / max(1, |x_oracle64|_inf)):
  fp64: 1e-9   (the reference's own FD/ID tolerance is 1e-10 absolute on O(1) values, test_mechanism_algorithms.jl:739;
                here |v̇| reaches 1e3-1e4 on Atlas' light distal links, hence the relative form)
  fp32: 2e-5   (the reference's fp32 CRBA + Cholesky path itself is ~3e-4, tests/test_hostsim.py)
"""
import numpy as np
import pytest
import torch

import rigidbodydynamics.jl_b200 as rbd
from oracle import Oracle
from tests.util import axis_aligned_tree, config_distance, make_duals, rand_inputs, randmech, rel_err

pytestmark = pytest.mark.gpu
TOL = {torch.float64: 1e-9, torch.float32: 2e-5}


def gpu_dynamics(mech, q, v, tau, dtype, wext=None, want_qd=True):
    B = q.shape[1]
    state = rbd.MechanismState(mech, B, dtype)
    state.q.copy_(torch.from_numpy(q).to(dtype))
    state.v.copy_(torch.from_numpy(v).to(dtype))
    t = None if tau is None else torch.from_numpy(tau).to(dtype).cuda()
    w = None if wext is None else torch.from_numpy(wext).to(dtype).cuda()
    res = rbd.DynamicsResult(mech, B, dtype)
    rbd.dynamics_(res, state, t, w, want_qd=want_qd)
    torch.cuda.synchronize()
    return res.vd.double().cpu().numpy(), res.qd.double().cpu().numpy()


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("name,floating", [("atlas", True), ("atlas", False), ("valkyrie", True), ("iiwa14", False),
                                           ("double_pendulum", False)])
def test_dynamics_matches_oracle(built, name, floating, dtype):
    mech = rbd.load_model(name, floating=floating)
    q, v, tau, _, _ = rand_inputs(mech, 193, 17)
    ref, ref_qd = Oracle(mech.flatten()).dynamics(q, v, tau, want_qd=True)
    got, got_qd = gpu_dynamics(mech, q, v, tau, dtype)
    assert rel_err(got, ref) < TOL[dtype]
    assert np.abs(got_qd - ref_qd).max() < (1e-12 if dtype == torch.float64 else 1e-5)


def test_quickstart_numbers_on_gpu(built):
    """Config 1 (examples/1 quick start): v̇ for q=(0.3,0.4), v=(1,2), tau=0 -- SURVEY 8(c)(1)."""
    from tests.util import double_pendulum
    mech = double_pendulum()
    got, _ = gpu_dynamics(mech, np.array([[0.3], [0.4]]), np.array([[1.0], [2.0]]), None, torch.float64)
    assert np.allclose(got.ravel(), [2.935110215118255, -17.068157341777777], atol=1e-11)


@pytest.mark.parametrize("B", [1, 31, 32, 33, 1000])
def test_ragged_batch_sizes(built, B):
    mech = rbd.load_model("atlas", floating=True)
    q, v, tau, _, _ = rand_inputs(mech, B, B)
    ref = Oracle(mech.flatten()).dynamics(q, v, tau)
    got, _ = gpu_dynamics(mech, q, v, tau, torch.float64)
    assert got.shape == ref.shape and rel_err(got, ref) < 1e-9


@pytest.mark.parametrize("seed", range(4))
def test_general_trees_all_joint_types(built, seed):
    mech = randmech(seed, shuffle=seed % 2 == 1)
    q, v, tau, _, _ = rand_inputs(mech, 65, seed)
    ref, ref_qd = Oracle(mech.flatten()).dynamics(q, v, tau, want_qd=True)
    for dtype in (torch.float64, torch.float32):
        got, got_qd = gpu_dynamics(mech, q, v, tau, dtype)
        assert rel_err(got, ref) < (1e-9 if dtype == torch.float64 else 1e-3)
        assert np.abs(got_qd - ref_qd).max() < (1e-12 if dtype == torch.float64 else 1e-5)


def test_host_pointer_entry_point(built):
    """rbd_dynamics_host (pinned host buffers in, host buffers out, chunked copies inside) == device-pointer path."""
    mech = rbd.load_model("atlas", floating=True)
    B = (1 << 16) + 777                       # more than one chunk, ragged tail
    q, v, tau, _, _ = rand_inputs(mech, 64, 3)
    reps = -(-B // 64)
    q, v, tau = (np.tile(a, (1, reps))[:, :B].copy() for a in (q, v, tau))
    got_dev, _ = gpu_dynamics(mech, q, v, tau, torch.float32, want_qd=False)
    lib = rbd.load_library()
    state = rbd.MechanismState(mech, 1, torch.float32)
    hq, hv, ht = (torch.from_numpy(a).float().pin_memory() for a in (q, v, tau))
    out = torch.empty((36, B), dtype=torch.float32).pin_memory()
    rbd._cabi.check(lib.rbd_dynamics_host(state.handle.ptr, 0, B, B, hq.data_ptr(), hv.data_ptr(), ht.data_ptr(), None,
                                          out.data_ptr(), None))
    assert np.array_equal(out.numpy().astype(np.float64), got_dev)
    # two chunks, one kernel each (each followed by the gated generic fallback when the model-specialised kernel serves the call)
    assert 2 <= rbd.launch_info().kernels_launched <= 4


def test_errors_match_reference_behaviour(built):
    mech = rbd.load_model("iiwa14")
    state = rbd.MechanismState(mech, 8, torch.float32)
    res = rbd.DynamicsResult(mech, 8, torch.float32)
    with pytest.raises(rbd.DimensionMismatch):
        rbd.dynamics_(res, state, torch.zeros((6, 8), dtype=torch.float32, device="cuda"))
    # a Mechanism edited after the state was built -> ModificationCountMismatch (util.jl:56-72)
    mech.attach(mech.bodies[-1], rbd.RigidBody("tool", rbd.SpatialInertia.rand(np.random.default_rng(0))),
                rbd.Joint("tool_joint", rbd.Fixed()))
    with pytest.raises(rbd.RbdError) as e:
        rbd.dynamics_(res, state)
    assert e.value.status == rbd._cabi.RBD_ESTALE


def test_full_size_properties(built):
    """At BASELINE.json's full batch (2^20, fp32): size-independent checks -- every output finite, sample b's result does not
    depend on the batch it sits in (re-evaluating slices reproduces it bit-for-bit), and a strided sub-sample matches the oracle."""
    mech = rbd.load_model("atlas", floating=True)
    B = 1 << 20
    rng = np.random.default_rng(1)
    state = rbd.MechanismState(mech, B, torch.float32)
    rbd.rand_(state, rng)
    tau = torch.rand((36, B), dtype=torch.float32, device="cuda")
    res = rbd.DynamicsResult(mech, B, torch.float32)
    rbd.dynamics_(res, state, tau, want_qd=False)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(res.vd).all())
    idx = torch.arange(0, B, 4099, device="cuda")
    sub = rbd.MechanismState(mech, idx.numel(), torch.float32)
    sub.q.copy_(state.q[:, idx]); sub.v.copy_(state.v[:, idx])
    res2 = rbd.DynamicsResult(mech, idx.numel(), torch.float32)
    rbd.dynamics_(res2, sub, tau[:, idx].contiguous(), want_qd=False)
    assert torch.equal(res2.vd, res.vd[:, idx])
    ref = Oracle(mech.flatten()).dynamics(sub.q.double().cpu().numpy(), sub.v.double().cpu().numpy(),
                                          tau[:, idx].double().cpu().numpy())
    assert rel_err(res2.vd.double().cpu().numpy(), ref) < 2e-5


def _state(mech, q, v, dtype):
    st = rbd.MechanismState(mech, q.shape[1], dtype)
    st.q.copy_(torch.from_numpy(q).to(dtype)); st.v.copy_(torch.from_numpy(v).to(dtype))
    return st


def _cu(a, dtype):
    return None if a is None else torch.from_numpy(a).to(dtype).cuda()


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("name,floating", [("atlas", True), ("atlas", False), ("iiwa14", False), ("double_pendulum", False)])
def test_inverse_dynamics_bias_mass_matrix(built, name, floating, dtype):
    """inverse_dynamics!, dynamics_bias!, mass_matrix! (+ external wrenches) vs the oracle.  fp32 tolerance 2e-5 relative."""
    mech = rbd.load_model(name, floating=floating)
    o = Oracle(mech.flatten())
    q, v, tau, vd, w = rand_inputs(mech, 130, 31, wext=True)
    st = _state(mech, q, v, dtype)
    tol = TOL[dtype]
    for wext in (None, w):
        got = rbd.inverse_dynamics(st, _cu(vd, dtype), _cu(wext, dtype)).double().cpu().numpy()
        assert rel_err(got, o.inverse_dynamics(q, v, vd, wext)) < tol
        got = rbd.dynamics_bias(st, _cu(wext, dtype)).double().cpu().numpy()
        assert rel_err(got, o.dynamics_bias(q, v, wext)) < tol
        res = rbd.DynamicsResult(mech, q.shape[1], dtype)
        rbd.dynamics_(res, st, _cu(tau, dtype), _cu(wext, dtype))
        assert rel_err(res.vd.double().cpu().numpy(), o.dynamics(q, v, tau, wext)) < tol
    M = rbd.mass_matrix(st).double().cpu().numpy()
    assert rel_err(M, o.mass_matrix(q)) < tol


def test_quickstart_closed_form_values_gpu(built):
    """Config 1 numbers through the CUDA path: M, c, inverse dynamics of the examples/1 pendulum (SURVEY 8(c)(1))."""
    from tests.util import double_pendulum
    mech = double_pendulum()
    st = _state(mech, np.array([[0.3], [0.4]]), np.array([[1.0], [2.0]]), torch.float64)
    M = rbd.mass_matrix(st).cpu().numpy().reshape(2, 2)
    assert np.allclose(M, [[2.587060994002885, 0.7935304970014425], [0.7935304970014425, 0.333]], atol=1e-12)
    assert np.allclose(rbd.dynamics_bias(st).cpu().numpy().ravel(), [5.950794227687885, 3.3545969270552], atol=1e-12)
    vd = torch.tensor([[1.0], [2.0]], dtype=torch.float64, device="cuda")
    assert np.allclose(rbd.inverse_dynamics(st, vd).cpu().numpy().ravel(), [10.124916215693656, 4.814127424056642], atol=1e-12)


@pytest.mark.parametrize("seed", range(3))
def test_general_trees_rnea_crba_wext(built, seed):
    mech = randmech(seed, shuffle=seed % 2 == 1)
    o = Oracle(mech.flatten())
    q, v, tau, vd, w = rand_inputs(mech, 40, seed, wext=True)
    st = _state(mech, q, v, torch.float64)
    assert rel_err(rbd.inverse_dynamics(st, _cu(vd, torch.float64), _cu(w, torch.float64)).cpu().numpy(),
                   o.inverse_dynamics(q, v, vd, w)) < 1e-10
    assert rel_err(rbd.mass_matrix(st).cpu().numpy(), o.mass_matrix(q)) < 1e-10
    res = rbd.DynamicsResult(mech, q.shape[1], torch.float64)
    rbd.dynamics_(res, st, _cu(tau, torch.float64), _cu(w, torch.float64))
    assert rel_err(res.vd.cpu().numpy(), o.dynamics(q, v, tau, w)) < 1e-9


def test_identities_at_scale_fp32(built):
    """Reference identities at a large batch (2^17, fp32, iiwa14 = config 3): FD o ID round trip and M v̇ + c = tau."""
    mech = rbd.load_model("iiwa14")
    B = 1 << 17
    st = rbd.MechanismState(mech, B, torch.float32)
    rbd.rand_(st, np.random.default_rng(7))
    tau = torch.rand((7, B), dtype=torch.float32, device="cuda")
    res = rbd.DynamicsResult(mech, B, torch.float32)
    rbd.dynamics_(res, st, tau)
    back = rbd.inverse_dynamics(st, res.vd)
    scale = 1 + tau.abs().amax(0) + back.abs().amax(0)
    assert float(((back - tau).abs().amax(0) / scale).max()) < 1e-3
    M = rbd.mass_matrix(st).reshape(7, 7, B)
    c = rbd.dynamics_bias(st)
    resid = torch.einsum("jib,jb->ib", M, res.vd) + c - tau
    assert float((resid.abs().amax(0) / scale).max()) < 1e-3
    assert bool(torch.equal(M, M.transpose(0, 1)))


def test_host_entry_points_rnea_crba(built):
    mech = rbd.load_model("iiwa14")
    lib = rbd.load_library()
    B = 70000
    q, v, tau, vd, _ = rand_inputs(mech, 50, 5)
    reps = -(-B // 50)
    q, v, vd = (np.tile(a, (1, reps))[:, :B].copy() for a in (q, v, vd))
    st = _state(mech, q, v, torch.float32)
    ref_tau = rbd.inverse_dynamics(st, _cu(vd, torch.float32)).cpu()
    ref_M = rbd.mass_matrix(st).cpu()
    hq, hv, hvd = (torch.from_numpy(a).float().pin_memory() for a in (q, v, vd))
    out = torch.empty((7, B), dtype=torch.float32).pin_memory()
    rbd._cabi.check(lib.rbd_inverse_dynamics_host(st.handle.ptr, 0, B, B, hq.data_ptr(), hv.data_ptr(), hvd.data_ptr(), None, out.data_ptr()))
    assert torch.equal(out, ref_tau)
    outM = torch.empty((49, B), dtype=torch.float32).pin_memory()
    rbd._cabi.check(lib.rbd_mass_matrix_host(st.handle.ptr, 0, B, B, hq.data_ptr(), outM.data_ptr()))
    assert torch.equal(outM, ref_M)


@pytest.mark.parametrize("name,floating,B", [("atlas", True, 8192), ("iiwa14", False, 1000)])
def test_dual_number_dynamics_gpu(built, name, floating, B):
    """Config 4 (Atlas ABA with ForwardDiff.Dual{Tag,Float64,6} inputs, batch 8192): values and all 6 partials vs the oracle's
    dual-number run of the reference's algorithm on a sub-sample, plus finite differences; tolerance 1e-8 relative."""
    mech = rbd.load_model(name, floating=floating)
    o = Oracle(mech.flatten())
    q, v, tau, _, _ = rand_inputs(mech, 64, 4)
    reps = -(-B // 64)
    q, v, tau = (np.tile(a, (1, reps))[:, :B].copy() for a in (q, v, tau))
    Q, V, T = make_duals(mech, q, v, tau, 5)
    st = rbd.MechanismState(mech, 1, torch.float64)
    out = torch.full((st.nv, B, 7), float("nan"), dtype=torch.float64, device="cuda")
    rbd.dynamics_dual_(out, st, torch.from_numpy(Q).cuda(), torch.from_numpy(V).cuda(), torch.from_numpy(T).cuda())
    got = out.cpu().numpy()
    assert not np.isnan(got).any()
    n = 96
    ref = o.dynamics_dual6(Q[:, :n], V[:, :n], T[:, :n])
    assert np.abs(got[:, :n, 0] - ref[..., 0]).max() / np.abs(ref[..., 0]).max() < 1e-10
    assert np.abs(got[:, :n, 1:] - ref[..., 1:]).max() / np.abs(ref[..., 1:]).max() < 1e-8
    # the value part equals the plain fp64 kernel bit-for-bit
    st2 = _state(mech, q, v, torch.float64)
    res = rbd.DynamicsResult(mech, B, torch.float64)
    rbd.dynamics_(res, st2, _cu(tau, torch.float64), want_qd=False)
    # the value part is the plain fp64 kernel's result up to the different FMA contraction of Dual arithmetic
    scale = float(res.vd.abs().max())
    assert float((res.vd - out[..., 0]).abs().max()) < 1e-11 * scale


def test_edge_cases_empty_padded_and_defaults(built):
    """Edge cases of the C ABI: empty batch (no launch), leading dimension larger than the batch, default (NULL) torques,
    optional q̇ output, single-body model, and the largest supported model (64-body chain)."""
    lib = rbd.load_library()
    mech = rbd.load_model("iiwa14")
    o = Oracle(mech.flatten())
    st = rbd.MechanismState(mech, 1, torch.float64)
    # B = 0: RBD_OK, nothing launched
    z = torch.empty((7, 0), dtype=torch.float64, device="cuda")
    assert lib.rbd_dynamics(st.handle.ptr, 1, 0, 0, z.data_ptr(), z.data_ptr(), None, None, z.data_ptr(), None, None) == 0
    assert rbd.launch_info().kernels_launched == 0
    # ld > B: rows are 50 apart, only the first 37 columns are a batch
    B, ld = 37, 50
    q, v, tau, _, _ = rand_inputs(mech, B, 8)
    pad = lambda a: torch.from_numpy(np.pad(a, ((0, 0), (0, ld - B)), constant_values=np.nan)).cuda()
    Q, V, T = pad(q), pad(v), pad(tau)
    out = torch.full((7, ld), float("nan"), dtype=torch.float64, device="cuda")
    rbd._cabi.check(lib.rbd_dynamics(st.handle.ptr, 1, B, ld, Q.data_ptr(), V.data_ptr(), T.data_ptr(), None,
                                     out.data_ptr(), None, None))
    torch.cuda.synchronize()
    assert rel_err(out[:, :B].cpu().numpy(), o.dynamics(q, v, tau)) < 1e-9
    assert bool(torch.isnan(out[:, B:]).all())                       # the padding is never written
    # default torques (NULL) == zero torques
    got, _ = gpu_dynamics(mech, q, v, None, torch.float64)
    assert rel_err(got, o.dynamics(q, v, np.zeros_like(tau))) < 1e-9
    # one revolute body
    rng = np.random.default_rng(3)
    one = rbd.rand_chain_mechanism(rng, [rbd.Revolute])
    q1, v1, t1, _, _ = rand_inputs(one, 5, 1)
    got, _ = gpu_dynamics(one, q1, v1, t1, torch.float64)
    assert rel_err(got, Oracle(one.flatten()).dynamics(q1, v1, t1)) < 1e-10
    # RBD_MAX_BODIES-long chain (fp64 and fp32 kernels; a stash beyond 256 rows -> generic kernel)
    big = rbd.rand_chain_mechanism(rng, [rbd.Revolute] * 64)
    qb, vb, tb, _, _ = rand_inputs(big, 40, 2)
    ref = Oracle(big.flatten()).dynamics(qb, vb, tb)
    got, _ = gpu_dynamics(big, qb, vb, tb, torch.float64)
    assert rel_err(got, ref) < 1e-8
    got32, _ = gpu_dynamics(big, qb, vb, tb, torch.float32)
    assert rel_err(got32, ref) < 5e-3


def test_concurrent_streams_and_cuda_graph(built):
    """The plain entry points are asynchronous on the caller's stream: two streams evaluate different batches concurrently,
    and a call can be captured into a CUDA graph and replayed."""
    mech = rbd.load_model("atlas", floating=True)
    o = Oracle(mech.flatten())
    B = 1 << 16
    rng = np.random.default_rng(5)
    states, taus, results, streams = [], [], [], [torch.cuda.Stream(), torch.cuda.Stream()]
    for k in range(2):
        st = rbd.MechanismState(mech, B, torch.float32)
        rbd.rand_(st, rng)
        states.append(st)
        taus.append(torch.rand((36, B), dtype=torch.float32, device="cuda"))
        results.append(rbd.DynamicsResult(mech, B, torch.float32))
    torch.cuda.synchronize()
    for _ in range(3):
        for k in range(2):
            with torch.cuda.stream(streams[k]):
                rbd.dynamics_(results[k], states[k], taus[k], want_qd=False)
    torch.cuda.synchronize()
    for k in range(2):
        n = 64
        ref = o.dynamics(states[k].q[:, :n].double().cpu().numpy(), states[k].v[:, :n].double().cpu().numpy(),
                         taus[k][:, :n].double().cpu().numpy())
        assert rel_err(results[k].vd[:, :n].double().cpu().numpy(), ref) < 2e-5
    # CUDA graph: capture one evaluation, change the inputs in place, replay
    g = torch.cuda.CUDAGraph()
    expected = results[0].vd.clone()
    results[0].vd.zero_()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        rbd.dynamics_(results[0], states[0], taus[0], want_qd=False)      # warm-up outside capture
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            rbd.dynamics_(results[0], states[0], taus[0], want_qd=False)
    results[0].vd.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(results[0].vd, expected)
    taus[0].mul_(0.5)
    g.replay()
    torch.cuda.synchronize()
    n = 32
    ref = o.dynamics(states[0].q[:, :n].double().cpu().numpy(), states[0].v[:, :n].double().cpu().numpy(),
                     taus[0][:, :n].double().cpu().numpy())
    assert rel_err(results[0].vd[:, :n].double().cpu().numpy(), ref) < 2e-5


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_large_batch_matches_small_batch_path(built, dtype):
    """At batch 2^16 (config 2's size) the default path is one persistent kernel; whichever block evaluates a sample, the
    result must match the oracle and be bit-identical to the small-batch path on the same sample."""
    mech = rbd.load_model("atlas", floating=True)
    B = 1 << 16
    st = rbd.MechanismState(mech, B, dtype)
    rbd.rand_(st, np.random.default_rng(21))
    tau = torch.rand((36, B), dtype=dtype, device="cuda")
    res = rbd.DynamicsResult(mech, B, dtype)
    rbd.dynamics_(res, st, tau, want_qd=False)
    info = rbd.launch_info()
    # one kernel, plus -- when the fp32 model-specialised kernel serves the call -- the gated generic fallback behind it
    assert info.kernels_launched == (2 if info.specialised and dtype == torch.float32 else 1)
    idx = torch.arange(0, B, 509, device="cuda")
    sub = rbd.MechanismState(mech, idx.numel(), dtype)
    sub.q.copy_(st.q[:, idx]); sub.v.copy_(st.v[:, idx])
    res2 = rbd.DynamicsResult(mech, idx.numel(), dtype)
    rbd.dynamics_(res2, sub, tau[:, idx].contiguous(), want_qd=False)
    info2 = rbd.launch_info()
    assert info2.kernels_launched == (2 if info2.specialised and dtype == torch.float32 else 1)
    assert torch.equal(res2.vd, res.vd[:, idx])
    ref = Oracle(mech.flatten()).dynamics(sub.q.double().cpu().numpy(), sub.v.double().cpu().numpy(),
                                          tau[:, idx].double().cpu().numpy())
    assert rel_err(res2.vd.double().cpu().numpy(), ref) < TOL[dtype]


@pytest.mark.parametrize("name,floating", [("atlas", True), ("iiwa14", False)])
def test_simulate_rk4_matches_oracle(built, name, floating):
    """rbd_integrate = simulate() / MuntheKaasIntegrator with the RK4 tableau (SURVEY 8(f) rank 1): q, v after several steps
    vs the oracle's restatement; fp64 1e-9, fp32 1e-4 (quaternion sign-insensitive configuration distance)."""
    mech = rbd.load_model(name, floating=floating)
    o = Oracle(mech.flatten())
    q, v, tau, _, _ = rand_inputs(mech, 150, 14)
    qr, vr = o.integrate(q, v, tau, dt=1e-3, nsteps=5)
    for dtype, tq, tv in ((torch.float64, 1e-9, 1e-9), (torch.float32, 5e-5, 5e-4)):
        st = _state(mech, q, v, dtype)
        n = rbd.simulate_(st, 5e-3 - 1e-9, _cu(tau, dtype), dt=1e-3)
        assert n == 5
        assert config_distance(mech, st.q.double().cpu().numpy(), qr) < tq
        assert rel_err(st.v.double().cpu().numpy(), vr) < tv
    # passive (no torques) run keeps unit quaternions on the manifold
    st = _state(mech, q, v, torch.float64)
    rbd.simulate_(st, 0.01, None, dt=1e-3)
    if floating:
        assert float((st.q[:4].norm(dim=0) - 1).abs().max()) < 1e-12


def test_simulate_all_joint_types_and_energy(built):
    mech = randmech(2)
    o = Oracle(mech.flatten())
    q, v, tau, _, _ = rand_inputs(mech, 33, 3)
    qr, vr = o.integrate(q, v, tau, dt=5e-4, nsteps=3)
    st = _state(mech, q, v, torch.float64)
    rbd.simulate_(st, 1.5e-3 - 1e-9, _cu(tau, torch.float64), dt=5e-4)
    assert config_distance(mech, st.q.cpu().numpy(), qr) < 1e-9
    assert rel_err(st.v.cpu().numpy(), vr) < 1e-8
    # energy conservation of the passive double pendulum (test/test_simulate.jl:5-13, atol 1e-3), batch of 1000 on the GPU
    from tests.util import double_pendulum
    pend = double_pendulum()
    B = 1000
    stp = rbd.MechanismState(pend, B, torch.float64)
    rbd.rand_(stp, np.random.default_rng(60))

    def energy(s):
        M = rbd.mass_matrix(s).reshape(2, 2, B)
        ke = 0.5 * torch.einsum("ib,ijb,jb->b", s.v, M, s.v)
        z1 = -0.5 * torch.cos(s.q[0]); z2 = -torch.cos(s.q[0]) - 0.5 * torch.cos(s.q[0] + s.q[1])
        return ke + 9.81 * (z1 + z2)
    e0 = energy(stp)
    rbd.simulate_(stp, 0.1, None, dt=1e-2)
    assert float((energy(stp) - e0).abs().max()) < 1e-3


# ---- kinematics by-products (SURVEY 8(f) rank 2) ---------------------------------------------------------------------
KIN_NAMES = {"transforms": "transforms_to_root", "com": "center_of_mass", "ke": "kinetic_energy",
             "pe": "gravitational_potential_energy", "momentum": "momentum", "mrb": "momentum_rate_bias",
             "A": "momentum_matrix", "J": "geometric_jacobian"}


def _gpu_state(mech, q, v, dtype):
    state = rbd.MechanismState(mech, q.shape[1], dtype)
    state.q.copy_(torch.from_numpy(q).to(dtype))
    state.v.copy_(torch.from_numpy(v).to(dtype))
    return state


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("name,floating", [("atlas", True), ("valkyrie", False), ("iiwa14", False), ("double_pendulum", False)])
def test_kinematics_matches_oracle(built, name, floating, dtype):
    mech = rbd.load_model(name, floating=floating)
    desc = mech.flatten()
    q, v, _, _, _ = rand_inputs(mech, 257, 23)
    p = rbd.path(mech, mech.joints[-1].successor, mech.joints[min(2, desc.nb - 1)].successor)
    ref = Oracle(desc).kinematics(q, v, p.sign)
    state = _gpu_state(mech, q, v, dtype)
    outs = {KIN_NAMES[k]: torch.full((a.shape[0], q.shape[1]), float("nan"), dtype=dtype, device="cuda") for k, a in ref.items()}
    rbd.kinematics_(state, p, **outs)                     # fused: all eight outputs from one launch
    assert rbd.launch_info().kernels_launched == 1
    torch.cuda.synchronize()
    tol = 1e-11 if dtype == torch.float64 else 2e-5
    for k, a in ref.items():
        got = outs[KIN_NAMES[k]].double().cpu().numpy()
        assert np.abs(got - a).max() / max(1.0, np.abs(a).max()) < tol, k
    # the reference-named single-output calls
    assert np.allclose(rbd.center_of_mass(state).double().cpu().numpy(), ref["com"], atol=tol * 10)
    assert np.allclose(rbd.kinetic_energy(state).double().cpu().numpy(), ref["ke"][0], rtol=tol * 10, atol=tol * 10)
    assert np.allclose(rbd.gravitational_potential_energy(state).double().cpu().numpy(), ref["pe"][0], rtol=tol * 10, atol=tol * 10)
    assert np.allclose(rbd.momentum(state).double().cpu().numpy(), ref["momentum"], rtol=tol * 10, atol=tol * 10)
    assert np.allclose(rbd.momentum_rate_bias(state).double().cpu().numpy(), ref["mrb"], rtol=tol * 100, atol=tol * 100)
    assert np.allclose(rbd.momentum_matrix(state).double().cpu().numpy(), ref["A"], rtol=tol * 10, atol=tol * 10)
    assert np.allclose(rbd.geometric_jacobian(state, p).double().cpu().numpy(), ref["J"], atol=tol * 10)
    assert np.allclose(rbd.transforms_to_root(state).double().cpu().numpy(), ref["transforms"], atol=tol * 10)


@pytest.mark.parametrize("seed", [17, 18, 19])
def test_kinematics_all_joint_types(built, seed):
    mech = randmech(seed, shuffle=seed % 2 == 1)
    desc = mech.flatten()
    q, v, _, _, _ = rand_inputs(mech, 97, seed)
    rng = np.random.default_rng(seed)
    a, b = rng.choice(desc.nb, 2, replace=False)
    p = rbd.path(mech, mech.joints[a].successor, mech.joints[b].successor)
    ref = Oracle(desc).kinematics(q, v, p.sign)
    state = _gpu_state(mech, q, v, torch.float64)
    outs = {KIN_NAMES[k]: torch.empty((r.shape[0], q.shape[1]), dtype=torch.float64, device="cuda") for k, r in ref.items()}
    rbd.kinematics_(state, p, **outs)
    torch.cuda.synchronize()
    for k, r in ref.items():
        assert np.abs(outs[KIN_NAMES[k]].cpu().numpy() - r).max() / max(1.0, np.abs(r).max()) < 1e-11, k


def test_kinematics_identities_at_scale_and_errors(built):
    """Atlas, fp32, 2^18 samples: 1/2 v'Mv = KE and A v = momentum (size-independent properties); error behaviour."""
    mech = rbd.load_model("atlas", floating=True)
    B = 1 << 18
    state = rbd.MechanismState(mech, B, torch.float32)
    rng = np.random.default_rng(3)
    rbd.rand_(state, rng)
    nv = state.nv
    ke = rbd.kinetic_energy(state)
    A = rbd.momentum_matrix(state).view(nv, 6, B)
    h = rbd.momentum(state)
    M = rbd.mass_matrix(state).view(nv, nv, B)
    torch.cuda.synchronize()
    ke2 = 0.5 * torch.einsum("ib,ijb,jb->b", state.v.double(), M.double(), state.v.double())
    assert float(((ke.double() - ke2).abs() / ke2.abs().clamp(min=1)).max()) < 1e-4
    Av = torch.einsum("kcb,kb->cb", A.double(), state.v.double())
    assert float(((Av - h.double()).abs().max(0).values / h.double().abs().max(0).values.clamp(min=1)).max()) < 1e-4
    # errors: wrong size -> DimensionMismatch; jacobian without a path; path of another mechanism
    with pytest.raises(rbd.DimensionMismatch):
        rbd.kinematics_(state, None, center_of_mass=torch.empty((4, B), dtype=torch.float32, device="cuda"))
    with pytest.raises(ValueError):
        rbd.kinematics_(state, None, geometric_jacobian=torch.empty((6 * nv, B), dtype=torch.float32, device="cuda"))
    lib = rbd.load_library()
    from rigidbodydynamics.jl_b200 import _cabi
    ko = _cabi.RbdKinematicsOut()
    ko.kinetic_energy = ke.data_ptr()
    import ctypes
    rc = lib.rbd_kinematics(state.handle.ptr, 0, B, B, state.q.data_ptr(), None, None, ctypes.byref(ko), None)
    assert rc == _cabi.RBD_EINVAL                                    # kinetic energy without v
    assert lib.rbd_kinematics(state.handle.ptr, 2, B, B, state.q.data_ptr(), None, None, ctypes.byref(ko), None) == _cabi.RBD_EUNSUPPORTED
    assert lib.rbd_kinematics(state.handle.ptr, 0, 0, 0, None, None, None, ctypes.byref(ko), None) == _cabi.RBD_OK


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_large_batch_rnea_and_extwrench_match_small_batch_path(built, dtype):
    """inverse_dynamics! (with and without external wrenches) and dynamics! with external wrenches at batch 2^16: results must
    be bit-identical to the small-batch path on the same samples and match the oracle."""
    mech = rbd.load_model("atlas", floating=True)
    desc = mech.flatten()
    B = 1 << 16
    st = rbd.MechanismState(mech, B, dtype)
    rbd.rand_(st, np.random.default_rng(22))
    g = torch.Generator(device="cuda").manual_seed(5)
    vd = torch.rand((36, B), dtype=dtype, device="cuda", generator=g)
    tau = torch.rand((36, B), dtype=dtype, device="cuda", generator=g)
    wext = torch.rand((6 * desc.nb, B), dtype=dtype, device="cuda", generator=g)
    idx = torch.arange(0, B, 733, device="cuda")
    sub = rbd.MechanismState(mech, idx.numel(), dtype)
    sub.q.copy_(st.q[:, idx]); sub.v.copy_(st.v[:, idx])
    o = Oracle(desc)
    qn, vn = sub.q.double().cpu().numpy(), sub.v.double().cpu().numpy()
    vdn, taun, wn = (t[:, idx].double().cpu().numpy() for t in (vd, tau, wext))
    for w in (None, wext):
        out = torch.empty_like(vd)
        rbd.inverse_dynamics_(out, st, vd, w)
        # one kernel (for the fp32 model-specialised kernel, followed by the gated generic fallback)
        assert rbd.launch_info().kernels_launched in (1, 2)
        out2 = torch.empty((36, idx.numel()), dtype=dtype, device="cuda")
        rbd.inverse_dynamics_(out2, sub, vd[:, idx].contiguous(), None if w is None else w[:, idx].contiguous())
        assert rbd.launch_info().kernels_launched in (1, 2)
        assert torch.equal(out2, out[:, idx])
        ref = o.inverse_dynamics(qn, vn, vdn, None if w is None else wn)
        assert rel_err(out2.double().cpu().numpy(), ref) < TOL[dtype]
    res = rbd.DynamicsResult(mech, B, dtype)
    rbd.dynamics_(res, st, tau, wext, want_qd=False)
    assert rbd.launch_info().kernels_launched == 1
    res2 = rbd.DynamicsResult(mech, idx.numel(), dtype)
    rbd.dynamics_(res2, sub, tau[:, idx].contiguous(), wext[:, idx].contiguous(), want_qd=False)
    assert torch.equal(res2.vd, res.vd[:, idx])
    assert rel_err(res2.vd.double().cpu().numpy(), o.dynamics(qn, vn, taun, wn)) < TOL[dtype]


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_axis_aligned_trees_fast_classes_gpu(built, seed):
    """Random trees with coordinate-axis joints and 90-degree tree rotations (fast joint classes mixed with general bodies,
    prismatic / fixed / sin-cos joints, zero tree offsets), fp64 and fp32, with and without external wrenches."""
    mech = axis_aligned_tree(seed)
    desc = mech.flatten()
    q, v, tau, vd, w = rand_inputs(mech, 161, seed, wext=True)
    o = Oracle(desc)
    ref, ref_w, ref_id = o.dynamics(q, v, tau), o.dynamics(q, v, tau, w), o.inverse_dynamics(q, v, vd, w)
    for dtype in (torch.float64, torch.float32):
        got, _ = gpu_dynamics(mech, q, v, tau, dtype)
        assert rel_err(got, ref) < (1e-9 if dtype == torch.float64 else 5e-4)
        got_w, _ = gpu_dynamics(mech, q, v, tau, dtype, wext=w)
        assert rel_err(got_w, ref_w) < (1e-9 if dtype == torch.float64 else 5e-4)
        st = _gpu_state(mech, q, v, dtype)
        out = rbd.inverse_dynamics(st, torch.from_numpy(vd).to(dtype).cuda(), torch.from_numpy(w).to(dtype).cuda())
        assert rel_err(out.double().cpu().numpy(), ref_id) < (1e-9 if dtype == torch.float64 else 2e-4)


# ---- the reference's remaining identity tests through the GPU path (restated against the oracle in tests/test_oracle.py) ----
def test_external_wrench_momentum_balance_gpu(built):
    """test/test_mechanism_algorithms.jl:707-727 with tau from the GPU's inverse_dynamics! and the GPU's own kinematics by-products."""
    from tests.test_oracle import momentum_balance_residual
    rng = np.random.default_rng(39)
    mech = rbd.rand_floating_tree_mechanism(rng, [rbd.Revolute] * 10 + [rbd.Planar] * 10 + [rbd.SinCosRevolute] * 5)
    B = 40
    q, v, _, vd, w = rand_inputs(mech, B, 39, wext=True)
    st = _state(mech, q, v, torch.float64)
    tau = torch.empty((st.nv, B), dtype=torch.float64, device="cuda")
    rbd.inverse_dynamics_(tau, st, _cu(vd, torch.float64), _cu(w, torch.float64))
    outs = {"transforms_to_root": torch.empty((12 * len(mech.joints), B), dtype=torch.float64, device="cuda"),
            "center_of_mass": torch.empty((3, B), dtype=torch.float64, device="cuda"),
            "momentum_rate_bias": torch.empty((6, B), dtype=torch.float64, device="cuda"),
            "momentum_matrix": torch.empty((6 * st.nv, B), dtype=torch.float64, device="cuda")}
    rbd.kinematics_(st, None, **outs)
    torch.cuda.synchronize()
    kin = {"transforms": outs["transforms_to_root"].cpu().numpy(), "com": outs["center_of_mass"].cpu().numpy(),
           "mrb": outs["momentum_rate_bias"].cpu().numpy(), "A": outs["momentum_matrix"].cpu().numpy()}
    taun = tau.cpu().numpy()
    for b in range(B):
        r = momentum_balance_residual(mech, q[:, b], v[:, b], vd[:, b], w[:, b], taun[:, b], {k: a[:, b] for k, a in kin.items()})
        assert np.abs(r).max() < 1e-9


def test_power_flow_gpu(built):
    """:773-798 with v̇, q̇ and the energies from the GPU path: tau . v + sum_b w_b . twist_b == dE/dt."""
    from tests.test_oracle import body_twists
    mech = randmech(43)
    o = Oracle(mech.flatten())
    B = 6
    q, v, tau, _, w = rand_inputs(mech, B, 43, wext=True)
    vd, qd = gpu_dynamics(mech, q, v, tau, torch.float64, wext=w)
    tw = body_twists(o, mech, q, v)
    power = np.einsum("ib,ib->b", tau, v) + np.einsum("ncb,ncb->b", w.reshape(-1, 6, B), tw)

    def energy(qq, vv):
        st = _state(mech, qq, vv, torch.float64)
        ke = torch.empty((1, B), dtype=torch.float64, device="cuda"); pe = torch.empty_like(ke)
        rbd.kinematics_(st, None, kinetic_energy=ke, gravitational_potential_energy=pe)
        return (ke + pe).cpu().numpy().ravel()
    h = 1e-6
    dE = (energy(q + h * qd, v + h * vd) - energy(q - h * qd, v - h * vd)) / (2 * h)
    assert np.allclose(power, dE, rtol=1e-6, atol=1e-5)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_free_rigid_body_closed_form_gpu(built, dtype):
    """Euler / Newton-Euler closed form of a single QuaternionFloating body (tests/test_oracle.py) through the GPU path."""
    from tests.test_oracle import free_body_closed_form, free_body_mechanism
    mech, J, c, m = free_body_mechanism(np.random.default_rng(7), True)
    q, v, _, _, _ = rand_inputs(mech, 70, 8)
    got, _ = gpu_dynamics(mech, q, v, None, dtype)
    ref = np.stack([free_body_closed_form(J, c, m, mech.gravitational_acceleration, q[:4, b], v[:, b]) for b in range(70)], 1)
    assert rel_err(got, ref) < (1e-11 if dtype == torch.float64 else 2e-5)


def test_config3_at_full_batch_gpu(built):
    """BASELINE config 3 at its stated size: 7-DoF arm, fp32, batch 2^20 -- inverse_dynamics! AND mass_matrix! against the oracle
    on a strided sub-sample (the oracle takes seconds for ~2000 samples), every entry finite, M symmetric to the last bit."""
    mech = rbd.load_model("iiwa14")
    B = 1 << 20
    st = rbd.MechanismState(mech, B, torch.float32)
    rbd.rand_(st, np.random.default_rng(3))
    vd = torch.rand((7, B), dtype=torch.float32, device="cuda")
    tau = torch.empty_like(vd)
    rbd.inverse_dynamics_(tau, st, vd)
    M = torch.empty((49, B), dtype=torch.float32, device="cuda")
    rbd.mass_matrix_(M, st)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(tau).all()) and bool(torch.isfinite(M).all())
    M3 = M.view(7, 7, B)
    assert torch.equal(M3, M3.transpose(0, 1))
    idx = torch.arange(0, B, 509, device="cuda")
    o = Oracle(mech.flatten())
    qn, vn, vdn = (t[:, idx].double().cpu().numpy() for t in (st.q, st.v, vd))
    assert rel_err(tau[:, idx].double().cpu().numpy(), o.inverse_dynamics(qn, vn, vdn)) < 2e-5
    assert rel_err(M[:, idx].double().cpu().numpy(), o.mass_matrix(qn)) < 2e-5


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_per_body_outputs_and_dynamics_byproducts_gpu(built, dtype):
    """The reference's per-body arguments of inverse_dynamics! (jointwrenchesout, accelerations) and the by-products dynamics!
    leaves in the DynamicsResult (massmatrix, dynamicsbias, accelerations, jointwrenches) against the oracle's caches."""
    tol = TOL[dtype] * (1 if dtype == torch.float64 else 5)
    for mech in (rbd.load_model("atlas", floating=True), randmech(3, shuffle=True)):
        o = Oracle(mech.flatten())
        B = 70
        q, v, tau, vd, w = rand_inputs(mech, B, 12, wext=True)
        st = _state(mech, q, v, dtype)
        nb6 = 6 * len(mech.joints)
        for wext in (None, w):
            out = torch.empty((st.nv, B), dtype=dtype, device="cuda")
            jw = torch.full((nb6, B), float("nan"), dtype=dtype, device="cuda"); acc = torch.full_like(jw, float("nan"))
            rbd.inverse_dynamics_(out, st, _cu(vd, dtype), _cu(wext, dtype), jointwrenchesout=jw, accelerations=acc)
            ra, rw = o.inverse_dynamics_bodies(q, v, vd, wext)
            assert rel_err(acc.double().cpu().numpy(), ra) < tol and rel_err(jw.double().cpu().numpy(), rw) < tol
        res = rbd.DynamicsResult(mech, B, dtype)
        rbd.dynamics_(res, st, _cu(tau, dtype), _cu(w, dtype), byproducts="all")
        vdn = res.vd.double().cpu().numpy()
        assert rel_err(vdn, o.dynamics(q, v, tau, w)) < tol
        assert rel_err(res.dynamicsbias.double().cpu().numpy(), o.dynamics_bias(q, v, w)) < tol
        assert rel_err(res.massmatrix.double().cpu().numpy(), o.mass_matrix(q)) < tol
        ra, rw = o.inverse_dynamics_bodies(q, v, vdn, w)               # at the v̇ the GPU returned
        assert rel_err(res.accelerations.double().cpu().numpy(), ra) < tol
        assert rel_err(res.jointwrenches.double().cpu().numpy(), rw) < tol
        # M v̇ + c = tau with the by-products themselves (what the reference's dynamics! solves)
        M = res.massmatrix.double().view(st.nv, st.nv, B)
        lhs = torch.einsum("jib,jb->ib", M, res.vd.double()) + res.dynamicsbias.double()
        assert rel_err(lhs.cpu().numpy(), tau) < (1e-8 if dtype == torch.float64 else 2e-3)


@pytest.mark.parametrize("name,floating", [("atlas", True), ("iiwa14", False)])
def test_mass_matrix_lower_triangle_only_gpu(built, name, floating):
    """rbd_mass_matrix_uplo(RBD_UPLO_LOWER): exactly the lower triangle the reference's mass_matrix! fills, bit-identical to the
    full result there, everything above the diagonal left untouched."""
    mech = rbd.load_model(name, floating=floating)
    B = 300
    st = rbd.MechanismState(mech, B, torch.float64)
    rbd.rand_(st, np.random.default_rng(4))
    nv = st.nv
    full = rbd.mass_matrix(st).view(nv, nv, B)                   # [j, i, b] = entry (i, j)
    low = torch.full((nv * nv, B), float("nan"), dtype=torch.float64, device="cuda")
    rbd.mass_matrix_(low, st, uplo="L")
    low = low.view(nv, nv, B)
    jj, ii = torch.meshgrid(torch.arange(nv), torch.arange(nv), indexing="ij")
    lower = (ii >= jj).cuda()                                    # row i >= column j
    assert torch.equal(low[lower], full[lower])
    assert bool(torch.isnan(low[~lower]).all())


def test_simulate_with_torque_schedule_gpu(built):
    """rbd_integrate_schedule: time-varying open-loop torques without a host round trip per step.  A per-step schedule must equal
    calling simulate_ once per step with that step's torques (bit for bit), and a per-stage schedule whose four blocks are equal
    must equal the per-step one."""
    mech = rbd.load_model("atlas", floating=True)
    B, nsteps, dt = 96, 4, 1e-3
    q, v, _, _, _ = rand_inputs(mech, B, 15)
    g = torch.Generator(device="cuda").manual_seed(3)
    sched = torch.rand((nsteps, 36, B), dtype=torch.float64, device="cuda", generator=g)
    a = _state(mech, q, v, torch.float64)
    assert rbd.simulate_(a, nsteps * dt - 1e-9, sched, dt=dt) == nsteps
    b = _state(mech, q, v, torch.float64)
    for s in range(nsteps):
        rbd.simulate_(b, dt - 1e-9, sched[s].contiguous(), dt=dt)
    assert torch.equal(a.q, b.q) and torch.equal(a.v, b.v)
    c = _state(mech, q, v, torch.float64)
    rbd.simulate_(c, nsteps * dt - 1e-9, sched[:, None].expand(-1, 4, -1, -1).contiguous(), dt=dt)
    assert torch.equal(a.q, c.q) and torch.equal(a.v, c.v)
    # and against the oracle, step by step
    o = Oracle(mech.flatten())
    qr, vr = q, v
    for s in range(nsteps):
        qr, vr = o.integrate(qr, vr, sched[s].cpu().numpy(), dt=dt, nsteps=1)
    assert config_distance(mech, a.q.cpu().numpy(), qr) < 1e-9 and np.abs(a.v.cpu().numpy() - vr).max() < 1e-8
