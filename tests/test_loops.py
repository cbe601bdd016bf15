"""Mechanisms with kinematic loops (SURVEY 8(f) rank 4, second half): dynamics! with the constraint Jacobian, the Baumgarte bias and
the KKT solve.  CPU tier + GPU parity.

The host restatement (tests/loops_oracle.py: numpy / scipy over the CPU oracle, LAPACK gelsy for λ) is pinned by
  * the basis property of every joint type's constraint wrench subspace      test/test_mechanism_algorithms.jl:419-438
  * the reference's four-bar linkage simulation                                test/test_simulate.jl:127-227
  * the maximal-coordinates equivalence test                                   test/test_mechanism_modification.jl:274-318
  * the identities K v̇ = -k and M v̇ + c + K^T λ = τ
Then the kernel's per-sample function (csrc/rbd_loops.cuh compiled for the host) and the CUDA kernel through the C ABI must agree
with it.  λ is compared with the same wrench basis on both sides; for revolute / prismatic / sin-cos loop joints that basis depends on
Rotations.jl's rotation_between, which the reference tree does not contain, so there only v̇, K^T λ and the row space of K are the
reference's own.
"""
import ctypes

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from oracle import Oracle
from rigidbodydynamics.jl_b200 import _cabi
from rigidbodydynamics.jl_b200.spatial import Transform3D
from tests.loops_oracle import (FOUR_BAR_Q0, LoopOracle, atlas_double_support, body_accelerations, closure_distance, energy,
                                four_bar, hostsim_dynamics_loops, maximal_coordinate_pair, mc_state_from_tree)
from tests.util import rand_inputs, rel_err

# fp32 vs the fp64 oracle, relative.  Max measured: 1.9e-4 (λ, Atlas double support, 512 samples of a 2^20 batch on an H100,
# tools/time_loops.py); 3e-5 on the CPU tier's fixtures.
F32_TOL = 5e-4


def _four_bar_inputs(B, seed):
    rng = np.random.default_rng(seed)
    q = FOUR_BAR_Q0[:, None] + 0.2 * rng.standard_normal((3, B))
    return q, rng.standard_normal((3, B)), rng.standard_normal((3, B))


def _fixtures():
    """(name, mechanism, q, v, tau, wext) of the three parity cases."""
    out = []
    m = four_bar()
    q, v, tau = _four_bar_inputs(9, 1)
    out.append(("four_bar", m, q, v, tau, None))
    m = atlas_double_support()
    q, v, tau, _, w = rand_inputs(m, 6, 2, wext=True)
    out.append(("atlas_double_support", m, q, v, tau, w))
    for seed in (3, 4):
        _, mc, _ = maximal_coordinate_pair(seed, 12)
        q, v, tau, _, _ = rand_inputs(mc, 4, seed)
        out.append((f"maximal_coordinates_{seed}", mc, q, v, tau, None))
    return out


FIXTURES = _fixtures()


# ------------------------------------------------------------------------------------------------------------------
# CPU tier: the restatement
# ------------------------------------------------------------------------------------------------------------------
def _motion_subspace(jt):
    """motion_subspace in the frame after the joint (revolute.jl:44, prismatic.jl:49, planar.jl:87-93, quaternion_spherical.jl:52,
    floating: identity, fixed: none)."""
    z = np.zeros(3)
    if isinstance(jt, rbd.Fixed):
        return np.zeros((6, 0))
    if isinstance(jt, rbd.Prismatic):
        return np.concatenate([z, jt.axis])[:, None]
    if isinstance(jt, rbd.Revolute):
        return np.concatenate([jt.axis, z])[:, None]
    if isinstance(jt, rbd.Planar):
        return np.column_stack([np.concatenate([z, jt.x_axis]), np.concatenate([z, jt.y_axis]), np.concatenate([jt.rot_axis, z])])
    if isinstance(jt, rbd.QuaternionSpherical):
        return np.vstack([np.eye(3), np.zeros((3, 3))])
    return np.eye(6)


@pytest.mark.parametrize("jtype", [rbd.Revolute, rbd.Prismatic, rbd.SinCosRevolute, rbd.Fixed, rbd.Planar, rbd.QuaternionSpherical,
                                   rbd.QuaternionFloating, rbd.SPQuatFloating])
def test_constraint_wrench_subspace_is_the_complement(jtype):
    """test/test_mechanism_algorithms.jl:419-438: 6 - nv columns and T^T S = 0.  Both are constant in the frame after the joint
    (has_fixed_subspaces), so the configuration does not enter."""
    rng = np.random.default_rng(11)
    for _ in range(5):
        jt = jtype.rand(rng)
        T, S = rbd.constraint_wrench_subspace(jt), _motion_subspace(jt)
        assert T.shape == (6, 6 - jt.nv) and S.shape == (6, jt.nv)
        assert np.abs(T.T @ S).max(initial=0.0) <= 1e-12
        if T.shape[1]:
            assert np.linalg.matrix_rank(np.hstack([T, S])) == 6


def _rk4(f, q, v, dt, n):
    for _ in range(n):
        k1q, k1v = v, f(q, v)
        k2q, k2v = v + 0.5 * dt * k1v, f(q + 0.5 * dt * k1q, v + 0.5 * dt * k1v)
        k3q, k3v = v + 0.5 * dt * k2v, f(q + 0.5 * dt * k2q, v + 0.5 * dt * k2v)
        k4q, k4v = v + dt * k3v, f(q + dt * k3q, v + dt * k3v)
        q = q + dt / 6 * (k1q + 2 * k2q + 2 * k3q + k4q)
        v = v + dt / 6 * (k1v + 2 * k2v + 2 * k3v + k4v)
    return q, v


def test_four_bar_without_stabilization_on_the_oracle():
    """test_simulate.jl:199-209: from rest, 1 s at dt = 1e-3 (RK4; for an all-revolute mechanism the Munthe-Kaas steps are the
    plain ones): motion, energy conserved to 1e-8, no separation beyond 1e-10."""
    lo = LoopOracle(four_bar())
    q, v = FOUR_BAR_Q0[:, None].copy(), np.zeros((3, 1))
    e0 = energy(lo, q, v)
    q, v = _rk4(lambda q, v: lo.dynamics(q, v, stabilization_gains=None)["vd"], q, v, 1e-3, 1000)
    ke = lo.oracle.kinematics(q, v, want=("ke",))["ke"][0, 0]
    assert ke > 1e-2
    assert abs(energy(lo, q, v)[0] - e0[0]) <= 1e-8
    assert closure_distance(lo, q)[0] <= 1e-10


def test_four_bar_stabilization_with_the_device_code():
    """test_simulate.jl:211-226 with the default gains from the separated start (q1 = 1.7): separation <= 1e-5 after 15 s and the
    energy settles (drift <= 1e-5 over the next 10 s).  25 s of RK4 are 1e5 dynamics evaluations: they run on loops_sample compiled
    for the host (which matches the oracle to 1e-13 in test_hostsim_matches_the_oracle); the oracle checks the separation."""
    m = four_bar()
    lo = LoopOracle(m)
    q = FOUR_BAR_Q0.copy()
    q[0] = 1.7
    q, v = q[:, None], np.array([[0.5], [-0.47295], [0.341]])
    assert closure_distance(lo, q)[0] > 1e-2
    ld = rbd.loop_desc(m)

    def f(q, v):
        rc, out = hostsim_dynamics_loops(m, q, v, ld=ld)
        assert rc == 0
        return out["vd"]
    q, v = _rk4(f, q, v, 1e-3, 15000)
    assert closure_distance(lo, q)[0] <= 1e-5
    e15 = energy(lo, q, v)[0]
    q, v = _rk4(f, q, v, 1e-3, 10000)
    assert abs(energy(lo, q, v)[0] - e15) <= 1e-5


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_maximal_coordinates_on_the_oracle(seed):
    """test_mechanism_modification.jl:274-318: a random tree (every joint type, 12 bodies) and the same bodies floating with every
    tree joint as a loop joint (nl = 48 rows, full-rank A) give the same body accelerations relative to the root, to 1e-10."""
    tree, mc, bodymap = maximal_coordinate_pair(seed, 12)
    lt, lm = LoopOracle(tree), LoopOracle(mc)
    q, v, _, _, _ = rand_inputs(tree, 1, seed + 100)
    vd = lt.oracle.dynamics(q, v)
    qm, vm = mc_state_from_tree(tree, mc, bodymap, q[:, 0], v[:, 0])
    out = lm.dynamics(qm[:, None], vm[:, None])
    assert out["lam"].shape[0] == 48 and np.linalg.matrix_rank(out["A"][0]) == 48
    at = body_accelerations(lt, q, v, vd)
    am = body_accelerations(lm, qm[:, None], vm[:, None], out["vd"])
    for body, copy in bodymap.items():
        if body is tree.root_body:
            continue
        i, k = lt.index[id(body)], lm.index[id(copy)]
        assert np.abs(at[6 * i:6 * i + 6] - am[6 * k:6 * k + 6]).max() <= 1e-10


@pytest.mark.parametrize("case", range(len(FIXTURES)), ids=[f[0] for f in FIXTURES])
def test_identities_on_the_oracle(case):
    """K v̇ = -k, M v̇ + c + K^T λ = τ (mechanism_algorithms.jl:831-843)."""
    _, m, q, v, tau, w = FIXTURES[case]
    out = LoopOracle(m).dynamics(q, v, tau, w)
    nv = m.num_velocities()
    for b in range(q.shape[1]):
        K, M = out["Kb"][b], out["M"][:, b].reshape(nv, nv, order="F")
        scale = max(1.0, np.abs(out["vd"][:, b]).max())
        assert np.abs(K @ out["vd"][:, b] + out["k"][:, b]).max() <= 1e-8 * scale
        assert np.abs(M @ out["vd"][:, b] + out["c"][:, b] + K.T @ out["lam"][:, b] - tau[:, b]).max() <= 1e-8 * scale


def test_four_bar_rank_rule_drops_the_structural_zeros():
    """All axes along -y: three of the loop joint's five rows of K vanish identically, A has rank 2, and λ is gelsy's minimum-norm
    solution (zero in the dropped directions)."""
    m = four_bar()
    q, v, tau = _four_bar_inputs(4, 5)
    out = LoopOracle(m).dynamics(q, v, tau)
    for b in range(4):
        assert np.linalg.matrix_rank(out["A"][b], tol=1e-8 * np.abs(out["A"][b]).max()) == 2
    for dt, tol in ((np.float64, 1e-9), (np.float32, F32_TOL)):
        rc, h = hostsim_dynamics_loops(m, q.astype(dt), v, tau)
        assert rc == 0
        assert rel_err(h["lam"], out["lam"]) <= tol and rel_err(h["vd"], out["vd"]) <= tol


def test_no_loops_is_plain_dynamics():
    """nloops = 0: v̇ = M^-1 (τ - c), the reference's no-loop branch == Oracle.dynamics."""
    m = rbd.load_model("atlas", floating=True)
    q, v, tau, _, w = rand_inputs(m, 5, 7, wext=True)
    ref = Oracle(m.flatten()).dynamics(q, v, tau, w)
    assert rel_err(LoopOracle(m).dynamics(q, v, tau, w)["vd"], ref) <= 1e-10
    rc, h = hostsim_dynamics_loops(m, q, v, tau, w)
    assert rc == 0 and h["lam"].shape == (0, 5)
    assert rel_err(h["vd"], ref) <= 1e-9


@pytest.mark.parametrize("case", range(len(FIXTURES)), ids=[f[0] for f in FIXTURES])
def test_hostsim_matches_the_oracle(case):
    """loops_sample (csrc/rbd_loops.cuh) on the CPU: fp64 <= 1e-9 relative; fp32 <= F32_TOL."""
    _, m, q, v, tau, w = FIXTURES[case]
    ref = LoopOracle(m).dynamics(q, v, tau, w)
    qd_ref = Oracle(m.flatten()).dynamics(q, v, tau, w, want_qd=True)[1]
    for dt, tol in ((np.float64, 1e-9), (np.float32, F32_TOL)):
        rc, h = hostsim_dynamics_loops(m, q.astype(dt), v, tau, w)
        assert rc == 0
        for key in ("vd", "lam", "K", "k"):
            assert rel_err(h[key], ref[key]) <= tol, (dt, key, rel_err(h[key], ref[key]))
        assert rel_err(h["qd"], qd_ref) <= tol


def test_null_optional_outputs():
    """Only v̇ requested: the same v̇, and nothing is written through the NULL outputs."""
    _, m, q, v, tau, w = FIXTURES[1]
    rc, full = hostsim_dynamics_loops(m, q, v, tau, w)
    rc2, only = hostsim_dynamics_loops(m, q, v, tau, w, want=())
    assert rc == rc2 == 0 and np.array_equal(full["vd"], only["vd"])


def test_descriptor_errors(built):
    """rbd_dynamics_loops: RBD_EINVAL for malformed descriptors, RBD_EUNSUPPORTED beyond the limits and for Dual arrays; all are
    decided on the host before anything touches the device."""
    lib = rbd.load_library()
    m = four_bar()
    h = _cabi.ModelHandle(m.flatten())
    good = rbd.loop_desc(m)

    def call(ld, dtype=_cabi.RBD_F64):
        st, keep = ld.c_struct() if ld is not None else (None, None)
        return lib.rbd_dynamics_loops(h.ptr, dtype, 1, 1, None, None, None, None, ctypes.byref(st) if st is not None else None,
                                      None, None, None, None, None, None)

    def edited(**kw):
        d = rbd.LoopDesc(**{k: getattr(good, k) for k in ("predecessor", "successor", "joint_to_predecessor", "joint_to_successor",
                                                          "nconstraints", "wrench_basis", "gains")})
        for k, val in kw.items():
            setattr(d, k, val)
        return d

    assert call(None) == _cabi.RBD_EINVAL
    assert call(edited(successor=np.array([7], np.int32))) == _cabi.RBD_EINVAL          # out of range
    assert call(edited(predecessor=np.array([-2], np.int32))) == _cabi.RBD_EINVAL
    assert call(edited(successor=good.predecessor.copy())) == _cabi.RBD_EINVAL           # predecessor == successor
    assert call(edited(nconstraints=np.array([7], np.int32))) == _cabi.RBD_EINVAL
    assert call(good, _cabi.RBD_DUAL64X6) == _cabi.RBD_EUNSUPPORTED
    n = _cabi.RBD_MAX_LOOP_JOINTS + 1
    eye = np.tile(Transform3D.identity().flat12(), (n, 1))
    many = rbd.LoopDesc(np.full(n, -1, np.int32), np.zeros(n, np.int32), eye, eye, np.ones(n, np.int32), np.tile(np.eye(6)[:1], (n, 1)), None)
    assert call(many) == _cabi.RBD_EUNSUPPORTED
    assert call(good) == _cabi.RBD_EINVAL                                                   # q / v / vd_out NULL


def test_guarded_paths_refuse_loops_before_launching(built):
    """The paths that cannot honour loop constraints raise RBD_ELOOP (inverse_dynamics! does, mechanism_algorithms.jl:549) instead of
    evaluating the spanning tree; the state itself can be built."""
    m = four_bar()
    state = rbd.MechanismState(m, 2, device="cpu")
    result = rbd.DynamicsResult(m, 2, device="cpu")
    from rigidbodydynamics.jl_b200 import sharding
    calls = [lambda: rbd.inverse_dynamics_(state.v.clone(), state, state.v.clone()),
             lambda: rbd.inverse_dynamics(state, state.v.clone()),
             lambda: rbd.simulate_(state, 0.01),
             lambda: rbd.dynamics_derivatives_(state.v.clone(), state.v.clone(), result, state),
             lambda: rbd.dynamics_dual_(None, state, None, None),
             lambda: rbd.dynamics_contact_(result, state),
             lambda: sharding.dynamics_gather_(None, state)]
    for c in calls:
        with pytest.raises(rbd.RbdError) as e:
            c()
        assert e.value.status == _cabi.RBD_ELOOP and "tree Mechanisms" in str(e.value)


def test_attach_and_remove_fixed_tree_joints_keep_joint_to_successor():
    """attach stores inv(successor_pose) for a loop joint (mechanism_modification.jl:34) and the identity for tree joints;
    remove_fixed_tree_joints re-targets a loop joint welded through a Fixed tree joint and composes the weld's transform, which
    leaves the dynamics unchanged."""
    m = four_bar()
    assert np.allclose(m.findjoint("joint4").joint_to_successor.trans, [0.75, 0, 0])
    assert all(np.allclose(j.joint_to_successor.mat(), np.eye(4)) for j in m.joints)

    rng = np.random.default_rng(21)
    mech = rbd.Mechanism(rbd.RigidBody("world"))
    b1, b2 = rbd.RigidBody("b1", rbd.SpatialInertia.rand(rng)), rbd.RigidBody("b2", rbd.SpatialInertia.rand(rng))
    b3 = rbd.RigidBody("b3", rbd.SpatialInertia.rand(rng))
    mech.attach(mech.root_body, b1, rbd.Joint("j1", rbd.Revolute.rand(rng)), joint_pose=Transform3D.rand(rng))
    weld = Transform3D.rand(rng)
    mech.attach(b1, b2, rbd.Joint("weld", rbd.Fixed()), joint_pose=weld)
    mech.attach(b2, b3, rbd.Joint("j3", rbd.Revolute.rand(rng)), joint_pose=Transform3D.rand(rng))
    sp = Transform3D.rand(rng)
    mech.attach(mech.root_body, b2, rbd.Joint("loop", rbd.QuaternionSpherical()), joint_pose=Transform3D.rand(rng), successor_pose=sp)
    loop = mech.findjoint("loop")
    q, v, tau, _, _ = rand_inputs(mech, 3, 22)
    before = LoopOracle(mech).dynamics(q, v, tau)
    mech.remove_fixed_tree_joints()
    assert loop.successor is b1
    assert np.allclose(loop.joint_to_successor.mat(), (weld * sp.inv()).mat())
    after = LoopOracle(mech).dynamics(q, v, tau)
    assert rel_err(after["vd"], before["vd"]) <= 1e-10 and rel_err(after["lam"], before["lam"]) <= 1e-10


# ------------------------------------------------------------------------------------------------------------------
# GPU tier
# ------------------------------------------------------------------------------------------------------------------
def _state(m, q, v, dtype):
    import torch
    st = rbd.MechanismState(m, q.shape[1], dtype)
    st.q.copy_(torch.from_numpy(np.ascontiguousarray(q)))
    st.v.copy_(torch.from_numpy(np.ascontiguousarray(v)))
    return st


def _cuda(a, dtype):
    import torch
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dtype).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(FIXTURES)), ids=[f[0] for f in FIXTURES])
@pytest.mark.parametrize("prec", ["f64", "f32"])
def test_gpu_parity_with_the_oracle(built, case, prec):
    """v̇, q̇, λ, K, k against the oracle; fp64 <= 1e-9 relative, fp32 <= F32_TOL (first H100 run: see DESIGN.md 4.11)."""
    import torch
    name, m, q, v, tau, w = FIXTURES[case]
    dtype, tol = (torch.float64, 1e-9) if prec == "f64" else (torch.float32, F32_TOL)
    ref = LoopOracle(m).dynamics(q, v, tau, w)
    qd_ref = Oracle(m.flatten()).dynamics(q, v, tau, w, want_qd=True)[1]
    st = _state(m, q, v, dtype)
    res = rbd.DynamicsResult(m, q.shape[1], dtype)
    rbd.dynamics_loops_(res, st, _cuda(tau, dtype), _cuda(w, dtype))
    torch.cuda.synchronize()
    got = {"vd": res.vd, "qd": res.qd, "lam": res.lam, "K": res.constraintjacobian, "k": res.constraintbias}
    for key, r in (("vd", ref["vd"]), ("qd", qd_ref), ("lam", ref["lam"]), ("K", ref["K"]), ("k", ref["k"])):
        err = rel_err(got[key].double().cpu().numpy(), r)
        assert err <= tol, (name, prec, key, err)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["f64", "f32"])
def test_gpu_ragged_batch_leading_dimension_and_null_outputs(built, prec):
    """Atlas double support through the C ABI with B = 45 columns of an ld = 64 array and only v̇ requested: equal to the full
    call on the same columns, and the padding columns are left alone."""
    import torch
    dtype = torch.float64 if prec == "f64" else torch.float32
    m = atlas_double_support()
    B, ld = 45, 64
    q, v, tau, _, _ = rand_inputs(m, ld, 31)
    st = _state(m, q[:, :B], v[:, :B], dtype)
    res = rbd.DynamicsResult(m, B, dtype)
    rbd.dynamics_loops_(res, st, _cuda(tau[:, :B], dtype))
    lib = rbd.load_library()
    qg, vg, tg = _cuda(q, dtype), _cuda(v, dtype), _cuda(tau, dtype)
    vd = torch.full((m.num_velocities(), ld), 7.0, dtype=dtype, device="cuda")
    desc, keep = rbd.loop_desc(m).c_struct()
    rc = lib.rbd_dynamics_loops(st.handle.ptr, 1 if prec == "f64" else 0, B, ld, qg.data_ptr(), vg.data_ptr(), tg.data_ptr(), None,
                                ctypes.byref(desc), vd.data_ptr(), None, None, None, None, torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    assert torch.equal(vd[:, :B], res.vd)
    assert bool((vd[:, B:] == 7.0).all())


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["f64", "f32"])
def test_gpu_no_loops_matches_rbd_dynamics(built, prec):
    import torch
    dtype, tol = (torch.float64, 1e-9) if prec == "f64" else (torch.float32, 2e-4)
    m = rbd.load_model("atlas", floating=True)
    q, v, tau, _, w = rand_inputs(m, 100, 41, wext=True)
    st = _state(m, q, v, dtype)
    a, b = rbd.DynamicsResult(m, 100, dtype), rbd.DynamicsResult(m, 100, dtype)
    rbd.dynamics_(a, st, _cuda(tau, dtype), _cuda(w, dtype))
    rbd.dynamics_loops_(b, st, _cuda(tau, dtype), _cuda(w, dtype))
    torch.cuda.synchronize()
    assert rel_err(b.vd.double().cpu().numpy(), a.vd.double().cpu().numpy()) <= tol
    assert torch.equal(a.qd, b.qd)


@pytest.mark.gpu
def test_gpu_dynamics_dispatches_to_the_loop_solver(built):
    """dynamics_ on a mechanism with loops == dynamics_loops_ with the default gains, bit for bit."""
    import torch
    m = atlas_double_support()
    q, v, tau, _, _ = rand_inputs(m, 33, 51)
    st = _state(m, q, v, torch.float64)
    a, b = rbd.DynamicsResult(m, 33), rbd.DynamicsResult(m, 33)
    rbd.dynamics_(a, st, _cuda(tau, torch.float64))
    rbd.dynamics_loops_(b, st, _cuda(tau, torch.float64), stabilization_gains=rbd.default_constraint_stabilization_gains())
    torch.cuda.synchronize()
    assert torch.equal(a.vd, b.vd) and torch.equal(a.qd, b.qd) and torch.equal(a.lam, b.lam)


@pytest.mark.gpu
def test_gpu_four_bar_energy_and_closure(built):
    """test_simulate.jl:199-209 through the GPU path: 1 s from rest without stabilisation, RK4 at dt = 1e-3."""
    import torch
    m = four_bar()
    lo = LoopOracle(m)
    st = _state(m, FOUR_BAR_Q0[:, None], np.zeros((3, 1)), torch.float64)
    res = rbd.DynamicsResult(m, 1)
    ld = rbd.loop_desc(m, None)
    e0 = energy(lo, FOUR_BAR_Q0[:, None], np.zeros((3, 1)))[0]

    def f(q, v):
        st.q.copy_(q)
        st.v.copy_(v)
        rbd.dynamics_loops_(res, st, loops=ld, want_qd=False)
        return res.vd.clone()
    q, v = _rk4(f, st.q.clone(), st.v.clone(), 1e-3, 1000)
    qn, vn = q.cpu().numpy(), v.cpu().numpy()
    assert lo.oracle.kinematics(qn, vn, want=("ke",))["ke"][0, 0] > 1e-2
    assert abs(energy(lo, qn, vn)[0] - e0) <= 1e-8
    assert closure_distance(lo, qn)[0] <= 1e-10


@pytest.mark.gpu
def test_gpu_large_batch_atlas_double_support_fp32(built):
    """2^20 samples (the workspace is per resident thread, not per sample): a strided subsample against the oracle, and the same
    columns bit-identical to a small-batch run."""
    import torch
    m = atlas_double_support()
    B = 1 << 20
    rng = np.random.default_rng(61)
    st = rbd.MechanismState(m, B, torch.float32)
    rbd.rand_(st, rng)
    tau = torch.rand((st.nv, B), dtype=torch.float32, device="cuda")
    res = rbd.DynamicsResult(m, B, torch.float32)
    rbd.dynamics_loops_(res, st, tau)
    torch.cuda.synchronize()
    idx = torch.arange(5, B, 4099, device="cuda")
    q, v, t = (x[:, idx].contiguous() for x in (st.q, st.v, tau))
    ref = LoopOracle(m).dynamics(q.double().cpu().numpy(), v.double().cpu().numpy(), t.double().cpu().numpy())
    assert rel_err(res.vd[:, idx].double().cpu().numpy(), ref["vd"]) <= F32_TOL
    assert rel_err(res.lam[:, idx].double().cpu().numpy(), ref["lam"]) <= F32_TOL
    small_state = rbd.MechanismState(m, idx.numel(), torch.float32)
    small_state.q.copy_(q)
    small_state.v.copy_(v)
    small = rbd.DynamicsResult(m, idx.numel(), torch.float32)
    rbd.dynamics_loops_(small, small_state, t)
    torch.cuda.synchronize()
    assert torch.equal(small.vd, res.vd[:, idx]) and torch.equal(small.lam, res.lam[:, idx])
