"""simulate for mechanisms with kinematic loops (DESIGN 4.16): rbd_integrate_loops / simulate_loops_, with and without contact.

The host integrator below is the Munthe-Kaas RK4 step of tests/contact_oracle.py with LoopOracle.dynamics (tests/loops_oracle.py) as
the stage dynamics and Oracle.contact_dynamics' wrenches as its external wrenches -- dynamics! as mechanism_algorithms.jl:845-864 runs
it.  It is pinned on the CPU by
  * integrate_contact when there are no loops (the same step on the tree path),
  * the reference's four-bar test without stabilisation (test/test_simulate.jl:199-209).
The kernel's per-stage device code (loops_contact_sample compiled for the host: tests/hostsim/hostsim_loops_rollout.cpp) must agree
with the host integrator's stage dynamics, and the GPU rollout with the host integrator.
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
from rigidbodydynamics.jl_b200._cabi import RbdModelDesc, make_desc
from rigidbodydynamics.jl_b200.loops import _DEFAULT
from rigidbodydynamics.jl_b200.spatial import Transform3D
from tests.contact_oracle import RK4_A, RK4_B, global_coordinates, integrate_contact, local_rate
from tests.loops_oracle import (FOUR_BAR_Q0, LoopOracle, _pose, atlas_double_support, closure_distance, energy, four_bar,
                                maximal_coordinate_pair, mc_state_from_tree)
from tests.test_contact import _with_contacts
from tests.util import config_distance, rand_inputs, rel_err

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "..", "rigidbodydynamics", "jl_b200", "csrc")
_lib = None

TOL64 = 1e-9          # GPU rollout against the fp64 host integrator, relative (the contact rollout's bound)
# fp32 rollout against the fp64 host integrator, 5 steps at dt = 1e-3.  Measured on an H100: q 2.3e-7 / v 1.5e-7 (four-bar),
# 1.8e-7 / 1.3e-6 (Atlas double support), 4.1e-7 / 2.9e-6 (maximal coordinates), 2.2e-7 / 7.0e-6 (Atlas single support with
# contact), up to 5.0e-7 / 3.5e-5 for Atlas double support at 2^20 (two runs); the bound is the contact rollout's, 57x above the largest.
TOL32 = 2e-3
# Maximal-coordinate twin against the tree after 10 steps (pose gap, closure): tightened from 1e-6.  Measured on an H100: pose gap
# 2.7e-12 / 3.9e-13, position closure 2.3e-13 / 2.2e-13, velocity closure 2.8e-12 / 2.7e-12 (seeds 3 / 4).
MC_GAP = 1e-9


# ------------------------------------------------------------------------------------------------------------------
# the host integrator
# ------------------------------------------------------------------------------------------------------------------
def stage_dynamics(lo, q, v, s, cd, tau, gains=_DEFAULT):
    """dynamics! with loops and contact at one stage state: (v̇, ṡ) -- ṡ has 0 rows without contact."""
    wr, sd = None, np.zeros((0, q.shape[1]))
    if cd is not None and cd.nstates:
        wr, sd, _ = lo.oracle.contact_dynamics(q, v, cd, s)            # the reset does not survive the stage
    return lo.dynamics(q, v, tau, wr, stabilization_gains=gains)["vd"], sd


def integrate_loops_step(lo, q, v, s, cd, tau=None, dt=1e-4, stage_tau=None, gains=_DEFAULT):
    """One Munthe-Kaas RK4 step (contact_oracle.integrate_contact_step) with stage_dynamics; returns (q, v, s)."""
    desc = lo.desc
    q0, v0, s0 = np.array(q, float), np.array(v, float), np.array(s, float)
    phid, vd, sd = [None] * 4, [None] * 4, [None] * 4
    for i in range(4):
        wa = dt * RK4_A[i]
        phi = wa * phid[i - 1] if i else np.zeros_like(v0)
        vs = v0 + wa * vd[i - 1] if i else v0.copy()
        ss = s0 + wa * sd[i - 1] if i else s0.copy()
        qs = global_coordinates(desc, q0, phi)
        t = stage_tau(i) if stage_tau is not None else tau
        vd[i], sd[i] = stage_dynamics(lo, qs, vs, ss, cd, t, gains)
        qd = lo.oracle.dynamics(qs, vs, want_qd=True)[1]
        phid[i] = local_rate(desc, q0, qs, vs, qd)
    phi, vn, sn = np.zeros_like(v0), v0.copy(), s0.copy()
    for i in range(4):
        phi += dt * RK4_B[i] * phid[i]
        vn += dt * RK4_B[i] * vd[i]
    if s0.shape[0]:
        sn = s0 + dt * (RK4_B[0] * sd[0] + RK4_B[1] * sd[1] + RK4_B[2] * sd[2] + RK4_B[3] * sd[3])
    return global_coordinates(desc, q0, phi), vn, sn


def integrate_loops(lo, q, v, s, cd, tau=None, *, dt=1e-4, nsteps=1, gains=_DEFAULT):
    """``nsteps`` steps; ``tau``: None, constant [nv, B], per step [nsteps, nv, B] or per stage [nsteps, 4, nv, B]."""
    q, v = np.array(q, float), np.array(v, float)
    ns = 0 if cd is None else cd.nstates
    s = np.zeros((ns, q.shape[1])) if s is None else np.array(s, float)
    tau = None if tau is None else np.asarray(tau, float)
    for n in range(nsteps):
        if tau is None or tau.ndim == 2:
            q, v, s = integrate_loops_step(lo, q, v, s, cd, tau, dt, gains=gains)
        elif tau.ndim == 3:
            q, v, s = integrate_loops_step(lo, q, v, s, cd, tau[n], dt, gains=gains)
        else:
            q, v, s = integrate_loops_step(lo, q, v, s, cd, None, dt, stage_tau=lambda i, n=n: tau[n, i], gains=gains)
    return q, v, s


# ------------------------------------------------------------------------------------------------------------------
# fixtures
# ------------------------------------------------------------------------------------------------------------------
def _foot_model():
    return rbd.SoftContactModel(rbd.hunt_crossley_hertz(), rbd.ViscoelasticCoulombModel(0.8, 20e3, 100.0))


def atlas_single_support():
    """Atlas (floating base) with the left foot welded to the world (one Fixed loop joint, nl = 6) and 4 contact points on the
    right foot over the floor."""
    mech = rbd.load_model("atlas", floating=True)
    mech.attach(mech.root_body, mech.findbody("l_foot"), rbd.Joint("l_foot_weld", rbd.Fixed()),
                joint_pose=Transform3D(trans=(0.0, 0.12, 0.0)), successor_pose=Transform3D.identity())
    foot = mech.findbody("r_foot")
    for x in (-0.08, 0.17):
        for y in (-0.06, 0.06):
            rbd.add_contact_point(foot, rbd.ContactPoint(np.array([x, y, -0.08]), _foot_model()))
    rbd.add_environment_primitive(mech, rbd.HalfSpace3D(np.zeros(3), [0, 0, 1.0]))
    return mech, rbd.contact_desc(mech)


def atlas_on_floor():
    """Atlas without loops, 4 points under each foot, floor (as tests/test_contact_rollout.py)."""
    mech = rbd.load_model("atlas", floating=True)
    for foot in ("l_foot", "r_foot"):
        for x in (-0.08, 0.17):
            for y in (-0.06, 0.06):
                rbd.add_contact_point(mech.findbody(foot), rbd.ContactPoint(np.array([x, y, -0.08]), _foot_model()))
    rbd.add_environment_primitive(mech, rbd.HalfSpace3D(np.zeros(3), [0, 0, 1.0]))
    return mech, rbd.contact_desc(mech)


def atlas_states(mech, B, seed):
    """Atlas near upright, the pelvis at a height that puts the feet around the floor, small joint motion."""
    rng = np.random.default_rng(seed)
    q, v, tau, _, _ = rand_inputs(mech, B, seed)
    q[:4] = np.array([[1.0], [0], [0], [0]]) + 0.05 * rng.standard_normal((4, B)); q[:4] /= np.linalg.norm(q[:4], axis=0)
    q[4:6] = 0.02 * rng.standard_normal((2, B)); q[6] = 0.93 + 0.03 * rng.standard_normal(B)
    q[7:] *= 0.1; v *= 0.2
    return q, v, tau - 0.5


def four_bar_with_contact():
    """The four-bar with one point on link2 and a half-space that about half of the states of _four_bar_inputs penetrate."""
    mech = four_bar()
    rbd.add_contact_point(mech.findbody("link2"), rbd.ContactPoint(np.array([0.3, 0.0, 0.0]),
                                                                   rbd.SoftContactModel(rbd.hunt_crossley_hertz(k=1e3, alpha=0.2),
                                                                                        rbd.ViscoelasticCoulombModel(0.5, 100.0, 20.0))))
    rbd.add_environment_primitive(mech, rbd.HalfSpace3D([0.29, 0.0, 0.53], [0.2, 0.0, 1.0]))
    return mech, rbd.contact_desc(mech)


def _four_bar_inputs(B, seed):
    rng = np.random.default_rng(seed)
    q = FOUR_BAR_Q0[:, None] + 0.2 * rng.standard_normal((3, B))
    return q, rng.standard_normal((3, B)), rng.standard_normal((3, B))


def _case(which, B, seed):
    """(mechanism, contact desc or None, q, v, tau, s) of the rollout fixtures."""
    cd = None
    if which == "four_bar":
        mech = four_bar()
        q, v, tau = _four_bar_inputs(B, seed)
    elif which == "atlas_ds":
        mech = atlas_double_support()
        q, v, tau = atlas_states(mech, B, seed)
    elif which == "atlas_ss":
        mech, cd = atlas_single_support()
        q, v, tau = atlas_states(mech, B, seed)
    elif which.startswith("mc"):
        _, mech, _ = maximal_coordinate_pair(int(which[2:]), 12)
        q, v, tau, _, _ = rand_inputs(mech, B, seed)
    else:
        raise ValueError(which)
    s = None if cd is None else np.random.default_rng(seed).standard_normal((cd.nstates, B)) * 1e-3
    return mech, cd, q, v, tau, s


# ------------------------------------------------------------------------------------------------------------------
# CPU tier: the host integrator
# ------------------------------------------------------------------------------------------------------------------
def test_host_integrator_without_loops_is_integrate_contact():
    """No loops: the host integrator is contact_oracle.integrate_contact (KKT path = CRBA + Cholesky against the oracle's forward
    dynamics; Atlas' cond(M) ~ 5e5 leaves rounding above 1e-12)."""
    mech, cd = atlas_on_floor()
    q, v, tau = atlas_states(mech, 6, 4)
    s = np.random.default_rng(4).standard_normal((cd.nstates, 6)) * 1e-3
    lo = LoopOracle(mech)
    qr, vr, sr = integrate_contact(lo.oracle, q, v, s, cd, tau, dt=1e-3, nsteps=3)
    ql, vl, sl = integrate_loops(lo, q, v, s, cd, tau, dt=1e-3, nsteps=3)
    assert np.any(sr != s)
    assert config_distance(mech, ql, qr) < 1e-10 and rel_err(vl, vr) < 1e-10
    assert np.abs(sl - sr).max() < 1e-10 * max(1.0, np.abs(sr).max())


def test_host_integrator_four_bar_without_stabilization():
    """test_simulate.jl:199-209 on the host integrator: from rest, 1 s at dt = 1e-3 without stabilisation: motion, energy conserved
    to 1e-8, no separation beyond 1e-10."""
    lo = LoopOracle(four_bar())
    q, v = FOUR_BAR_Q0[:, None].copy(), np.zeros((3, 1))
    e0 = energy(lo, q, v)[0]
    q, v, _ = integrate_loops(lo, q, v, None, None, dt=1e-3, nsteps=1000, gains=None)
    assert lo.oracle.kinematics(q, v, want=("ke",))["ke"][0, 0] > 1e-2
    assert abs(energy(lo, q, v)[0] - e0) <= 1e-8
    assert closure_distance(lo, q)[0] <= 1e-10


# ------------------------------------------------------------------------------------------------------------------
# CPU tier: the kernel's per-stage code compiled for the host
# ------------------------------------------------------------------------------------------------------------------
def _shim():
    """tests/hostsim/hostsim_loops_rollout.cpp, compiled on first use into a temporary directory."""
    global _lib
    if _lib is not None:
        return _lib
    srcs = [os.path.join(_HERE, "hostsim", "hostsim_loops_rollout.cpp")] + sorted(
        os.path.join(_CSRC, f) for f in os.listdir(_CSRC) if f.endswith((".cuh", ".h")) or f == "rbd_model.cpp")
    srcs.append(os.path.join(_HERE, "..", "include", "rbd_b200.h"))
    h = hashlib.sha1(b"".join(open(s, "rb").read() for s in srcs)).hexdigest()[:16]
    d = os.path.join(tempfile.gettempdir(), f"rbd_hostsim_loops_rollout_{os.getuid()}")
    os.makedirs(d, exist_ok=True)
    so = os.path.join(d, f"hostsim_loops_rollout_{h}.so")
    if not os.path.exists(so):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so + f".{os.getpid()}",
                               srcs[0], os.path.join(_CSRC, "rbd_model.cpp")])
        os.replace(so + f".{os.getpid()}", so)
    lib = ctypes.CDLL(so)
    vp = ctypes.c_void_p
    lib.hostsim_loops_contact_stage.argtypes = [ctypes.POINTER(RbdModelDesc), vp, vp, ctypes.c_int, ctypes.c_int64, vp, vp, vp, vp, vp,
                                                ctypes.c_double, vp, vp]
    _lib = lib
    return lib


def hostsim_stage(mech, cd, q, v, tau, s0, sdp, wa):
    dt = q.dtype
    c = lambda a: None if a is None else np.ascontiguousarray(a, dt)     # noqa: E731
    p = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)   # noqa: E731
    desc = mech.flatten()
    B = q.shape[1]
    vd = np.full((desc.nv, B), np.nan, dt)
    sd = np.full((cd.nstates, B), np.nan, dt)
    d, keep = make_desc(desc)
    lst, keep2 = rbd.loop_desc(mech).c_struct()
    cst, keep3 = cd.c_struct()
    q, v, tau, s0, sdp = c(q), c(v), c(tau), c(s0), c(sdp)
    assert _shim().hostsim_loops_contact_stage(ctypes.byref(d), ctypes.byref(lst), ctypes.byref(cst), 0 if dt == np.float32 else 1, B,
                                               p(q), p(v), p(tau), p(s0), p(sdp), float(wa), p(vd), p(sd)) == 0
    return vd, sd


def _stage_fixture(which):
    if which == "atlas_ss":
        mech, cd = atlas_single_support()
        q, v, tau = atlas_states(mech, 16, 7)
    elif which == "mc":
        _, mech, _ = maximal_coordinate_pair(5, 12)
        cd = _with_contacts(mech, 5, npoints=6, nhalf=2)
        q, v, tau, _, _ = rand_inputs(mech, 8, 5)
    else:
        mech, cd = four_bar_with_contact()
        q, v, tau = _four_bar_inputs(16, 3)
    return mech, cd, q, v, tau


@pytest.mark.parametrize("which", ["atlas_ss", "mc", "four_bar"])
def test_hostsim_stage_matches_host_integrator(which):
    """The contact pass + loops_sample of one stage: v̇ and ṡ to 1e-10 in fp64, at stage 0 (no previous ṡ) and a later stage, with
    pairs in and out of contact."""
    mech, cd, q, v, tau = _stage_fixture(which)
    assert mech.has_loops() and len({int(b) for b in cd.body}) >= (2 if which == "mc" else 1)
    rng = np.random.default_rng(12)
    B = q.shape[1]
    s0 = rng.standard_normal((cd.nstates, B)) * 0.05
    sdp = rng.standard_normal((cd.nstates, B))
    wa = 5e-4
    lo = LoopOracle(mech)
    for prev in (None, sdp):
        ss = s0 if prev is None else s0 + wa * prev
        vd_o, sd_o = stage_dynamics(lo, q, v, ss, cd, tau)
        vd, sd = hostsim_stage(mech, cd, q, v, tau, s0, prev, wa)
        assert np.any(sd_o == 0) and np.any(sd_o != 0)                        # pairs in and out of contact
        assert np.abs(vd - vd_o).max() < 1e-10 * max(1.0, np.abs(vd_o).max())
        assert np.abs(sd - sd_o).max() < 1e-10 * max(1.0, np.abs(sd_o).max())


# ------------------------------------------------------------------------------------------------------------------
# CPU tier: C-ABI argument checks (host only, nothing launched)
# ------------------------------------------------------------------------------------------------------------------
def test_integrate_loops_argument_checks(built):
    lib = rbd.load_library()
    mech, cd = atlas_single_support()
    h = _cabi.ModelHandle(mech.flatten())
    good = rbd.loop_desc(mech)
    lst, keep = good.c_struct()
    cst, keep2 = cd.c_struct()
    fake = ctypes.c_void_p(64)                  # never dereferenced by the checks below
    F32, F64 = _cabi.RBD_F32, _cabi.RBD_F64

    def call(dtype=F64, B=4, ld=4, s=fake, step=0, stage=0, loops=ctypes.byref(lst), contact=ctypes.byref(cst), dt=1e-3, n=1,
             traj=(None, None, None)):
        return lib.rbd_integrate_loops(h.ptr, dtype, B, ld, fake, fake, s, None, step, stage, loops, contact, dt, n, *traj, None)

    assert call(dtype=_cabi.RBD_DUAL64X6) == _cabi.RBD_EUNSUPPORTED
    assert call(dtype=7) == _cabi.RBD_EUNSUPPORTED
    assert call(loops=None) == _cabi.RBD_EINVAL
    assert call(n=-1) == _cabi.RBD_EINVAL
    assert call(dt=0.0) == _cabi.RBD_EINVAL and call(dt=-1e-3) == _cabi.RBD_EINVAL
    assert call(step=-1) == _cabi.RBD_EINVAL and call(stage=-4) == _cabi.RBD_EINVAL
    assert call(s=None) == _cabi.RBD_EINVAL and b"s must not be NULL" in lib.rbd_last_error()
    assert call(B=8, ld=4) == _cabi.RBD_EDIM
    assert call(traj=(fake, None, None)) == _cabi.RBD_EINVAL
    assert call(traj=(fake, fake, None)) == _cabi.RBD_EINVAL
    assert call(B=0, ld=0, s=None) == _cabi.RBD_OK                       # empty batch: nothing to do
    assert lib.rbd_integrate_loops(None, F32, 1, 1, fake, fake, fake, None, 0, 0, ctypes.byref(lst), ctypes.byref(cst), 1e-3, 1, None,
                                   None, None, None) == _cabi.RBD_EINVAL
    # malformed / oversized loop descriptors
    bad = rbd.LoopDesc(good.predecessor, np.array([999], np.int32), good.joint_to_predecessor, good.joint_to_successor,
                       good.nconstraints, good.wrench_basis, good.gains)
    b1, k1 = bad.c_struct()
    assert call(loops=ctypes.byref(b1)) == _cabi.RBD_EINVAL
    n = _cabi.RBD_MAX_LOOP_JOINTS + 1
    eye = np.tile(Transform3D.identity().flat12(), (n, 1))
    many = rbd.LoopDesc(np.full(n, -1, np.int32), np.zeros(n, np.int32), eye, eye, np.ones(n, np.int32), np.tile(np.eye(6)[:1], (n, 1)), None)
    b2, k2 = many.c_struct()
    assert call(loops=ctypes.byref(b2)) == _cabi.RBD_EUNSUPPORTED
    m = 17                                                                # 17 Fixed loops of 6 rows: more than 96 rows
    eye = np.tile(Transform3D.identity().flat12(), (m, 1))
    rows = rbd.LoopDesc(np.full(m, -1, np.int32), np.arange(m, dtype=np.int32) % 20, eye, eye, np.full(m, 6, np.int32),
                        np.tile(np.eye(6), (m, 1)), None)
    b3, k3 = rows.c_struct()
    assert call(loops=ctypes.byref(b3)) == _cabi.RBD_EUNSUPPORTED
    # malformed / oversized contact descriptors
    badc = rbd.ContactDesc(cd.body.copy(), cd.location, cd.normal_model, cd.friction_model, cd.halfspace)
    badc.body[0] = 99
    c1, kc1 = badc.c_struct()
    assert call(contact=ctypes.byref(c1)) == _cabi.RBD_EINVAL and b"body index" in lib.rbd_last_error()
    manyc = rbd.ContactDesc(np.zeros(33, np.int32), np.zeros((33, 3)), np.ones((33, 3)), np.ones((33, 3)), cd.halfspace)
    c2, kc2 = manyc.c_struct()
    assert call(contact=ctypes.byref(c2)) == _cabi.RBD_EUNSUPPORTED
    halfs = rbd.ContactDesc(cd.body, cd.location, cd.normal_model, cd.friction_model, np.tile(cd.halfspace, (5, 1)))
    c3, kc3 = halfs.c_struct()
    assert call(contact=ctypes.byref(c3)) == _cabi.RBD_EUNSUPPORTED
    # no contact: s may be NULL
    assert call(contact=None, s=None, B=0, ld=0) == _cabi.RBD_OK
    h.close()


def test_existing_rollouts_keep_refusing_loops(built):
    """simulate_ / simulate_contact_* / dynamics_contact_ / autodiff.simulate* still refuse loops; simulate_loops_ is the way."""
    from rigidbodydynamics.jl_b200 import autodiff
    m = four_bar()
    state = rbd.MechanismState(m, 2, device="cpu")
    result = rbd.DynamicsResult(m, 2, device="cpu")
    for c in (lambda: rbd.simulate_(state, 0.01), lambda: rbd.simulate_trajectory_(state, 1),
              lambda: rbd.simulate_contact_(state, 0.01, None), lambda: rbd.simulate_contact_trajectory_(state, 1, None),
              lambda: rbd.dynamics_contact_(result, state)):
        with pytest.raises(rbd.RbdError) as e:
            c()
        assert e.value.status == _cabi.RBD_ELOOP
    for c in (lambda: autodiff.simulate(m, state.q, state.v, dt=1e-3, nsteps=1),
              lambda: autodiff.simulate_contact(m, state.q, state.v, None, dt=1e-3, nsteps=1)):
        with pytest.raises(rbd.RbdError) as e:
            c()
        assert e.value.status == _cabi.RBD_ELOOP


# ------------------------------------------------------------------------------------------------------------------
# GPU tier
# ------------------------------------------------------------------------------------------------------------------
def _tau_arg(tau, kind, nsteps, rng):
    nv, B = tau.shape
    if kind == "none":
        return None
    if kind == "const":
        return tau
    if kind == "step":
        return tau[None] * (0.5 + rng.random((nsteps, 1, 1)))
    return tau[None, None] * (0.5 + rng.random((nsteps, 4, 1, 1)))


def _cabi_rollout(mech, cd, q, v, s, tau, dtype, dt, nsteps, ld, record=False):
    """rbd_integrate_loops through the C ABI on arrays with leading dimension ld (> B: NaN padding that must stay untouched)."""
    import torch
    B = q.shape[1]
    st = rbd.MechanismState(mech, batch=1, dtype=dtype)

    def pad(a):
        t = torch.full(a.shape[:-1] + (ld,), float("nan"), dtype=dtype, device="cuda")
        t[..., :B] = torch.from_numpy(np.ascontiguousarray(a)).to(dtype)
        return t
    qd, vd = pad(q), pad(v)
    sd = None if s is None else pad(s)
    td = None if tau is None else pad(tau)
    blk = mech.num_velocities() * ld
    step, stage = (0, 0) if tau is None or tau.ndim == 2 else ((blk, 0) if tau.ndim == 3 else (4 * blk, blk))
    lst, keep = rbd.loop_desc(mech).c_struct()
    cst, keep2 = (None, None) if cd is None else cd.c_struct()
    lib = rbd.load_library()
    _cabi.check(lib.rbd_integrate_loops(st.handle.ptr, _cabi.RBD_F32 if dtype == torch.float32 else _cabi.RBD_F64, B, ld,
                                        qd.data_ptr(), vd.data_ptr(), None if sd is None else sd.data_ptr(),
                                        None if td is None else td.data_ptr(), step, stage, ctypes.byref(lst),
                                        None if cst is None else ctypes.byref(cst), dt, nsteps, None, None, None,
                                        torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    for t in (qd, vd) + (() if sd is None else (sd,)):
        assert bool(torch.isnan(t[:, B:]).all())
    out = tuple(t[:, :B].double().cpu().numpy() for t in (qd, vd))
    return out + (None if sd is None else sd[:, :B].double().cpu().numpy(),)


def _max_rel(a, b):
    return float(np.abs(a - b).max() / max(1.0, np.abs(b).max()))


def _state(m, q, v, dtype):
    import torch
    st = rbd.MechanismState(m, q.shape[1], dtype)
    st.q.copy_(torch.from_numpy(np.ascontiguousarray(q)))
    st.v.copy_(torch.from_numpy(np.ascontiguousarray(v)))
    return st


@pytest.mark.gpu
def test_gpu_four_bar_reference_testset(built):
    """test/test_simulate.jl:127-227 verbatim through simulate_loops_ on 64 identical states: 1 s from rest without stabilisation
    (motion, energy to 1e-8, closure 1e-10); from q1 = 1.7 with the default gains, 15 s (closure 1e-5), then 10 s more (energy drift
    1e-5).  Every column equals column 0, bit for bit."""
    import torch
    m = four_bar()
    lo = LoopOracle(m)
    B = 64
    st = _state(m, np.tile(FOUR_BAR_Q0[:, None], (1, B)), np.zeros((3, B)), torch.float64)
    e0 = energy(lo, FOUR_BAR_Q0[:, None], np.zeros((3, 1)))[0]
    assert rbd.simulate_loops_(st, 1.0, dt=1e-3, stabilization_gains=None) == 1000

    def check_columns():
        assert bool((st.q == st.q[:, :1]).all()) and bool((st.v == st.v[:, :1]).all())
        return st.q[:, :1].cpu().numpy(), st.v[:, :1].cpu().numpy()
    q, v = check_columns()
    assert lo.oracle.kinematics(q, v, want=("ke",))["ke"][0, 0] > 1e-2
    assert abs(energy(lo, q, v)[0] - e0) <= 1e-8
    assert closure_distance(lo, q)[0] <= 1e-10
    q0 = FOUR_BAR_Q0.copy()
    q0[0] = 1.7
    st.q.copy_(torch.from_numpy(np.tile(q0[:, None], (1, B))))
    st.v.copy_(torch.from_numpy(np.tile(np.array([[0.5], [-0.47295], [0.341]]), (1, B))))
    assert closure_distance(lo, q0[:, None])[0] > 1e-2
    rbd.simulate_loops_(st, 15.0, dt=1e-3)
    q, v = check_columns()
    assert closure_distance(lo, q)[0] <= 1e-5
    e15 = energy(lo, q, v)[0]
    rbd.simulate_loops_(st, 10.0, dt=1e-3)
    q, v = check_columns()
    assert abs(energy(lo, q, v)[0] - e15) <= 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize("which,nsteps,torque", [("four_bar", 1, "none"), ("four_bar", 20, "stage"), ("atlas_ds", 5, "const"),
                                                 ("atlas_ds", 1, "step"), ("atlas_ds", 20, "none"), ("mc3", 5, "stage"),
                                                 ("mc4", 20, "const"), ("mc5", 1, "none"), ("atlas_ss", 1, "stage"),
                                                 ("atlas_ss", 5, "step"), ("atlas_ss", 20, "const")])
def test_gpu_rollout_matches_host_integrator_fp64(built, which, nsteps, torque):
    import torch
    B = 45 if which.startswith("atlas") else 37                 # ragged: not a multiple of the block size
    mech, cd, q, v, tau, s = _case(which, B, 32)
    tau = _tau_arg(tau, torque, nsteps, np.random.default_rng(2))
    dt = 1e-3
    qr, vr, sr = integrate_loops(LoopOracle(mech), q, v, s, cd, tau, dt=dt, nsteps=nsteps)
    qg, vg, sg = _cabi_rollout(mech, cd, q, v, s, tau, torch.float64, dt, nsteps, ld=B + 13)
    assert config_distance(mech, qg, qr) < TOL64
    assert rel_err(vg, vr) < TOL64
    if cd is not None:
        assert np.any(sr != s)                                  # something touched
        assert _max_rel(sg, sr) < TOL64


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["four_bar", "atlas_ds", "mc3", "atlas_ss"])
def test_gpu_rollout_fp32(built, which):
    import torch
    mech, cd, q, v, tau, s = _case(which, 33, 35)
    r = lambda a: None if a is None else a.astype(np.float32).astype(np.float64)    # noqa: E731
    q, v, tau, s = r(q), r(v), r(tau), r(s)
    qr, vr, sr = integrate_loops(LoopOracle(mech), q, v, s, cd, tau, dt=1e-3, nsteps=5)
    qg, vg, sg = _cabi_rollout(mech, cd, q, v, s, tau, torch.float32, 1e-3, 5, ld=33)
    eq, ev = config_distance(mech, qg, qr), rel_err(vg, vr)
    print(f"fp32 {which}: q {eq:.2e}  v {ev:.2e}" + ("" if cd is None else f"  s {_max_rel(sg, sr):.2e}"))
    assert eq < TOL32 and ev < TOL32


def _body_poses(lo, q):
    return lo.oracle.kinematics(q, want=("transforms",))["transforms"]


def _closure(lo, q, v):
    """(position, velocity) closure of the loop joints: the largest distance between the origins of the frames before and after
    the joints that keep them together (revolute, sin-cos revolute, spherical, fixed), and max |K v|."""
    tr = _body_poses(lo, q)
    pos = 0.0
    for j in lo.mech.non_tree_joints:
        if type(j.joint_type) not in (rbd.Revolute, rbd.SinCosRevolute, rbd.QuaternionSpherical, rbd.Fixed):    # Prismatic is a Revolute
            continue
        for b in range(q.shape[1]):
            Rp, pp = _pose(tr, lo.body(j.predecessor), b)
            Rs, ps = _pose(tr, lo.body(j.successor), b)
            gap = (Rp @ j.joint_to_predecessor.trans + pp) - (Rs @ j.joint_to_successor.trans + ps)
            pos = max(pos, float(np.linalg.norm(gap)))
    K, _ = lo.constraints(q, v)
    return pos, float(np.abs(np.einsum("bcj,jb->bc", K, v)).max())


@pytest.mark.gpu
def test_gpu_maximal_coordinates_match_the_tree(built):
    """The maximal-coordinate twin's rollout (default gains) and simulate_ of the tree give the same body poses after 10 steps at
    dt = 1e-3; the closure stays small."""
    import torch
    for seed in (3, 4):
        tree, mc, bodymap = maximal_coordinate_pair(seed, 12)
        B = 4
        q, v, _, _, _ = rand_inputs(tree, B, seed + 50)
        v *= 0.3
        qm, vm = zip(*(mc_state_from_tree(tree, mc, bodymap, q[:, b], v[:, b]) for b in range(B)))
        qm, vm = np.stack(qm, 1), np.stack(vm, 1)
        a = _state(tree, q, v, torch.float64)
        rbd.simulate_(a, 10e-3 - 1e-9, dt=1e-3)
        b = _state(mc, qm, vm, torch.float64)
        assert rbd.simulate_loops_(b, 10e-3 - 1e-9, dt=1e-3) == 10
        lt, lm = LoopOracle(tree), LoopOracle(mc)
        tt, tm = _body_poses(lt, a.q.cpu().numpy()), _body_poses(lm, b.q.cpu().numpy())
        gap = 0.0
        for body, copy in bodymap.items():
            if body is tree.root_body:
                continue
            i, k = lt.index[id(body)], lm.index[id(copy)]
            gap = max(gap, float(np.abs(tt[12 * i:12 * i + 12] - tm[12 * k:12 * k + 12]).max()))
        cpos, cvel = _closure(lm, b.q.cpu().numpy(), b.v.cpu().numpy())
        print(f"maximal coordinates seed {seed}: pose gap {gap:.2e}, closure {cpos:.2e} (position) {cvel:.2e} (velocity)")
        assert gap < MC_GAP and cpos < MC_GAP and cvel < MC_GAP


@pytest.mark.gpu
def test_gpu_tree_and_contact_without_loops_match_the_tree_rollouts(built):
    """nloops = 0: simulate_loops_ against simulate_ (Atlas, no contact) and against simulate_contact_ (Atlas on the floor), fp64, to
    1e-9 relative -- CRBA + Cholesky against ABA, so equal to rounding only."""
    import torch
    B = 100
    mech = rbd.load_model("atlas", floating=True)
    q, v, tau = atlas_states(mech, B, 41)
    tq = torch.from_numpy(tau).cuda()
    a, b = _state(mech, q, v, torch.float64), _state(mech, q, v, torch.float64)
    rbd.simulate_(a, 5e-3 - 1e-9, tq, dt=1e-3)
    assert rbd.simulate_loops_(b, 5e-3 - 1e-9, tq, dt=1e-3) == 5
    assert config_distance(mech, b.q.cpu().numpy(), a.q.cpu().numpy()) < 1e-9
    assert rel_err(b.v.cpu().numpy(), a.v.cpu().numpy()) < 1e-9
    mech, cd = atlas_on_floor()
    q, v, tau = atlas_states(mech, B, 42)
    s0 = torch.from_numpy(np.random.default_rng(3).standard_normal((cd.nstates, B)) * 1e-3).cuda()
    a, b = _state(mech, q, v, torch.float64), _state(mech, q, v, torch.float64)
    sa, sb = s0.clone(), s0.clone()
    rbd.simulate_contact_(a, 5e-3 - 1e-9, sa, tq, dt=1e-3)
    rbd.simulate_loops_(b, 5e-3 - 1e-9, tq, dt=1e-3, contact_state=sb)
    assert not torch.equal(sa, s0)
    assert config_distance(mech, b.q.cpu().numpy(), a.q.cpu().numpy()) < 1e-9
    assert rel_err(b.v.cpu().numpy(), a.v.cpu().numpy()) < 1e-9
    assert _max_rel(sb.cpu().numpy(), sa.cpu().numpy()) < 1e-9


@pytest.mark.gpu
def test_gpu_recording_and_split_calls(built):
    """Atlas single support with foot contact: recording does not change the result and its last block is it; two calls equal one
    call of the summed steps, bit for bit, including s."""
    import torch
    B = 200
    mech, cd, q, v, tau, s = _case("atlas_ss", B, 38)
    dt, n = 1e-3, 6
    tq = torch.from_numpy(tau).cuda()

    def state():
        return _state(mech, q, v, torch.float64), torch.from_numpy(s).cuda()
    c, sc = state()
    qt, vt, st_ = rbd.simulate_loops_trajectory_(c, n, tq, dt=dt, contact_state=sc)
    d, sd = state()
    assert rbd.simulate_loops_(d, n * dt - 1e-9, tq, dt=dt, contact_state=sd) == n
    assert torch.equal(c.q, d.q) and torch.equal(c.v, d.v) and torch.equal(sc, sd)
    assert torch.equal(qt[-1], c.q) and torch.equal(vt[-1], c.v) and torch.equal(st_[-1], sc)
    assert torch.equal(qt[0].cpu(), torch.from_numpy(q)) and torch.equal(st_[0].cpu(), torch.from_numpy(s))
    assert not torch.equal(sc, torch.from_numpy(s).cuda())
    e, se = state()
    rbd.simulate_loops_(e, 2 * dt - 1e-9, tq, dt=dt, contact_state=se)
    rbd.simulate_loops_(e, (n - 2) * dt - 1e-9, tq, dt=dt, contact_state=se)
    assert torch.equal(e.q, c.q) and torch.equal(e.v, c.v) and torch.equal(se, sc)


@pytest.mark.gpu
@pytest.mark.parametrize("which,B,per_step", [("four_bar", 64, 9), ("atlas_ds", 4096, 14), ("atlas_ds", 777, 9), ("atlas_ss", 4096, 15),
                                              ("atlas_ss", 777, 10)])
def test_gpu_launch_count(built, which, B, per_step):
    """Per step: per stage 1 or 2 coordinate-map kernels and one KKT kernel, then 1 or 2 finishing kernels and, with contact, the
    contact-state kernel (include/rbd_b200.h)."""
    import torch
    mech, cd, q, v, tau, s = _case(which, B, 3)
    st = _state(mech, q, v, torch.float64)
    sg = None if s is None else torch.from_numpy(s).cuda()
    for n in (1, 3):
        rbd.simulate_loops_(st, n * 1e-3 - 1e-9, dt=1e-3, contact_state=sg)
        assert rbd.launch_info().kernels_launched == per_step * n


@pytest.mark.gpu
def test_gpu_atlas_double_support_fp32_large_batch(built):
    """2^20 samples, 5 steps: finite; strided columns agree with the host integrator and are bit-identical to a small-batch run of
    the same columns (the workspace is per resident thread, not per sample).  The small batch has 1024 columns, so that it takes
    the same vectorised RK4 stage / finishing kernels as the large one (include/rbd_b200.h)."""
    import torch
    m = atlas_double_support()
    B = 1 << 20
    rng = np.random.default_rng(61)
    st = rbd.MechanismState(m, B, torch.float32)
    rbd.rand_(st, rng)
    st.v.mul_(0.2)
    tau = torch.rand((st.nv, B), dtype=torch.float32, device="cuda")
    idx = torch.arange(5, B, 1021, device="cuda")[:1024]
    q0, v0, t = (x[:, idx].contiguous() for x in (st.q, st.v, tau))
    assert rbd.simulate_loops_(st, 5e-3 - 1e-9, tau, dt=1e-3) == 5
    assert bool(torch.isfinite(st.q).all()) and bool(torch.isfinite(st.v).all())
    sub = idx[::16]
    qr, vr, _ = integrate_loops(LoopOracle(m), q0[:, ::16].double().cpu().numpy(), v0[:, ::16].double().cpu().numpy(), None, None,
                                t[:, ::16].double().cpu().numpy(), dt=1e-3, nsteps=5)
    eq = config_distance(m, st.q[:, sub].double().cpu().numpy(), qr)
    ev = rel_err(st.v[:, sub].double().cpu().numpy(), vr)
    print(f"Atlas double support fp32 2^20, 5 steps: q {eq:.2e}  v {ev:.2e}")
    assert eq < TOL32 and ev < TOL32
    small = rbd.MechanismState(m, idx.numel(), torch.float32)
    small.q.copy_(q0)
    small.v.copy_(v0)
    rbd.simulate_loops_(small, 5e-3 - 1e-9, t, dt=1e-3)
    assert torch.equal(small.q, st.q[:, idx]) and torch.equal(small.v, st.v[:, idx])
