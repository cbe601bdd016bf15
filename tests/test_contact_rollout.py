"""simulate for mechanisms with contact points (DESIGN 4.14): rbd_integrate_contact / simulate_contact_.

The reference integrator with the contact state (tests/contact_oracle.py) is pinned on the CPU by
  * Oracle.integrate when no pair is ever in contact (it restates the same Munthe-Kaas step),
  * the reference's two contact simulation tests, re-run on it:
      "elastic ball drop"  energy balance at every step + bounces      test/test_simulate.jl:34-89
      "inclined plane"     stick above / slip below mu_crit, two calls  test/test_simulate.jl:91-125
  * the reset semantics of simulate: a pair out of contact keeps its state, frozen, across the step.
The kernel's per-stage device code (contact_stage_pass + aba_sample, compiled for the host: tests/hostsim/hostsim_contact_rollout.cpp)
must agree with the oracle's contact_dynamics + dynamics at random stage states, and the GPU rollout with the oracle integrator.
"""
import ctypes
import functools

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from oracle import Oracle
from rigidbodydynamics.jl_b200 import _cabi
from rigidbodydynamics.jl_b200._cabi import RbdModelDesc, make_desc
from tests import hostsim
from tests.contact_oracle import integrate_contact
from tests.test_contact import _free_body, _with_contacts
from tests.util import config_distance, rand_inputs, randmech, rel_err


TOL64 = 1e-9          # GPU rollout against the fp64 oracle integrator, relative (rel_err)
# fp32 rollout against the fp64 oracle, 5 steps at dt = 1e-3.  Measured on an H100: 9.7e-6 (q) / 9.4e-6 (v) on the random tree,
# 2.6e-7 / 8.6e-6 on Atlas standing on the floor, 7.2e-7 / 7.6e-6 for Atlas at 2^20 over 10 steps; the bound leaves the
# headroom of about 200x that the single-call fp32 tests keep (2e-4 against 1e-6).
TOL32 = 2e-3


@functools.cache
def _shim():
    """tests/hostsim/hostsim_contact_rollout.cpp, compiled and loaded by hostsim.shim."""
    lib = hostsim.shim("hostsim_contact_rollout")
    vp = ctypes.c_void_p
    lib.hostsim_contact_stage.argtypes = [ctypes.POINTER(RbdModelDesc), ctypes.c_int, ctypes.c_int64, vp, vp, vp, vp, vp, vp,
                                          ctypes.c_double, vp, vp]
    return lib


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def hostsim_stage(desc, cd, q, v, tau, s0, sdp, wa):
    dt = q.dtype
    c = lambda a: None if a is None else np.ascontiguousarray(a, dt)     # noqa: E731
    B = q.shape[1]
    vd = np.full((desc.nv, B), np.nan, dt)
    sd = np.full((cd.nstates, B), np.nan, dt)
    d, keep = make_desc(desc)
    st, keep2 = cd.c_struct()
    assert _shim().hostsim_contact_stage(ctypes.byref(d), 0 if dt == np.float32 else 1, B, _p(c(q)), _p(c(v)), _p(c(tau)),
                                         ctypes.byref(st), _p(c(s0)), _p(c(sdp)), float(wa), _p(vd), _p(sd)) == 0
    return vd, sd


def _atlas_on_floor(per_foot=4):
    mech = rbd.load_model("atlas", floating=True)
    model = rbd.SoftContactModel(rbd.hunt_crossley_hertz(), rbd.ViscoelasticCoulombModel(0.8, 20e3, 100.0))
    for foot in ("l_foot", "r_foot"):
        body = mech.findbody(foot)
        xs = (-0.08, 0.17) if per_foot == 4 else (-0.08, 0.045, 0.17, 0.0)[:per_foot // 2]
        for x in xs:
            for y in (-0.06, 0.06):
                rbd.add_contact_point(body, rbd.ContactPoint(np.array([x, y, -0.08]), model))
    rbd.add_environment_primitive(mech, rbd.HalfSpace3D(np.zeros(3), [0, 0, 1.0]))
    return mech, rbd.contact_desc(mech)


def _atlas_states(mech, B, seed, vectorised=False):
    """Atlas near upright with the pelvis at a height that puts the feet around the floor, small joint motion.  ``vectorised``:
    joint inputs drawn in one call each instead of per sample (for batches of 2^20)."""
    rng = np.random.default_rng(seed)
    if vectorised:
        nq, nv = mech.num_positions(), mech.num_velocities()
        q, v, tau = rng.uniform(-np.pi, np.pi, (nq, B)), rng.random((nv, B)), rng.random((nv, B))
    else:
        q, v, tau, _, _ = rand_inputs(mech, B, seed)
    q[:4] = np.array([[1.0], [0], [0], [0]]) + 0.05 * rng.standard_normal((4, B)); q[:4] /= np.linalg.norm(q[:4], axis=0)
    q[4:6] = rng.standard_normal((2, B)); q[6] = 0.93 + 0.03 * rng.standard_normal(B)
    q[7:] *= 0.1; v *= 0.2
    return q, v, tau - 0.5


def _empty_desc():
    return rbd.ContactDesc(np.zeros(0, np.int32), np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 6)))


# ------------------------------------------------------------------------------------------------------------------
# CPU tier: the oracle integrator
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["tree", "atlas"])
def test_oracle_without_contact_is_oracle_integrate(which):
    """No pair ever in contact: the contact integrator is the oracle's Munthe-Kaas RK4 step (its coordinate maps restated in
    numpy), and the contact state does not move, bit for bit."""
    mech = randmech(4) if which == "tree" else rbd.load_model("atlas", floating=True)
    cd = _with_contacts(mech, 5, npoints=4, nhalf=1)
    cd.halfspace[:] = [0, 0, -100.0, 0, 0, 1.0]                          # far below everything
    orc = Oracle(mech.flatten())
    q, v, tau, _, _ = rand_inputs(mech, 17, 6)
    s = np.random.default_rng(1).standard_normal((cd.nstates, 17))
    qr, vr = orc.integrate(q, v, tau, dt=1e-3, nsteps=3)
    qc, vc, sc = integrate_contact(orc, q, v, s, cd, tau, dt=1e-3, nsteps=3)
    assert config_distance(mech, qc, qr) < 1e-12 and rel_err(vc, vr) < 1e-12
    assert np.array_equal(sc, s)
    qe, ve, _ = integrate_contact(orc, q, v, None, _empty_desc(), tau, dt=1e-3, nsteps=3)
    assert config_distance(mech, qe, qr) < 1e-12 and rel_err(ve, vr) < 1e-12


def _ball(alpha=0.0, mu=0.5):
    rng = np.random.default_rng(61)
    mech, body = _free_body(rng=rng)
    com = body.inertia.cross_part / body.inertia.mass
    model = rbd.SoftContactModel(rbd.hunt_crossley_hertz(alpha=alpha), rbd.ViscoelasticCoulombModel(mu, 1e3, 1e3))
    rbd.add_contact_point(body, rbd.ContactPoint(com, model))
    rbd.add_environment_primitive(mech, rbd.HalfSpace3D(np.zeros(3), [0, 0, 1.0]))
    return mech, rbd.contact_desc(mech), com, model


def _ball_energy(orc, model, q, v):
    k = orc.kinematics(q, v, want=("com", "ke", "pe"))
    pen = np.maximum(-k["com"][2], 0.0)
    n = model.normal.n
    return model.normal.k * pen ** (n + 1) / (n + 1) + k["ke"][0] + k["pe"][0]


def test_oracle_elastic_ball_drop():
    """test/test_simulate.jl:34-89 on the contact integrator: energy within 1e-2 at every step, more than 3 bounces."""
    mech, cd, com, model = _ball()
    orc = Oracle(mech.flatten())
    q = np.zeros((7, 1)); q[0] = 1; q[4:, 0] = [1.0, 2.0, 0.05 - com[2]]
    energies, vz = [], []

    def record(n, q, v, s):
        energies.append(_ball_energy(orc, model, q, v)[0])
        vz.append(v[5, 0])
    integrate_contact(orc, q, np.zeros((6, 1)), None, cd, dt=1e-3, nsteps=500, record=record)
    energies = np.asarray(energies)
    assert np.abs(energies - energies[0]).max() < 1e-2
    sg = np.sign(vz)
    assert np.count_nonzero(sg[1:] != sg[:-1]) > 3


def _incline(stick):
    theta = 0.5
    mu = np.tan(theta) + (1e-2 if stick else -1e-2)
    mech, body = _free_body(rbd.SpatialInertia(np.eye(3), np.zeros(3), 2.0))
    rbd.add_environment_primitive(mech, rbd.HalfSpace3D(np.zeros(3), [np.sin(theta), 0, np.cos(theta)]))
    rbd.add_environment_primitive(mech, rbd.HalfSpace3D([0, 0, -100.0], [0, 0, 1.0]))
    model = rbd.SoftContactModel(rbd.hunt_crossley_hertz(k=50e3, alpha=1.0), rbd.ViscoelasticCoulombModel(mu, 50e3, 1e4))
    rbd.add_contact_point(body, rbd.ContactPoint(np.zeros(3), model))
    return mech, rbd.contact_desc(mech), theta


@pytest.mark.parametrize("stick", [True, False])
def test_oracle_inclined_plane(stick):
    """test/test_simulate.jl:91-125: sticks to 1e-4 above mu_crit, slips beyond 5e-2 below; the second call continues from the
    contact state the first one left (it is not zero: the point sticks through the tangential spring)."""
    mech, cd, _ = _incline(stick)
    orc = Oracle(mech.flatten())
    q = np.zeros((7, 1)); q[0] = 1
    q, v, s = integrate_contact(orc, q, np.zeros((6, 1)), None, cd, dt=1e-3, nsteps=1000)
    assert np.abs(s[:3]).max() > 0 and np.all(s[3:] == 0)            # the far half-space never touches
    x1 = q[4:, 0].copy()
    q, v, s = integrate_contact(orc, q, v, s, cd, dt=1e-3, nsteps=500)
    if stick:
        assert np.allclose(x1, q[4:, 0], atol=1e-4)
    else:
        assert not np.allclose(x1, q[4:, 0], atol=5e-2)


def test_oracle_reset_semantics():
    """A pair out of contact in all four stages keeps its state bit for bit (not zeroed); a bouncing ball that slides while in
    contact leaves the floor with a non-zero tangential state that stays frozen in the air."""
    mech, cd, com, model = _ball(alpha=0.2, mu=0.3)
    orc = Oracle(mech.flatten())
    q = np.zeros((7, 2)); q[0] = 1; q[4:6] = [[0.3, -1.0], [0.2, 0.5]]; q[6] = [0.5, 0.05 - com[2]]
    v = np.zeros((6, 2)); v[3] = 1.5                                   # sliding along x
    s = np.full((3, 2), 0.25)
    q1, v1, s1 = integrate_contact(orc, q, v, s, cd, dt=1e-3, nsteps=1)
    assert np.array_equal(s1[:, 0], s[:, 0])                           # high above the floor: frozen, not reset
    zs, ss = [], []
    integrate_contact(orc, q[:, 1:], v[:, 1:], np.zeros((3, 1)), cd, dt=1e-3, nsteps=300,
                      record=lambda n, q, v, s: (zs.append(orc.kinematics(q, v, want=("com",))["com"][2, 0]), ss.append(s[:, 0].copy())))
    zs, ss = np.asarray(zs), np.asarray(ss)
    touched = np.flatnonzero(zs < 0)
    assert touched.size > 0
    air = [n for n in range(touched[0], len(zs) - 1) if zs[n] > 2e-3 and zs[n + 1] > 2e-3]    # no stage can reach the floor
    assert len(air) > 10
    for n in air:
        assert np.array_equal(ss[n + 1], ss[n])
    assert np.abs(ss[air[-1]]).max() > 1e-6


# ------------------------------------------------------------------------------------------------------------------
# CPU tier: the kernel's device code compiled for the host
# ------------------------------------------------------------------------------------------------------------------
def _stage_case(mech, cd, B, seed, atlas=False):
    rng = np.random.default_rng(seed + 100)
    if atlas:
        q, v, tau = _atlas_states(mech, B, seed)
    else:
        q, v, tau, _, _ = rand_inputs(mech, B, seed)
    s0 = rng.standard_normal((cd.nstates, B)) * 0.05
    sdp = rng.standard_normal((cd.nstates, B))
    return q, v, tau, s0, sdp, float(rng.uniform(1e-4, 1e-3))


@pytest.mark.parametrize("seed", [32, 33, 35, 38])
def test_hostsim_stage_matches_oracle(seed):
    mech = randmech(seed)
    cd = _with_contacts(mech, seed, npoints=7, nhalf=3)
    desc = mech.flatten()
    orc = Oracle(desc)
    q, v, tau, s0, sdp, wa = _stage_case(mech, cd, 24, seed)
    for prev in (None, sdp):
        ss = s0 if prev is None else s0 + wa * prev
        wr, sd_o, _ = orc.contact_dynamics(q, v, cd, ss)
        vd_o = orc.dynamics(q, v, tau, wr)
        vd, sd = hostsim_stage(desc, cd, q, v, tau, s0, prev, wa)
        assert np.abs(wr).max() > 0 and np.any(sd_o == 0) and np.any(sd_o != 0)      # pairs in and out of contact
        assert np.abs(vd - vd_o).max() < 1e-10 * max(1.0, np.abs(vd_o).max())
        assert np.abs(sd - sd_o).max() < 1e-10 * max(1.0, np.abs(sd_o).max())


def test_hostsim_stage_atlas_eight_foot_points():
    mech, cd = _atlas_on_floor()
    assert cd.npoints == 8
    desc = mech.flatten()
    orc = Oracle(desc)
    q, v, tau, s0, sdp, wa = _stage_case(mech, cd, 64, 7, atlas=True)
    wr, sd_o, _ = orc.contact_dynamics(q, v, cd, s0 + wa * sdp)
    vd_o = orc.dynamics(q, v, tau, wr)
    vd, sd = hostsim_stage(desc, cd, q, v, tau, s0, sdp, wa)
    assert 0 < np.count_nonzero(np.abs(wr).sum(0)) < 64
    assert np.abs(vd - vd_o).max() < 1e-10 * max(1.0, np.abs(vd_o).max())
    assert np.abs(sd - sd_o).max() < 1e-10 * max(1.0, np.abs(sd_o).max())


# ------------------------------------------------------------------------------------------------------------------
# CPU tier: C-ABI argument checks (host only, nothing launched)
# ------------------------------------------------------------------------------------------------------------------
def test_integrate_contact_argument_checks(built):
    lib = rbd.load_library()
    mech = randmech(33)
    cd = _with_contacts(mech, 3, npoints=2, nhalf=1)
    h = _cabi.ModelHandle(mech.flatten())
    st, keep = cd.c_struct()
    fake = ctypes.c_void_p(64)                  # never dereferenced by the checks below
    F32, F64 = _cabi.RBD_F32, _cabi.RBD_F64

    def call(dtype=F64, B=4, ld=4, s=fake, step=0, stage=0, contact=ctypes.byref(st), dt=1e-3, n=1, traj=(None, None, None)):
        return lib.rbd_integrate_contact(h.ptr, dtype, B, ld, fake, fake, s, None, step, stage, contact, dt, n, *traj, None)

    assert call(dtype=_cabi.RBD_DUAL64X6) == _cabi.RBD_EUNSUPPORTED
    assert call(dtype=7) == _cabi.RBD_EUNSUPPORTED
    assert call(n=-1) == _cabi.RBD_EINVAL
    assert call(dt=0.0) == _cabi.RBD_EINVAL and call(dt=-1e-3) == _cabi.RBD_EINVAL
    assert call(step=-1) == _cabi.RBD_EINVAL and call(stage=-4) == _cabi.RBD_EINVAL
    assert call(s=None) == _cabi.RBD_EINVAL and b"s must not be NULL" in lib.rbd_last_error()
    assert call(contact=None) == _cabi.RBD_EINVAL
    assert call(B=8, ld=4) == _cabi.RBD_EDIM
    assert call(traj=(fake, None, None)) == _cabi.RBD_EINVAL
    assert call(traj=(fake, fake, None)) == _cabi.RBD_EINVAL
    assert call(B=0, ld=0, s=None) == _cabi.RBD_OK                       # empty batch: nothing to do
    assert lib.rbd_integrate_contact(None, F32, 1, 1, fake, fake, fake, None, 0, 0, ctypes.byref(st), 1e-3, 1, None, None, None,
                                     None) == _cabi.RBD_EINVAL
    bad = rbd.ContactDesc(cd.body.copy(), cd.location, cd.normal_model, cd.friction_model, cd.halfspace)
    bad.body[0] = 99
    st2, keep2 = bad.c_struct()
    assert call(contact=ctypes.byref(st2)) == _cabi.RBD_EINVAL and b"body index" in lib.rbd_last_error()
    many = rbd.ContactDesc(np.zeros(33, np.int32), np.zeros((33, 3)), np.ones((33, 3)), np.ones((33, 3)), cd.halfspace)
    st3, keep3 = many.c_struct()
    assert call(contact=ctypes.byref(st3)) == _cabi.RBD_EUNSUPPORTED
    h.close()


def test_simulate_contact_refuses_loops(built):
    """Mechanisms with loops are refused before anything is launched (no GPU needed)."""
    from tests.loops_oracle import four_bar
    mech = four_bar()
    assert mech.has_loops()
    for call in (lambda: rbd.simulate_contact_(_LoopStub(mech), 1e-3, None),
                 lambda: rbd.simulate_contact_trajectory_(_LoopStub(mech), 1, None)):
        with pytest.raises(rbd.RbdError) as e:
            call()
        assert e.value.status == _cabi.RBD_ELOOP


class _LoopStub:
    """The part of a MechanismState that the loop refusal reads (a real state needs a GPU)."""

    def __init__(self, mech):
        self.mechanism = mech


# ------------------------------------------------------------------------------------------------------------------
# GPU tier
# ------------------------------------------------------------------------------------------------------------------
def _tau_arg(tau, kind, nsteps, rng):
    """None / constant / per-step / per-stage torque arrays (numpy) for the oracle and the device."""
    nv, B = tau.shape
    if kind == "none":
        return None
    if kind == "const":
        return tau
    if kind == "step":
        return tau[None] * (0.5 + rng.random((nsteps, 1, 1)))
    return tau[None, None] * (0.5 + rng.random((nsteps, 4, 1, 1)))


def _cabi_rollout(mech, cd, q, v, s, tau, dtype, dt, nsteps, ld, record=False):
    """rbd_integrate_contact through the C ABI on arrays with leading dimension ld (> B: NaN padding that must stay untouched)."""
    import torch
    B = q.shape[1]
    st = rbd.MechanismState(mech, batch=1, dtype=dtype)

    def pad(a):
        t = torch.full(a.shape[:-1] + (ld,), float("nan"), dtype=dtype, device="cuda")
        t[..., :B] = torch.from_numpy(np.ascontiguousarray(a)).to(dtype)
        return t
    qd, vd, sd = pad(q), pad(v), pad(s)
    td = None if tau is None else pad(tau)
    blk = mech.num_velocities() * ld
    step, stage = (0, 0) if tau is None or tau.ndim == 2 else ((blk, 0) if tau.ndim == 3 else (4 * blk, blk))
    traj = [None, None, None]
    if record:
        traj = [torch.empty((nsteps + 1, r, B), dtype=dtype, device="cuda") for r in (q.shape[0], v.shape[0], s.shape[0])]
    c, keep = cd.c_struct()
    lib = rbd.load_library()
    _cabi.check(lib.rbd_integrate_contact(st.handle.ptr, _cabi.RBD_F32 if dtype == torch.float32 else _cabi.RBD_F64, B, ld,
                                          qd.data_ptr(), vd.data_ptr(), sd.data_ptr(), None if td is None else td.data_ptr(), step, stage,
                                          ctypes.byref(c), dt, nsteps, *[None if t is None else t.data_ptr() for t in traj],
                                          torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    for t in (qd, vd, sd):
        assert bool(torch.isnan(t[:, B:]).all())
    out = tuple(t[:, :B].double().cpu().numpy() for t in (qd, vd, sd))
    return out + (tuple(t.double().cpu().numpy() for t in traj),) if record else out


def _case(which, B, seed):
    if which == "tree":
        mech = randmech(seed)
        cd = _with_contacts(mech, seed, npoints=7, nhalf=3)
        q, v, tau, _, _ = rand_inputs(mech, B, seed)
    else:
        mech, cd = _atlas_on_floor()
        q, v, tau = _atlas_states(mech, B, seed)
    s = np.random.default_rng(seed).standard_normal((cd.nstates, B)) * 1e-3
    return mech, cd, q, v, tau, s


def _max_rel(a, b):
    return float(np.abs(a - b).max() / max(1.0, np.abs(b).max()))


@pytest.mark.gpu
@pytest.mark.parametrize("which,nsteps,torque", [("tree", 1, "none"), ("tree", 5, "const"), ("tree", 20, "step"), ("tree", 5, "stage"),
                                                 ("atlas", 1, "stage"), ("atlas", 5, "none"), ("atlas", 20, "const"),
                                                 ("atlas", 5, "step")])
def test_gpu_rollout_matches_oracle_fp64(built, which, nsteps, torque):
    import torch
    B = 77 if which == "tree" else 333                          # ragged: not a multiple of the block size
    mech, cd, q, v, tau, s = _case(which, B, 32)
    tau = _tau_arg(tau, torque, nsteps, np.random.default_rng(2))
    orc = Oracle(mech.flatten())
    dt = 1e-3
    qr, vr, sr = integrate_contact(orc, q, v, s, cd, tau, dt=dt, nsteps=nsteps)
    assert np.any(sr != s)                                    # something touched
    qg, vg, sg = _cabi_rollout(mech, cd, q, v, s, tau, torch.float64, dt, nsteps, ld=B + 13)
    assert config_distance(mech, qg, qr) < TOL64
    assert rel_err(vg, vr) < TOL64
    assert _max_rel(sg, sr) < TOL64


@pytest.mark.gpu
@pytest.mark.parametrize("which,torque", [("tree", "const"), ("atlas", "step")])
def test_gpu_rollout_fp32(built, which, torque):
    import torch
    mech, cd, q, v, tau, s = _case(which, 129, 35)
    q = q.astype(np.float32).astype(np.float64); v = v.astype(np.float32).astype(np.float64)
    s = s.astype(np.float32).astype(np.float64)
    tau = _tau_arg(tau.astype(np.float32).astype(np.float64), torque, 5, np.random.default_rng(3))
    tau = None if tau is None else tau.astype(np.float32).astype(np.float64)
    orc = Oracle(mech.flatten())
    qr, vr, sr = integrate_contact(orc, q, v, s, cd, tau, dt=1e-3, nsteps=5)
    qg, vg, sg = _cabi_rollout(mech, cd, q, v, s, tau, torch.float32, 1e-3, 5, ld=129)
    eq, ev = config_distance(mech, qg, qr), rel_err(vg, vr)
    print(f"fp32 {which}: q {eq:.2e}  v {ev:.2e}  s {_max_rel(sg, sr):.2e}")
    assert eq < TOL32 and ev < TOL32


@pytest.mark.gpu
def test_gpu_ball_drop_batch():
    """test/test_simulate.jl:34-89 for a batch of initial positions, fp64, every step of the recorded trajectory."""
    import torch
    mech, cd, com, model = _ball()
    orc = Oracle(mech.flatten())
    B = 48
    rng = np.random.default_rng(5)
    q = np.zeros((7, B)); q[0] = 1; q[4:6] = rng.uniform(-2, 2, (2, B)); q[6] = rng.uniform(0.03, 0.08, B) - com[2]
    st = rbd.MechanismState(mech, batch=B, dtype=torch.float64)
    st.q.copy_(torch.from_numpy(q)); st.v.zero_()
    s = torch.zeros((cd.nstates, B), dtype=torch.float64, device="cuda")
    qt, vt, _ = rbd.simulate_contact_trajectory_(st, 500, s, dt=1e-3)
    qt, vt = qt.cpu().numpy(), vt.cpu().numpy()
    energies = np.stack([_ball_energy(orc, model, qt[n], vt[n]) for n in range(501)])
    assert np.abs(energies - energies[0]).max(0).max() < 1e-2
    sg = np.sign(vt[:, 5])
    assert (np.count_nonzero(sg[1:] != sg[:-1], axis=0) > 3).all()


@pytest.mark.gpu
@pytest.mark.parametrize("stick", [True, False])
def test_gpu_inclined_plane_batch(stick):
    import torch
    mech, cd, theta = _incline(stick)
    B = 40
    rng = np.random.default_rng(9)
    q = np.zeros((7, B)); q[0] = 1
    q[4:6] = rng.uniform(-1, 1, (2, B)); q[6] = -np.tan(theta) * q[4]           # on the plane
    st = rbd.MechanismState(mech, batch=B, dtype=torch.float64)
    st.q.copy_(torch.from_numpy(q)); st.v.zero_()
    s = torch.zeros((cd.nstates, B), dtype=torch.float64, device="cuda")
    assert rbd.simulate_contact_(st, 1.0, s, dt=1e-3) == 1000
    x1 = st.q[4:].cpu().numpy().copy()
    assert float(s[:3].abs().max()) > 0
    rbd.simulate_contact_(st, 0.5, s, dt=1e-3)
    d = np.abs(st.q[4:].cpu().numpy() - x1).max(0)
    if stick:
        assert (d < 1e-4).all()
    else:
        assert (d > 5e-2).all()


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["tree", "atlas"])
def test_gpu_consistency(built, which):
    """Far half-space: s bit for bit, q / v as simulate_ (generic vs specialised kernels: to rounding).  Recording does not change
    the result and its last block is it; two calls equal one call of the summed steps, bit for bit."""
    import torch
    B = 200
    mech, cd, q, v, tau, s = _case(which, B, 38)
    dt, n = 1e-3, 6
    tq = torch.from_numpy(tau).cuda()

    def state():
        st = rbd.MechanismState(mech, batch=B, dtype=torch.float64)
        st.q.copy_(torch.from_numpy(q)); st.v.copy_(torch.from_numpy(v))
        return st, torch.from_numpy(s).cuda()
    far = rbd.ContactDesc(cd.body, cd.location, cd.normal_model, cd.friction_model, cd.halfspace.copy())
    far.halfspace[:] = [0, 0, -100.0, 0, 0, 1.0]
    a, sa = state()
    rbd.simulate_contact_trajectory_(a, n, sa, tq, dt=dt, contact=far)
    assert torch.equal(sa, torch.from_numpy(s).cuda())
    b, _ = state()
    rbd.simulate_trajectory_(b, n, tq, dt=dt)
    assert config_distance(mech, a.q.cpu().numpy(), b.q.cpu().numpy()) < 1e-12
    assert rel_err(a.v.cpu().numpy(), b.v.cpu().numpy()) < 1e-12
    # recording vs not, and one call vs two
    c, sc = state()
    qt, vt, st_ = rbd.simulate_contact_trajectory_(c, n, sc, tq, dt=dt)
    d, sd = state()
    rbd.simulate_contact_(d, n * dt - 1e-9, sd, tq, dt=dt)
    assert torch.equal(c.q, d.q) and torch.equal(c.v, d.v) and torch.equal(sc, sd)
    assert torch.equal(qt[-1], c.q) and torch.equal(vt[-1], c.v) and torch.equal(st_[-1], sc)
    assert torch.equal(qt[0].cpu(), torch.from_numpy(q)) and torch.equal(st_[0].cpu(), torch.from_numpy(s))
    assert not torch.equal(sc, torch.from_numpy(s).cuda())
    e, se = state()
    rbd.simulate_contact_(e, 2 * dt - 1e-9, se, tq, dt=dt)
    rbd.simulate_contact_(e, (n - 2) * dt - 1e-9, se, tq, dt=dt)
    assert torch.equal(e.q, c.q) and torch.equal(e.v, c.v) and torch.equal(se, sc)


@pytest.mark.gpu
@pytest.mark.parametrize("B,per_step", [(4096, 15), (777, 10)])
def test_gpu_launch_count(built, B, per_step):
    """Per step: per stage 1 or 2 coordinate-map kernels and the contact forward-dynamics kernel, then 1 or 2 finishing kernels
    and the contact-state kernel (include/rbd_b200.h): 4 (2 + 1) + 2 + 1 = 15 when the vectorised kernels apply (B >= 1024, a
    multiple of the vector width), 4 (1 + 1) + 1 + 1 = 10 otherwise."""
    import torch
    mech, cd = _atlas_on_floor()
    q, v, tau = _atlas_states(mech, B, 3)
    st = rbd.MechanismState(mech, batch=B, dtype=torch.float64)
    st.q.copy_(torch.from_numpy(q)); st.v.copy_(torch.from_numpy(v))
    s = torch.zeros((cd.nstates, B), dtype=torch.float64, device="cuda")
    for n in (1, 3):
        rbd.simulate_contact_(st, n * 1e-3 - 1e-9, s, dt=1e-3)
        assert rbd.launch_info().kernels_launched == per_step * n


@pytest.mark.gpu
def test_gpu_atlas_fp32_large_batch(built):
    """Atlas with 8 foot points, fp32 at 2^20, 10 steps: finite, and strided samples agree with the fp64 oracle integrator."""
    import torch
    mech, cd = _atlas_on_floor()
    B = 1 << 20
    q, v, tau = _atlas_states(mech, B, 11, vectorised=True)
    q = q.astype(np.float32); v = v.astype(np.float32); tau = tau.astype(np.float32)
    st = rbd.MechanismState(mech, batch=B, dtype=torch.float32)
    st.q.copy_(torch.from_numpy(q)); st.v.copy_(torch.from_numpy(v))
    s = torch.zeros((cd.nstates, B), dtype=torch.float32, device="cuda")
    tg = torch.from_numpy(tau).cuda()
    assert rbd.simulate_contact_(st, 10e-3 - 1e-9, s, tg, dt=1e-3) == 10
    assert bool(torch.isfinite(st.q).all()) and bool(torch.isfinite(st.v).all()) and bool(torch.isfinite(s).all())
    idx = np.arange(0, B, 4099)
    orc = Oracle(mech.flatten())
    qr, vr, sr = integrate_contact(orc, q[:, idx].astype(np.float64), v[:, idx].astype(np.float64), np.zeros((cd.nstates, idx.size)), cd,
                                   tau[:, idx].astype(np.float64), dt=1e-3, nsteps=10)
    eq = config_distance(mech, st.q[:, idx].double().cpu().numpy(), qr)
    ev = rel_err(st.v[:, idx].double().cpu().numpy(), vr)
    print(f"Atlas fp32 2^20, 10 steps: q {eq:.2e}  v {ev:.2e}")
    assert eq < TOL32 and ev < TOL32
