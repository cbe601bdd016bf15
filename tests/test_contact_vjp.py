"""Reverse mode through contact rollouts (DESIGN 4.15): rbd_integrate_contact_vjp (csrc/rbd_contact_adjoint.cuh) and
rigidbodydynamics.jl_b200.autodiff.simulate_contact.

The loss of every check is  L = sum_s q̄_s . q_s + v̄_s . v_s + s̄_s . s_s  over the recorded trajectory.
CPU tier: the adjoint of the force law against central differences, branch by branch; the whole backward pass run on the CPU
(tests/hostsim/hostsim_contact_vjp.cpp) against central differences of the fp64 oracle integrator (tests/contact_oracle.py) along
random directions of q (as q̇(u)), v, s and the torques.  GPU tier: the kernels against that CPU run and the torch.autograd function."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from oracle import Oracle
from rigidbodydynamics.jl_b200 import _cabi
from rigidbodydynamics.jl_b200._cabi import RbdModelDesc, make_desc
from tests.contact_oracle import integrate_contact
from tests.test_contact import _free_body, _with_contacts
from tests.test_contact_rollout import _atlas_on_floor, _atlas_states, _empty_desc
from tests.test_integrate_vjp import host_ivjp, host_traj
from tests.util import rand_inputs, randmech, rel_err

# central differences of the fp64 oracle at eps = 1e-5, the precedent of DESIGN 4.13 (tests/test_integrate_vjp.py)
TOL_FD = 1e-6
EPS_FD = 1e-5
TOL64 = 1e-10        # GPU kernels against the CPU run of the same code, fp64
# The single-body cases sit 1 cm deep in a stiff contact; there the fp64 kernels differ from the CPU run (compiled without fused
# multiply-adds) by up to 3.1e-9, measured on an H100 (ball drop, B = 1 and 161), and their fp32 runs are not compared (see
# DESIGN 4.15); their fp64 gradients are also checked by gradcheck below.
TOL64_STIFF = 1e-8
# fp32 kernels against the fp64 CPU run on Atlas and the random tree.  Bound of the single-call VJPs (tests/test_vjp.py) x 4.
TOL32 = 2e-2
DT = 1e-3

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "..", "rigidbodydynamics", "jl_b200", "csrc")
_lib = None


def _shim():
    """tests/hostsim/hostsim_contact_vjp.cpp, compiled on first use into a temporary directory."""
    global _lib
    if _lib is not None:
        return _lib
    srcs = [os.path.join(_HERE, "hostsim", "hostsim_contact_vjp.cpp")] + sorted(
        os.path.join(_CSRC, f) for f in os.listdir(_CSRC) if f.endswith((".cuh", ".h")) or f == "rbd_model.cpp")
    h = hashlib.sha1(b"".join(open(s, "rb").read() for s in srcs)).hexdigest()[:16]
    d = os.path.join(tempfile.gettempdir(), f"rbd_hostsim_contact_vjp_{os.getuid()}")
    os.makedirs(d, exist_ok=True)
    so = os.path.join(d, f"hostsim_contact_vjp_{h}.so")
    if not os.path.exists(so):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so + f".{os.getpid()}",
                               srcs[0], os.path.join(_CSRC, "rbd_model.cpp")])
        os.replace(so + f".{os.getpid()}", so)
    lib = ctypes.CDLL(so)
    vp, i64, c_int, c_double = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_double
    lib.hostsim_integrate_contact_vjp.argtypes = [ctypes.POINTER(RbdModelDesc), c_int, i64, vp, vp, vp, vp, i64, i64, vp, c_double,
                                                  c_int] + [vp] * 8
    lib.hostsim_contact_force.argtypes = [vp, vp, vp, c_double, vp, vp, vp, vp]
    lib.hostsim_contact_force_adjoint.argtypes = [vp, vp, vp, c_double] + [vp] * 7
    _lib = lib
    return lib


def _p(a):
    return None if a is None or a.size == 0 else a.ctypes.data


def _sched(tau, nv, B):
    if tau is None:
        return None, 0, 0
    blk = nv * B
    return np.ascontiguousarray(tau), {2: 0, 3: blk, 4: 4 * blk}[tau.ndim], blk if tau.ndim == 4 else 0


def host_cvjp(desc, cd, qt, vt, st, tau, n, qtb, vtb, stb, dt=DT):
    """The CPU run of rbd_integrate_contact_vjp: dict q0t, q0c, v0b, s0b, taub (shape of tau)."""
    dt_ = qt.dtype
    B = qt.shape[2]
    c = lambda a: None if a is None else np.ascontiguousarray(a, dt_)      # noqa: E731
    t, step, stage = _sched(c(tau), desc.nv, B)
    out = {"q0t": np.full((desc.nv, B), np.nan, dt_), "q0c": np.full((desc.nq, B), np.nan, dt_), "v0b": np.full((desc.nv, B), np.nan, dt_),
           "s0b": np.full((cd.nstates, B), np.nan, dt_), "taub": None if tau is None else np.zeros(tau.shape, dt_)}
    d, keep = make_desc(desc)
    cs, keep2 = cd.c_struct()
    assert _shim().hostsim_integrate_contact_vjp(ctypes.byref(d), 0 if dt_ == np.float32 else 1, B, _p(c(qt)), _p(c(vt)), _p(c(st)), _p(t),
                                                 step, stage, ctypes.byref(cs), dt, n, _p(c(qtb)), _p(c(vtb)), _p(c(stb)), _p(out["q0t"]),
                                                 _p(out["q0c"]), _p(out["v0b"]), _p(out["s0b"]), _p(out["taub"])) == 0
    return out


def oracle_traj(orc, cd, q, v, s, tau, n, dt=DT):
    qs, vs, ss = [], [], []
    integrate_contact(orc, q, v, s, cd, tau, dt=dt, nsteps=n,
                      record=lambda k, q_, v_, s_: (qs.append(q_.copy()), vs.append(v_.copy()), ss.append(s_.copy())))
    return np.stack(qs), np.stack(vs), np.stack(ss)


def _loss(orc, cd, q, v, s, tau, n, qtb, vtb, stb, dt=DT):
    qt, vt, st = oracle_traj(orc, cd, q, v, s, tau, n, dt)
    return (qt * qtb).sum((0, 1)) + (vt * vtb).sum((0, 1)) + (st * stb).sum((0, 1))


# ----------------------------------------------------------------------------------------------------------------------
# cases
# ----------------------------------------------------------------------------------------------------------------------
def _ball_case(B):
    rng = np.random.default_rng(61)
    mech, body = _free_body(rng=rng)
    com = body.inertia.cross_part / body.inertia.mass
    model = rbd.SoftContactModel(rbd.hunt_crossley_hertz(k=5e3, alpha=0.2), rbd.ViscoelasticCoulombModel(0.5, 1e3, 1e3))
    rbd.add_contact_point(body, rbd.ContactPoint(com, model))
    rbd.add_environment_primitive(mech, rbd.HalfSpace3D(np.zeros(3), [0, 0, 1.0]))
    q = np.zeros((7, B)); q[0] = 1; q[4:6] = rng.uniform(-1, 1, (2, B)); q[6] = -0.01 - com[2]     # 1 cm into the floor
    v = np.zeros((6, B)); v[5] = -0.2                                                                 # still going down
    return mech, rbd.contact_desc(mech), q, v, np.zeros((3, B))


def _incline_case(stick, B):
    theta = 0.5
    mu = np.tan(theta) + (0.3 if stick else -0.3)
    mech, body = _free_body(rbd.SpatialInertia(np.eye(3), np.zeros(3), 2.0))
    rbd.add_environment_primitive(mech, rbd.HalfSpace3D(np.zeros(3), [np.sin(theta), 0, np.cos(theta)]))
    model = rbd.SoftContactModel(rbd.hunt_crossley_hertz(k=5e3, alpha=1.0), rbd.ViscoelasticCoulombModel(mu, 5e3, 1e2))
    rbd.add_contact_point(body, rbd.ContactPoint(np.zeros(3), model))
    rng = np.random.default_rng(9)
    q = np.zeros((7, B)); q[0] = 1
    q[4] = rng.uniform(-1, 1, B); q[6] = -np.tan(theta) * q[4] - 0.01 / np.cos(theta)               # 1 cm into the plane
    v = np.zeros((6, B)); v[3] = 0.05 * np.cos(theta); v[5] = -0.05 * np.sin(theta)                  # sliding down the plane
    s = np.zeros((3, B))
    if stick:
        s[:] = np.array([[0.0], [0.0], [0.0]])
    return mech, rbd.contact_desc(mech), q, v, s


def _atlas_case(B):
    mech, cd = _atlas_on_floor()
    q, v, _ = _atlas_states(mech, B, 21)
    q[4:6] = 0.0
    q[6] = 0.9                                                           # feet a few mm into the floor
    s = np.random.default_rng(3).standard_normal((cd.nstates, B)) * 1e-4
    return mech, cd, q, v, s


def _tree_case(B):
    rng = np.random.default_rng(5)
    mech = rbd.rand_tree_mechanism(rng, [rbd.QuaternionFloating, rbd.Revolute, rbd.Prismatic, rbd.Planar, rbd.QuaternionSpherical,
                                         rbd.SPQuatFloating, rbd.SinCosRevolute, rbd.Fixed, rbd.Revolute])
    cd = _with_contacts(mech, 8, npoints=6, nhalf=2)
    q, v, _, _, _ = rand_inputs(mech, B, 5)
    v *= 0.3
    s = np.random.default_rng(6).standard_normal((cd.nstates, B)) * 1e-2
    return mech, cd, q, v, s


CASES = {"ball": _ball_case, "incline_stick": lambda B: _incline_case(True, B), "incline_slip": lambda B: _incline_case(False, B),
         "atlas": _atlas_case, "tree": _tree_case}


def _tau(kind, nv, B, n, rng, scale):
    return {"none": None, "const": rng.standard_normal((nv, B)) * scale, "step": rng.standard_normal((n, nv, B)) * scale,
            "stage": rng.standard_normal((n, 4, nv, B)) * scale}[kind]


# ----------------------------------------------------------------------------------------------------------------------
# CPU tier: the force law
# ----------------------------------------------------------------------------------------------------------------------
def _force(hc, fr, nrm, z, vel, x):
    f, xd = np.zeros(3), np.zeros(3)
    _shim().hostsim_contact_force(_p(hc), _p(fr), _p(nrm), z, _p(vel), _p(x), _p(f), _p(xd))
    return np.concatenate([f, xd])


def _force_branch(hc, fr, nrm, z, vel, x):
    """(f_n clamped, slipping) as contact_force decides them"""
    zd = -vel @ nrm
    zn = z ** hc[2]
    fn = max(hc[1] * zn * zd + hc[0] * zn, 0.0)
    ft = -fr[1] * x - fr[2] * (vel + zd * nrm)
    return fn == 0.0, ft @ ft > (fr[0] * fn) ** 2


@pytest.mark.parametrize("branch", ["stick", "slip", "clamped", "surface"])
def test_contact_force_adjoint_matches_finite_differences(branch):
    """The adjoint of contact_force against central differences of the same fp64 code, on each branch; at z = 0 (a point exactly on
    the surface) it is finite and equals the one-sided difference."""
    lib = _shim()
    rng = np.random.default_rng({"stick": 1, "slip": 2, "clamped": 3, "surface": 4}[branch])
    nrm = rng.standard_normal(3); nrm /= np.linalg.norm(nrm)
    hc, fr = np.array([5e3, 1.5 * 0.2 * 5e3, 1.5]), np.array([0.6, 1e3, 50.0])
    z, vel, x = 0.01, 0.05 * rng.standard_normal(3), 1e-4 * rng.standard_normal(3)
    if branch == "stick":
        vel = 0.1 * vel
    elif branch == "slip":
        vel = vel + 3.0 * np.cross(nrm, rng.standard_normal(3))        # fast tangential motion
    elif branch == "clamped":
        vel = vel + 20.0 * nrm                                          # separating faster than the spring pushes
    elif branch == "surface":
        z = 0.0
    clamped, slip = _force_branch(hc, fr, nrm, z, vel, x)
    assert (clamped, slip) == {"stick": (False, False), "slip": (False, True), "clamped": (True, True), "surface": (True, True)}[branch]
    fb, xdb = rng.standard_normal(3), rng.standard_normal(3)
    w = np.concatenate([fb, xdb])
    zb, velb, xb = np.zeros(1), np.zeros(3), np.zeros(3)
    lib.hostsim_contact_force_adjoint(_p(hc), _p(fr), _p(nrm), z, _p(vel), _p(x), _p(fb), _p(xdb), _p(zb), _p(velb), _p(xb))
    assert np.isfinite(zb).all() and np.isfinite(velb).all() and np.isfinite(xb).all()
    eps = 1e-7
    F = lambda z_=z, vel_=vel, x_=x: w @ _force(hc, fr, nrm, z_, vel_, x_)      # noqa: E731
    e = lambda k: np.eye(3)[k] * eps                                            # noqa: E731
    for k in range(3):                       # the branch holds within ±eps
        for sg in (1, -1):
            assert _force_branch(hc, fr, nrm, z, vel + sg * e(k), x) == (clamped, slip)
            assert _force_branch(hc, fr, nrm, z, vel, x + sg * e(k)) == (clamped, slip)
    ref_vel = [(F(vel_=vel + e(k)) - F(vel_=vel - e(k))) / (2 * eps) for k in range(3)]
    ref_x = [(F(x_=x + e(k)) - F(x_=x - e(k))) / (2 * eps) for k in range(3)]
    scale = max(1.0, np.abs(ref_vel).max(), np.abs(ref_x).max())
    assert np.abs(velb - ref_vel).max() < 1e-6 * scale, (velb, ref_vel)
    assert np.abs(xb - ref_x).max() < 1e-6 * scale, (xb, ref_x)
    if branch == "surface":
        # one-sided (z < 0 is out of contact): the differences fall like sqrt(h) (n = 1.5) to their limit, 0
        one = [abs(F(z_=h) - F(z_=0.0)) / h for h in (1e-8, 1e-10, 1e-12)]
        assert one[1] < one[0] / 5 and one[2] < one[1] / 5 and one[2] < 1e-2, one
        assert zb[0] == 0.0
    else:
        ref_z = (F(z_=z + eps) - F(z_=z - eps)) / (2 * eps)
        assert abs(zb[0] - ref_z) < 1e-6 * max(1.0, abs(ref_z)), (zb, ref_z)


# ----------------------------------------------------------------------------------------------------------------------
# CPU tier: the whole backward pass
# ----------------------------------------------------------------------------------------------------------------------
FD_PARAMS = [("ball", 1, "none"), ("ball", 5, "const"), ("incline_stick", 1, "step"), ("incline_stick", 5, "stage"),
             ("incline_slip", 1, "const"), ("incline_slip", 5, "none"), ("atlas", 1, "stage"), ("atlas", 5, "step"),
             ("tree", 1, "const"), ("tree", 5, "stage")]


@pytest.mark.parametrize("which,n,tmode", FD_PARAMS)
def test_rollout_vjp_hostsim_matches_oracle_finite_differences(which, n, tmode):
    """Directional derivatives of L along q̇(u), v, s and the torques: the CPU run of the backward pass against central differences
    of the fp64 oracle integrator.  No pair may change contact, clamping or stick / slip mode within ±eps anywhere in the rollout:
    that is asserted by requiring the gap between the two one-sided differences to shrink with the step (a mode change is a kink,
    whose gap does not)."""
    B = 2
    mech, cd, q, v, s = CASES[which](B)
    d = mech.flatten()
    orc = Oracle(d)
    rng = np.random.default_rng(len(which) + n)
    tau = _tau(tmode, d.nv, B, n, rng, 0.5)
    qt, vt, st = oracle_traj(orc, cd, q, v, s, tau, n)
    assert np.any(st != st[0]) or which == "ball" and np.any(vt[-1] != vt[0])      # something touched
    qtb, vtb, stb = rng.standard_normal(qt.shape), rng.standard_normal(vt.shape), rng.standard_normal(st.shape)
    r = host_cvjp(d, cd, qt, vt, st, tau, n, qtb, vtb, stb)
    f = lambda q_=q, v_=v, s_=s, t_=tau: _loss(orc, cd, q_, v_, s_, t_, n, qtb, vtb, stb)     # noqa: E731
    eps = EPS_FD
    L0 = f()

    def check(got, g):
        fp, fm = g(eps), g(-eps)
        ref = (fp - fm) / (2 * eps)
        # the gap between the one-sided slopes is curvature x h on a smooth branch, but does not shrink with h across a kink
        gap = lambda h: np.abs((g(h) - L0) / h - (L0 - g(-h)) / h)      # noqa: E731
        g1, g2 = gap(eps), gap(eps / 10)
        # (or stays at the level of the oracle's rounding noise over h)
        assert ((g2 < 0.2 * g1) | (g2 < 1e-3 * np.maximum(1.0, np.abs(ref)))).all(), ("mode change within eps", g1, g2, ref)
        assert rel_err(got, ref) < TOL_FD, (rel_err(got, ref), got, ref)

    u = rng.standard_normal((d.nv, B))
    qd = orc.dynamics(q, u, None, want_qd=True)[1]
    check((r["q0t"] * u).sum(0), lambda h: f(q_=q + h * qd))
    dv = rng.standard_normal((d.nv, B))
    check((r["v0b"] * dv).sum(0), lambda h: f(v_=v + h * dv))
    if cd.nstates:
        ds = rng.standard_normal((cd.nstates, B)) * 1e-2
        check((r["s0b"] * ds).sum(0), lambda h: f(s_=s + h * ds))
    if tau is not None:
        dtau = rng.standard_normal(tau.shape)
        check((r["taub"] * dtau).sum(tuple(range(tau.ndim - 1))), lambda h: f(t_=tau + h * dtau))
    # the configuration form pairs with q̇ like the tangent form with v
    assert np.abs((r["q0c"] * qd).sum(0) - (r["q0t"] * u).sum(0)).max() < 1e-10 * max(1.0, np.abs(r["q0t"]).max() * np.abs(u).max() * d.nv)


@pytest.mark.parametrize("which", ["tree", "atlas"])
def test_no_pair_in_contact_is_the_contact_free_vjp(which):
    """Every half-space far below: the backward pass equals rbd_integrate_vjp's CPU run to 1e-12, and s̄0 is the sum of the
    s_traj_bar blocks (frozen pairs pass their adjoint through)."""
    B, n = 3, 4
    mech, cd, q, v, s = CASES[which](B)
    cd.halfspace[:] = [0, 0, -100.0, 0, 0, 1.0]
    d = mech.flatten()
    rng = np.random.default_rng(2)
    tau = rng.standard_normal((n, d.nv, B))
    qt, vt = host_traj(d, q, v, tau, n, dt=DT)
    st = np.repeat(s[None], n + 1, 0)
    qtb, vtb, stb = rng.standard_normal(qt.shape), rng.standard_normal(vt.shape), rng.standard_normal(st.shape)
    r = host_cvjp(d, cd, qt, vt, st, tau, n, qtb, vtb, stb)
    ref = host_ivjp(d, qt, vt, tau, n, qtb, vtb, dt=DT)
    for k in ("q0t", "q0c", "v0b", "taub"):
        assert rel_err(r[k], ref[k]) < 1e-12, (k, rel_err(r[k], ref[k]))
    assert np.allclose(r["s0b"], stb.sum(0), rtol=0, atol=1e-12)


def test_zero_steps_is_the_identity():
    mech, cd, q, v, s = CASES["ball"](3)
    d = mech.flatten()
    rng = np.random.default_rng(0)
    qtb, vtb, stb = rng.standard_normal((1, d.nq, 3)), rng.standard_normal((1, d.nv, 3)), rng.standard_normal((1, cd.nstates, 3))
    r = host_cvjp(d, cd, q[None], v[None], s[None], None, 0, qtb, vtb, stb)
    assert np.array_equal(r["v0b"], vtb[0]) and np.array_equal(r["s0b"], stb[0])


# ----------------------------------------------------------------------------------------------------------------------
# CPU tier: C-ABI argument checks (host only, nothing launched)
# ----------------------------------------------------------------------------------------------------------------------
def test_integrate_contact_vjp_argument_checks(built):
    lib = rbd.load_library()
    mech = randmech(33)
    cd = _with_contacts(mech, 3, npoints=2, nhalf=1)
    h = _cabi.ModelHandle(mech.flatten())
    st, keep = cd.c_struct()
    fake = ctypes.c_void_p(64)                  # never dereferenced by the checks below
    F32, F64 = _cabi.RBD_F32, _cabi.RBD_F64

    def call(dtype=F64, B=4, qt=fake, vt=fake, s=fake, tau=None, step=0, stage=0, contact=ctypes.byref(st), dt=1e-3, n=1, tb=None):
        return lib.rbd_integrate_contact_vjp(h.ptr, dtype, B, qt, vt, s, tau, step, stage, contact, dt, n, None, None, None, None, None,
                                             None, None, tb, None)

    assert call(dtype=_cabi.RBD_DUAL64X6) == _cabi.RBD_EUNSUPPORTED
    assert call(dtype=7) == _cabi.RBD_EINVAL
    assert call(n=-1) == _cabi.RBD_EINVAL
    assert call(dt=0.0) == _cabi.RBD_EINVAL and call(dt=-1e-3) == _cabi.RBD_EINVAL
    assert call(step=-1) == _cabi.RBD_EINVAL and call(stage=-4) == _cabi.RBD_EINVAL
    assert call(tb=fake) == _cabi.RBD_EINVAL and b"tau_bar needs tau" in lib.rbd_last_error()
    assert call(qt=None) == _cabi.RBD_EINVAL and call(vt=None) == _cabi.RBD_EINVAL
    assert call(s=None) == _cabi.RBD_EINVAL and b"s_traj must not be NULL" in lib.rbd_last_error()
    assert call(contact=None) == _cabi.RBD_EINVAL
    assert call(B=-1) == _cabi.RBD_EDIM
    assert call(B=0, qt=None, vt=None, s=None) == _cabi.RBD_OK                # empty batch: nothing to do
    assert lib.rbd_integrate_contact_vjp(None, F32, 1, fake, fake, fake, None, 0, 0, ctypes.byref(st), 1e-3, 1, None, None, None, None, None,
                                         None, None, None, None) == _cabi.RBD_EINVAL
    bad = rbd.ContactDesc(cd.body.copy(), cd.location, cd.normal_model, cd.friction_model, cd.halfspace)
    bad.body[0] = 99
    st2, keep2 = bad.c_struct()
    assert call(contact=ctypes.byref(st2)) == _cabi.RBD_EINVAL and b"body index" in lib.rbd_last_error()
    many = rbd.ContactDesc(np.zeros(33, np.int32), np.zeros((33, 3)), np.ones((33, 3)), np.ones((33, 3)), cd.halfspace)
    st3, keep3 = many.c_struct()
    assert call(contact=ctypes.byref(st3)) == _cabi.RBD_EUNSUPPORTED
    e = _empty_desc()
    st4, keep4 = e.c_struct()
    assert call(s=None, contact=ctypes.byref(st4), B=0) == _cabi.RBD_OK
    h.close()


def test_simulate_contact_refuses_loops(built):
    """Mechanisms with loops are refused before anything is launched (no GPU needed)."""
    from rigidbodydynamics.jl_b200 import autodiff
    from tests.loops_oracle import four_bar
    mech = four_bar()
    with pytest.raises(rbd.RbdError) as e:
        autodiff.simulate_contact(mech, None, None, None, contact=_empty_desc(), dt=DT, nsteps=1)
    assert e.value.status == _cabi.RBD_ELOOP


# ----------------------------------------------------------------------------------------------------------------------
# GPU tier
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch():
    import torch as t
    assert t.cuda.is_available()
    rbd.load_library()
    return t


def _gpu_traj(torch, mech, cd, q, v, s, tau, n, dtype):
    st = rbd.MechanismState(mech, q.shape[1], dtype)
    st.q.copy_(torch.from_numpy(q)); st.v.copy_(torch.from_numpy(v))
    sc = torch.from_numpy(np.ascontiguousarray(s)).to(dtype).cuda()
    t = None if tau is None else torch.from_numpy(np.ascontiguousarray(tau)).to(dtype).cuda()
    qt, vt, stj = rbd.simulate_contact_trajectory_(st, n, sc, t, dt=DT, contact=cd)
    return t, qt, vt, stj


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["ball", "incline_slip", "atlas", "tree"])
@pytest.mark.parametrize("B", [1, 161])
def test_kernels_vs_hostsim(torch, which, B):
    """rbd_integrate_contact_vjp against the CPU run of the same code: fp64 and fp32, every torque shape."""
    n = 3
    mech, cd, q, v, s = CASES[which](B)
    d = mech.flatten()
    rng = np.random.default_rng(B)
    worst = 0.0
    for tmode in ("none", "const", "step", "stage"):
        tau = _tau(tmode, d.nv, B, n, rng, 0.5)
        stiff = which in ("ball", "incline_slip")
        for dtype in (torch.float64,) if stiff else (torch.float64, torch.float32):
            t, qt, vt, stj = _gpu_traj(torch, mech, cd, q, v, s, tau, n, dtype)
            qtb, vtb, stb = (rng.standard_normal(tuple(x.shape)) for x in (qt, vt, stj))
            T = lambda a: torch.from_numpy(a).to(dtype).cuda()      # noqa: E731
            e = lambda rows: torch.full((rows, B), float("nan"), dtype=dtype, device="cuda")      # noqa: E731
            out = {"q0t": e(d.nv), "q0c": e(d.nq), "v0b": e(d.nv), "s0b": e(cd.nstates), "taub": None if t is None else torch.zeros_like(t)}
            rbd.integrate_contact_vjp_(mech, qt, vt, stj, t, contact=cd, dt=DT, q_traj_bar=T(qtb), v_traj_bar=T(vtb), s_traj_bar=T(stb),
                                       q0_bar_tan=out["q0t"], q0_bar_cfg=out["q0c"], v0_bar=out["v0b"], s0_bar=out["s0b"],
                                       tau_bar=out["taub"])
            torch.cuda.synchronize()
            np64 = lambda x: x.double().cpu().numpy()      # noqa: E731
            ref = host_cvjp(d, cd, np64(qt), np64(vt), np64(stj), None if t is None else np64(t), n, qtb, vtb, stb)
            tol = (TOL64_STIFF if stiff else TOL64) if dtype == torch.float64 else TOL32
            for k in ("q0t", "q0c", "v0b", "s0b", "taub"):
                if out[k] is None:
                    continue
                err = rel_err(np64(out[k]).reshape(ref[k].shape), ref[k])
                if dtype == torch.float32:
                    worst = max(worst, err)
                assert err < tol, (tmode, dtype, k, err)
    print(f"{which} B={B}: worst fp32 rel_err {worst:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("which,trajectory", [("ball", True), ("incline_stick", False), ("incline_slip", True)])
def test_simulate_contact_gradcheck(torch, which, trajectory):
    from rigidbodydynamics.jl_b200 import autodiff
    B, n = 2, 3
    mech, cd, q, v, s = CASES[which](B)
    d = mech.flatten()
    tau = np.random.default_rng(1).standard_normal((n, d.nv, B)) * 0.1
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda().requires_grad_(True)      # noqa: E731
    f = lambda q_, v_, s_, t_: autodiff.simulate_contact(mech, q_, v_, s_, t_, contact=cd, dt=DT, nsteps=n, trajectory=trajectory)  # noqa
    # q0 moves along the configuration space, not along q̇ directions: gradcheck's raw perturbation of a quaternion is a
    # perturbation of the unnormalised formula, whose radial part the gradient deliberately omits -- so check q through v only
    fq = lambda v_, s_, t_: f(torch.from_numpy(q).cuda(), v_, s_, t_)      # noqa: E731
    assert torch.autograd.gradcheck(fq, (T(v), T(s), T(tau)), eps=1e-7, atol=1e-5, rtol=1e-4)


@pytest.mark.gpu
def test_autograd_equals_direct_call_and_checkpointing(torch):
    """autograd equals the direct call bit for bit; checkpointed runs and split calls are bit-identical, tau_bar accumulation
    included; the q0 gradient along q̇ directions matches the oracle."""
    from rigidbodydynamics.jl_b200 import autodiff
    B, n = 5, 6
    mech, cd, q, v, s = CASES["atlas"](B)
    d = mech.flatten()
    rng = np.random.default_rng(4)
    tau = rng.standard_normal((n, d.nv, B)) * 0.5
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda().requires_grad_(True)      # noqa: E731
    tq, tv, ts, tt = T(q), T(v), T(s), T(tau)
    qt, vt, stj = autodiff.simulate_contact(mech, tq, tv, ts, tt, contact=cd, dt=DT, nsteps=n)
    qtb, vtb, stb = torch.randn_like(qt), torch.randn_like(vt), torch.randn_like(stj)
    ((qt * qtb).sum() + (vt * vtb).sum() + (stj * stb).sum()).backward()
    outs = {"q": torch.empty_like(tq), "v": torch.empty_like(tv), "s": torch.empty_like(ts), "t": torch.zeros_like(tt)}
    rbd.integrate_contact_vjp_(mech, qt.detach(), vt.detach(), stj.detach(), tt.detach(), contact=cd, dt=DT, q_traj_bar=qtb,
                               v_traj_bar=vtb, s_traj_bar=stb, q0_bar_cfg=outs["q"], v0_bar=outs["v"], s0_bar=outs["s"], tau_bar=outs["t"])
    torch.cuda.synchronize()
    for k, x in (("q", tq), ("v", tv), ("s", ts), ("t", tt)):
        assert torch.equal(x.grad, outs[k]), k
    # checkpointing and the trajectory form give the same gradients of the final state, bit for bit
    grads = []
    for k in (None, 1, 4, n):
        tq.grad = tv.grad = ts.grad = tt.grad = None
        if k is None:
            qf, vf, sf = (x[-1] for x in autodiff.simulate_contact(mech, tq, tv, ts, tt, contact=cd, dt=DT, nsteps=n))
        else:
            qf, vf, sf = autodiff.simulate_contact(mech, tq, tv, ts, tt, contact=cd, dt=DT, nsteps=n, trajectory=False, checkpoint_every=k)
        ((qf * qtb[-1]).sum() + (vf * vtb[-1]).sum() + (sf * stb[-1]).sum()).backward()
        grads.append((tq.grad.clone(), tv.grad.clone(), ts.grad.clone(), tt.grad.clone()))
    for g in grads[1:]:
        assert all(torch.equal(a, b) for a, b in zip(g, grads[0]))
    # a double backward raises
    tq.grad = None
    qf, _, _ = autodiff.simulate_contact(mech, tq, tv, ts, None, contact=cd, dt=DT, nsteps=2, trajectory=False)
    g, = torch.autograd.grad(qf.sum(), tq, create_graph=True)
    with pytest.raises(RuntimeError):
        g.sum().backward()


@pytest.mark.gpu
def test_no_contact_points_matches_simulate(torch):
    """npoints = 0: the gradients of autodiff.simulate, to 1e-12 in fp64 (generic against specialised dynamics)."""
    from rigidbodydynamics.jl_b200 import autodiff
    mech = rbd.load_model("atlas", floating=True)
    d = mech.flatten()
    B, n = 64, 4
    q, v, tau, _, _ = rand_inputs(mech, B, 3)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda().requires_grad_(True)      # noqa: E731
    tq, tv, tt = T(q), T(v), T(tau)
    qt, vt = autodiff.simulate(mech, tq, tv, tt, dt=DT, nsteps=n)
    qtb, vtb = torch.randn_like(qt), torch.randn_like(vt)
    ((qt * qtb).sum() + (vt * vtb).sum()).backward()
    ref = (tq.grad.clone(), tv.grad.clone(), tt.grad.clone())
    tq.grad = tv.grad = tt.grad = None
    s0 = torch.zeros((0, B), dtype=torch.float64, device="cuda")
    qc, vc, sc = autodiff.simulate_contact(mech, tq, tv, s0, tt, contact=_empty_desc(), dt=DT, nsteps=n)
    assert rel_err(qc.detach().cpu().numpy(), qt.detach().cpu().numpy()) < 1e-12
    ((qc * qtb).sum() + (vc * vtb).sum()).backward()
    for a, b in zip((tq.grad, tv.grad, tt.grad), ref):
        assert rel_err(a.cpu().numpy(), b.cpu().numpy()) < 1e-12


@pytest.mark.gpu
def test_split_calls_are_bit_identical(torch):
    """Two consecutive calls over the segments of one rollout give one call's gradients bit for bit, tau_bar accumulated."""
    B, n = 300, 6
    mech, cd, q, v, s = CASES["atlas"](B)
    d = mech.flatten()
    tau = torch.from_numpy(np.random.default_rng(2).standard_normal((d.nv, B)) * 0.5).cuda()
    _, qt, vt, stj = _gpu_traj(torch, mech, cd, q, v, s, tau.cpu().numpy(), n, torch.float64)
    bars = [torch.randn_like(x) for x in (qt, vt, stj)]
    e = lambda x: torch.empty_like(x[0])      # noqa: E731
    one = [e(qt), e(vt), e(stj), torch.zeros_like(tau)]
    rbd.integrate_contact_vjp_(mech, qt, vt, stj, tau, contact=cd, dt=DT, q_traj_bar=bars[0], v_traj_bar=bars[1], s_traj_bar=bars[2],
                               q0_bar_cfg=one[0], v0_bar=one[1], s0_bar=one[2], tau_bar=one[3])
    k = 2
    tail = [e(qt), e(vt), e(stj)]
    tb = torch.zeros_like(tau)
    sl = lambda x, a, b: x[a:b].contiguous()      # noqa: E731
    rbd.integrate_contact_vjp_(mech, sl(qt, k, n + 1), sl(vt, k, n + 1), sl(stj, k, n + 1), tau, contact=cd, dt=DT,
                               q_traj_bar=sl(bars[0], k, n + 1), v_traj_bar=sl(bars[1], k, n + 1), s_traj_bar=sl(bars[2], k, n + 1),
                               q0_bar_cfg=tail[0], v0_bar=tail[1], s0_bar=tail[2], tau_bar=tb)
    head_bars = [sl(x, 0, k + 1) for x in bars]
    for hb, t in zip(head_bars, tail):
        hb[-1] = t
    two = [e(qt), e(vt), e(stj)]
    rbd.integrate_contact_vjp_(mech, sl(qt, 0, k + 1), sl(vt, 0, k + 1), sl(stj, 0, k + 1), tau, contact=cd, dt=DT, q_traj_bar=head_bars[0],
                               v_traj_bar=head_bars[1], s_traj_bar=head_bars[2], q0_bar_cfg=two[0], v0_bar=two[1], s0_bar=two[2], tau_bar=tb)
    torch.cuda.synchronize()
    for a, b in zip(two + [tb], one):
        assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [4096, 777])
def test_launch_count_linear_in_nsteps(torch, B):
    mech, cd, q, v, s = CASES["atlas"](B)
    counts = []
    for n in (1, 2, 3):
        _, qt, vt, stj = _gpu_traj(torch, mech, cd, q, v, s, None, n, torch.float64)
        rbd.integrate_contact_vjp_(mech, qt, vt, stj, None, contact=cd, dt=DT, v_traj_bar=torch.randn_like(vt),
                                   v0_bar=torch.empty_like(vt[0]))
        counts.append(rbd.launch_info().kernels_launched)
    assert counts[2] - counts[1] == counts[1] - counts[0] > 0, counts


@pytest.mark.gpu
def test_atlas_fp32_large_batch_point_on_floor(torch):
    """Atlas with 8 foot points, fp32 at 2^20: finite gradients, with one foot point exactly on the floor in every sample."""
    mech, cd = _atlas_on_floor()
    d = mech.flatten()
    B, n = 1 << 20, 2
    q, v, tau = _atlas_states(mech, B, 11, vectorised=True)
    q[:4] = np.array([[1.0], [0], [0], [0]]); q[4:6] = 0; q[7:] = 0; v[:] = 0
    # upright with zero joint angles: lower the robot until the first foot point sits exactly on z = 0
    k = Oracle(d).kinematics(q[:, :1].astype(np.float64), None, want=("transforms",))["transforms"]
    foot = cd.body[0]
    R, p = k[12 * foot:12 * foot + 9, 0].reshape(3, 3), k[12 * foot + 9:12 * foot + 12, 0]
    q[6] -= (R @ cd.location[0] + p)[2]
    qg = torch.from_numpy(q.astype(np.float32)).cuda(); vg = torch.from_numpy(v.astype(np.float32)).cuda()
    sg = torch.zeros((cd.nstates, B), dtype=torch.float32, device="cuda")
    tg = torch.from_numpy(tau.astype(np.float32)).cuda()
    from rigidbodydynamics.jl_b200 import autodiff
    qg.requires_grad_(True); vg.requires_grad_(True); sg.requires_grad_(True); tg.requires_grad_(True)
    qf, vf, sf = autodiff.simulate_contact(mech, qg, vg, sg, tg, contact=cd, dt=DT, nsteps=n, trajectory=False)
    (qf.sum() + vf.sum() + sf.sum()).backward()
    torch.cuda.synchronize()
    for x in (qg, vg, sg, tg):
        assert bool(torch.isfinite(x.grad).all())
