"""TEST INFRASTRUCTURE -- simulate() for mechanisms with contact points, restated on the host over the CPU oracle (oracle/).

integrate_contact_step is MuntheKaasIntegrator.step (src/ode_integrators.jl:233-300) with the runge_kutta_4 tableau, on the
configuration, the velocity AND the additional state s of the MechanismState (3 tangential-displacement rows per (contact point,
half-space) pair, the layout of rbd_contact_dynamics):
    stage i   phi_i = dt a_i phid_{i-1},  q_i = global(q0, phi_i),  v_i = v0 + dt a_i vd_{i-1},  s_i = s0 + dt a_i sd_{i-1}
              (wr, sd_i) = contact_dynamics!(q_i, v_i, s_i),  vd_i = dynamics!(q_i, v_i, tau_i, wr),  phid_i = d/dt local(q0, q_i, v_i)
    step      q = global(q0, dt sum_i b_i phid_i),  v = v0 + dt sum_i b_i vd_i,  s = s0 + dt sum_i b_i sd_i
The reset that contact_dynamics! applies to pairs out of contact (mechanism_algorithms.jl:714-716) acts on a view of state.s, which
the integrator overwrites with a copy of the stage value at every stage and with the step result at its end
(set_additional_state!, mechanism_state.jl:440-443; ode_integrators.jl:268, 296): within simulate a reset never survives, so the
oracle's reset output is discarded here.

The per-joint coordinate maps are the oracle's closed forms (oracle/rbd_oracle.hpp, o_global_coordinates / o_local_rate) vectorised
over the batch; q̇ of the joints whose local rate is q̇ comes from the oracle's dynamics (configuration_derivative).  With no
contact pair this integrator equals Oracle.integrate (tests/test_contact_rollout.py pins that).
"""
from __future__ import annotations

import numpy as np

from oracle import Oracle

K_REV, K_PRIS, K_FIXED, K_PLANAR, K_QFLOAT, K_SPQFLOAT, K_QSPH, K_SINCOS = range(8)
NQ = (1, 1, 0, 3, 7, 6, 4, 2)
RK4_A, RK4_B = (0.0, 0.5, 0.5, 1.0), (1.0 / 6, 1.0 / 3, 1.0 / 3, 1.0 / 6)
EPS = 2.220446049250313e-16


def _quat_mul(a, b):
    return np.stack([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
                     a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                     a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1],
                     a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0]])


def _conj(a):
    return np.stack([a[0], -a[1], -a[2], -a[3]])


def _rot(q):
    """[3, 3, B], no normalisation (quaternion_floating.jl:81-83)."""
    w, x, y, z = q[:4]
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _mv(R, v):
    return np.einsum("ijb,jb->ib", R, v)


def _mtv(R, v):
    return np.einsum("jib,jb->ib", R, v)


def _cross(a, b):
    return np.cross(a, b, axis=0)


def _small(th):
    """|remainder(th, 2 pi)| < eps (std::remainder: nearest multiple)."""
    return np.abs(th - 2 * np.pi * np.round(th / (2 * np.pi))) < EPS


def _rotvec_to_quat(r):
    th = np.sqrt((r * r).sum(0))
    zero = th < 1e-300
    ths = np.where(zero, 1.0, th)
    s = np.sin(ths / 2) / ths
    q = np.concatenate([np.cos(ths / 2)[None], s * r])
    q[:, zero] = np.array([1.0, 0, 0, 0])[:, None]
    return q


def _quat_to_rotvec(qin):
    """(rotation vector, angle in [0, pi])."""
    q = np.where(qin[0] < 0, -qin, qin)
    sn = np.sqrt((q[1:] ** 2).sum(0))
    th = 2 * np.arctan2(sn, q[0])
    k = np.where(sn < 1e-300, 0.0, th / np.where(sn < 1e-300, 1.0, sn))
    return k * q[1:], th


def _se3_exp(pr, pt):
    """exp(::Twist), spatialmotion.jl:306-326 -> (relative quaternion, translation)."""
    th = np.sqrt((pr * pr).sum(0))
    dq = _rotvec_to_quat(pr)
    small = _small(th)
    ths = np.where(small, 1.0, th)
    w, v = pr / ths, pt / ths
    t = _cross(w, v)
    t = t - _mv(_rot(dq), t)
    tr = t + w * ((w * v).sum(0) * ths)
    return dq, np.where(small, pt, tr)


def _commutator(x, y):
    return _cross(x[0], y[0]), _cross(x[0], y[1]) + _cross(x[1], y[0])


def _se3_log_rate(dq, p, w, v):
    """log_with_time_derivative, spatialmotion.jl:262-300: rate of the exponential coordinates."""
    psi, th = _quat_to_rotvec(dq)
    small = _small(th)
    ths = np.where(small, 1.0, th)
    th2, h = ths * ths, ths / 2
    sh, ch = np.sin(h), np.cos(h)
    alpha = np.where(small, 1.0, h * ch / sh)
    qq = np.where(small, p, p - _cross(psi, p) * 0.5 + _cross(psi, _cross(psi, p)) * ((1 - alpha) / th2))
    X, V = (psi, qq), (w, v)
    beta = h * h / (sh * sh)
    A = (2 * (1 - alpha) + (alpha - beta) / 2) / th2
    Bc = ((1 - alpha) + (alpha - beta) / 2) / (th2 * th2)
    a1 = _commutator(X, V)
    a2 = _commutator(X, a1)
    a4 = _commutator(X, _commutator(X, a2))
    out = [V[k] + a1[k] * 0.5 + a2[k] * A + a4[k] * Bc for k in range(2)]
    return np.concatenate([np.where(small, V[k], out[k]) for k in range(2)])


def global_coordinates(desc, q0, phi):
    """global_coordinates! of every joint (o_global_coordinates): [nq, B]."""
    q = np.empty_like(q0)
    for i, jt in enumerate(desc.jtype):
        a = q0[desc.qstart[i]:desc.qstart[i] + NQ[jt]]
        f = phi[desc.vstart[i]:]
        o = q[desc.qstart[i]:desc.qstart[i] + NQ[jt]]
        if jt == K_QFLOAT:
            dq, tr = _se3_exp(f[:3], f[3:6])
            o[:4] = _quat_mul(a[:4], dq)
            o[4:7] = a[4:7] + _mv(_rot(a), tr)
        elif jt == K_QSPH:
            o[:] = _quat_mul(a, _rotvec_to_quat(f[:3]))
        elif jt == K_SINCOS:
            s, c = np.sin(f[0]), np.cos(f[0])
            o[0] = a[0] * c + a[1] * s
            o[1] = a[1] * c - a[0] * s
        else:
            o[:] = a + f[:NQ[jt]]
    return q


def local_rate(desc, q0, q, v, qd):
    """d/dt local_coordinates!(q0, q) along v (o_local_rate): [nv, B].  qd = q̇ at (q, v)."""
    out = np.empty_like(v)
    for i, jt in enumerate(desc.jtype):
        qs, vs = desc.qstart[i], desc.vstart[i]
        a, b, w = q0[qs:qs + NQ[jt]], q[qs:qs + NQ[jt]], v[vs:]
        if jt == K_QFLOAT:
            dq = _quat_mul(_conj(a[:4]), b[:4])
            dp = _mtv(_rot(a), b[4:7] - a[4:7])
            out[vs:vs + 6] = _se3_log_rate(dq, dp, w[:3], w[3:6])
        elif jt == K_QSPH:
            phi, th = _quat_to_rotvec(_quat_mul(_conj(a), b))
            om = w[:3]
            r = om + _cross(phi, om) * 0.5
            big = th > EPS
            ths = np.where(big, th, 1.0)
            s, c = np.sin(ths), np.cos(ths)
            k = np.where(big, 1 / (ths * ths) * (1 - (ths * s) / (2 * (1 - np.where(big, c, 0.0)))), 0.0)
            out[vs:vs + 3] = r + _cross(phi, _cross(phi, om)) * k
        elif jt == K_SINCOS:
            out[vs] = w[0]
        elif NQ[jt]:
            out[vs:vs + NQ[jt]] = qd[qs:qs + NQ[jt]]
    return out


def integrate_contact_step(orc: Oracle, q, v, s, contact, tau=None, dt=1e-4, stage_tau=None):
    """One MuntheKaasIntegrator step with contact (see the module docstring); returns (q, v, s).  ``stage_tau(i)`` (optional) gives
    the torques of stage i; else ``tau`` (or None) is held over the step."""
    desc = orc.desc
    q0, v0, s0 = np.array(q, float), np.array(v, float), np.array(s, float)
    phid, vd, sd = [None] * 4, [None] * 4, [None] * 4
    for i in range(4):
        wa = dt * RK4_A[i]
        phi = wa * phid[i - 1] if i else np.zeros_like(v0)
        vs = v0 + wa * vd[i - 1] if i else v0.copy()
        ss = s0 + wa * sd[i - 1] if i else s0.copy()
        qs = global_coordinates(desc, q0, phi)
        wr, sd[i], _ = orc.contact_dynamics(qs, vs, contact, ss)          # the reset does not survive the stage
        t = stage_tau(i) if stage_tau is not None else tau
        vd[i], qd = orc.dynamics(qs, vs, t, wr, want_qd=True)
        phid[i] = local_rate(desc, q0, qs, vs, qd)
    phi = np.zeros_like(v0)
    vn = v0.copy()
    for i in range(4):
        phi += dt * RK4_B[i] * phid[i]
        vn += dt * RK4_B[i] * vd[i]
    sn = s0 + dt * (RK4_B[0] * sd[0] + RK4_B[1] * sd[1] + RK4_B[2] * sd[2] + RK4_B[3] * sd[3])
    return global_coordinates(desc, q0, phi), vn, sn


def integrate_contact(orc: Oracle, q, v, s, contact, tau=None, *, dt=1e-4, nsteps=1, record=None):
    """``nsteps`` steps of integrate_contact_step; ``tau``: None, constant [nv, B], per step [nsteps, nv, B] or per stage
    [nsteps, 4, nv, B] (the blocks of rbd_integrate_schedule).  ``record(step, q, v, s)`` (optional) sees the state before every step
    and after the last.  Returns (q, v, s)."""
    q, v = np.array(q, float), np.array(v, float)
    s = np.zeros((3 * len(contact.body) * len(contact.halfspace), q.shape[1])) if s is None else np.array(s, float)
    tau = None if tau is None else np.asarray(tau, float)
    for n in range(nsteps):
        if record is not None:
            record(n, q, v, s)
        if tau is None or tau.ndim == 2:
            q, v, s = integrate_contact_step(orc, q, v, s, contact, tau, dt)
        elif tau.ndim == 3:
            q, v, s = integrate_contact_step(orc, q, v, s, contact, tau[n], dt)
        else:
            q, v, s = integrate_contact_step(orc, q, v, s, contact, None, dt, stage_tau=lambda i, n=n: tau[n, i])
    if record is not None:
        record(nsteps, q, v, s)
    return q, v, s
