// Reverse mode through the Munthe-Kaas RK4 step (rbd_integrate_vjp, DESIGN 4.13): the per-joint adjoints of the coordinate maps
// of rbd_integrate.cuh and the elementwise part of one backward step.
//
// Per joint the RK4 step is (a = (0, 1/2, 1/2, 1), b = (1/6, 1/3, 1/3, 1/6), φ̇_{-1} = v̇_{-1} = 0)
//   φ_i = dt a_i φ̇_{i-1},  qs_i = G(q0, φ_i),  vs_i = v0 + dt a_i v̇_{i-1},  φ̇_i = L(q0, qs_i, vs_i),  v̇_i = FD(qs_i, vs_i, τ_i)
//   q1 = G(q0, dt Σ b_i φ̇_i),  v1 = v0 + dt Σ b_i v̇_i
// with G / L the global / local coordinate maps of joint_stage.  The backward step runs, from (q̄1, v̄1):
//   finish:  q̄0 = G_q0^T q̄1,  Φ̄ = G_φ^T q̄1,  v̄0 = v̄1
//   i = 3..0:  φ̇̄_i = dt b_i Φ̄ + dt a_{i+1} φ̄_{i+1},  v̇̄_i = dt b_i v̄1 + dt a_{i+1} v̄s_{i+1}
//              L:  q̄0 += L_q0^T φ̇̄_i,  q̄s_i = L_qs^T φ̇̄_i,  v̄s_i = L_vs^T φ̇̄_i
//              FD VJP at (qs_i, vs_i, v̇_i) with ν̄ = v̇̄_i:  q̄s_i += q̄_cfg, v̄s_i += v̄, τ̄_i = μ          (rbd_adjoint.cuh)
//              G:  q̄0 += G_q0^T q̄s_i,  φ̄_i = G_φ^T q̄s_i,  v̄0 += v̄s_i
// Configuration adjoints are carried in configuration coordinates, brought to the minimal-norm form at every step boundary (adj_out).  The VJP's q̄_cfg has no radial part on quaternion / sin-cos
// blocks; that is sound because G maps tangent directions at q0 to tangent directions at qs (|q0 ⊗ exp(φ)| = |q0|) and Φ̄ only
// sees the tangent part of q̄s: the radial parts never reach a tangent component.  At the end q̄0 is mapped to the tangent form
// N(q0)^T q̄0 and from there to the minimal-norm configuration covector (cfg_adjoint).
//
// The Jacobian products of G and L are forward-mode dual numbers (Dual1, one direction per pass) through the SAME templated
// code the forward pass runs, so they are the derivative of the function as implemented, on the branch the forward pass took
// (the thresholds key on ScalarOf<T>, the dual's value type).  Revolute and prismatic joints -- G = q0 + φ, L = vs -- take the
// closed forms of adj_lin instead.
#pragma once
#include "rbd_adjoint.cuh"
#include "rbd_dual.cuh"
#include "rbd_integrate.cuh"

namespace rbd {

template <class F> struct ScalarOf<Dual1<F>> { using type = F; };

template <class F> RBD_HD bool operator<(const Dual1<F>& a, const Dual1<F>& b) { return a.v < b.v; }
template <class F> RBD_HD bool operator>(const Dual1<F>& a, const Dual1<F>& b) { return a.v > b.v; }
template <class F> RBD_HD Dual1<F> sqrt_t(const Dual1<F>& x) {
  const F r = sqrt_t(x.v);
  return {r, r > F(0) ? x.d * F(0.5) / r : F(0)};      // sqrt(0): only the Taylor branches read it, with a zero derivative
}
template <class F> RBD_HD Dual1<F> atan2_t(const Dual1<F>& y, const Dual1<F>& x) {
  return {atan2_t(y.v, x.v), (x.v * y.d - y.v * x.d) / (x.v * x.v + y.v * y.v)};
}
RBD_HD void sincos_t(const Dual1<float>& x, Dual1<float>& s, Dual1<float>& c) {
  float sv, cv;
  sincos_t(x.v, sv, cv);
  s = {sv, cv * x.d};
  c = {cv, -sv * x.d};
}

// G and L of one joint on local arrays (rows of this joint only)
template <class T> RBD_HD void joint_global_arr(int kind, const T* q0, const T* phi, T* qs) {
  switch (kind) {
    case K_REV: case K_PRIS: qs[0] = q0[0] + phi[0]; break;
    case K_SINCOS: sincos_global(q0[0], q0[1], phi[0], qs[0], qs[1]); break;
    case K_PLANAR:
      for (int k = 0; k < 3; ++k) qs[k] = q0[k] + phi[k];
      break;
    case K_SPQFLOAT:
      for (int k = 0; k < 6; ++k) qs[k] = q0[k] + phi[k];
      break;
    case K_QFLOAT: qfloat_global(q0, phi, qs); break;
    case K_QSPH: qsph_global(q0, phi, qs); break;
    default: break;
  }
}
template <class T> RBD_HD void joint_rate_arr(int kind, const T* q0, const T* qs, const T* vs, T* pd) {
  switch (kind) {
    case K_REV: case K_PRIS: case K_SINCOS: pd[0] = vs[0]; break;
    case K_PLANAR: planar_rate(qs[2], vs[0], vs[1], pd[0], pd[1]); pd[2] = vs[2]; break;
    case K_SPQFLOAT: spq_rate(qs, vs, pd); break;
    case K_QFLOAT: qfloat_local_rate(q0, qs, vs, pd); break;
    case K_QSPH: qsph_local_rate(q0, qs, vs, pd); break;
    default: break;
  }
}

// G adjoint: q0b[k] += (G_q0^T qsb)_k;  phib = G_φ^T qsb (skipped when phib is NULL)
template <class T> RBD_HD void g_adjoint(int kind, const T* q0, const T* phi, const T* qsb, T* q0b, T* phib) {
  using D = Dual1<T>;
  const int nq = kind_nq_dev(kind), nv = kind_nv_dev(kind);
  const int ndir = phib ? nq + nv : nq;
  for (int dir = 0; dir < ndir; ++dir) {
    D dq0[7], dphi[6], dqs[7];
    for (int k = 0; k < nq; ++k) dq0[k] = D(q0[k], dir == k ? T(1) : T(0));
    for (int k = 0; k < nv; ++k) dphi[k] = D(phi[k], dir == nq + k ? T(1) : T(0));
    joint_global_arr<D>(kind, dq0, dphi, dqs);
    T s = T(0);
    for (int k = 0; k < nq; ++k) s += qsb[k] * dqs[k].d;
    if (dir < nq) q0b[dir] += s;
    else phib[dir - nq] = s;
  }
}
// L adjoint: q0b += L_q0^T pdb;  qsb = L_qs^T pdb;  vsb = L_vs^T pdb
template <class T> RBD_HD void l_adjoint(int kind, const T* q0, const T* qs, const T* vs, const T* pdb, T* q0b, T* qsb, T* vsb) {
  using D = Dual1<T>;
  const int nq = kind_nq_dev(kind), nv = kind_nv_dev(kind);
  for (int dir = 0; dir < 2 * nq + nv; ++dir) {
    D dq0[7], dqs[7], dvs[6], dpd[6];
    for (int k = 0; k < nq; ++k) {
      dq0[k] = D(q0[k], dir == k ? T(1) : T(0));
      dqs[k] = D(qs[k], dir == nq + k ? T(1) : T(0));
    }
    for (int k = 0; k < nv; ++k) dvs[k] = D(vs[k], dir == 2 * nq + k ? T(1) : T(0));
    joint_rate_arr<D>(kind, dq0, dqs, dvs, dpd);
    T s = T(0);
    for (int k = 0; k < nv; ++k) s += pdb[k] * dpd[k].d;
    if (dir < nq) q0b[dir] += s;
    else if (dir < 2 * nq) qsb[dir - nq] = s;
    else vsb[dir - 2 * nq] = s;
  }
}

// f = N(q)^T g: the tangent covector of a configuration covector g (N: q̇ = N(q) v, qdot_joint)
template <class T> RBD_HD void cfg_to_tan(int kind, const T* q, const T* g, T* f) {
  switch (kind) {
    case K_REV: case K_PRIS: f[0] = g[0]; break;
    case K_SINCOS: f[0] = q[1] * g[0] - q[0] * g[1]; break;
    case K_PLANAR: {
      T s, c;
      sincos_t(q[2], s, c);
      f[0] = c * g[0] + s * g[1];
      f[1] = -s * g[0] + c * g[1];
      f[2] = g[2];
      break;
    }
    case K_QFLOAT: case K_QSPH: {
      const T w = q[0], x = q[1], y = q[2], z = q[3];
      f[0] = T(0.5) * (-x * g[0] + w * g[1] + z * g[2] - y * g[3]);
      f[1] = T(0.5) * (-y * g[0] - z * g[1] + w * g[2] + x * g[3]);
      f[2] = T(0.5) * (-z * g[0] + y * g[1] - x * g[2] + w * g[3]);
      if (kind == K_QFLOAT) {
        T R[9];
        rot_quat(w, x, y, z, R);
        matT_vec(R, g + 4, f + 3);
      }
      break;
    }
    case K_SPQFLOAT: {     // f_k = g . N e_k, the MRP rate columns as spq_rate forms them
      for (int k = 0; k < 6; ++k) {
        const T e[6] = {T(k == 0), T(k == 1), T(k == 2), T(k == 3), T(k == 4), T(k == 5)};
        T pd[6];
        spq_rate(q, e, pd);
        f[k] = g[0] * pd[0] + g[1] * pd[1] + g[2] * pd[2] + g[3] * pd[3] + g[4] * pd[4] + g[5] * pd[5];
      }
      break;
    }
    default: break;
  }
}

// ---- one backward phase of one joint ------------------------------------------------------------------------------------
// Every array is [rows][ld] (one sample per column); a thread owns its joint's rows of each.  One phase = the G adjoint of stage
// g (g = 4: the finishing step) followed by the L adjoint of stage l (l = -1: none) -- the two elementwise halves that meet
// between two forward-dynamics VJPs.
template <class T> struct AdjStepArgs {
  const T* q0;                            // configuration at the start of the step [nq]
  const T* qs[4]; const T* vs[4];         // recomputed stages [nq] / [nv]
  const T* pd[4];                         // φ̇_i [nv]
  const T* qcb; const T* vvb;             // the VJP of stage g: q̄_cfg [nq], v̄ [nv]
  const T* taub;                          // ... and τ̄ [nv], or NULL (no torque gradient wanted)
  T* tau_bar;                             // torque-gradient block of (step, stage g) [nv] (+= τ̄), or NULL
  T* qb; T* vb;                           // (q̄1, v̄1): read by the finish phase; (q̄0, v̄0) + trajectory adjoints written by g = 0
  T* qb0; T* vb0;                         // accumulated (q̄0, v̄0) of the step
  T* qsb; T* vsb;                         // L_qs^T φ̇̄, L_vs^T φ̇̄ of stage l, read by the G phase of the same stage
  T* vdb;                                 // v̇̄_l: ν̄ of the next VJP
  T* phib;                                // Φ̄
  const T* qtb; const T* vtb;             // trajectory adjoints of the step's start state (g = 0), or NULL
  int64_t ld;
  T dt;
  T wa[4];                                // (T)(dt a_i), as the forward stage kernels round it
  T wb[4];                                // (T) b_i
  int g, l;
};

// revolute / prismatic rows (q row = v row): G = q0 + φ, L = vs; one scalar lane, shared by the vectorised kernel
template <class T> struct LinIn { T qb, vb, qcb, vvb, vsb, taub, phib, qtb, vtb, qb0, vb0; };
template <class T> struct LinOut { T qb, vb, qb0, vb0, phib, vdb, vsb, tau; };
template <class T> RBD_HD void adj_lin(const AdjStepArgs<T>& a, const LinIn<T>& x, LinOut<T>& o) {
  T pn = T(0), vn = T(0);
  o.phib = x.phib;
  if (a.g == 4) {
    o.qb0 = x.qb; o.phib = x.qb; o.vb0 = x.vb;
  } else {
    const T qs = x.qcb, vs = x.vsb + x.vvb;
    o.qb0 = x.qb0 + qs; o.vb0 = x.vb0 + vs;
    pn = a.wa[a.g] * qs; vn = a.wa[a.g] * vs;
    o.tau = x.taub;
    if (a.g == 0) { o.qb = o.qb0 + x.qtb; o.vb = o.vb0 + x.vtb; }
  }
  if (a.l >= 0) {
    o.vsb = a.dt * a.wb[a.l] * o.phib + pn;     // L = vs: φ̇̄ passes straight to v̄s
    o.vdb = a.dt * a.wb[a.l] * x.vb + vn;
  }
}

// any joint at sample column b
template <class T> RBD_HD void adj_joint(const BodyDev<T>& bd, const AdjStepArgs<T>& a, int64_t b) {
  const int kind = bd.kind, qr = bd.qrow, vr = bd.vrow, nq = kind_nq_dev(kind), nv = kind_nv_dev(kind);
  if (nv == 0) return;
  auto Q = [&](int k) { return (int64_t)(qr + k) * a.ld + b; };
  auto V = [&](int k) { return (int64_t)(vr + k) * a.ld + b; };
  if (kind == K_REV || kind == K_PRIS) {
    LinIn<T> x;
    LinOut<T> o;
    x.qb = a.qb[Q(0)]; x.vb = a.vb[V(0)]; x.phib = a.phib[V(0)];
    if (a.g < 4) {
      x.qcb = a.qcb[Q(0)]; x.vvb = a.vvb[V(0)]; x.vsb = a.vsb[V(0)]; x.qb0 = a.qb0[Q(0)]; x.vb0 = a.vb0[V(0)];
      x.taub = a.tau_bar ? a.taub[V(0)] : T(0);
      x.qtb = a.qtb ? a.qtb[Q(0)] : T(0); x.vtb = a.vtb ? a.vtb[V(0)] : T(0);
    }
    adj_lin(a, x, o);
    a.qb0[Q(0)] = o.qb0; a.vb0[V(0)] = o.vb0;
    if (a.g == 4) a.phib[V(0)] = o.phib;
    if (a.g < 4 && a.tau_bar) a.tau_bar[V(0)] += o.tau;
    if (a.g == 0) { a.qb[Q(0)] = o.qb; a.vb[V(0)] = o.vb; }
    if (a.l >= 0) { a.vsb[V(0)] = o.vsb; a.vdb[V(0)] = o.vdb; }
    return;
  }
  T q0[7], q0b[7], pn[6], vn[6];
  for (int k = 0; k < nq; ++k) q0[k] = a.q0[Q(k)];
  for (int k = 0; k < nv; ++k) pn[k] = vn[k] = T(0);
  if (a.g == 4) {
    T phi[6], qsb[7], phib[6];
    for (int k = 0; k < nv; ++k) {
      const int64_t e = V(k);
      phi[k] = a.dt * (a.wb[0] * a.pd[0][e] + a.wb[1] * a.pd[1][e] + a.wb[2] * a.pd[2][e] + a.wb[3] * a.pd[3][e]);
      a.vb0[e] = a.vb[e];
    }
    for (int k = 0; k < nq; ++k) { qsb[k] = a.qb[Q(k)]; q0b[k] = T(0); }
    g_adjoint(kind, q0, phi, qsb, q0b, phib);
    for (int k = 0; k < nv; ++k) a.phib[V(k)] = phib[k];
  } else {
    const int g = a.g;
    T phi[6], qsb[7], vsb[6], phib[6];
    for (int k = 0; k < nq; ++k) { qsb[k] = a.qsb[Q(k)] + a.qcb[Q(k)]; q0b[k] = a.qb0[Q(k)]; }
    for (int k = 0; k < nv; ++k) {
      const int64_t e = V(k);
      phi[k] = g ? a.wa[g] * a.pd[g - 1][e] : T(0);
      vsb[k] = a.vsb[e] + a.vvb[e];
      a.vb0[e] += vsb[k];
      if (a.tau_bar) a.tau_bar[e] += a.taub[e];
    }
    g_adjoint(kind, q0, phi, qsb, q0b, g ? phib : (T*)nullptr);
    for (int k = 0; k < nv && g; ++k) { pn[k] = a.wa[g] * phib[k]; vn[k] = a.wa[g] * vsb[k]; }
    if (g == 0) {
      for (int k = 0; k < nq; ++k) a.qb[Q(k)] = q0b[k] + (a.qtb ? a.qtb[Q(k)] : T(0));
      for (int k = 0; k < nv; ++k) a.vb[V(k)] = a.vb0[V(k)] + (a.vtb ? a.vtb[V(k)] : T(0));
    }
  }
  if (a.l >= 0) {
    const int l = a.l;
    T qs[7], vs[6], pdb[6], qsb[7], vsb[6];
    for (int k = 0; k < nq; ++k) qs[k] = a.qs[l][Q(k)];
    for (int k = 0; k < nv; ++k) {
      const int64_t e = V(k);
      vs[k] = a.vs[l][e];
      pdb[k] = a.dt * a.wb[l] * a.phib[e] + pn[k];
      a.vdb[e] = a.dt * a.wb[l] * a.vb[e] + vn[k];
    }
    l_adjoint(kind, q0, qs, vs, pdb, q0b, qsb, vsb);
    for (int k = 0; k < nq; ++k) a.qsb[Q(k)] = qsb[k];
    for (int k = 0; k < nv; ++k) a.vsb[V(k)] = vsb[k];
  }
  for (int k = 0; k < nq; ++k) a.qb0[Q(k)] = q0b[k];
}

// q̄ of one joint at configuration q (configuration coordinates) -> its tangent form qt (may be NULL) and minimal-norm configuration
// form qc (may be NULL, may alias qb).  Also applied to the running q̄ between two steps, so that a rollout split into consecutive
// calls (checkpointing) carries bit for bit what one call carries.
template <class T> RBD_HD void adj_out(const BodyDev<T>& bd, const T* q, const T* qb, T* qt, T* qc, int64_t ld, int64_t b) {
  const int nq = kind_nq_dev(bd.kind), nv = kind_nv_dev(bd.kind);
  if (nv == 0) return;
  T qq[7], g[7], f[6];
  for (int k = 0; k < nq; ++k) { qq[k] = q[(int64_t)(bd.qrow + k) * ld + b]; g[k] = qb[(int64_t)(bd.qrow + k) * ld + b]; }
  cfg_to_tan(bd.kind, qq, g, f);
  if (qt)
    for (int k = 0; k < nv; ++k) qt[(int64_t)(bd.vrow + k) * ld + b] = f[k];
  if (qc) cfg_adjoint(bd, Col<T>{q + b, ld}, f, ColOut<T>{qc + b, ld, true});
}

}  // namespace rbd
