// Forward mode through one Munthe-Kaas RK4 step (rbd_integrate_derivatives, DESIGN 4.25): the Jacobians
//   A = ∂x1/∂x0 (2nv x 2nv),  B = ∂x1/∂τ (2nv x nv),  x = (q, v), configuration rows and columns in the tangent space.
//
// Per sample there are 3nv seed columns j: δq0 = N(q0) e_j (j < nv), δv0 = e_{j-nv} (nv <= j < 2nv), δτ = e_{j-2nv} (2nv <= j),
// with the torque held over the four stages.  With a = (0, 1/2, 1/2, 1), b = (1/6, 1/3, 1/3, 1/6) and G / L the global / local
// coordinate maps of joint_stage, per stage i:
//   δφ_i  = dt a_i δφ̇_{i-1}
//   δqs_i = G_q0 δq0 + G_φ δφ_i                               (configuration coordinates, per joint)
//   δvs_i = δv0 + dt a_i δv̇_{i-1}
//   δφ̇_i  = L_q0 δq0 + L_qs δqs_i + L_vs δvs_i                (per joint)
//   δv̇_i  = Dq_i N⁺(qs_i) δqs_i + Dv_i δvs_i + Dτ_i δτ        (dense; (Dq, Dv, Dτ) = ∂v̇/∂(q, v, τ) at the stage state)
// and at the end  δq1 = G_q0 δq0 + G_φ(q0, Φ) δΦ,  δΦ = dt Σ b_i δφ̇_i,  δv1 = δv0 + dt Σ b_i δv̇_i,  [A | B] = [N⁺(q1) δq1 ; δv1].
// At stage 0 the state is x0 itself and δv̇_0 = [Dq_0 | Dv_0 | Dτ_0] needs no product.  N⁺ is configuration_derivative_to_velocity:
// exact on tangent directions, which G and L produce for unit quaternions / (sin, cos) pairs.
//
// The Jacobian products of G and L are Dual1 passes (one seed column each) through the SAME templated maps the forward pass and
// rbd_integrate_adjoint.cuh's adjoints run; revolute and prismatic joints take the closed forms G = q0 + φ, L = vs.
//
// Every array is [rows x ld] with the sample fastest; the tangent state of a sample is column-major, entry (row r, column j) at row
// r + j nv of a [3 nv^2 x ld] array.  The stage Jacobians [Dq | Dv | Dτ] share that layout (rbd_dynamics_derivatives_ext's
// column-major blocks one after the other), so column j of D is the seed column j of δv̇_0.
#pragma once
#include "rbd_integrate_adjoint.cuh"

namespace rbd {

// q̇ = N(q) v of one joint on local arrays (velocity_to_configuration_derivative!, as qdot_joint)
template <class T> RBD_HD void vel_to_cfg(int kind, const T* q, const T* v, T* qd) {
  switch (kind) {
    case K_REV: case K_PRIS: qd[0] = v[0]; break;
    case K_SINCOS: qd[0] = q[1] * v[0]; qd[1] = -q[0] * v[0]; break;
    case K_PLANAR: planar_rate(q[2], v[0], v[1], qd[0], qd[1]); qd[2] = v[2]; break;
    case K_QFLOAT: case K_QSPH: {
      T o[4];
      quat_Q(q[0], q[1], q[2], q[3], v, o);
      for (int k = 0; k < 4; ++k) qd[k] = T(0.5) * o[k];
      if (kind == K_QFLOAT) {
        T R[9];
        rot_quat(q[0], q[1], q[2], q[3], R);
        mat_vec(R, v + 3, qd + 4);
      }
      break;
    }
    case K_SPQFLOAT: spq_rate(q, v, qd); break;
    default: break;
  }
}

// v = N⁺(q) q̇ of one joint on local arrays (configuration_derivative_to_velocity!); cfg_adjoint applies its transpose
template <class T> RBD_HD void cfg_to_vel(int kind, const T* q, const T* qd, T* v) {
  switch (kind) {
    case K_REV: case K_PRIS: v[0] = qd[0]; break;
    case K_SINCOS: v[0] = (q[1] * qd[0] - q[0] * qd[1]) / (q[0] * q[0] + q[1] * q[1]); break;
    case K_PLANAR: {
      T s, c;
      sincos_t(q[2], s, c);
      v[0] = c * qd[0] + s * qd[1];
      v[1] = -s * qd[0] + c * qd[1];
      v[2] = qd[2];
      break;
    }
    case K_QFLOAT: case K_QSPH: {      // ω = 2 Q(q)^T q̇ / |q|^2;  linear: R^-1 ṗ
      const T w = q[0], x = q[1], y = q[2], z = q[3];
      const T sc = T(2) / (w * w + x * x + y * y + z * z);
      v[0] = sc * (-x * qd[0] + w * qd[1] + z * qd[2] - y * qd[3]);
      v[1] = sc * (-y * qd[0] - z * qd[1] + w * qd[2] + x * qd[3]);
      v[2] = sc * (-z * qd[0] + y * qd[1] - x * qd[2] + w * qd[3]);
      if (kind == K_QFLOAT) {
        T R[9], Rt[9];
        rot_quat(w, x, y, z, R);
        for (int r = 0; r < 3; ++r)
          for (int c = 0; c < 3; ++c) Rt[3 * r + c] = R[3 * c + r];
        inv_t3(Rt, qd + 4, v + 3);      // inv_t3(A, x) = A^-T x
      }
      break;
    }
    case K_SPQFLOAT: {                  // the inverse of spq_rate's blocks, columns formed as spq_rate forms them
      T Nt[9];
      for (int k = 0; k < 3; ++k) {
        const T e[6] = {T(k == 0), T(k == 1), T(k == 2), T(0), T(0), T(0)};
        T pd[6];
        spq_rate(q, e, pd);
        for (int r = 0; r < 3; ++r) Nt[3 * k + r] = pd[r];
      }
      inv_t3(Nt, qd, v);
      T qq[4], R[9], Rt[9];
      mrp_to_quat(q[0], q[1], q[2], qq);
      rot_quat(qq[0], qq[1], qq[2], qq[3], R);
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) Rt[3 * r + c] = R[3 * c + r];
      inv_t3(Rt, qd + 3, v + 3);
      break;
    }
    default: break;
  }
}

// G JVP: qs = G(q0, φ), dqs = G_q0 dq0 + G_φ dphi
template <class T> RBD_HD void g_jvp(int kind, const T* q0, const T* dq0, const T* phi, const T* dphi, T* qs, T* dqs) {
  using D = Dual1<T>;
  const int nq = kind_nq_dev(kind), nv = kind_nv_dev(kind);
  D a[7], p[6], o[7];
  for (int k = 0; k < nq; ++k) a[k] = D(q0[k], dq0[k]);
  for (int k = 0; k < nv; ++k) p[k] = D(phi[k], dphi[k]);
  joint_global_arr<D>(kind, a, p, o);
  for (int k = 0; k < nq; ++k) { qs[k] = o[k].v; dqs[k] = o[k].d; }
}
// L JVP: dpd = L_q0 dq0 + L_qs dqs + L_vs dvs at (q0, qs, vs)
template <class T> RBD_HD void l_jvp(int kind, const T* q0, const T* dq0, const T* qs, const T* dqs, const T* vs, const T* dvs, T* dpd) {
  using D = Dual1<T>;
  const int nq = kind_nq_dev(kind), nv = kind_nv_dev(kind);
  D a[7], s[7], w[6], o[6];
  for (int k = 0; k < nq; ++k) { a[k] = D(q0[k], dq0[k]); s[k] = D(qs[k], dqs[k]); }
  for (int k = 0; k < nv; ++k) w[k] = D(vs[k], dvs[k]);
  joint_rate_arr<D>(kind, a, s, w, o);
  for (int k = 0; k < nv; ++k) dpd[k] = o[k].d;
}

template <class T> struct LinArgs {
  const T* q0;                            // the step's start configuration [nq]
  const T* qs[4]; const T* vs[4];         // the recomputed stages [nq] / [nv]
  const T* pd[4];                         // φ̇_i [nv]
  const T* D;                             // [Dq | Dv | Dτ] of the current stage [3 nv^2]
  const T* vdp;                           // δv̇ of the previous stage [3 nv^2] (stage 1: D of stage 0)
  T* X; T* Y;                             // N⁺(qs_i) δqs_i and δvs_i: the product's right-hand sides [3 nv^2]
  T* P;                                   // δφ̇ of the latest stage [3 nv^2]
  T* SP; T* SV;                           // Σ b_i δφ̇_i, Σ b_i δv̇_i [3 nv^2]
  T* vd;                                  // the product's output δv̇_i [3 nv^2]
  T* A; T* Bt;                            // outputs [nsteps x 4 nv^2 x B] / [nsteps x 2 nv^2 x B], or NULL
  int64_t ld;                             // samples in this chunk
  int64_t n0, B;                          // the chunk's first (step, sample) pair, flattened step-major; samples per step
  int nv;
  T dt;
  T wa[4];                                // (T)(dt a_i), as the forward stage kernels round it
  T wb[4];                                // (T) b_i
  int i;                                  // stage
};

// the seed δq0 of column j on one joint: N(q0) e_{j - vrow} when j is one of its velocity coordinates, else 0
template <class T> RBD_HD void lin_seed(int kind, int vrow, int j, const T* q0, T* dq0) {
  const int nq = kind_nq_dev(kind), nv = kind_nv_dev(kind);
  for (int k = 0; k < nq; ++k) dq0[k] = T(0);
  if (j < vrow || j >= vrow + nv) return;
  T e[6] = {T(0), T(0), T(0), T(0), T(0), T(0)};
  e[j - vrow] = T(1);
  vel_to_cfg(kind, q0, e, dq0);
}

// stage a.i of one joint, seed column j, sample b: δqs, δvs and δφ̇ of the stage, the product's right-hand sides (stages 1..3)
// and the b-weighted sums (δv̇ of the previous stage enters Σ b δv̇ here)
template <class T> RBD_HD void lin_stage_joint(const BodyDev<T>& bd, const LinArgs<T>& a, int64_t b, int j) {
  const int kind = bd.kind, nq = kind_nq_dev(kind), nvj = kind_nv_dev(kind), i = a.i;
  if (nvj == 0) return;
  auto Q = [&](int k) { return (int64_t)(bd.qrow + k) * a.ld + b; };
  auto V = [&](int k) { return (int64_t)(bd.vrow + k) * a.ld + b; };
  auto C = [&](int k) { return ((int64_t)bd.vrow + k + (int64_t)j * a.nv) * a.ld + b; };
  T q0[7], dq0[7], dqs[7], dvs[6], dpd[6], x[6];
  for (int k = 0; k < nq; ++k) q0[k] = a.q0[Q(k)];
  lin_seed(kind, bd.vrow, j, q0, dq0);
  for (int k = 0; k < nvj; ++k) {
    dvs[k] = j == a.nv + bd.vrow + k ? T(1) : T(0);
    if (i) dvs[k] += a.wa[i] * a.vdp[C(k)];
  }
  if (kind == K_REV || kind == K_PRIS) {
    dqs[0] = i ? dq0[0] + a.wa[i] * a.P[C(0)] : dq0[0];
    dpd[0] = dvs[0];
    x[0] = dqs[0];
  } else {
    T phi[6], dphi[6], qv[7], qs[7], vs[6];
    for (int k = 0; k < nvj; ++k) {
      phi[k] = i ? a.wa[i] * a.pd[i - 1][V(k)] : T(0);
      dphi[k] = i ? a.wa[i] * a.P[C(k)] : T(0);
      vs[k] = a.vs[i][V(k)];
    }
    g_jvp(kind, q0, dq0, phi, dphi, qv, dqs);
    for (int k = 0; k < nq; ++k) qs[k] = a.qs[i][Q(k)];
    l_jvp(kind, q0, dq0, qs, dqs, vs, dvs, dpd);
    if (i) cfg_to_vel(kind, qs, dqs, x);
  }
  for (int k = 0; k < nvj; ++k) {
    const int64_t e = C(k);
    if (i) {
      a.X[e] = x[k];
      a.Y[e] = dvs[k];
      a.SV[e] = (i == 1 ? T(0) : a.SV[e]) + a.wb[i - 1] * a.vdp[e];
      a.SP[e] += a.wb[i] * dpd[k];
    } else {
      a.SP[e] = a.wb[0] * dpd[k];
    }
    a.P[e] = dpd[k];
  }
}

// the finishing step of one joint, seed column j, sample b: δq1 (through N⁺(q1)) and δv1 into the rows of A (j < 2nv) or B
template <class T> RBD_HD void lin_finish_joint(const BodyDev<T>& bd, const LinArgs<T>& a, int64_t b, int j) {
  const int kind = bd.kind, nq = kind_nq_dev(kind), nvj = kind_nv_dev(kind), nv = a.nv;
  if (nvj == 0) return;
  auto Q = [&](int k) { return (int64_t)(bd.qrow + k) * a.ld + b; };
  auto V = [&](int k) { return (int64_t)(bd.vrow + k) * a.ld + b; };
  auto C = [&](int k) { return ((int64_t)bd.vrow + k + (int64_t)j * nv) * a.ld + b; };
  T q0[7], dq0[7], oq[6], ov[6];
  for (int k = 0; k < nq; ++k) q0[k] = a.q0[Q(k)];
  lin_seed(kind, bd.vrow, j, q0, dq0);
  for (int k = 0; k < nvj; ++k) {
    const int64_t e = C(k);
    ov[k] = (j == nv + bd.vrow + k ? T(1) : T(0)) + a.dt * (a.SV[e] + a.wb[3] * a.vdp[e]);
  }
  if (kind == K_REV || kind == K_PRIS) {
    oq[0] = dq0[0] + a.dt * a.SP[C(0)];
  } else {
    T phi[6], dphi[6], q1[7], dq1[7];
    for (int k = 0; k < nvj; ++k) {
      const int64_t e = V(k);
      phi[k] = a.dt * (a.wb[0] * a.pd[0][e] + a.wb[1] * a.pd[1][e] + a.wb[2] * a.pd[2][e] + a.wb[3] * a.pd[3][e]);
      dphi[k] = a.dt * a.SP[C(k)];
    }
    g_jvp(kind, q0, dq0, phi, dphi, q1, dq1);
    cfg_to_vel(kind, q1, dq1, oq);
  }
  const int64_t n = a.n0 + b, s = n / a.B, bb = n - s * a.B, nv2 = 2 * (int64_t)nv;
  T* out = j < 2 * nv ? a.A : a.Bt;
  if (!out) return;
  const int64_t col = j < 2 * nv ? j : j - 2 * nv;
  const int64_t base = s * nv2 * (j < 2 * nv ? nv2 : nv) + col * nv2;
  for (int k = 0; k < nvj; ++k) {
    out[(base + bd.vrow + k) * a.B + bb] = oq[k];
    out[(base + nv + bd.vrow + k) * a.B + bb] = ov[k];
  }
}

// δv̇_i = Dq X + Dv Y + Dτ Z (Z = [0 | 0 | I]) for rows r0 .. r0 + R - 1 and seed columns c0 .. c0 + CG - 1 of sample b
template <class T, int R, int CG> RBD_HD void lin_product_tile(const LinArgs<T>& a, int64_t b, int r0, int c0) {
  const int nv = a.nv, nc = 3 * nv;
  const int64_t ld = a.ld, nv2 = (int64_t)nv * nv;
  int rr[R], cc[CG];
#pragma unroll
  for (int r = 0; r < R; ++r) rr[r] = r0 + r < nv ? r0 + r : nv - 1;      // rows / columns past the end repeat the last one, stores
#pragma unroll                                                            // are masked
  for (int c = 0; c < CG; ++c) cc[c] = c0 + c < nc ? c0 + c : nc - 1;
  T acc[R][CG];
#pragma unroll
  for (int c = 0; c < CG; ++c)
#pragma unroll
    for (int r = 0; r < R; ++r)
      acc[r][c] = cc[c] >= 2 * nv ? a.D[(2 * nv2 + rr[r] + (int64_t)(cc[c] - 2 * nv) * nv) * ld + b] : T(0);
  for (int k = 0; k < nv; ++k) {
    T dq[R], dv[R], x[CG], y[CG];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      dq[r] = a.D[(rr[r] + (int64_t)k * nv) * ld + b];
      dv[r] = a.D[(nv2 + rr[r] + (int64_t)k * nv) * ld + b];
    }
#pragma unroll
    for (int c = 0; c < CG; ++c) {
      x[c] = a.X[(k + (int64_t)cc[c] * nv) * ld + b];
      y[c] = a.Y[(k + (int64_t)cc[c] * nv) * ld + b];
    }
#pragma unroll
    for (int c = 0; c < CG; ++c)
#pragma unroll
      for (int r = 0; r < R; ++r) acc[r][c] += dq[r] * x[c] + dv[r] * y[c];
  }
#pragma unroll
  for (int c = 0; c < CG; ++c)
#pragma unroll
    for (int r = 0; r < R; ++r)
      if (r0 + r < nv && c0 + c < nc) a.vd[(r0 + r + (int64_t)(c0 + c) * nv) * ld + b] = acc[r][c];
}

}  // namespace rbd
