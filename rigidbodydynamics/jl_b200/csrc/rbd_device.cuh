// Per-sample rigid-body dynamics in body-local coordinates: the code every GPU thread runs for its sample.
//
// One thread owns one sample (q, v, tau).  All spatial quantities of the three passes live in registers; the
// only per-sample memory is the shared-memory "stash" (one row = one scalar per sample, private to the thread)
// that carries  v_i, (sin, cos)_i  from the outward pass to the inward pass and  U~_i, u~_i  from the inward pass
// to the second outward pass, plus one pending slot per simultaneously-open branch node of the tree.
//
// What is computed, in the reference's terms (citations relative to the reference's src/):
//   joint transforms / twists      joint_types/*.jl (joint_transform, joint_twist), mechanism_state.jl:687-780
//   velocity-product accelerations mechanism_state.jl:814-830 (bias_accelerations_wrt_world), spatialmotion.jl:375-401
//   Newton-Euler wrench            spatial/motion_force_interaction.jl:244-263, spatial/util.jl:110-114
//   RNEA                           mechanism_algorithms.jl:387-459  (spatial_accelerations!, newton_euler!,
//                                  joint_wrenches_and_torques!), :484-498, :542-553
//   CRBA                           mechanism_algorithms.jl:248-272, mechanism_state.jl:852-868
//   forward dynamics               mechanism_algorithms.jl:845-864 -- the reference solves M v̇ = tau - c with CRBA +
//                                  RNEA + Cholesky; here Featherstone's Articulated-Body Algorithm gives the same v̇
//   q̇ = N(q) v                     mechanism_state.jl:905-910 + velocity_to_configuration_derivative! per joint type
//
// The reference keeps every cache in the WORLD frame (mechanism_state.jl:604-682).  This implementation keeps every
// quantity in the BODY frame (re-oriented on the host so 1-DoF joint axes are e_z, see rbd_model.cpp): in fp32 the
// world-frame form loses ~|p|^2 m / I_local (1e3-1e4 for Atlas' wrists) in S^T I^A S by cancellation; the body-frame
// form has no such cancellation, and one-hot motion subspaces make U = I^A S a column read.
//
// The functions are __host__ __device__ so that tests/hostsim can run THE SAME CODE on the CPU against the oracle
// (test infrastructure only; the shipped library has no CPU path).
#pragma once
#include <stdint.h>

#include "rbd_types.h"

#if defined(__CUDACC__)
#define RBD_HD __host__ __device__ __forceinline__
#else
#include <cmath>
#include <cstring>
#define RBD_HD inline
#endif

#include "rbd_sincos.cuh"

namespace rbd {

// Per-thread view of the shared-memory stash: row k of this sample is p[k * STRIDE].
template <class T, int STRIDE> struct Stash {
  T* p;
  RBD_HD T ld(int row) const { return p[row * STRIDE]; }
  RBD_HD void st(int row, T v) const { p[row * STRIDE] = v; }
  RBD_HD void add(int row, T v) const { p[row * STRIDE] += v; }
  template <int N> RBD_HD void ldv(int row, T* out) const {
#pragma unroll
    for (int k = 0; k < N; ++k) out[k] = p[(row + k) * STRIDE];
  }
  RBD_HD void fence_st() const {}                          // stores are visible to later loads of the same thread
  RBD_HD const Stash& slots() const { return *this; }     // pending slots live in the same array
};
// Read-only view of one sample's column in a rows x batch array (element (k, b) at base[k * ld + b]).
template <class T> struct Col {
  const T* p;      // already offset by the sample index
  int64_t ld;
  RBD_HD T operator()(int row) const {
#if defined(__CUDA_ARCH__)
    return __ldg(p + (int64_t)row * ld);
#else
    return p[(int64_t)row * ld];
#endif
  }
  RBD_HD bool valid() const { return p != nullptr; }
};
// Same view with plain (coherent) loads: for rows the SAME kernel has written earlier (ld.global.nc / __ldg must not be used
// on data that is written during the kernel's lifetime).
template <class T> struct ColRW {
  const T* p;
  int64_t ld;
  RBD_HD T operator()(int row) const { return p[(int64_t)row * ld]; }
  RBD_HD bool valid() const { return p != nullptr; }
};
template <class T> struct ColOut {
  T* p;
  int64_t ld;
  bool active;
  RBD_HD void st(int row, T v) const { if (active) p[(int64_t)row * ld] = v; }
  RBD_HD bool valid() const { return p != nullptr; }
};

// Read-write view of one sample's column in a global scratch array (same rows x batch layout).
template <class T> struct Scr {
  T* p;
  int64_t ld;
  RBD_HD T get(int row) const { return p[(int64_t)row * ld]; }
  RBD_HD void st(int row, T v) const { p[(int64_t)row * ld] = v; }
  RBD_HD bool valid() const { return p != nullptr; }
};

// ------------------------------------------------------------------------------------------------------------------
// 3-vector helpers on plain arrays (constant indices only => registers)
// ------------------------------------------------------------------------------------------------------------------
template <class T> RBD_HD void cross3(const T* a, const T* b, T* o) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}
template <class T> RBD_HD void mat_vec(const T* R, const T* v, T* o) {       // o = R v
  o[0] = R[0] * v[0] + R[1] * v[1] + R[2] * v[2];
  o[1] = R[3] * v[0] + R[4] * v[1] + R[5] * v[2];
  o[2] = R[6] * v[0] + R[7] * v[1] + R[8] * v[2];
}
template <class T> RBD_HD void matT_vec(const T* R, const T* v, T* o) {      // o = R^T v
  o[0] = R[0] * v[0] + R[3] * v[1] + R[6] * v[2];
  o[1] = R[1] * v[0] + R[4] * v[1] + R[7] * v[2];
  o[2] = R[2] * v[0] + R[5] * v[1] + R[8] * v[2];
}

// Spatial motion vector in body coordinates: w = angular, l = linear.
template <class T> struct Mot { T w[3]; T l[3]; };
// Articulated-body inertia [[A, B], [B^T, C]] (A, C symmetric: xx xy xz yy yz zz; B row-major, row = angular index)
// together with the articulated bias force (n = moment, f = force).
template <class T> struct Art { T A[6]; T B[9]; T C[6]; T n[3]; T f[3]; };

// index of (i, j) in the packed symmetric storage
RBD_HD constexpr int sidx(int i, int j) {
  // (0,0)=0 (0,1)=1 (0,2)=2 (1,1)=3 (1,2)=4 (2,2)=5 -- no recursion: must fold to a constant after unrolling
  return (i < j ? i : j) == 0 ? (i < j ? j : i) : ((i < j ? i : j) == 1 ? 2 + (i < j ? j : i) : 5);
}

// Motion transform parent -> child.  R: child->parent rotation, r: child origin in parent coordinates.
//   w_c = R^T w_p ;  l_c = R^T (l_p + w_p x r)          (inverse of transform_spatial_motion, spatial/util.jl:104-108)
template <class T> RBD_HD void motion_to_child(const T* R, const T* r, const Mot<T>& p, Mot<T>& c) {
  matT_vec(R, p.w, c.w);
  T t[3];
  cross3(p.w, r, t);
  t[0] += p.l[0]; t[1] += p.l[1]; t[2] += p.l[2];
  matT_vec(R, t, c.l);
}
// Force transform child -> parent:  f_p = R f ;  n_p = R n + r x f_p        (spatialforce.jl:152-158)
template <class T> RBD_HD void force_to_parent(const T* R, const T* r, const T* n, const T* f, T* np, T* fp) {
  mat_vec(R, f, fp);
  mat_vec(R, n, np);
  np[0] += r[1] * fp[2] - r[2] * fp[1];
  np[1] += r[2] * fp[0] - r[0] * fp[2];
  np[2] += r[0] * fp[1] - r[1] * fp[0];
}

// Rigid-body inertia times motion (mul_inertia, spatial/util.jl:110-114): n = J w + h x l ; f = m l - h x w
template <class T> RBD_HD void inertia_mul(const BodyDev<T>& bd, const Mot<T>& v, T* n, T* f) {
  const T* J = bd.J;
  const T* h = bd.h;
  n[0] = J[0] * v.w[0] + J[1] * v.w[1] + J[2] * v.w[2] + (h[1] * v.l[2] - h[2] * v.l[1]);
  n[1] = J[1] * v.w[0] + J[3] * v.w[1] + J[4] * v.w[2] + (h[2] * v.l[0] - h[0] * v.l[2]);
  n[2] = J[2] * v.w[0] + J[4] * v.w[1] + J[5] * v.w[2] + (h[0] * v.l[1] - h[1] * v.l[0]);
  f[0] = bd.m * v.l[0] - (h[1] * v.w[2] - h[2] * v.w[1]);
  f[1] = bd.m * v.l[1] - (h[2] * v.w[0] - h[0] * v.w[2]);
  f[2] = bd.m * v.l[2] - (h[0] * v.w[1] - h[1] * v.w[0]);
}
// Velocity-dependent part of newton_euler (motion_force_interaction.jl:258-260):  p = v x* (I v)
template <class T> RBD_HD void bias_force(const BodyDev<T>& bd, const Mot<T>& v, T* n, T* f) {
  T hn[3], hf[3];
  inertia_mul(bd, v, hn, hf);
  T a[3], b[3];
  cross3(v.w, hn, a);
  cross3(v.l, hf, b);
  n[0] = a[0] + b[0]; n[1] = a[1] + b[1]; n[2] = a[2] + b[2];
  cross3(v.w, hf, f);
}

// ------------------------------------------------------------------------------------------------------------------
// joint kinematics in the canonical frames (joint_transform / joint_twist of joint_types/*.jl)
// ------------------------------------------------------------------------------------------------------------------
// 1-DoF joints: rotation Rz(s, c) and displacement d along e_z after the constant tree transform.
//   R = Rt Rz ;  r = pt + d Rt e_z
template <class T> RBD_HD void frame_1dof(const BodyDev<T>& bd, T s, T c, T d, T* R, T* r) {
  const T* Rt = bd.Rt;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    R[3 * i + 0] = c * Rt[3 * i + 0] + s * Rt[3 * i + 1];
    R[3 * i + 1] = c * Rt[3 * i + 1] - s * Rt[3 * i + 0];
    R[3 * i + 2] = Rt[3 * i + 2];
    r[i] = bd.pt[i] + d * Rt[3 * i + 2];
  }
}
// quaternion [w x y z] -> rotation, not normalised (quaternion_floating.jl:29-32,81-83)
template <class T> RBD_HD void rot_quat(T w, T x, T y, T z, T* R) {
  R[0] = T(1) - T(2) * (y * y + z * z); R[1] = T(2) * (x * y - w * z);        R[2] = T(2) * (x * z + w * y);
  R[3] = T(2) * (x * y + w * z);        R[4] = T(1) - T(2) * (x * x + z * z); R[5] = T(2) * (y * z - w * x);
  R[6] = T(2) * (x * z - w * y);        R[7] = T(2) * (y * z + w * x);        R[8] = T(1) - T(2) * (x * x + y * y);
}
template <class T> RBD_HD void mrp_to_quat(T x, T y, T z, T* q) {              // spquat_floating.jl:30-32
  T n2 = x * x + y * y + z * z;
  T inv = T(1) / (T(1) + n2);
  q[0] = (T(1) - n2) * inv; q[1] = T(2) * x * inv; q[2] = T(2) * y * inv; q[3] = T(2) * z * inv;
}
template <class T> RBD_HD void mat_mul3(const T* a, const T* b, T* o) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) o[3 * i + j] = a[3 * i] * b[j] + a[3 * i + 1] * b[3 + j] + a[3 * i + 2] * b[6 + j];
}
// Multi-DoF joints: R = Rt R_J(q), r = pt + Rt p_J(q), from the q column (re-read from global memory each pass).
template <class T> RBD_HD void frame_multi(const BodyDev<T>& bd, const Col<T>& q, T* R, T* r) {
  T RJ[9], pJ[3] = {T(0), T(0), T(0)};
  const int q0 = bd.qrow;
  switch (bd.kind) {
    case K_PLANAR: {                                                            // planar.jl:65-70 in canonical axes
      T s, c;
      sincos_t(q(q0 + 2), s, c);
      RJ[0] = c; RJ[1] = -s; RJ[2] = T(0); RJ[3] = s; RJ[4] = c; RJ[5] = T(0); RJ[6] = T(0); RJ[7] = T(0); RJ[8] = T(1);
      pJ[0] = q(q0); pJ[1] = q(q0 + 1);
      break;
    }
    case K_QFLOAT:
      rot_quat(q(q0), q(q0 + 1), q(q0 + 2), q(q0 + 3), RJ);
      pJ[0] = q(q0 + 4); pJ[1] = q(q0 + 5); pJ[2] = q(q0 + 6);
      break;
    case K_SPQFLOAT: {
      T qq[4];
      mrp_to_quat(q(q0), q(q0 + 1), q(q0 + 2), qq);
      rot_quat(qq[0], qq[1], qq[2], qq[3], RJ);
      pJ[0] = q(q0 + 3); pJ[1] = q(q0 + 4); pJ[2] = q(q0 + 5);
      break;
    }
    default:  // K_QSPH
      rot_quat(q(q0), q(q0 + 1), q(q0 + 2), q(q0 + 3), RJ);
      break;
  }
  mat_mul3(bd.Rt, RJ, R);
  T t[3];
  mat_vec(bd.Rt, pJ, t);
  r[0] = bd.pt[0] + t[0]; r[1] = bd.pt[1] + t[1]; r[2] = bd.pt[2] + t[2];
}

// One-hot motion subspace of the multi-DoF kinds: velocity coordinate k drives component sub_index(kind, k) of
// [w; l] (planar.jl:87-93 in canonical axes; quaternion_floating.jl:85-91; quaternion_spherical.jl:52-58).
RBD_HD constexpr int sub_index(int kind, int k) { return kind == K_PLANAR ? (k == 0 ? 3 : (k == 1 ? 4 : 2)) : k; }

// Joint velocity S x in body coordinates for a multi-DoF joint (x = v or v̇ rows starting at `row`).
template <class T, int K> RBD_HD void joint_motion_multi(int kind, const T* x, Mot<T>& m) {
  T e[6] = {T(0), T(0), T(0), T(0), T(0), T(0)};
#pragma unroll
  for (int k = 0; k < K; ++k) {
#pragma unroll
    for (int c = 0; c < 6; ++c) if (sub_index(kind, k) == c) e[c] = x[k];
  }
  m.w[0] = e[0]; m.w[1] = e[1]; m.w[2] = e[2]; m.l[0] = e[3]; m.l[1] = e[4]; m.l[2] = e[5];
}

// q̇ = N(q) v per joint type (velocity_to_configuration_derivative!)
template <class T, bool ONLY1 = false>
RBD_HD void qdot_joint(const BodyDev<T>& bd, const Col<T>& q, const Col<T>& v, const ColOut<T>& qd) {
  const int q0 = bd.qrow, v0 = bd.vrow;
  if (ONLY1) {                                    // caller guarantees a 1-DoF / fixed joint: keep the multi-DoF code out of its loop
    if (bd.kind == K_REV || bd.kind == K_PRIS) qd.st(q0, v(v0));
    else if (bd.kind == K_SINCOS) {
      T w = v(v0);
      qd.st(q0, q(q0 + 1) * w);
      qd.st(q0 + 1, -q(q0) * w);
    }
    return;
  }
  switch (bd.kind) {
    case K_REV: case K_PRIS: qd.st(q0, v(v0)); break;                           // joint_types.jl:29-32
    case K_FIXED: break;
    case K_SINCOS: {                                                            // sin_cos_revolute.jl:160-165
      T w = v(v0);
      qd.st(q0, q(q0 + 1) * w);
      qd.st(q0 + 1, -q(q0) * w);
      break;
    }
    case K_PLANAR: {                                                            // planar.jl:123-129
      T s, c;
      sincos_t(q(q0 + 2), s, c);
      T a = v(v0), b = v(v0 + 1);
      qd.st(q0, c * a - s * b);
      qd.st(q0 + 1, s * a + c * b);
      qd.st(q0 + 2, v(v0 + 2));
      break;
    }
    case K_QFLOAT: case K_QSPH: {                                               // quaternion_floating.jl:126-136, util.jl:127-134
      T w = q(q0), x = q(q0 + 1), y = q(q0 + 2), z = q(q0 + 3);
      T a = v(v0), b = v(v0 + 1), c = v(v0 + 2);
      qd.st(q0, T(0.5) * (-x * a - y * b - z * c));
      qd.st(q0 + 1, T(0.5) * (w * a - z * b + y * c));
      qd.st(q0 + 2, T(0.5) * (z * a + w * b - x * c));
      qd.st(q0 + 3, T(0.5) * (-y * a + x * b + w * c));
      if (bd.kind == K_QFLOAT) {
        T R[9], l[3] = {v(v0 + 3), v(v0 + 4), v(v0 + 5)}, t[3];
        rot_quat(w, x, y, z, R);
        mat_vec(R, l, t);
        qd.st(q0 + 4, t[0]); qd.st(q0 + 5, t[1]); qd.st(q0 + 6, t[2]);
      }
      break;
    }
    case K_SPQFLOAT: {                                                          // spquat_floating.jl:128-138, util.jl:136-141
      T qq[4];
      mrp_to_quat(q(q0), q(q0 + 1), q(q0 + 2), qq);
      T w = qq[0], x = qq[1], y = qq[2], z = qq[3];
      T a = v(v0), b = v(v0 + 1), c = v(v0 + 2);
      T dw = T(0.5) * (-x * a - y * b - z * c);
      T dx = T(0.5) * (w * a - z * b + y * c);
      T dy = T(0.5) * (z * a + w * b - x * c);
      T dz = T(0.5) * (-y * a + x * b + w * c);
      T inv = T(1) / (T(1) + w);
      qd.st(q0, (dx - x * dw * inv) * inv);
      qd.st(q0 + 1, (dy - y * dw * inv) * inv);
      qd.st(q0 + 2, (dz - z * dw * inv) * inv);
      T R[9], l[3] = {v(v0 + 3), v(v0 + 4), v(v0 + 5)}, t[3];
      rot_quat(w, x, y, z, R);
      mat_vec(R, l, t);
      qd.st(q0 + 3, t[0]); qd.st(q0 + 4, t[1]); qd.st(q0 + 5, t[2]);
      break;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// articulated inertia: own inertia, child -> parent transform
// ------------------------------------------------------------------------------------------------------------------
template <class T> RBD_HD void art_set_body(const BodyDev<T>& bd, Art<T>& a) {     // 6x6 [J h^; h^T m1], :102-107
  a.A[0] = bd.J[0]; a.A[1] = bd.J[1]; a.A[2] = bd.J[2]; a.A[3] = bd.J[3]; a.A[4] = bd.J[4]; a.A[5] = bd.J[5];
  a.B[0] = T(0);     a.B[1] = -bd.h[2]; a.B[2] = bd.h[1];
  a.B[3] = bd.h[2];  a.B[4] = T(0);     a.B[5] = -bd.h[0];
  a.B[6] = -bd.h[1]; a.B[7] = bd.h[0];  a.B[8] = T(0);
  a.C[0] = bd.m; a.C[1] = T(0); a.C[2] = T(0); a.C[3] = bd.m; a.C[4] = T(0); a.C[5] = bd.m;
}
template <class T> RBD_HD void art_add(Art<T>& a, const Art<T>& b) {
#pragma unroll
  for (int k = 0; k < 6; ++k) { a.A[k] += b.A[k]; a.C[k] += b.C[k]; }
#pragma unroll
  for (int k = 0; k < 9; ++k) a.B[k] += b.B[k];
#pragma unroll
  for (int k = 0; k < 3; ++k) { a.n[k] += b.n[k]; a.f[k] += b.f[k]; }
}
template <class T, class S> RBD_HD void art_store(const S& st, int row, const Art<T>& a) {
#pragma unroll
  for (int k = 0; k < 6; ++k) { st.st(row + k, a.A[k]); st.st(row + 15 + k, a.C[k]); }
#pragma unroll
  for (int k = 0; k < 9; ++k) st.st(row + 6 + k, a.B[k]);
#pragma unroll
  for (int k = 0; k < 3; ++k) { st.st(row + 21 + k, a.n[k]); st.st(row + 24 + k, a.f[k]); }
}
template <class T, class S> RBD_HD void art_accum(const S& st, int row, const Art<T>& a) {
  // all loads first, then all stores: a store to the stash may alias a later load as far as the compiler can tell, and
  // interleaving them would serialise 27 memory round trips
  T t[27];
  st.fence_st();
  st.template ldv<27>(row, t);
#pragma unroll
  for (int k = 0; k < 6; ++k) { t[k] += a.A[k]; t[15 + k] += a.C[k]; }
#pragma unroll
  for (int k = 0; k < 9; ++k) t[6 + k] += a.B[k];
#pragma unroll
  for (int k = 0; k < 3; ++k) { t[21 + k] += a.n[k]; t[24 + k] += a.f[k]; }
#pragma unroll
  for (int k = 0; k < 27; ++k) st.st(row + k, t[k]);
}
template <class T, class S> RBD_HD void art_add_from(const S& st, int row, Art<T>& a) {
  T t[27];
  st.fence_st();
  st.template ldv<27>(row, t);
#pragma unroll
  for (int k = 0; k < 6; ++k) { a.A[k] += t[k]; a.C[k] += t[15 + k]; }
#pragma unroll
  for (int k = 0; k < 9; ++k) a.B[k] += t[6 + k];
#pragma unroll
  for (int k = 0; k < 3; ++k) { a.n[k] += t[21 + k]; a.f[k] += t[24 + k]; }
}

// X^T I X and X^T p for the child -> parent hand-over: rotate the 3x3 blocks by R, then shift the origin by r.
//   C' = Cr ;  B' = Br + r^ Cr ;  A' = Ar + P + P^T + W  with  P = r^ Br^T,  W = r^ (r^ Cr)^T
// ZAZ: the angular-z row/column of the child's inertia is structurally zero (after eliminating a revolute-z DoF).
template <class T, bool ZAZ> RBD_HD void art_to_parent(const T* R, const T* r, const Art<T>& c, Art<T>& o) {
  constexpr int LA = ZAZ ? 2 : 3;   // live angular rows
  T Ar[6], Br[9], Cr[6];
  {  // Ar = R A R^T
    T t[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int k = 0; k < LA; ++k) {
        T s = R[3 * i] * c.A[sidx(0, k)];
#pragma unroll
        for (int l = 1; l < LA; ++l) s += R[3 * i + l] * c.A[sidx(l, k)];
        t[3 * i + k] = s;
      }
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = i; j < 3; ++j) {
        T s = t[3 * i] * R[3 * j];
#pragma unroll
        for (int k = 1; k < LA; ++k) s += t[3 * i + k] * R[3 * j + k];
        Ar[sidx(i, j)] = s;
      }
  }
  {  // Br = R B R^T
    T t[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        T s = R[3 * i] * c.B[k];
#pragma unroll
        for (int l = 1; l < LA; ++l) s += R[3 * i + l] * c.B[3 * l + k];
        t[3 * i + k] = s;
      }
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) Br[3 * i + j] = t[3 * i] * R[3 * j] + t[3 * i + 1] * R[3 * j + 1] + t[3 * i + 2] * R[3 * j + 2];
  }
  {  // Cr = R C R^T
    T t[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int k = 0; k < 3; ++k)
        t[3 * i + k] = R[3 * i] * c.C[sidx(0, k)] + R[3 * i + 1] * c.C[sidx(1, k)] + R[3 * i + 2] * c.C[sidx(2, k)];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = i; j < 3; ++j) Cr[sidx(i, j)] = t[3 * i] * R[3 * j] + t[3 * i + 1] * R[3 * j + 1] + t[3 * i + 2] * R[3 * j + 2];
  }
  // Q = r^ Cr (column-wise cross), B' = Br + Q
  T Q[9];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const T m0 = Cr[sidx(0, j)], m1 = Cr[sidx(1, j)], m2 = Cr[sidx(2, j)];
    Q[0 + j] = r[1] * m2 - r[2] * m1;
    Q[3 + j] = r[2] * m0 - r[0] * m2;
    Q[6 + j] = r[0] * m1 - r[1] * m0;
  }
#pragma unroll
  for (int k = 0; k < 9; ++k) o.B[k] = Br[k] + Q[k];
#pragma unroll
  for (int k = 0; k < 6; ++k) o.C[k] = Cr[k];
  // P[:, j] = r x row_j(Br) ;  W[:, j] = r x row_j(Q)
  T P[9], W[9];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    P[0 + j] = r[1] * Br[3 * j + 2] - r[2] * Br[3 * j + 1];
    P[3 + j] = r[2] * Br[3 * j + 0] - r[0] * Br[3 * j + 2];
    P[6 + j] = r[0] * Br[3 * j + 1] - r[1] * Br[3 * j + 0];
    W[0 + j] = r[1] * Q[3 * j + 2] - r[2] * Q[3 * j + 1];
    W[3 + j] = r[2] * Q[3 * j + 0] - r[0] * Q[3 * j + 2];
    W[6 + j] = r[0] * Q[3 * j + 1] - r[1] * Q[3 * j + 0];
  }
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = i; j < 3; ++j) o.A[sidx(i, j)] = Ar[sidx(i, j)] + P[3 * i + j] + P[3 * j + i] + W[3 * i + j];
  force_to_parent(R, r, c.n, c.f, o.n, o.f);
}

// ------------------------------------------------------------------------------------------------------------------
// Fast classes (F_ZPAR / F_ZPERP): joint transform E = [P] Rz(s, c), origin r = pt.  PERM = 1 applies the cyclic
// permutation P after the z-rotation (P v = (v_z, v_x, v_y)); PERM = 0 is a plain z-rotation.
// ------------------------------------------------------------------------------------------------------------------
template <class T, int PERM> RBD_HD void zrot_fwd(T s, T c, const T* v, T* o) {          // o = E v
  const T t0 = c * v[0] - s * v[1], t1 = s * v[0] + c * v[1];
  if (PERM) { o[0] = v[2]; o[1] = t0; o[2] = t1; } else { o[0] = t0; o[1] = t1; o[2] = v[2]; }
}
template <class T, int PERM> RBD_HD void zrot_inv(T s, T c, const T* w, T* o) {          // o = E^T w
  const T u0 = PERM ? w[1] : w[0], u1 = PERM ? w[2] : w[1], u2 = PERM ? w[0] : w[2];
  o[0] = c * u0 + s * u1; o[1] = c * u1 - s * u0; o[2] = u2;
}
template <class T, int PERM> RBD_HD void motion_to_child_z(T s, T c, const T* r, const Mot<T>& p, Mot<T>& ch) {
  zrot_inv<T, PERM>(s, c, p.w, ch.w);
  T t[3];
  cross3(p.w, r, t);
  t[0] += p.l[0]; t[1] += p.l[1]; t[2] += p.l[2];
  zrot_inv<T, PERM>(s, c, t, ch.l);
}
template <class T, int PERM> RBD_HD void force_to_parent_z(T s, T c, const T* r, const T* n, const T* f, T* np, T* fp) {
  zrot_fwd<T, PERM>(s, c, f, fp);
  zrot_fwd<T, PERM>(s, c, n, np);
  np[0] += r[1] * fp[2] - r[2] * fp[1];
  np[1] += r[2] * fp[0] - r[0] * fp[2];
  np[2] += r[0] * fp[1] - r[1] * fp[0];
}
// Shared tail of the child -> parent hand-over: blocks already rotated into the parent's axes, now shift the origin by r.
//   C' = Cr ;  B' = Br + r^ Cr ;  A' = Ar + P + P^T + W  with  P = r^ Br^T,  W = r^ (r^ Cr)^T ;  f' = fr ;  n' = nr + r x fr
template <class T>
RBD_HD void art_shift(const T* r, const T* Ar, const T* Br, const T* Cr, const T* nr, const T* fr, Art<T>& o) {
  T Q[9];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const T m0 = Cr[sidx(0, j)], m1 = Cr[sidx(1, j)], m2 = Cr[sidx(2, j)];
    Q[0 + j] = r[1] * m2 - r[2] * m1;
    Q[3 + j] = r[2] * m0 - r[0] * m2;
    Q[6 + j] = r[0] * m1 - r[1] * m0;
  }
#pragma unroll
  for (int k = 0; k < 9; ++k) o.B[k] = Br[k] + Q[k];
#pragma unroll
  for (int k = 0; k < 6; ++k) o.C[k] = Cr[k];
  T P[9], W[9];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    P[0 + j] = r[1] * Br[3 * j + 2] - r[2] * Br[3 * j + 1];
    P[3 + j] = r[2] * Br[3 * j + 0] - r[0] * Br[3 * j + 2];
    P[6 + j] = r[0] * Br[3 * j + 1] - r[1] * Br[3 * j + 0];
    W[0 + j] = r[1] * Q[3 * j + 2] - r[2] * Q[3 * j + 1];
    W[3 + j] = r[2] * Q[3 * j + 0] - r[0] * Q[3 * j + 2];
    W[6 + j] = r[0] * Q[3 * j + 1] - r[1] * Q[3 * j + 0];
  }
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = i; j < 3; ++j) o.A[sidx(i, j)] = Ar[sidx(i, j)] + P[3 * i + j] + P[3 * j + i] + W[3 * i + j];
#pragma unroll
  for (int k = 0; k < 3; ++k) o.f[k] = fr[k];
  o.n[0] = nr[0] + r[1] * fr[2] - r[2] * fr[1];
  o.n[1] = nr[1] + r[2] * fr[0] - r[0] * fr[2];
  o.n[2] = nr[2] + r[0] * fr[1] - r[1] * fr[0];
}
// Child -> parent hand-over for the fast classes.  The child's inertia `b` has a vanishing angular-z row / column (a
// revolute-z DoF was just eliminated).  Congruence by Rz acts on the xy-plane only: a symmetric 2x2 block turns by the
// double angle ( (xx-yy)/2, xy ), the (xz, yz) pairs turn by the single angle, zz stays; P is an index relabelling.
// Origin shift with r = 0: the rotated blocks are the result.
template <class T>
RBD_HD void art_noshift(const T* Ar, const T* Br, const T* Cr, const T* nr, const T* fr, Art<T>& o) {
#pragma unroll
  for (int k = 0; k < 6; ++k) { o.A[k] = Ar[k]; o.C[k] = Cr[k]; }
#pragma unroll
  for (int k = 0; k < 9; ++k) o.B[k] = Br[k];
#pragma unroll
  for (int k = 0; k < 3; ++k) { o.n[k] = nr[k]; o.f[k] = fr[k]; }
}
template <class T, int PERM, bool ZERO_R = false>
RBD_HD void art_to_parent_z(T s, T c, const T* r, const Art<T>& b, Art<T>& o) {
  const T c2 = c * c - s * s, s2 = (s + s) * c;
  T Ya[6], Yb[9], Yc[6], yn[3], yf[3];
  {  // A: only xx, xy, yy are non-zero
    const T m = T(0.5) * (b.A[0] + b.A[3]), d = T(0.5) * (b.A[0] - b.A[3]);
    const T dn = c2 * d - s2 * b.A[1];
    Ya[0] = m + dn; Ya[1] = s2 * d + c2 * b.A[1]; Ya[3] = m - dn;
    Ya[2] = T(0); Ya[4] = T(0); Ya[5] = T(0);
  }
  {  // C: full symmetric
    const T m = T(0.5) * (b.C[0] + b.C[3]), d = T(0.5) * (b.C[0] - b.C[3]);
    const T dn = c2 * d - s2 * b.C[1];
    Yc[0] = m + dn; Yc[1] = s2 * d + c2 * b.C[1]; Yc[3] = m - dn;
    Yc[2] = c * b.C[2] - s * b.C[4]; Yc[4] = s * b.C[2] + c * b.C[4]; Yc[5] = b.C[5];
  }
  {  // B: rows x, y (row z vanishes):  Rz2 B Rz3^T
    T t[6];
#pragma unroll
    for (int i = 0; i < 2; ++i) {        // columns
      t[3 * i + 0] = c * b.B[3 * i + 0] - s * b.B[3 * i + 1];
      t[3 * i + 1] = s * b.B[3 * i + 0] + c * b.B[3 * i + 1];
      t[3 * i + 2] = b.B[3 * i + 2];
    }
#pragma unroll
    for (int j = 0; j < 3; ++j) {        // rows
      Yb[0 + j] = c * t[0 + j] - s * t[3 + j];
      Yb[3 + j] = s * t[0 + j] + c * t[3 + j];
      Yb[6 + j] = T(0);
    }
  }
  yn[0] = c * b.n[0] - s * b.n[1]; yn[1] = s * b.n[0] + c * b.n[1]; yn[2] = b.n[2];
  yf[0] = c * b.f[0] - s * b.f[1]; yf[1] = s * b.f[0] + c * b.f[1]; yf[2] = b.f[2];
  if (PERM) {
    // X'[i][j] = Y[sg(i)][sg(j)], sg = (2, 0, 1)
    constexpr int sg[3] = {2, 0, 1};
    T Ar[6], Br[9], Cr[6], nr[3], fr[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
      for (int j = i; j < 3; ++j) { Ar[sidx(i, j)] = Ya[sidx(sg[i], sg[j])]; Cr[sidx(i, j)] = Yc[sidx(sg[i], sg[j])]; }
#pragma unroll
      for (int j = 0; j < 3; ++j) Br[3 * i + j] = Yb[3 * sg[i] + sg[j]];
      nr[i] = yn[sg[i]]; fr[i] = yf[sg[i]];
    }
    if (ZERO_R) art_noshift(Ar, Br, Cr, nr, fr, o);
    else art_shift(r, Ar, Br, Cr, nr, fr, o);
  } else {
    if (ZERO_R) art_noshift(Ya, Yb, Yc, yn, yf, o);
    else art_shift(r, Ya, Yb, Yc, yn, yf, o);
  }
}

// Hooks for the expression tracer (rbd_sym.h specialises them for its scalar type; for float / double they compile to nothing):
// trace_step marks where the step of body `i` in ABA pass `pass` begins (i = -1: the pass is over), trace_conn brackets the
// nodes that connect a body to its parent through the stash (the parent's v / (v, a), or the pending slot the articulated
// inertia is handed over in) -- the code generator shares one program image between mirror-image limbs and keeps those
// connections per instance.
template <class T> RBD_HD void trace_step(int pass, int i) { (void)pass; (void)i; }
template <class T> RBD_HD void trace_conn(bool begin) { (void)begin; }

// Hand a finished child contribution (already in `carry`, written there by art_to_parent) to its parent: a first child's
// stays in registers; any other child's goes to the parent's pending slot.  Writing every contribution into `carry` is safe
// because a non-first child is followed (in reverse preorder) by the last body of a sibling subtree, a leaf, which does not
// read `carry` -- and it saves a 27-register copy per body.
template <class T, class ST>
RBD_HD void hand_over(const ModelDev<T>& M, const BodyDev<T>& bd, const ST& st, const Art<T>& carry) {
  trace_conn<T>(true);
  if (!(bd.flags & F_FIRST_CHILD)) {
    const int row = M.slot_base + bd.pslot * kSlotRowsAba;
    if (bd.flags & F_SLOT_INIT) art_store(st.slots(), row, carry);
    else art_accum(st.slots(), row, carry);
  }
  trace_conn<T>(false);
}

// ------------------------------------------------------------------------------------------------------------------
// small dense SPD solves (joint-space blocks of multi-DoF joints, 6x6 floating base)
// ------------------------------------------------------------------------------------------------------------------
// LDL^T of a small SPD matrix: L (unit lower) overwrites D below the diagonal, dinv[] = 1/d.
template <class T, int K> RBD_HD void ldlt(T (&D)[K][K], T (&dinv)[K]) {
  T dd[K];
#pragma unroll
  for (int j = 0; j < K; ++j) {
    T d = D[j][j];
#pragma unroll
    for (int k = 0; k < j; ++k) d -= D[j][k] * D[j][k] * dd[k];
    dd[j] = d;
    dinv[j] = T(1) / d;
#pragma unroll
    for (int i = j + 1; i < K; ++i) {
      T s = D[i][j];
#pragma unroll
      for (int k = 0; k < j; ++k) s -= D[i][k] * D[j][k] * dd[k];
      D[i][j] = s * dinv[j];
    }
  }
}
template <class T, int K> RBD_HD void ldlt_solve(const T (&D)[K][K], const T (&dinv)[K], T (&x)[K]) {
#pragma unroll
  for (int i = 0; i < K; ++i) {
#pragma unroll
    for (int k = 0; k < i; ++k) x[i] -= D[i][k] * x[k];
  }
#pragma unroll
  for (int i = 0; i < K; ++i) x[i] *= dinv[i];
#pragma unroll
  for (int i = K - 1; i >= 0; --i) {
#pragma unroll
    for (int k = i + 1; k < K; ++k) x[i] -= D[k][i] * x[k];
  }
}

template <class T> RBD_HD void art_to_full(const Art<T>& a, T (&I)[6][6], T (&p)[6]) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      I[i][j] = a.A[sidx(i, j)];
      I[i][3 + j] = a.B[3 * i + j];
      I[3 + j][i] = a.B[3 * i + j];
      I[3 + i][3 + j] = a.C[sidx(i, j)];
    }
#pragma unroll
  for (int k = 0; k < 3; ++k) { p[k] = a.n[k]; p[3 + k] = a.f[k]; }
}
template <class T> RBD_HD void full_to_art(const T (&I)[6][6], const T (&p)[6], Art<T>& a) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      if (i <= j) { a.A[sidx(i, j)] = I[i][j]; a.C[sidx(i, j)] = I[3 + i][3 + j]; }
      a.B[3 * i + j] = I[i][3 + j];
    }
#pragma unroll
  for (int k = 0; k < 3; ++k) { a.n[k] = p[k]; a.f[k] = p[3 + k]; }
}

// spatial motion cross product  c = v x (S qd)   (se3_commutator, spatial/util.jl:117-121)
template <class T> RBD_HD void motion_cross(const Mot<T>& v, const Mot<T>& j, Mot<T>& c) {
  cross3(v.w, j.w, c.w);
  T a[3], b[3];
  cross3(v.w, j.l, a);
  cross3(v.l, j.w, b);
  c.l[0] = a[0] + b[0]; c.l[1] = a[1] + b[1]; c.l[2] = a[2] + b[2];
}

// ==================================================================================================================
// Articulated-Body Algorithm
// ==================================================================================================================
// Compile-time promise about the 1-DoF kinds a model contains, so kernels for all-revolute robots (the common case) carry
// no prismatic / fixed code in their hot loops (smaller instruction footprint).
constexpr int kHasPris = 1, kHasFixed = 2, kAllKinds = 3;

template <class T, bool EXT = false, int KINDS = kAllKinds> struct AbaIO {
  static constexpr bool kExt = EXT;   // external wrenches present (compile-time so the common path carries no extra state)
  static constexpr int kKinds = KINDS;
  Col<T> q, v, tau, wext;   // tau may be invalid (NULL): zero torques
  ColOut<T> vd, qd;         // qd may be invalid
  Scr<T> ext;               // [6 * nb] body-frame external wrenches, written by ext_wrench_pass (EXT only)
};

// Scalars of one 1-DoF body that come from global memory.  They are requested one body AHEAD of their use (software
// pipelining in aba_sample) so the load latency overlaps the previous body's arithmetic instead of stalling the warp.
template <class T> struct Pre { T q0, q1, qd, tau; T w[6]; T qoff; int32_t zflags; };

template <class T, int PASS, class IO>
RBD_HD void prefetch_body(const ModelDev<T>& M, int i, const IO& io, Pre<T>& p) {
  p.q0 = T(0); p.q1 = T(0); p.qd = T(0); p.tau = T(0);
#pragma unroll
  for (int k = 0; k < 6; ++k) p.w[k] = T(0);
  p.zflags = 0; p.qoff = T(0);
  if (i < 0 || i >= M.nb) return;
  const BodyDev<T>& bd = M.body[i];
  const int kind = bd.kind;
  p.zflags = bd.flags & (F_ZPAR | F_ZPERP | F_ZERO_R);      // fast-class bits and angle offset, fetched a body ahead like the joint scalars
  p.qoff = bd.qoff;
  if (PASS == 2 && IO::kExt) {
#pragma unroll
    for (int k = 0; k < 6; ++k) p.w[k] = io.ext.get(6 * i + k);
  }
  if (kind == K_REV || kind == K_PRIS || kind == K_SINCOS) {     // multi-DoF bodies read their rows directly
    p.q0 = io.q(bd.qrow);                 // the joint angle is re-read (and sin/cos recomputed) in every pass:
    if (kind == K_SINCOS) p.q1 = io.q(bd.qrow + 1);   // two stash rows per body buy ~40 % more resident warps
    p.qd = io.v(bd.vrow);
    if (PASS == 2 && io.tau.valid()) p.tau = io.tau(bd.vrow);
  }
}

// sin / cos / displacement of a 1-DoF joint from its prefetched configuration scalars
// (`qoff`: the constant z-rotation of the fast classes, added HERE and not where q is loaded, so that the load issued one body
//  ahead is not consumed before it has arrived)
template <class T> RBD_HD void joint_scd(int kind, const Pre<T>& pre, T& s, T& c, T& d, T qoff = T(0)) {
  s = T(0); c = T(1); d = T(0);
  if (kind == K_REV) sincos_t(pre.q0 + qoff, s, c);
  else if (kind == K_SINCOS) { s = pre.q0; c = pre.q1; }
  else if (kind == K_PRIS) d = pre.q0;
}

// ---- pass 1 (outward): velocities ---------------------------------------------------------------------------------
// ANY: the body may carry a multi-DoF joint (always possible for body 0; elsewhere only in GENERAL models)
template <class T, class ST, bool ANY, class IO>
RBD_HD void aba_pass1_body(const ModelDev<T>& M, int i, const IO& io, const ST& st, Mot<T>& vcur,
                           const Pre<T>& pre) {
  const BodyDev<T>& bd = M.body[i];
  Mot<T> vp;
  trace_conn<T>(true);
  if (bd.flags & F_ROOT_CHILD) {
#pragma unroll
    for (int k = 0; k < 3; ++k) { vp.w[k] = T(0); vp.l[k] = T(0); }
  } else if (bd.flags & F_FIRST_CHILD) {
    vp = vcur;
  } else {
    const int pr = M.body[bd.parent].row0;
    T t[6];
    st.fence_st();
    st.template ldv<6>(pr, t);
#pragma unroll
    for (int k = 0; k < 3; ++k) { vp.w[k] = t[k]; vp.l[k] = t[3 + k]; }
  }
  trace_conn<T>(false);
  const int kind = bd.kind;
  T R[9], r[3];
  Mot<T> v;
  if (pre.zflags) {                                  // revolute, E = [P] Rz(q + qoff)
    T s, c;
    sincos_t(pre.q0 + pre.qoff, s, c);
    if (pre.zflags & F_ZPERP) motion_to_child_z<T, 1>(s, c, bd.pt, vp, v);
    else motion_to_child_z<T, 0>(s, c, bd.pt, vp, v);
    v.w[2] += pre.qd;
  } else if (!ANY || kind == K_REV || kind == K_PRIS || kind == K_SINCOS || kind == K_FIXED) {
    T s, c, d, qd = T(0);
    joint_scd(kind, pre, s, c, d);
    if (!(IO::kKinds & kHasFixed) || kind != K_FIXED) qd = pre.qd;
    frame_1dof(bd, s, c, d, R, r);
    motion_to_child(R, r, vp, v);
    if ((IO::kKinds & kHasPris) && kind == K_PRIS) v.l[2] += qd;
    else if (!(IO::kKinds & kHasFixed) || kind != K_FIXED) v.w[2] += qd;
  } else {
    frame_multi(bd, io.q, R, r);
    motion_to_child(R, r, vp, v);
    const int K = kind == K_QSPH || kind == K_PLANAR ? 3 : 6;
    T x[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) x[k] = k < K ? io.v(bd.vrow + k) : T(0);
    Mot<T> vj;
    if (kind == K_PLANAR) joint_motion_multi<T, 3>(K_PLANAR, x, vj);
    else joint_motion_multi<T, 6>(K_QFLOAT, x, vj);
#pragma unroll
    for (int k = 0; k < 3; ++k) { v.w[k] += vj.w[k]; v.l[k] += vj.l[k]; }
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) { st.st(bd.row0 + k, v.w[k]); st.st(bd.row0 + 3 + k, v.l[k]); }
  vcur = v;
  if (io.qd.valid()) qdot_joint<T, !ANY>(bd, io.q, io.v, io.qd);
}

// Eliminate a revolute-z DoF from the assembled articulated quantities `a` of a body moving with `v`:
//   U = IA e_z (a column), D = U_z, u = tau - pA_z;  U~ = U / D (returned without its unit entry: ang x, ang y, lin x, lin y,
//   lin z), u~ = (u - U.c) / D with c = v x (e_z qd);  b = (Ia, pa) = (IA - U U~^T, pA + Ia c + U u / D), whose angular-z
//   row / column vanish.  Straight-line code (no branches) so two calls in one block interleave.
template <class T>
RBD_HD void rev_eliminate(const Art<T>& a, const Mot<T>& v, T qd, T tau, T (&tU)[5], T& tu, Art<T>& b) {
  const T Ux = a.A[2], Uy = a.A[4], D = a.A[5];
  const T Ulx = a.B[6], Uly = a.B[7], Ulz = a.B[8];
  const T Dinv = T(1) / D;
  const T cax = qd * v.w[1], cay = -qd * v.w[0];     // c = v x (e_z qd): [w x e_z qd ; l x e_z qd]
  const T clx = qd * v.l[1], cly = -qd * v.l[0];
  const T u = tau - a.n[2];
  const T Uc = Ux * cax + Uy * cay + Ulx * clx + Uly * cly;
  const T tUx = Ux * Dinv, tUy = Uy * Dinv, tLx = Ulx * Dinv, tLy = Uly * Dinv, tLz = Ulz * Dinv;
  tU[0] = tUx; tU[1] = tUy; tU[2] = tLx; tU[3] = tLy; tU[4] = tLz;
  tu = (u - Uc) * Dinv;
  b.A[0] = a.A[0] - Ux * tUx; b.A[1] = a.A[1] - Ux * tUy; b.A[3] = a.A[3] - Uy * tUy;
  b.A[2] = T(0); b.A[4] = T(0); b.A[5] = T(0);
  b.B[0] = a.B[0] - Ux * tLx; b.B[1] = a.B[1] - Ux * tLy; b.B[2] = a.B[2] - Ux * tLz;
  b.B[3] = a.B[3] - Uy * tLx; b.B[4] = a.B[4] - Uy * tLy; b.B[5] = a.B[5] - Uy * tLz;
  b.B[6] = T(0); b.B[7] = T(0); b.B[8] = T(0);
  b.C[0] = a.C[0] - Ulx * tLx; b.C[1] = a.C[1] - Ulx * tLy; b.C[2] = a.C[2] - Ulx * tLz;
  b.C[3] = a.C[3] - Uly * tLy; b.C[4] = a.C[4] - Uly * tLz; b.C[5] = a.C[5] - Ulz * tLz;
  const T du = u * Dinv;
  b.n[0] = a.n[0] + b.A[0] * cax + b.A[1] * cay + b.B[0] * clx + b.B[1] * cly + Ux * du;
  b.n[1] = a.n[1] + b.A[1] * cax + b.A[3] * cay + b.B[3] * clx + b.B[4] * cly + Uy * du;
  b.n[2] = a.n[2] + u;
  b.f[0] = a.f[0] + b.B[0] * cax + b.B[3] * cay + b.C[0] * clx + b.C[1] * cly + Ulx * du;
  b.f[1] = a.f[1] + b.B[1] * cax + b.B[4] * cay + b.C[1] * clx + b.C[3] * cly + Uly * du;
  b.f[2] = a.f[2] + b.B[2] * cax + b.B[5] * cay + b.C[2] * clx + b.C[4] * cly + Ulz * du;
}

// ---- pass 2 (inward): articulated inertias ------------------------------------------------------------------------
// 1-DoF / fixed body.  On exit the body's rows hold U~ (5 non-unit entries) and u~; `carry` / the parent's slot hold
// its contribution to the parent.
template <class T, class ST, class IO>
RBD_HD void aba_pass2_1dof(const ModelDev<T>& M, int i, const IO& io, const ST& st, Art<T>& carry,
                           const Pre<T>& pre) {
  const BodyDev<T>& bd = M.body[i];
  const int kind = bd.kind;
  Mot<T> v;
  {
    T t[6];
    st.template ldv<6>(bd.row0, t);
#pragma unroll
    for (int k = 0; k < 3; ++k) { v.w[k] = t[k]; v.l[k] = t[3 + k]; }
  }
  Art<T> a;
  art_set_body(bd, a);
  bias_force(bd, v, a.n, a.f);
  if (IO::kExt) {
#pragma unroll
    for (int k = 0; k < 3; ++k) { a.n[k] -= pre.w[k]; a.f[k] -= pre.w[3 + k]; }   // - w_ext in body coordinates
  }
  if (!(bd.flags & F_LEAF)) art_add(a, carry);
  if (bd.flags & F_HAS_PENDING) art_add_from(st.slots(), M.slot_base + bd.oslot * kSlotRowsAba, a);

  if ((IO::kKinds & kHasFixed) && kind == K_FIXED) {
    if (!(bd.flags & F_ROOT_CHILD)) {
      T R[9], r[3];
      frame_1dof(bd, T(0), T(1), T(0), R, r);
      const Art<T> src = a;
      art_to_parent<T, false>(R, r, src, carry);
      hand_over(M, bd, st, carry);
    }
    return;
  }
  T sn, c, dd;
  joint_scd(kind, pre, sn, c, dd, pre.qoff);
  const T qd = pre.qd;
  const T tau = pre.tau;
  if (!(IO::kKinds & kHasPris) || kind != K_PRIS) {
    // ---- revolute about e_z: S = e_{ang z} ----
    T tU[5], tu;
    Art<T> b;
    rev_eliminate(a, v, qd, tau, tU, tu, b);
#pragma unroll
    for (int k = 0; k < 5; ++k) st.st(bd.row0 + k, tU[k]);
    st.st(bd.row0 + 5, tu);
    if (bd.flags & F_ROOT_CHILD) return;
    if (pre.zflags & F_ZERO_R) {
      if (pre.zflags & F_ZPERP) art_to_parent_z<T, 1, true>(sn, c, bd.pt, b, carry);
      else art_to_parent_z<T, 0, true>(sn, c, bd.pt, b, carry);
    } else if (pre.zflags & F_ZPERP) art_to_parent_z<T, 1>(sn, c, bd.pt, b, carry);
    else if (pre.zflags & F_ZPAR) art_to_parent_z<T, 0>(sn, c, bd.pt, b, carry);
    else {
      T R[9], r[3];
      frame_1dof(bd, sn, c, T(0), R, r);
      art_to_parent<T, true>(R, r, b, carry);
    }
    hand_over(M, bd, st, carry);
  } else {
    // ---- prismatic along e_z: S = e_{lin z} ----
    const T Ux = a.B[2], Uy = a.B[5], Uz = a.B[8];
    const T Ulx = a.C[2], Uly = a.C[4], D = a.C[5];
    const T Dinv = T(1) / D;
    // c = v x (e_{lin z} qd) = [0 ; w x e_z qd]
    const T clx = qd * v.w[1], cly = -qd * v.w[0];
    const T u = tau - a.f[2];
    const T Uc = Ulx * clx + Uly * cly;
    const T tUx = Ux * Dinv, tUy = Uy * Dinv, tUz = Uz * Dinv, tLx = Ulx * Dinv, tLy = Uly * Dinv;
    st.st(bd.row0 + 0, tUx); st.st(bd.row0 + 1, tUy); st.st(bd.row0 + 2, tUz); st.st(bd.row0 + 3, tLx);
    st.st(bd.row0 + 4, tLy); st.st(bd.row0 + 5, (u - Uc) * Dinv);
    if (bd.flags & F_ROOT_CHILD) return;
    Art<T> b;
    b.A[0] = a.A[0] - Ux * tUx; b.A[1] = a.A[1] - Ux * tUy; b.A[2] = a.A[2] - Ux * tUz;
    b.A[3] = a.A[3] - Uy * tUy; b.A[4] = a.A[4] - Uy * tUz; b.A[5] = a.A[5] - Uz * tUz;
    b.B[0] = a.B[0] - Ux * tLx; b.B[1] = a.B[1] - Ux * tLy; b.B[2] = T(0);
    b.B[3] = a.B[3] - Uy * tLx; b.B[4] = a.B[4] - Uy * tLy; b.B[5] = T(0);
    b.B[6] = a.B[6] - Uz * tLx; b.B[7] = a.B[7] - Uz * tLy; b.B[8] = T(0);
    b.C[0] = a.C[0] - Ulx * tLx; b.C[1] = a.C[1] - Ulx * tLy; b.C[3] = a.C[3] - Uly * tLy;
    b.C[2] = T(0); b.C[4] = T(0); b.C[5] = T(0);
    const T du = u * Dinv;
    b.n[0] = a.n[0] + b.B[0] * clx + b.B[1] * cly + Ux * du;
    b.n[1] = a.n[1] + b.B[3] * clx + b.B[4] * cly + Uy * du;
    b.n[2] = a.n[2] + b.B[6] * clx + b.B[7] * cly + Uz * du;
    b.f[0] = a.f[0] + b.C[0] * clx + b.C[1] * cly + Ulx * du;
    b.f[1] = a.f[1] + b.C[1] * clx + b.C[3] * cly + Uly * du;
    b.f[2] = a.f[2] + u;
    T R[9], r[3];
    frame_1dof(bd, T(0), T(1), dd, R, r);
    art_to_parent<T, false>(R, r, b, carry);
    hand_over(M, bd, st, carry);
  }
}

// Multi-DoF body (K = 3 or 6, one-hot subspace).  ROOT0 = preorder position 0 under the world: nothing is stored or
// propagated; instead the joint acceleration is solved right away and the outward pass starts from registers.
template <class T, class ST, int K, int FAM, bool ROOT0, class IO>
RBD_HD void aba_pass2_multi(const ModelDev<T>& M, int i, const IO& io, const ST& st, Art<T>& carry,
                            Mot<T>& vout, Mot<T>& aout) {
  const BodyDev<T>& bd = M.body[i];
  constexpr int ck = FAM;   // subspace index family: K_PLANAR, or K_QFLOAT (spherical = first 3 of floating)
  Mot<T> v;
#pragma unroll
  for (int k = 0; k < 3; ++k) { v.w[k] = st.ld(bd.row0 + k); v.l[k] = st.ld(bd.row0 + 3 + k); }
  Art<T> a;
  art_set_body(bd, a);
  bias_force(bd, v, a.n, a.f);
  if (IO::kExt) {
#pragma unroll
    for (int k = 0; k < 3; ++k) { a.n[k] -= io.ext.get(6 * i + k); a.f[k] -= io.ext.get(6 * i + 3 + k); }
  }
  if (!(bd.flags & F_LEAF)) art_add(a, carry);
  if (bd.flags & F_HAS_PENDING) art_add_from(st.slots(), M.slot_base + bd.oslot * kSlotRowsAba, a);
  T I[6][6], p[6];
  art_to_full(a, I, p);
  T x[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) x[k] = k < K ? io.v(bd.vrow + k) : T(0);
  Mot<T> vj, cm;
  joint_motion_multi<T, K>(ck, x, vj);
  motion_cross(v, vj, cm);
  const T c[6] = {cm.w[0], cm.w[1], cm.w[2], cm.l[0], cm.l[1], cm.l[2]};
  T D[K][K], dinv[K], U[6][K], u[K];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const int sk = sub_index(ck, k);
#pragma unroll
    for (int rr = 0; rr < 6; ++rr) U[rr][k] = I[rr][sk];
#pragma unroll
    for (int l = 0; l < K; ++l) D[k][l] = I[sk][sub_index(ck, l)];
    u[k] = (io.tau.valid() ? io.tau(bd.vrow + k) : T(0)) - p[sk];
  }
  ldlt<T, K>(D, dinv);
  T tU[6][K];   // U~ = U D^-1 (row r = D^-1 U[r][:])
#pragma unroll
  for (int rr = 0; rr < 6; ++rr) {
    T y[K];
#pragma unroll
    for (int k = 0; k < K; ++k) y[k] = U[rr][k];
    ldlt_solve<T, K>(D, dinv, y);
#pragma unroll
    for (int k = 0; k < K; ++k) tU[rr][k] = y[k];
  }
  T tu[K];      // u~ = D^-1 (u - U^T c)
#pragma unroll
  for (int k = 0; k < K; ++k) {
    T s = u[k];
#pragma unroll
    for (int rr = 0; rr < 6; ++rr) s -= U[rr][k] * c[rr];
    tu[k] = s;
  }
  ldlt_solve<T, K>(D, dinv, tu);
  if (ROOT0) {
    // outward step for this body, straight from registers: parent = world, a_parent = -g (mechanism_algorithms.jl:405)
    T R[9], r[3];
    frame_multi(bd, io.q, R, r);
    Mot<T> ap, xa;
    ap.w[0] = ap.w[1] = ap.w[2] = T(0);
    ap.l[0] = -M.g[0]; ap.l[1] = -M.g[1]; ap.l[2] = -M.g[2];
    motion_to_child(R, r, ap, xa);
    const T xa6[6] = {xa.w[0], xa.w[1], xa.w[2], xa.l[0], xa.l[1], xa.l[2]};
    T vd[6] = {T(0), T(0), T(0), T(0), T(0), T(0)};
#pragma unroll
    for (int k = 0; k < K; ++k) {
      T s = tu[k];
#pragma unroll
      for (int rr = 0; rr < 6; ++rr) s -= tU[rr][k] * xa6[rr];
      vd[k] = s;
      io.vd.st(bd.vrow + k, s);
    }
    Mot<T> sa;
    joint_motion_multi<T, K>(ck, vd, sa);
#pragma unroll
    for (int k = 0; k < 3; ++k) { aout.w[k] = xa.w[k] + cm.w[k] + sa.w[k]; aout.l[k] = xa.l[k] + cm.l[k] + sa.l[k]; }
    vout = v;
    return;
  }
  if (!(bd.flags & F_ROOT_CHILD)) {
    // Ia = IA - U~ U^T ; pa = pA + Ia c + U~ u
    T Ia[6][6], pa[6];
#pragma unroll
    for (int rr = 0; rr < 6; ++rr)
#pragma unroll
      for (int cc = 0; cc < 6; ++cc) {
        T s = I[rr][cc];
#pragma unroll
        for (int k = 0; k < K; ++k) s -= tU[rr][k] * U[cc][k];
        Ia[rr][cc] = s;
      }
#pragma unroll
    for (int rr = 0; rr < 6; ++rr) {
      T s = p[rr];
#pragma unroll
      for (int cc = 0; cc < 6; ++cc) s += Ia[rr][cc] * c[cc];
#pragma unroll
      for (int k = 0; k < K; ++k) s += tU[rr][k] * u[k];
      pa[rr] = s;
    }
    Art<T> b;
    full_to_art(Ia, pa, b);
    T R[9], r[3];
    frame_multi(bd, io.q, R, r);
    art_to_parent<T, false>(R, r, b, carry);
    hand_over(M, bd, st, carry);
  }
  // rows: U~ (6K, row-major [r][k]) then u~ (K)
#pragma unroll
  for (int rr = 0; rr < 6; ++rr)
#pragma unroll
    for (int k = 0; k < K; ++k) st.st(bd.row0 + rr * K + k, tU[rr][k]);
#pragma unroll
  for (int k = 0; k < K; ++k) st.st(bd.row0 + 6 * K + k, tu[k]);
}

// ---- pass 3 (outward): accelerations ------------------------------------------------------------------------------
template <class T, class ST>
RBD_HD void load_parent_va(const ModelDev<T>& M, const BodyDev<T>& bd, const ST& st, const Mot<T>& vcur,
                           const Mot<T>& acur, Mot<T>& vp, Mot<T>& ap) {
  trace_conn<T>(true);
  if (bd.flags & F_ROOT_CHILD) {
#pragma unroll
    for (int k = 0; k < 3; ++k) { vp.w[k] = T(0); vp.l[k] = T(0); ap.w[k] = T(0); ap.l[k] = -M.g[k]; }
  } else if (bd.flags & F_FIRST_CHILD) {
    vp = vcur; ap = acur;
  } else {
    const int row = M.slot_base + bd.pslot * kSlotRowsAba;
    const auto sl = st.slots();
    T t[12];
    sl.fence_st();
    sl.template ldv<12>(row, t);
#pragma unroll
    for (int k = 0; k < 3; ++k) { vp.w[k] = t[k]; vp.l[k] = t[3 + k]; ap.w[k] = t[6 + k]; ap.l[k] = t[9 + k]; }
  }
  trace_conn<T>(false);
}
template <class T, class ST>
RBD_HD void save_own_va(const ModelDev<T>& M, const BodyDev<T>& bd, const ST& st, const Mot<T>& v, const Mot<T>& a) {
  if (bd.flags & F_HAS_PENDING) {
    const int row = M.slot_base + bd.oslot * kSlotRowsAba;
    const auto sl = st.slots();
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      sl.st(row + k, v.w[k]); sl.st(row + 3 + k, v.l[k]);
      sl.st(row + 6 + k, a.w[k]); sl.st(row + 9 + k, a.l[k]);
    }
  }
}

template <class T, class ST, class IO>
RBD_HD void aba_pass3_1dof(const ModelDev<T>& M, int i, const IO& io, const ST& st, Mot<T>& vcur, Mot<T>& acur,
                           const Pre<T>& pre) {
  const BodyDev<T>& bd = M.body[i];
  const int kind = bd.kind;
  Mot<T> vp, ap, v, xa;
  load_parent_va(M, bd, st, vcur, acur, vp, ap);
  T R[9], r[3];
  if ((IO::kKinds & kHasFixed) && kind == K_FIXED) {
    frame_1dof(bd, T(0), T(1), T(0), R, r);
    motion_to_child(R, r, vp, v);
    motion_to_child(R, r, ap, xa);
    vcur = v; acur = xa;
    save_own_va(M, bd, st, v, xa);
    return;
  }
  T sn, c, dd;
  joint_scd(kind, pre, sn, c, dd, pre.qoff);
  const T qd = pre.qd;
  T tt[6];
  st.template ldv<6>(bd.row0, tt);
  const T t0 = tt[0], t1 = tt[1], t2 = tt[2], t3 = tt[3], t4 = tt[4], tu = tt[5];
  Mot<T> a;
  if (!(IO::kKinds & kHasPris) || kind != K_PRIS) {
    if (pre.zflags & F_ZPERP) {
      motion_to_child_z<T, 1>(sn, c, bd.pt, vp, v);
      motion_to_child_z<T, 1>(sn, c, bd.pt, ap, xa);
    } else if (pre.zflags & F_ZPAR) {
      motion_to_child_z<T, 0>(sn, c, bd.pt, vp, v);
      motion_to_child_z<T, 0>(sn, c, bd.pt, ap, xa);
    } else {
      frame_1dof(bd, sn, c, T(0), R, r);
      motion_to_child(R, r, vp, v);
      motion_to_child(R, r, ap, xa);
    }
    v.w[2] += qd;
    // v̇ = u~ - U~ . (X a_parent), U~ = (t0, t1, 1 | t2, t3, t4)
    const T vd = tu - (t0 * xa.w[0] + t1 * xa.w[1] + xa.w[2] + t2 * xa.l[0] + t3 * xa.l[1] + t4 * xa.l[2]);
    io.vd.st(bd.vrow, vd);
    a.w[0] = xa.w[0] + qd * v.w[1]; a.w[1] = xa.w[1] - qd * v.w[0]; a.w[2] = xa.w[2] + vd;
    a.l[0] = xa.l[0] + qd * v.l[1]; a.l[1] = xa.l[1] - qd * v.l[0]; a.l[2] = xa.l[2];
  } else {
    frame_1dof(bd, T(0), T(1), dd, R, r);
    motion_to_child(R, r, vp, v);
    motion_to_child(R, r, ap, xa);
    v.l[2] += qd;
    // U~ = (t0, t1, t2 | t3, t4, 1)
    const T vd = tu - (t0 * xa.w[0] + t1 * xa.w[1] + t2 * xa.w[2] + t3 * xa.l[0] + t4 * xa.l[1] + xa.l[2]);
    io.vd.st(bd.vrow, vd);
    a.w[0] = xa.w[0]; a.w[1] = xa.w[1]; a.w[2] = xa.w[2];
    a.l[0] = xa.l[0] + qd * v.w[1]; a.l[1] = xa.l[1] - qd * v.w[0]; a.l[2] = xa.l[2] + vd;
  }
  vcur = v; acur = a;
  save_own_va(M, bd, st, v, a);
}

template <class T, class ST, int K, int FAM, class IO>
RBD_HD void aba_pass3_multi(const ModelDev<T>& M, int i, const IO& io, const ST& st, Mot<T>& vcur, Mot<T>& acur) {
  const BodyDev<T>& bd = M.body[i];
  constexpr int ck = FAM;
  Mot<T> vp, ap, v, xa;
  load_parent_va(M, bd, st, vcur, acur, vp, ap);
  T R[9], r[3];
  frame_multi(bd, io.q, R, r);
  motion_to_child(R, r, vp, v);
  motion_to_child(R, r, ap, xa);
  T x[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) x[k] = k < K ? io.v(bd.vrow + k) : T(0);
  Mot<T> vj, cm, sa;
  joint_motion_multi<T, K>(ck, x, vj);
#pragma unroll
  for (int k = 0; k < 3; ++k) { v.w[k] += vj.w[k]; v.l[k] += vj.l[k]; }
  motion_cross(v, vj, cm);
  const T xa6[6] = {xa.w[0], xa.w[1], xa.w[2], xa.l[0], xa.l[1], xa.l[2]};
  T vd[6] = {T(0), T(0), T(0), T(0), T(0), T(0)};
#pragma unroll
  for (int k = 0; k < K; ++k) {
    T s = st.ld(bd.row0 + 6 * K + k);
#pragma unroll
    for (int rr = 0; rr < 6; ++rr) s -= st.ld(bd.row0 + rr * K + k) * xa6[rr];
    vd[k] = s;
    io.vd.st(bd.vrow + k, s);
  }
  joint_motion_multi<T, K>(ck, vd, sa);
  Mot<T> a;
#pragma unroll
  for (int k = 0; k < 3; ++k) { a.w[k] = xa.w[k] + cm.w[k] + sa.w[k]; a.l[k] = xa.l[k] + cm.l[k] + sa.l[k]; }
  vcur = v; acur = a;
  save_own_va(M, bd, st, v, a);
}

// ---- whole algorithm for one sample -------------------------------------------------------------------------------
// GENERAL = false: bodies 1..nb-1 are 1-DoF or fixed (a multi-DoF joint is allowed only at position 0 under the world), so the
// loops carry 1-DoF code only.  GENERAL = true dispatches every body on its kind.
// (Tried and removed: walking two sibling revolute chains in lock-step for 2x instruction-level parallelism -- 601 M vs 666 M
// evals/s on Atlas, the second copy of the inlined step bodies overflowed the instruction cache.  DESIGN.md section 7.)
template <class T, class ST, bool GENERAL, class IO>
RBD_HD void aba_sample(const ModelDev<T>& M, const IO& io, const ST& st) {
  const int nb = M.nb;
  Mot<T> vcur, acur;
#pragma unroll
  for (int k = 0; k < 3; ++k) vcur.w[k] = vcur.l[k] = acur.w[k] = acur.l[k] = T(0);
  // ---- pass 1 (loads for the next body are in flight while this body is processed) ----
  Pre<T> cur, nxt;
  prefetch_body<T, 1>(M, 0, io, cur);
  prefetch_body<T, 1>(M, 1, io, nxt);
  aba_pass1_body<T, ST, true>(M, 0, io, st, vcur, cur);      // body 0 may be multi-DoF in any model: peeled
  cur = nxt;
  for (int i = 1; i < nb; ++i) {
    trace_step<T>(1, i);
    prefetch_body<T, 1>(M, i + 1, io, nxt);
    aba_pass1_body<T, ST, GENERAL>(M, i, io, st, vcur, cur);
    cur = nxt;
  }
  trace_step<T>(1, -1);
  // ---- pass 2 ----
  st.fence_st();
  Art<T> carry;
#pragma unroll
  for (int k = 0; k < 6; ++k) { carry.A[k] = T(0); carry.C[k] = T(0); }
#pragma unroll
  for (int k = 0; k < 9; ++k) carry.B[k] = T(0);
#pragma unroll
  for (int k = 0; k < 3; ++k) { carry.n[k] = T(0); carry.f[k] = T(0); }
  prefetch_body<T, 2>(M, nb - 1, io, cur);
  for (int i = nb - 1; i >= 1; --i) {
    const int kind = M.body[i].kind;
    trace_step<T>(2, i);
    prefetch_body<T, 2>(M, i - 1, io, nxt);
    const Pre<T> now = cur;
    cur = nxt;
    if (!GENERAL || kind == K_REV || kind == K_PRIS || kind == K_SINCOS || kind == K_FIXED) {
      aba_pass2_1dof(M, i, io, st, carry, now);
    } else if (kind == K_QFLOAT || kind == K_SPQFLOAT) {
      aba_pass2_multi<T, ST, 6, K_QFLOAT, false>(M, i, io, st, carry, vcur, acur);
    } else if (kind == K_PLANAR) {
      aba_pass2_multi<T, ST, 3, K_PLANAR, false>(M, i, io, st, carry, vcur, acur);
    } else {
      aba_pass2_multi<T, ST, 3, K_QFLOAT, false>(M, i, io, st, carry, vcur, acur);
    }
  }
  trace_step<T>(2, -1);
  // body 0: inward step, then the outward pass starts here
  {
    const BodyDev<T>& b0 = M.body[0];
    const int kind = b0.kind;
    prefetch_body<T, 3>(M, 1, io, nxt);
    if (kind == K_REV || kind == K_PRIS || kind == K_SINCOS || kind == K_FIXED) {
      aba_pass2_1dof(M, 0, io, st, carry, cur);
      st.fence_st();
      aba_pass3_1dof(M, 0, io, st, vcur, acur, cur);
    } else if (kind == K_QFLOAT || kind == K_SPQFLOAT) {
      aba_pass2_multi<T, ST, 6, K_QFLOAT, true>(M, 0, io, st, carry, vcur, acur);
      save_own_va(M, b0, st, vcur, acur);
    } else if (kind == K_PLANAR) {
      aba_pass2_multi<T, ST, 3, K_PLANAR, true>(M, 0, io, st, carry, vcur, acur);
      save_own_va(M, b0, st, vcur, acur);
    } else {
      aba_pass2_multi<T, ST, 3, K_QFLOAT, true>(M, 0, io, st, carry, vcur, acur);
      save_own_va(M, b0, st, vcur, acur);
    }
  }
  // ---- pass 3 ----
  st.fence_st();
  cur = nxt;
  for (int i = 1; i < nb; ++i) {
    const int kind = M.body[i].kind;
    trace_step<T>(3, i);
    prefetch_body<T, 3>(M, i + 1, io, nxt);
    const Pre<T> now = cur;
    cur = nxt;
    if (!GENERAL || kind == K_REV || kind == K_PRIS || kind == K_SINCOS || kind == K_FIXED) {
      aba_pass3_1dof(M, i, io, st, vcur, acur, now);
    } else if (kind == K_QFLOAT || kind == K_SPQFLOAT) {
      aba_pass3_multi<T, ST, 6, K_QFLOAT>(M, i, io, st, vcur, acur);
    } else if (kind == K_PLANAR) {
      aba_pass3_multi<T, ST, 3, K_PLANAR>(M, i, io, st, vcur, acur);
    } else {
      aba_pass3_multi<T, ST, 3, K_QFLOAT>(M, i, io, st, vcur, acur);
    }
  }
  trace_step<T>(3, -1);
}

}  // namespace rbd
