// Munthe-Kaas RK4 step around `dynamics` (SURVEY 8(f) rank 1): the per-joint local <-> global coordinate maps.
//
// Reference (relative to the reference's src/):
//   step(::MuntheKaasIntegrator, t, dt)      ode_integrators.jl:233-300   (stages in local coordinates phi around q0)
//   runge_kutta_4                            ode_integrators.jl:48-55     a21 = a32 = 1/2, a43 = 1, b = (1/6, 1/3, 1/3, 1/6)
//   local_coordinates! / global_coordinates! mechanism_state.jl:1057-1085, defaults joint_types/joint_types.jl:9-18
//     (phi = q - q0, phi_dot = q̇ = N(q) v, q = q0 + phi: Revolute, Prismatic, Planar, SPQuatFloating, Fixed),
//     quaternion_floating.jl:205-249 (SE(3) exp / log_with_time_derivative, spatial/spatialmotion.jl:226-331),
//     quaternion_spherical.jl:139-154 (rotation vector, rotation_vector_rate spatial/util.jl:83-101),
//     sin_cos_revolute.jl:173-196.
//
// The stage angles are small (dt * phi_dot), where the closed forms of Bullo & Murray divide differences of nearly equal
// numbers by theta^2 or theta^4; below a threshold the same coefficients are evaluated from their Taylor series
// (dexp^-1 = 1 + ad/2 + ad^2/12 - ad^4/720 + ...), which is what makes the fp32 path usable.
#pragma once
#include "rbd_device.cuh"

namespace rbd {

RBD_HD float sqrt_t(float x) { return sqrtf(x); }
RBD_HD double sqrt_t(double x) { return sqrt(x); }
RBD_HD float atan2_t(float y, float x) { return atan2f(y, x); }
RBD_HD double atan2_t(double y, double x) { return atan2(y, x); }
// The floating type a scalar type computes in: T itself, or the value type of a dual number (rbd_integrate_adjoint.cuh), so
// that the adjoints' dual-number runs take the branches the forward pass took.
template <class T> struct ScalarOf { using type = T; };
template <class T> RBD_HD constexpr bool is_f32() { return sizeof(typename ScalarOf<T>::type) == 4; }
template <class T> RBD_HD T small_angle2() { return is_f32<T>() ? T(2.5e-3) : T(1e-6); }   // theta^2 threshold

template <class T> RBD_HD void quat_mul(const T* a, const T* b, T* o) {   // Hamilton product, [w x y z]
  o[0] = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  o[1] = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  o[2] = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
  o[3] = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
}
// rotation vector -> unit quaternion
template <class T> RBD_HD void quat_from_rotvec(const T* r, T* q) {
  const T t2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
  T k, w;
  if (t2 < small_angle2<T>()) {
    k = T(0.5) - t2 / T(48);
    w = T(1) - t2 / T(8) + t2 * t2 / T(384);
  } else {
    const T th = sqrt_t(t2);
    T s, c;
    sincos_t(T(0.5) * th, s, c);
    k = s / th;
    w = c;
  }
  q[0] = w; q[1] = k * r[0]; q[2] = k * r[1]; q[3] = k * r[2];
}
// unit quaternion -> rotation vector with angle in [0, pi]  (AngleAxis(rot), RotationVec(quat))
template <class T> RBD_HD void rotvec_from_quat(const T* qin, T* r, T& theta2) {
  T q[4] = {qin[0], qin[1], qin[2], qin[3]};
  if (q[0] < T(0)) { q[0] = -q[0]; q[1] = -q[1]; q[2] = -q[2]; q[3] = -q[3]; }
  const T s2 = q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  const T sn = sqrt_t(s2);
  T k;
  if (s2 < small_angle2<T>() * T(0.25)) {
    k = T(2) + s2 / T(3);                       // theta / sin(theta/2) for small angles, w ~ 1
    theta2 = k * k * s2;
  } else {
    const T th = T(2) * atan2_t(sn, q[0]);
    k = th / sn;
    theta2 = th * th;
  }
  r[0] = k * q[1]; r[1] = k * q[2]; r[2] = k * q[3];
}

// Coefficients of dexp^-1 on SE(3) / SO(3) (Bullo & Murray, "PD control on the Euclidean group", eq. (2.5) and Lemma 4):
//   g = (1 - alpha) / theta^2,  A = (2 (1 - alpha) + (alpha - beta) / 2) / theta^2,  B = ((1 - alpha) + (alpha - beta) / 2) / theta^4
template <class T> RBD_HD void dexpinv_coeffs(T theta2, T& g, T& A, T& B) {
  if (theta2 < small_angle2<T>()) {
    g = T(1) / T(12) + theta2 / T(720) + theta2 * theta2 / T(30240);
    A = T(1) / T(12) - theta2 * theta2 / T(30240);            // the theta^2 term cancels exactly
    B = T(-1) / T(720) - theta2 / T(15120);
  } else {
    const T th = sqrt_t(theta2);
    T s, c;
    sincos_t(T(0.5) * th, s, c);
    const T alpha = T(0.5) * th * c / s;
    const T beta = T(0.25) * theta2 / (s * s);
    g = (T(1) - alpha) / theta2;
    A = (T(2) * (T(1) - alpha) + T(0.5) * (alpha - beta)) / theta2;
    B = ((T(1) - alpha) + T(0.5) * (alpha - beta)) / (theta2 * theta2);
  }
}

template <class T> RBD_HD void se3_comm(const T* xw, const T* xv, const T* yw, const T* yv, T* ow, T* ov) {   // util.jl:117-121
  cross3(xw, yw, ow);
  T a[3], b[3];
  cross3(xw, yv, a);
  cross3(xv, yw, b);
  ov[0] = a[0] + b[0]; ov[1] = a[1] + b[1]; ov[2] = a[2] + b[2];
}

// ---- QuaternionFloating --------------------------------------------------------------------------------------------
// global_coordinates!: q = q0 * exp(phi)  (quaternion_floating.jl:233-249, exp(::Twist) spatialmotion.jl:306-326)
template <class T> RBD_HD void qfloat_global(const T* q0, const T* phi, T* q) {
  const T* pr = phi;        // rotational part
  const T* pt = phi + 3;    // translational part
  const T t2 = pr[0] * pr[0] + pr[1] * pr[1] + pr[2] * pr[2];
  T dq[4];
  quat_from_rotvec(pr, dq);
  T R0[9], Rr[9], tr[3];
  rot_quat(q0[0], q0[1], q0[2], q0[3], R0);
  if (t2 < (is_f32<T>() ? T(1e-12) : T(1e-30))) {
    tr[0] = pt[0]; tr[1] = pt[1]; tr[2] = pt[2];
  } else {
    // trans = (1 - R) (w x v) + w (w . v) theta,  w = pr / theta, v = pt / theta
    rot_quat(dq[0], dq[1], dq[2], dq[3], Rr);
    const T it2 = T(1) / t2;
    T wxv[3], rw[3];
    cross3(pr, pt, wxv);
    wxv[0] *= it2; wxv[1] *= it2; wxv[2] *= it2;
    mat_vec(Rr, wxv, rw);
    const T wv = (pr[0] * pt[0] + pr[1] * pt[1] + pr[2] * pt[2]) * it2;
    tr[0] = wxv[0] - rw[0] + pr[0] * wv; tr[1] = wxv[1] - rw[1] + pr[1] * wv; tr[2] = wxv[2] - rw[2] + pr[2] * wv;
  }
  quat_mul(q0, dq, q);
  T t[3];
  mat_vec(R0, tr, t);
  q[4] = q0[4] + t[0]; q[5] = q0[5] + t[1]; q[6] = q0[6] + t[2];
}
// local_coordinates!: (phi, phi_dot) = log_with_time_derivative(q0^-1 q, twist v)   (quaternion_floating.jl:205-231)
template <class T> RBD_HD void qfloat_local_rate(const T* q0, const T* q, const T* v, T* phid) {
  const T q0c[4] = {q0[0], -q0[1], -q0[2], -q0[3]};
  T dq[4];
  quat_mul(q0c, q, dq);
  T R0[9], d[3] = {q[4] - q0[4], q[5] - q0[5], q[6] - q0[6]}, p[3];
  rot_quat(q0[0], q0[1], q0[2], q0[3], R0);
  matT_vec(R0, d, p);
  T psi[3], t2;
  rotvec_from_quat(dq, psi, t2);
  T g, A, B;
  dexpinv_coeffs(t2, g, A, B);
  // X = (psi, qq): qq = p - psi x p / 2 + g psi x (psi x p)     (_log, spatialmotion.jl:226-252)
  T c1[3], c2[3], qq[3];
  cross3(psi, p, c1);
  cross3(psi, c1, c2);
  qq[0] = p[0] - T(0.5) * c1[0] + g * c2[0]; qq[1] = p[1] - T(0.5) * c1[1] + g * c2[1]; qq[2] = p[2] - T(0.5) * c1[2] + g * c2[2];
  // X_dot = V + ad_X V / 2 + A ad_X^2 V + B ad_X^4 V            (Lemma 4, spatialmotion.jl:272-296)
  const T* w = v; const T* vl = v + 3;
  T a1w[3], a1v[3], a2w[3], a2v[3], a3w[3], a3v[3], a4w[3], a4v[3];
  se3_comm(psi, qq, w, vl, a1w, a1v);
  se3_comm(psi, qq, a1w, a1v, a2w, a2v);
  se3_comm(psi, qq, a2w, a2v, a3w, a3v);
  se3_comm(psi, qq, a3w, a3v, a4w, a4v);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    phid[k] = w[k] + T(0.5) * a1w[k] + A * a2w[k] + B * a4w[k];
    phid[3 + k] = vl[k] + T(0.5) * a1v[k] + A * a2v[k] + B * a4v[k];
  }
}

// ---- QuaternionSpherical (quaternion_spherical.jl:139-154, rotation_vector_rate util.jl:83-101) -----------------------
template <class T> RBD_HD void qsph_global(const T* q0, const T* phi, T* q) {
  T dq[4];
  quat_from_rotvec(phi, dq);
  quat_mul(q0, dq, q);
}
template <class T> RBD_HD void qsph_local_rate(const T* q0, const T* q, const T* w, T* phid) {
  const T q0c[4] = {q0[0], -q0[1], -q0[2], -q0[3]};
  T dq[4], phi[3], t2;
  quat_mul(q0c, q, dq);
  rotvec_from_quat(dq, phi, t2);
  // phi_dot = w + phi x w / 2 + 1/theta^2 (1 - theta s / (2 (1 - c))) phi x (phi x w);  the bracket / theta^2 equals g above
  T g, A, B;
  dexpinv_coeffs(t2, g, A, B);
  T c1[3], c2[3];
  cross3(phi, w, c1);
  cross3(phi, c1, c2);
#pragma unroll
  for (int k = 0; k < 3; ++k) phid[k] = w[k] + T(0.5) * c1[k] + g * c2[k];
}

// ---- SinCosRevolute, Planar, SPQuatFloating: the non-trivial halves of their coordinate maps ----------------------------
// (s, c) of the angle of (s0, c0) advanced by phi
template <class T> RBD_HD void sincos_global(T s0, T c0, T phi, T& s1, T& c1) {
  T s, c;
  sincos_t(phi, s, c);
  s1 = s0 * c + c0 * s;
  c1 = c0 * c - s0 * s;
}
// planar q̇ of the two translational velocity coordinates (a, b) at angle th
template <class T> RBD_HD void planar_rate(T th, T a, T b, T& pa, T& pb) {
  T s, c;
  sincos_t(th, s, c);
  pa = c * a - s * b;
  pb = s * a + c * b;
}
// SPQuatFloating q̇ = N(q) v (q: MRP, translation)
template <class T> RBD_HD void spq_rate(const T* qq, const T* vv, T* pd) {
  T e[4];
  mrp_to_quat(qq[0], qq[1], qq[2], e);
  const T w = e[0], x = e[1], y = e[2], z = e[3];
  const T dw = T(0.5) * (-x * vv[0] - y * vv[1] - z * vv[2]);
  const T dx = T(0.5) * (w * vv[0] - z * vv[1] + y * vv[2]);
  const T dy = T(0.5) * (z * vv[0] + w * vv[1] - x * vv[2]);
  const T dz = T(0.5) * (-y * vv[0] + x * vv[1] + w * vv[2]);
  const T inv = T(1) / (T(1) + w);
  pd[0] = (dx - x * dw * inv) * inv; pd[1] = (dy - y * dw * inv) * inv; pd[2] = (dz - z * dw * inv) * inv;
  T R[9];
  rot_quat(w, x, y, z, R);
  mat_vec(R, vv + 3, pd + 3);
}

// ---- one joint: stage configuration from local coordinates, and the rate of the local coordinates ---------------------
// q_stage = global(q0, phi);  phid = d/dt local(q0, q_stage, v_stage).  Rows are addressed through Col / ColOut views.
// CP / CV: any row accessor with operator()(row) -- Col<T>, ColRW<T>, or the on-the-fly combinations of the RK4 kernels.
template <class T, class CP, class CV>
RBD_HD void joint_stage(const BodyDev<T>& bd, const Col<T>& q0, const CP& phi, const CV& vs, const ColOut<T>& qs,
                        const ColOut<T>& phid) {
  const int q = bd.qrow, v = bd.vrow;
  switch (bd.kind) {
    case K_REV: case K_PRIS: {
      qs.st(q, q0(q) + phi(v));
      phid.st(v, vs(v));
      break;
    }
    case K_FIXED: break;
    case K_SINCOS: {                                   // sin_cos_revolute.jl:186-196, :173-184
      T s, c;
      sincos_global(q0(q), q0(q + 1), phi(v), s, c);
      qs.st(q, s);
      qs.st(q + 1, c);
      phid.st(v, vs(v));
      break;
    }
    case K_PLANAR: {                                   // defaults: q = q0 + phi, phi_dot = q̇ (planar.jl:123-129)
      const T x = q0(q) + phi(v), y = q0(q + 1) + phi(v + 1), th = q0(q + 2) + phi(v + 2);
      qs.st(q, x); qs.st(q + 1, y); qs.st(q + 2, th);
      T pa, pb;
      planar_rate(th, vs(v), vs(v + 1), pa, pb);
      phid.st(v, pa); phid.st(v + 1, pb); phid.st(v + 2, vs(v + 2));
      break;
    }
    case K_SPQFLOAT: {                                 // defaults with q̇ of spquat_floating.jl:128-138
      T qq[6], vv[6], pd[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) { qq[k] = q0(q + k) + phi(v + k); vv[k] = vs(v + k); qs.st(q + k, qq[k]); }
      spq_rate(qq, vv, pd);
#pragma unroll
      for (int k = 0; k < 6; ++k) phid.st(v + k, pd[k]);
      break;
    }
    case K_QFLOAT: {
      T a0[7], ph[6], vv[6], qn[7], pd[6];
#pragma unroll
      for (int k = 0; k < 7; ++k) a0[k] = q0(q + k);
#pragma unroll
      for (int k = 0; k < 6; ++k) { ph[k] = phi(v + k); vv[k] = vs(v + k); }
      qfloat_global(a0, ph, qn);
      qfloat_local_rate(a0, qn, vv, pd);
#pragma unroll
      for (int k = 0; k < 7; ++k) qs.st(q + k, qn[k]);
#pragma unroll
      for (int k = 0; k < 6; ++k) phid.st(v + k, pd[k]);
      break;
    }
    case K_QSPH: {
      T a0[4], ph[3], vv[3], qn[4], pd[3];
#pragma unroll
      for (int k = 0; k < 4; ++k) a0[k] = q0(q + k);
#pragma unroll
      for (int k = 0; k < 3; ++k) { ph[k] = phi(v + k); vv[k] = vs(v + k); }
      qsph_global(a0, ph, qn);
      qsph_local_rate(a0, qn, vv, pd);
#pragma unroll
      for (int k = 0; k < 4; ++k) qs.st(q + k, qn[k]);
#pragma unroll
      for (int k = 0; k < 3; ++k) phid.st(v + k, pd[k]);
      break;
    }
  }
}

#if defined(__CUDACC__)
// 16-byte vector of T for the kernels that treat revolute / prismatic rows VEC samples per thread (rbd_integrate, rbd_integrate_vjp)
template <class T> struct VecOf { using type = float4; static constexpr int N = 4; };
template <> struct VecOf<double> { using type = double2; static constexpr int N = 2; };
#endif

}  // namespace rbd
