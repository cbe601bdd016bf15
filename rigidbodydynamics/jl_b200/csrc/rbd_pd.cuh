// Joint-space feedback evaluated at every RK4 stage of a rollout (rbd_integrate_pd, DESIGN 4.18): the per-joint law, shared by the
// stage kernels of rbd_b200.cu and, compiled for the host, by tests/hostsim/hostsim_pd.cpp.
//
// Reference: pd(gains, e, ė) = -k e - d ė (src/pdcontrol.jl:35); the error of a joint is its local coordinates around the target,
// e = local_coordinates!(q_ref, q) (mechanism_state.jl:1057-1085 and the joint types cited in rbd_integrate.cuh), evaluated on
// the stage state (q_s, v_s) as the reference's simulate calls control!(τ, t, state) at every stage (src/simulate.jl:36-55).
//   q - q_ref                       Revolute, Prismatic, Planar, SPQuatFloating (the defaults, joint_types.jl:9-18)
//   angle of q_ref^-1 q             SinCosRevolute (sin_cos_revolute.jl:173-184)
//   rotation vector of q_ref^-1 q   QuaternionSpherical (quaternion_spherical.jl:139-154)
//   SE(3) log of q_ref^-1 q         QuaternionFloating (quaternion_floating.jl:205-231)
// The quaternions of q_ref must be unit quaternions: they are used as given, not normalised.
#pragma once
#include "rbd_integrate.cuh"

namespace rbd {

// e = local(q_ref, q) of one joint: nv(kind) entries from nq(kind) of each configuration
template <class T> RBD_HD void joint_error(int kind, const T* qref, const T* q, T* e) {
  switch (kind) {
    case K_REV: case K_PRIS: e[0] = q[0] - qref[0]; break;
    case K_PLANAR:
#pragma unroll
      for (int k = 0; k < 3; ++k) e[k] = q[k] - qref[k];
      break;
    case K_SPQFLOAT:
#pragma unroll
      for (int k = 0; k < 6; ++k) e[k] = q[k] - qref[k];
      break;
    case K_SINCOS: e[0] = atan2_t(qref[1] * q[0] - qref[0] * q[1], qref[1] * q[1] + qref[0] * q[0]); break;
    case K_QSPH: { T g; qsph_log(qref, q, e, g); break; }
    case K_QFLOAT: { T A, B; qfloat_log(qref, q, e, e + 3, A, B); break; }
    default: break;
  }
}

// one DoF of the law: ff - kp e - kd (v - v_ref)  (ff: the feedforward torque, or v̇_ref in computed-torque mode)
template <class T> RBD_HD T pd_law(T e, T v, T vref, T ff, T kp, T kd) { return ff - kp * e - kd * (v - vref); }
template <class T> RBD_HD T clamp_t(T x, T lo, T hi) { return x < lo ? lo : (x > hi ? hi : x); }

// One sample's view of the controller's inputs, each pointer already offset by the sample's column:
//   q, v       the stage state, leading dimension sld
//   qref, vref, ff   caller arrays at this (step, stage), leading dimension ld; vref / ff NULL = 0
//   kp, kd     gains, row stride gstride (1: one value per DoF shared by the batch; ld: per sample)
//   lo, hi     per-DoF saturation, NULL = none
template <class T> struct PdSample {
  const T* q; const T* v; int64_t sld;
  const T* qref; const T* vref; const T* ff; int64_t ld;
  const T* kp; const T* kd; int64_t gstride;
  const T* lo; const T* hi;
  RBD_HD T law(int row, T e) const {
    const int64_t r = (int64_t)row * ld, g = (int64_t)row * gstride;
    const T u = pd_law(e, v[(int64_t)row * sld], vref ? vref[r] : T(0), ff ? ff[r] : T(0), kp[g], kd[g]);
    return lo ? clamp_t(u, lo[row], hi[row]) : u;
  }
};

template <class T, int KIND, int NQ, int NV>
RBD_HD void pd_rows(int qrow, int vrow, const PdSample<T>& s, const ColOut<T>& out) {
  T q[NQ], qr[NQ], e[NV];
#pragma unroll
  for (int k = 0; k < NQ; ++k) { q[k] = s.q[(int64_t)(qrow + k) * s.sld]; qr[k] = s.qref[(int64_t)(qrow + k) * s.ld]; }
  joint_error(KIND, qr, q, e);
#pragma unroll
  for (int k = 0; k < NV; ++k) out.st(vrow + k, s.law(vrow + k, e[k]));
}

// The law of one joint at one sample: out rows vrow .. vrow + nv(kind) - 1 receive pd_law (clamped when s.lo is set).
template <class T> RBD_HD void pd_joint(const BodyDev<T>& bd, const PdSample<T>& s, const ColOut<T>& out) {
  const int q = bd.qrow, v = bd.vrow;
  switch (bd.kind) {
    case K_REV: pd_rows<T, K_REV, 1, 1>(q, v, s, out); break;
    case K_PRIS: pd_rows<T, K_PRIS, 1, 1>(q, v, s, out); break;
    case K_SINCOS: pd_rows<T, K_SINCOS, 2, 1>(q, v, s, out); break;
    case K_PLANAR: pd_rows<T, K_PLANAR, 3, 3>(q, v, s, out); break;
    case K_SPQFLOAT: pd_rows<T, K_SPQFLOAT, 6, 6>(q, v, s, out); break;
    case K_QSPH: pd_rows<T, K_QSPH, 4, 3>(q, v, s, out); break;
    case K_QFLOAT: pd_rows<T, K_QFLOAT, 7, 6>(q, v, s, out); break;
    default: break;
  }
}

}  // namespace rbd
