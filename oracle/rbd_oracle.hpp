// =====================================================================================================
// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
//
// CPU restatement ("oracle") of the reference's batched-dynamics hot path, RigidBodyDynamics.jl v2.5.0.
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load the
// library built from this file.  The product path (rigidbodydynamics/jl_b200 + csrc/) never calls it.
//
// PARITY PINNING: the reference cannot run here (no Julia) and its tests hold no stored numeric vectors
// for dynamics.  This restatement is pinned by (1) the closed-form double-pendulum test of the reference
// (test/test_double_pendulum.jl:2-11,51-65,72-75, atol 1e-12), (2) the rpy goldens (test/test_urdf.jl:85-100)
// via the host parser, and (3) the reference's own identity tests re-stated in tests/test_oracle.py
// (test/test_mechanism_algorithms.jl:564-572, 729-753).  For Atlas-sized models parity is therefore
// "pinned by identities + agreement of independent formulations", not by reference-produced vectors;
// quaternion/MRP -> rotation for NON-unit inputs is "parity unpinned" (Rotations.jl is not in the tree).
//
// What is restated (file:line relative to the reference's src/, RigidBodyDynamics.jl v2.5.0):
//   kinematic caches, world frame      mechanism_state.jl:687-868
//   CRBA  mass_matrix!                 mechanism_algorithms.jl:248-272
//   RNEA  bias/spatial accelerations   mechanism_algorithms.jl:377-417
//         newton_euler!                mechanism_algorithms.jl:428-439
//         joint_wrenches_and_torques!  mechanism_algorithms.jl:442-459
//   dynamics_bias! / inverse_dynamics! mechanism_algorithms.jl:484-498 / 542-553
//   dynamics_solve! (Cholesky, tree)   mechanism_algorithms.jl:747-766, 817-820
//   dynamics!                          mechanism_algorithms.jl:845-864
//   configuration_derivative!          mechanism_state.jl:905-910 + joint_types/*.jl
//   spatial device functions           spatial/util.jl:56-161, motion_force_interaction.jl:147-263,
//                                      spatialmotion.jl:375-401
// plus an INDEPENDENT world-frame Articulated-Body Algorithm (not in the reference; SURVEY 8(a) footnote)
// so that "algorithm change" and "hardware change" can be separated and the GPU ABA has a second check.
// =====================================================================================================
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace rbdo {

enum JointType : int32_t {
  JT_REVOLUTE = 0, JT_PRISMATIC = 1, JT_FIXED = 2, JT_PLANAR = 3, JT_QUAT_FLOATING = 4,
  JT_SPQUAT_FLOATING = 5, JT_QUAT_SPHERICAL = 6, JT_SINCOS_REVOLUTE = 7
};

// Forward-mode dual number with N partials (the ForwardDiff.Dual{Tag,Float64,N} the reference's generic-scalar path sees;
// examples/5, test "generic scalar dynamics").  Only what the templated code below needs.
template <int N> struct DualN {
  double v;
  double d[N];
  DualN() : v(0) { for (int i = 0; i < N; ++i) d[i] = 0; }
  DualN(double a) : v(a) { for (int i = 0; i < N; ++i) d[i] = 0; }
};
template <int N> inline DualN<N> operator+(const DualN<N>& a, const DualN<N>& b) { DualN<N> r; r.v = a.v + b.v; for (int i = 0; i < N; ++i) r.d[i] = a.d[i] + b.d[i]; return r; }
template <int N> inline DualN<N> operator-(const DualN<N>& a, const DualN<N>& b) { DualN<N> r; r.v = a.v - b.v; for (int i = 0; i < N; ++i) r.d[i] = a.d[i] - b.d[i]; return r; }
template <int N> inline DualN<N> operator-(const DualN<N>& a) { DualN<N> r; r.v = -a.v; for (int i = 0; i < N; ++i) r.d[i] = -a.d[i]; return r; }
template <int N> inline DualN<N> operator*(const DualN<N>& a, const DualN<N>& b) { DualN<N> r; r.v = a.v * b.v; for (int i = 0; i < N; ++i) r.d[i] = a.v * b.d[i] + a.d[i] * b.v; return r; }
template <int N> inline DualN<N> operator/(const DualN<N>& a, const DualN<N>& b) { DualN<N> r; r.v = a.v / b.v; for (int i = 0; i < N; ++i) r.d[i] = (a.d[i] - r.v * b.d[i]) / b.v; return r; }
template <int N> inline DualN<N>& operator+=(DualN<N>& a, const DualN<N>& b) { a = a + b; return a; }
template <int N> inline DualN<N>& operator-=(DualN<N>& a, const DualN<N>& b) { a = a - b; return a; }
template <int N> inline bool operator>(const DualN<N>& a, const DualN<N>& b) { return a.v > b.v; }
template <int N> inline DualN<N> sin(const DualN<N>& a) { DualN<N> r; r.v = std::sin(a.v); double c = std::cos(a.v); for (int i = 0; i < N; ++i) r.d[i] = c * a.d[i]; return r; }
template <int N> inline DualN<N> cos(const DualN<N>& a) { DualN<N> r; r.v = std::cos(a.v); double s = -std::sin(a.v); for (int i = 0; i < N; ++i) r.d[i] = s * a.d[i]; return r; }
template <int N> inline DualN<N> sqrt(const DualN<N>& a) { DualN<N> r; r.v = std::sqrt(a.v); for (int i = 0; i < N; ++i) r.d[i] = a.d[i] / (2 * r.v); return r; }

inline int joint_nq(int t) { static const int n[8] = {1, 1, 0, 3, 7, 6, 4, 2}; return n[t]; }
inline int joint_nv(int t) { static const int n[8] = {1, 1, 0, 3, 6, 6, 3, 1}; return n[t]; }

// ------------------------------------------------------------------------------------------------
// small fixed-size algebra
// ------------------------------------------------------------------------------------------------
template <class T> struct V3 {
  T x, y, z;
  V3() : x(0), y(0), z(0) {}
  V3(T a, T b, T c) : x(a), y(b), z(c) {}
  T operator[](int i) const { return i == 0 ? x : (i == 1 ? y : z); }
};
template <class T> inline V3<T> operator+(const V3<T>& a, const V3<T>& b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
template <class T> inline V3<T> operator-(const V3<T>& a, const V3<T>& b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
template <class T> inline V3<T> operator-(const V3<T>& a) { return {-a.x, -a.y, -a.z}; }
template <class T> inline V3<T> operator*(T s, const V3<T>& a) { return {s * a.x, s * a.y, s * a.z}; }
template <class T> inline V3<T> operator*(const V3<T>& a, T s) { return {s * a.x, s * a.y, s * a.z}; }
template <class T> inline T dot(const V3<T>& a, const V3<T>& b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
template <class T> inline V3<T> cross(const V3<T>& a, const V3<T>& b) {
  return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}

template <class T> struct M3 {   // row-major
  T m[9];
  M3() { for (int i = 0; i < 9; ++i) m[i] = T(0); }
  T& operator()(int r, int c) { return m[3 * r + c]; }
  T operator()(int r, int c) const { return m[3 * r + c]; }
  static M3 identity() { M3 r; r.m[0] = r.m[4] = r.m[8] = T(1); return r; }
};
template <class T> inline M3<T> operator*(const M3<T>& a, const M3<T>& b) {
  M3<T> r;
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) {
    T s = T(0);
    for (int k = 0; k < 3; ++k) s += a(i, k) * b(k, j);
    r(i, j) = s;
  }
  return r;
}
template <class T> inline V3<T> operator*(const M3<T>& a, const V3<T>& v) {
  return {a(0, 0) * v.x + a(0, 1) * v.y + a(0, 2) * v.z, a(1, 0) * v.x + a(1, 1) * v.y + a(1, 2) * v.z,
          a(2, 0) * v.x + a(2, 1) * v.y + a(2, 2) * v.z};
}
template <class T> inline M3<T> operator+(const M3<T>& a, const M3<T>& b) { M3<T> r; for (int i = 0; i < 9; ++i) r.m[i] = a.m[i] + b.m[i]; return r; }
template <class T> inline M3<T> operator-(const M3<T>& a, const M3<T>& b) { M3<T> r; for (int i = 0; i < 9; ++i) r.m[i] = a.m[i] - b.m[i]; return r; }
template <class T> inline M3<T> transpose(const M3<T>& a) { M3<T> r; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r(i, j) = a(j, i); return r; }
template <class T> inline M3<T> outer(const V3<T>& a, const V3<T>& b) {
  M3<T> r;
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r(i, j) = a[i] * b[j];
  return r;
}

// Transform3D (spatial/transform3d.jl:7-69): x_to = R x_from + p
template <class T> struct Xf {
  M3<T> R; V3<T> p;
  Xf() : R(M3<T>::identity()), p() {}
  Xf(const M3<T>& r, const V3<T>& t) : R(r), p(t) {}
};
template <class T> inline Xf<T> operator*(const Xf<T>& a, const Xf<T>& b) { return {a.R * b.R, a.R * b.p + a.p}; }
template <class T> inline Xf<T> inv(const Xf<T>& a) { M3<T> rt = transpose(a.R); return {rt, -(rt * a.p)}; }

// 6-vectors [angular; linear] (spatial/common.jl:13)
template <class T> struct S6 { V3<T> ang, lin; };
template <class T> inline S6<T> operator+(const S6<T>& a, const S6<T>& b) { return {a.ang + b.ang, a.lin + b.lin}; }
template <class T> inline S6<T> operator-(const S6<T>& a, const S6<T>& b) { return {a.ang - b.ang, a.lin - b.lin}; }
template <class T> inline S6<T> operator-(const S6<T>& a) { return {-a.ang, -a.lin}; }
template <class T> inline T dot(const S6<T>& a, const S6<T>& b) { return dot(a.ang, b.ang) + dot(a.lin, b.lin); }

// spatial/util.jl:104-108
template <class T> inline S6<T> transform_spatial_motion(const S6<T>& m, const M3<T>& R, const V3<T>& p) {
  V3<T> ang = R * m.ang;
  V3<T> lin = R * m.lin + cross(p, ang);
  return {ang, lin};
}
// spatial/util.jl:117-121 ("spatial motion cross product")
template <class T> inline S6<T> se3_commutator(const S6<T>& x, const S6<T>& y) {
  return {cross(x.ang, y.ang), cross(x.ang, y.lin) + cross(x.lin, y.ang)};
}

// SpatialInertia (motion_force_interaction.jl:28-37)
template <class T> struct Inertia {
  M3<T> J; V3<T> c; T m;
  Inertia() : J(), c(), m(0) {}
};
template <class T> inline Inertia<T> operator+(const Inertia<T>& a, const Inertia<T>& b) {   // :147-153
  Inertia<T> r; r.J = a.J + b.J; r.c = a.c + b.c; r.m = a.m + b.m; return r;
}
// motion_force_interaction.jl:160-176
template <class T> inline Inertia<T> transform(const Inertia<T>& I, const Xf<T>& t) {
  V3<T> Rmc = t.R * I.c;
  V3<T> mp = I.m * t.p;
  Inertia<T> r;
  r.c = Rmc + mp;
  M3<T> X = outer(Rmc, t.p);
  M3<T> Y = X + transpose(X) + outer(mp, t.p);
  T trY = Y(0, 0) + Y(1, 1) + Y(2, 2);
  r.J = t.R * I.J * transpose(t.R) - Y;
  r.J(0, 0) += trY; r.J(1, 1) += trY; r.J(2, 2) += trY;
  r.m = I.m;
  return r;
}
// spatial/util.jl:110-114
template <class T> inline S6<T> mul_inertia(const Inertia<T>& I, const S6<T>& v) {
  return {I.J * v.ang + cross(I.c, v.lin), I.m * v.lin - cross(I.c, v.ang)};
}
// motion_force_interaction.jl:244-263
template <class T> inline S6<T> newton_euler(const Inertia<T>& I, const S6<T>& accel, const S6<T>& tw) {
  S6<T> w = mul_inertia(I, accel);
  S6<T> h = mul_inertia(I, tw);
  w.ang = w.ang + cross(tw.ang, h.ang) + cross(tw.lin, h.lin);
  w.lin = w.lin + cross(tw.ang, h.lin);
  return w;
}

// ------------------------------------------------------------------------------------------------
// rotations supplied by Rotations.jl in the reference (not in tree; formulas per SURVEY 8(c))
// ------------------------------------------------------------------------------------------------
// AngleAxis -> RotMatrix, element order as restated in-tree at joint_types/sin_cos_revolute.jl:69-96
template <class T> inline M3<T> rot_sincos_axis(T s, T c, const V3<T>& a) {
  T c1 = T(1) - c;
  T c1x2 = c1 * a.x * a.x, c1y2 = c1 * a.y * a.y, c1z2 = c1 * a.z * a.z;
  T c1xy = c1 * a.x * a.y, c1xz = c1 * a.x * a.z, c1yz = c1 * a.y * a.z;
  T sx = s * a.x, sy = s * a.y, sz = s * a.z;
  M3<T> R;
  R(0, 0) = T(1) - c1y2 - c1z2; R(0, 1) = c1xy - sz;          R(0, 2) = c1xz + sy;
  R(1, 0) = c1xy + sz;          R(1, 1) = T(1) - c1x2 - c1z2; R(1, 2) = c1yz - sx;
  R(2, 0) = c1xz - sy;          R(2, 1) = c1yz + sx;          R(2, 2) = T(1) - c1x2 - c1y2;
  return R;
}
template <class T> inline M3<T> rot_quat(T w, T x, T y, T z) {   // no normalisation (quaternion_floating.jl:81-83)
  M3<T> R;
  R(0, 0) = T(1) - T(2) * (y * y + z * z); R(0, 1) = T(2) * (x * y - w * z);        R(0, 2) = T(2) * (x * z + w * y);
  R(1, 0) = T(2) * (x * y + w * z);        R(1, 1) = T(1) - T(2) * (x * x + z * z); R(1, 2) = T(2) * (y * z - w * x);
  R(2, 0) = T(2) * (x * z - w * y);        R(2, 1) = T(2) * (y * z + w * x);        R(2, 2) = T(1) - T(2) * (x * x + y * y);
  return R;
}
template <class T> inline void mrp_to_quat(T x, T y, T z, T q[4]) {
  T n2 = x * x + y * y + z * z;
  T f = T(2) / (T(1) + n2);
  q[0] = (T(1) - n2) / (T(1) + n2); q[1] = f * x; q[2] = f * y; q[3] = f * z;
}

// ------------------------------------------------------------------------------------------------
// model (flattened Mechanism, reference tree-joint order) -- same content as rbd_model_desc
// ------------------------------------------------------------------------------------------------
struct Model {
  int nb = 0, nq = 0, nv = 0;
  std::vector<int> parent, jtype, qstart, vstart;
  std::vector<double> X_tree;    // [nb][12]
  std::vector<double> jparam;    // [nb][9]
  std::vector<double> inertia;   // [nb][13]
  double gravity[3] = {0, 0, -9.81};
  std::vector<int> vjoint;       // [nv] velocity index -> joint
  std::vector<uint8_t> supports; // [nb][nb]: supports[j*nb+i] = joint j is an ancestor-or-self of body i (mechanism_state.jl:588-590)
  void finalize() {
    vjoint.assign(nv, 0);
    for (int i = 0; i < nb; ++i) for (int k = 0; k < joint_nv(jtype[i]); ++k) vjoint[vstart[i] + k] = i;
    supports.assign((size_t)nb * nb, 0);
    for (int i = 0; i < nb; ++i) for (int a = i; a >= 0; a = parent[a]) supports[(size_t)a * nb + i] = 1;
  }
};

template <class T> struct JointConsts {
  Xf<T> X_tree; V3<T> a0, a1, a2; Inertia<T> I;
};

// Per-evaluation workspace = the dirty-flag caches of MechanismState (mechanism_state.jl:35-78), all world frame.
template <class T> struct Workspace {
  const Model* mdl;
  std::vector<JointConsts<T>> jc;
  std::vector<Xf<T>> T_root;                 // transforms_to_root
  std::vector<S6<T>> joint_twist;            // in body frame
  std::vector<S6<T>> twist;                  // twists_wrt_world
  std::vector<S6<T>> bias;                   // bias_accelerations_wrt_world
  std::vector<S6<T>> S;                      // motion_subspaces, one per velocity index
  std::vector<Inertia<T>> Iw, Ic;            // inertias, crb_inertias
  std::vector<S6<T>> accel, wrench, wext;
  std::vector<T> M, L, c, rhs;
  V3<T> g;
  explicit Workspace(const Model& m) : mdl(&m) {
    int nb = m.nb, nv = m.nv;
    jc.resize(nb); T_root.resize(nb); joint_twist.resize(nb); twist.resize(nb); bias.resize(nb);
    S.resize(nv); Iw.resize(nb); Ic.resize(nb); accel.resize(nb); wrench.resize(nb); wext.resize(nb);
    M.resize((size_t)nv * nv); L.resize((size_t)nv * nv); c.resize(nv); rhs.resize(nv);
    for (int i = 0; i < nb; ++i) {
      const double* x = &m.X_tree[12 * i];
      for (int k = 0; k < 9; ++k) jc[i].X_tree.R.m[k] = T(x[k]);
      jc[i].X_tree.p = V3<T>(T(x[9]), T(x[10]), T(x[11]));
      const double* jp = &m.jparam[9 * i];
      jc[i].a0 = V3<T>(T(jp[0]), T(jp[1]), T(jp[2]));
      jc[i].a1 = V3<T>(T(jp[3]), T(jp[4]), T(jp[5]));
      jc[i].a2 = V3<T>(T(jp[6]), T(jp[7]), T(jp[8]));
      const double* in = &m.inertia[13 * i];
      for (int k = 0; k < 9; ++k) jc[i].I.J.m[k] = T(in[k]);
      jc[i].I.c = V3<T>(T(in[9]), T(in[10]), T(in[11]));
      jc[i].I.m = T(in[12]);
    }
    g = V3<T>(T(m.gravity[0]), T(m.gravity[1]), T(m.gravity[2]));
  }
};

// ------------------------------------------------------------------------------------------------
// per-joint-type functions (joint_types/*.jl)
// ------------------------------------------------------------------------------------------------
template <class T> inline Xf<T> joint_transform(int type, const JointConsts<T>& jc, const T* q) {
  using std::sin; using std::cos;
  switch (type) {
    case JT_REVOLUTE: return Xf<T>(rot_sincos_axis(T(sin(q[0])), T(cos(q[0])), jc.a0), V3<T>());      // revolute.jl:59-62
    case JT_PRISMATIC: return Xf<T>(M3<T>::identity(), q[0] * jc.a0);                                  // prismatic.jl:69-73
    case JT_FIXED: return Xf<T>();                                                                     // fixed.jl:18-22
    case JT_PLANAR:                                                                                    // planar.jl:65-70
      return Xf<T>(rot_sincos_axis(T(sin(q[2])), T(cos(q[2])), jc.a2), jc.a0 * q[0] + jc.a1 * q[1]);
    case JT_QUAT_FLOATING: return Xf<T>(rot_quat(q[0], q[1], q[2], q[3]), V3<T>(q[4], q[5], q[6]));   // quaternion_floating.jl:81-83
    case JT_SPQUAT_FLOATING: {                                                                         // spquat_floating.jl:78-81
      T qq[4]; mrp_to_quat(q[0], q[1], q[2], qq);
      return Xf<T>(rot_quat(qq[0], qq[1], qq[2], qq[3]), V3<T>(q[3], q[4], q[5]));
    }
    case JT_QUAT_SPHERICAL: return Xf<T>(rot_quat(q[0], q[1], q[2], q[3]), V3<T>());                   // quaternion_spherical.jl:47-50
    case JT_SINCOS_REVOLUTE: return Xf<T>(rot_sincos_axis(q[0], q[1], jc.a0), V3<T>());                // sin_cos_revolute.jl:69-96
  }
  return Xf<T>();
}

// joint_twist / joint_spatial_acceleration: S_loc * x, x = v or v̇ (e.g. revolute.jl:64-68,76-81)
template <class T> inline S6<T> joint_motion(int type, const JointConsts<T>& jc, const T* x) {
  switch (type) {
    case JT_REVOLUTE: case JT_SINCOS_REVOLUTE: return {jc.a0 * x[0], V3<T>()};
    case JT_PRISMATIC: return {V3<T>(), jc.a0 * x[0]};
    case JT_FIXED: return {V3<T>(), V3<T>()};
    case JT_PLANAR: return {jc.a2 * x[2], jc.a0 * x[0] + jc.a1 * x[1]};                  // planar.jl:72-77
    case JT_QUAT_FLOATING: case JT_SPQUAT_FLOATING: return {V3<T>(x[0], x[1], x[2]), V3<T>(x[3], x[4], x[5])};
    case JT_QUAT_SPHERICAL: return {V3<T>(x[0], x[1], x[2]), V3<T>()};
  }
  return {V3<T>(), V3<T>()};
}

// motion_subspace column k in the frame after the joint (e.g. revolute.jl:83-89, planar.jl:87-93)
template <class T> inline S6<T> subspace_col(int type, const JointConsts<T>& jc, int k) {
  T e[6] = {T(0), T(0), T(0), T(0), T(0), T(0)};
  e[k] = T(1);
  return joint_motion(type, jc, e);
}

// velocity_to_configuration_derivative! per type (q̇ = N(q) v)
template <class T> inline void qdot_joint(int type, const T* q, const T* v, T* qd) {
  using std::sin; using std::cos;
  switch (type) {
    case JT_REVOLUTE: case JT_PRISMATIC: qd[0] = v[0]; break;                             // joint_types.jl:29-32
    case JT_FIXED: break;
    case JT_PLANAR: {                                                                     // planar.jl:123-129
      T s = sin(q[2]), c = cos(q[2]);
      qd[0] = c * v[0] - s * v[1]; qd[1] = s * v[0] + c * v[1]; qd[2] = v[2];
      break;
    }
    case JT_QUAT_FLOATING: case JT_QUAT_SPHERICAL: {                                      // quaternion_floating.jl:126-136, util.jl:127-134
      T w = q[0], x = q[1], y = q[2], z = q[3];
      qd[0] = (-x * v[0] - y * v[1] - z * v[2]) / T(2);
      qd[1] = (w * v[0] - z * v[1] + y * v[2]) / T(2);
      qd[2] = (z * v[0] + w * v[1] - x * v[2]) / T(2);
      qd[3] = (-y * v[0] + x * v[1] + w * v[2]) / T(2);
      if (type == JT_QUAT_FLOATING) {
        V3<T> t = rot_quat(w, x, y, z) * V3<T>(v[3], v[4], v[5]);
        qd[4] = t.x; qd[5] = t.y; qd[6] = t.z;
      }
      break;
    }
    case JT_SPQUAT_FLOATING: {                                                            // spquat_floating.jl:128-138, util.jl:136-141
      T qq[4]; mrp_to_quat(q[0], q[1], q[2], qq);
      T w = qq[0], x = qq[1], y = qq[2], z = qq[3];
      T dq[4];
      dq[0] = (-x * v[0] - y * v[1] - z * v[2]) / T(2);
      dq[1] = (w * v[0] - z * v[1] + y * v[2]) / T(2);
      dq[2] = (z * v[0] + w * v[1] - x * v[2]) / T(2);
      dq[3] = (-y * v[0] + x * v[1] + w * v[2]) / T(2);
      // d/dt [vec/(1+w)]  (jacobian of the MRP w.r.t. the quaternion, Rotations.jacobian)
      T d = T(1) + w;
      qd[0] = dq[1] / d - x * dq[0] / (d * d);
      qd[1] = dq[2] / d - y * dq[0] / (d * d);
      qd[2] = dq[3] / d - z * dq[0] / (d * d);
      V3<T> t = rot_quat(w, x, y, z) * V3<T>(v[3], v[4], v[5]);
      qd[3] = t.x; qd[4] = t.y; qd[5] = t.z;
      break;
    }
    case JT_SINCOS_REVOLUTE: qd[0] = q[1] * v[0]; qd[1] = -q[0] * v[0]; break;            // sin_cos_revolute.jl:160-165
  }
}

// ------------------------------------------------------------------------------------------------
// cache updates (mechanism_state.jl:687-868) -- every call recomputes (setdirty! semantics)
// ------------------------------------------------------------------------------------------------
template <class T> void update_transforms(Workspace<T>& w, const T* q) {           // :687-714
  const Model& m = *w.mdl;
  for (int i = 0; i < m.nb; ++i) {
    Xf<T> J = joint_transform(m.jtype[i], w.jc[i], q + m.qstart[i]);
    int p = m.parent[i];
    if (p < 0) w.T_root[i] = w.jc[i].X_tree * J;     // transforms_to_root[world] = identity
    else w.T_root[i] = (w.T_root[p] * w.jc[i].X_tree) * J;
  }
}
template <class T> void update_twists(Workspace<T>& w, const T* v) {               // :720-726, :769-780
  const Model& m = *w.mdl;
  for (int i = 0; i < m.nb; ++i) {
    w.joint_twist[i] = joint_motion(m.jtype[i], w.jc[i], v + m.vstart[i]);
    S6<T> jw = transform_spatial_motion(w.joint_twist[i], w.T_root[i].R, w.T_root[i].p);
    int p = m.parent[i];
    w.twist[i] = p < 0 ? jw : w.twist[p] + jw;
  }
}
template <class T> void update_bias_accelerations(Workspace<T>& w) {               // :814-830 + spatialmotion.jl:375-401
  const Model& m = *w.mdl;
  for (int i = 0; i < m.nb; ++i) {
    Xf<T> ti = inv(w.T_root[i]);
    S6<T> tw_body = transform_spatial_motion(w.twist[i], ti.R, ti.p);   // twist wrt world, in body frame
    S6<T> cr = se3_commutator(tw_body, w.joint_twist[i]);               // + joint bias (zero for all types)
    S6<T> b = transform_spatial_motion(cr, w.T_root[i].R, w.T_root[i].p);
    int p = m.parent[i];
    w.bias[i] = p < 0 ? b : w.bias[p] + b;
  }
}
template <class T> void update_motion_subspaces(Workspace<T>& w) {                 // :749-763
  const Model& m = *w.mdl;
  for (int i = 0; i < m.nb; ++i)
    for (int k = 0; k < joint_nv(m.jtype[i]); ++k)
      w.S[m.vstart[i] + k] = transform_spatial_motion(subspace_col(m.jtype[i], w.jc[i], k), w.T_root[i].R, w.T_root[i].p);
}
template <class T> void update_spatial_inertias(Workspace<T>& w) {                 // :836-846
  for (int i = 0; i < w.mdl->nb; ++i) w.Iw[i] = transform(w.jc[i].I, w.T_root[i]);
}
template <class T> void update_crb_inertias(Workspace<T>& w) {                     // :852-868
  const Model& m = *w.mdl;
  for (int i = 0; i < m.nb; ++i) w.Ic[i] = w.Iw[i];
  for (int i = m.nb - 1; i >= 0; --i) if (m.parent[i] >= 0) w.Ic[m.parent[i]] = w.Ic[m.parent[i]] + w.Ic[i];
}

// ------------------------------------------------------------------------------------------------
// algorithms (mechanism_algorithms.jl)
// ------------------------------------------------------------------------------------------------
// mass_matrix! :248-272.  Writes the LOWER triangle of column-major M (M[i + j*nv], j <= i) like M.data,
// and mirrors it into the upper triangle for convenience.
template <class T> void mass_matrix(Workspace<T>& w, T* M) {
  const Model& m = *w.mdl;
  int nv = m.nv, nb = m.nb;
  for (int i = 0; i < nv; ++i) {
    int bi = m.vjoint[i];
    S6<T> F = mul_inertia(w.Ic[bi], w.S[i]);       // Ic * S_i  (motion_force_interaction.jl:223-233)
    for (int j = 0; j <= i; ++j) {
      T val = m.supports[(size_t)m.vjoint[j] * nb + bi] ? dot(F, w.S[j]) : T(0);
      M[i + (size_t)j * nv] = val;
      M[j + (size_t)i * nv] = val;
    }
  }
}

// newton_euler! :428-439 followed by joint_wrenches_and_torques! :442-459
template <class T> void wrenches_to_torques(Workspace<T>& w, const T* wext /*[nb][6] or null*/, T* tau) {
  const Model& m = *w.mdl;
  for (int i = 0; i < m.nb; ++i) {
    S6<T> f = newton_euler(w.Iw[i], w.accel[i], w.twist[i]);
    if (wext) {
      f.ang = f.ang - V3<T>(wext[6 * i + 0], wext[6 * i + 1], wext[6 * i + 2]);
      f.lin = f.lin - V3<T>(wext[6 * i + 3], wext[6 * i + 4], wext[6 * i + 5]);
    }
    w.wrench[i] = f;
  }
  for (int i = m.nb - 1; i >= 0; --i) {
    if (m.parent[i] >= 0) w.wrench[m.parent[i]] = w.wrench[m.parent[i]] + w.wrench[i];
    for (int k = 0; k < joint_nv(m.jtype[i]); ++k) tau[m.vstart[i] + k] = dot(w.S[m.vstart[i] + k], w.wrench[i]);
  }
}

template <class T> void update_kinematics(Workspace<T>& w, const T* q, const T* v) {
  update_transforms(w, q);
  update_twists(w, v);
  update_motion_subspaces(w);
  update_spatial_inertias(w);
}

// ------------------------------------------------------------------------------------------------
// kinematics by-products (SURVEY 8(f) rank 2): all world (root) frame, straight from the caches above
// ------------------------------------------------------------------------------------------------
//   transform_to_root             mechanism_state.jl:687-714 (the cache itself)
//   center_of_mass                mechanism_algorithms.jl:30-49
//   kinetic_energy                mechanism_state.jl:886-888, :989-994; motion_force_interaction.jl:337-346
//   gravitational_potential_energy mechanism_state.jl:897-903, :996-1000
//   momentum / momentum_rate_bias mechanism_state.jl:878-884, :975-987
//   momentum_matrix!              mechanism_algorithms.jl:313-327
//   geometric_jacobian!           mechanism_algorithms.jl:80-100 (sign[i] = +1 joint i traversed down, -1 up, 0 not on the path)
template <class T> struct KinOut {
  T* transforms = nullptr;   // [nb][12]: R row-major, p
  T* com = nullptr;          // [3]
  T* ke = nullptr;           // [1]
  T* pe = nullptr;           // [1]
  T* momentum = nullptr;     // [6]
  T* mrb = nullptr;          // [6]
  T* A = nullptr;            // [nv][6]
  T* J = nullptr;            // [nv][6]
};
template <class T> void kinematics(Workspace<T>& w, const T* q, const T* v, const signed char* sign, const KinOut<T>& o) {
  const Model& m = *w.mdl;
  update_transforms(w, q);
  update_motion_subspaces(w);
  update_spatial_inertias(w);
  if (v) { update_twists(w, v); update_bias_accelerations(w); }
  if (o.transforms)
    for (int i = 0; i < m.nb; ++i) {
      for (int k = 0; k < 9; ++k) o.transforms[12 * i + k] = w.T_root[i].R.m[k];
      o.transforms[12 * i + 9] = w.T_root[i].p.x; o.transforms[12 * i + 10] = w.T_root[i].p.y; o.transforms[12 * i + 11] = w.T_root[i].p.z;
    }
  if (o.com || o.pe) {
    V3<T> mc(T(0), T(0), T(0));
    T mass = T(0), pe = T(0);
    for (int i = 0; i < m.nb; ++i) {
      const Inertia<T>& I = w.jc[i].I;
      if (!(I.m > T(0))) continue;
      V3<T> c_body = (T(1) / I.m) * I.c;                                  // center_of_mass(inertia) = cross_part / mass
      V3<T> c_world = w.T_root[i].R * c_body + w.T_root[i].p;
      mc = mc + I.m * c_world;
      mass = mass + I.m;
      pe = pe - I.m * dot(w.g, c_world);
    }
    if (o.com) { V3<T> c = (T(1) / mass) * mc; o.com[0] = c.x; o.com[1] = c.y; o.com[2] = c.z; }
    if (o.pe) o.pe[0] = pe;
  }
  if (v && (o.ke || o.momentum || o.mrb)) {
    T ke = T(0);
    S6<T> h{V3<T>(T(0), T(0), T(0)), V3<T>(T(0), T(0), T(0))}, hb = h;
    for (int i = 0; i < m.nb; ++i) {
      const Inertia<T>& I = w.Iw[i];
      const S6<T>& tw = w.twist[i];
      ke = ke + (dot(tw.ang, I.J * tw.ang) + dot(tw.lin, I.m * tw.lin + T(2) * cross(tw.ang, I.c))) / T(2);
      h = h + mul_inertia(I, tw);
      hb = hb + newton_euler(I, w.bias[i], tw);
    }
    if (o.ke) o.ke[0] = ke;
    if (o.momentum) { for (int k = 0; k < 3; ++k) { o.momentum[k] = h.ang[k]; o.momentum[3 + k] = h.lin[k]; } }
    if (o.mrb) { for (int k = 0; k < 3; ++k) { o.mrb[k] = hb.ang[k]; o.mrb[3 + k] = hb.lin[k]; } }
  }
  if (o.A) {
    update_crb_inertias(w);
    for (int i = 0; i < m.nv; ++i) {
      S6<T> F = mul_inertia(w.Ic[m.vjoint[i]], w.S[i]);
      for (int k = 0; k < 3; ++k) { o.A[6 * i + k] = F.ang[k]; o.A[6 * i + 3 + k] = F.lin[k]; }
    }
  }
  if (o.J) {
    for (int i = 0; i < m.nv; ++i) {
      T sg = sign ? T((int)sign[m.vjoint[i]]) : T(0);
      for (int k = 0; k < 3; ++k) { o.J[6 * i + k] = sg * w.S[i].ang[k]; o.J[6 * i + 3 + k] = sg * w.S[i].lin[k]; }
    }
  }
}

// dynamics_bias! :484-498 (bias_accelerations! :377-385: a_i = -g + b_i)
template <class T> void dynamics_bias(Workspace<T>& w, const T* q, const T* v, const T* wext, T* c) {
  update_kinematics(w, q, v);
  update_bias_accelerations(w);
  S6<T> gb{V3<T>(), -w.g};
  for (int i = 0; i < w.mdl->nb; ++i) w.accel[i] = gb + w.bias[i];
  wrenches_to_torques(w, wext, c);
}

// inverse_dynamics! :542-553 (spatial_accelerations! :387-417)
template <class T> void inverse_dynamics(Workspace<T>& w, const T* q, const T* v, const T* vd, const T* wext, T* tau) {
  const Model& m = *w.mdl;
  update_kinematics(w, q, v);
  S6<T> root{V3<T>(), -w.g};
  for (int i = 0; i < m.nb; ++i) {
    S6<T> ja = joint_motion(m.jtype[i], w.jc[i], vd + m.vstart[i]);
    S6<T> jaw = transform_spatial_motion(ja, w.T_root[i].R, w.T_root[i].p);
    int p = m.parent[i];
    S6<T> ap = p < 0 ? root : w.accel[p];
    S6<T> tp = p < 0 ? S6<T>{V3<T>(), V3<T>()} : w.twist[p];
    w.accel[i] = ap + se3_commutator(-w.twist[i], tp) + jaw;           // :415
  }
  wrenches_to_torques(w, wext, tau);
}

// Cholesky M = L L^T (lower, column-major) and solve: what potrf!/potrs! do at :764, :819
template <class T> bool cholesky_solve(int n, const T* M, T* L, T* x /* in: rhs, out: solution */) {
  using std::sqrt;
  for (int j = 0; j < n; ++j) {
    T d = M[j + (size_t)j * n];
    for (int k = 0; k < j; ++k) d -= L[j + (size_t)k * n] * L[j + (size_t)k * n];
    if (!(d > T(0))) return false;               // PosDefException
    d = sqrt(d);
    L[j + (size_t)j * n] = d;
    for (int i = j + 1; i < n; ++i) {
      T s = M[i + (size_t)j * n];
      for (int k = 0; k < j; ++k) s -= L[i + (size_t)k * n] * L[j + (size_t)k * n];
      L[i + (size_t)j * n] = s / d;
    }
  }
  for (int i = 0; i < n; ++i) {                  // L y = b
    T s = x[i];
    for (int k = 0; k < i; ++k) s -= L[i + (size_t)k * n] * x[k];
    x[i] = s / L[i + (size_t)i * n];
  }
  for (int i = n - 1; i >= 0; --i) {             // L^T x = y
    T s = x[i];
    for (int k = i + 1; k < n; ++k) s -= L[k + (size_t)i * n] * x[k];
    x[i] = s / L[i + (size_t)i * n];
  }
  return true;
}

template <class T> void configuration_derivative(const Model& m, const T* q, const T* v, T* qd) {   // mechanism_state.jl:905-910
  for (int i = 0; i < m.nb; ++i) qdot_joint(m.jtype[i], q + m.qstart[i], v + m.vstart[i], qd + m.qstart[i]);
}

// dynamics! :845-864 (tree, no contact): q̇ ; bias (RNEA) ; M (CRBA) ; Cholesky solve
template <class T> bool dynamics(Workspace<T>& w, const T* q, const T* v, const T* tau, const T* wext, T* vd, T* qd) {
  const Model& m = *w.mdl;
  if (qd) configuration_derivative(m, q, v, qd);
  dynamics_bias(w, q, v, wext, w.c.data());
  update_crb_inertias(w);
  mass_matrix(w, w.M.data());
  for (int i = 0; i < m.nv; ++i) vd[i] = (tau ? tau[i] : T(0)) - w.c[i];
  return cholesky_solve(m.nv, w.M.data(), w.L.data(), vd);
}

// ------------------------------------------------------------------------------------------------
// INDEPENDENT check: world-frame Articulated-Body Algorithm (not in the reference; SURVEY 8(a) note).
// Dense symmetric 6x6 articulated inertias, k x k joint-space blocks solved by Cholesky.
// ------------------------------------------------------------------------------------------------
template <class T> struct Sym6 { T a[6][6]; };

template <class T> bool aba(Workspace<T>& w, const T* q, const T* v, const T* tau, const T* wext, T* vd) {
  const Model& m = *w.mdl;
  int nb = m.nb;
  update_kinematics(w, q, v);
  std::vector<Sym6<T>> IA(nb);
  std::vector<S6<T>> pA(nb), cb(nb);
  std::vector<T> U((size_t)m.nv * 6), Dinv_u(m.nv);
  std::vector<std::vector<T>> Lfac(nb);
  auto to6 = [](const S6<T>& s, T* o) { o[0] = s.ang.x; o[1] = s.ang.y; o[2] = s.ang.z; o[3] = s.lin.x; o[4] = s.lin.y; o[5] = s.lin.z; };
  auto from6 = [](const T* o) { return S6<T>{V3<T>(o[0], o[1], o[2]), V3<T>(o[3], o[4], o[5])}; };
  for (int i = 0; i < nb; ++i) {
    // 6x6 of the world-frame inertia [J c^; c^T m1]
    const Inertia<T>& I = w.Iw[i];
    Sym6<T>& A = IA[i];
    for (int r = 0; r < 6; ++r) for (int c = 0; c < 6; ++c) A.a[r][c] = T(0);
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) A.a[r][c] = I.J(r, c);
    T ch[3][3] = {{T(0), -I.c.z, I.c.y}, {I.c.z, T(0), -I.c.x}, {-I.c.y, I.c.x, T(0)}};
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { A.a[r][3 + c] = ch[r][c]; A.a[3 + c][r] = ch[r][c]; }
    for (int r = 0; r < 3; ++r) A.a[3 + r][3 + r] = I.m;
    // velocity-product acceleration c_i = v_parent x (S_i v_i) (world frame) and bias force
    int p = m.parent[i];
    S6<T> jw = transform_spatial_motion(w.joint_twist[i], w.T_root[i].R, w.T_root[i].p);
    S6<T> tp = p < 0 ? S6<T>{V3<T>(), V3<T>()} : w.twist[p];
    cb[i] = se3_commutator(tp, jw);
    S6<T> h = mul_inertia(I, w.twist[i]);
    S6<T> pf{cross(w.twist[i].ang, h.ang) + cross(w.twist[i].lin, h.lin), cross(w.twist[i].ang, h.lin)};
    if (wext) {
      pf.ang = pf.ang - V3<T>(wext[6 * i], wext[6 * i + 1], wext[6 * i + 2]);
      pf.lin = pf.lin - V3<T>(wext[6 * i + 3], wext[6 * i + 4], wext[6 * i + 5]);
    }
    pA[i] = pf;
  }
  for (int i = nb - 1; i >= 0; --i) {
    int k = joint_nv(m.jtype[i]), vs = m.vstart[i];
    T Sm[6][6], Um[6][6], D[36], pa6[6], c6[6];
    to6(pA[i], pa6); to6(cb[i], c6);
    for (int a = 0; a < k; ++a) to6(w.S[vs + a], Sm[a]);
    for (int a = 0; a < k; ++a) for (int r = 0; r < 6; ++r) {
      T s = T(0);
      for (int c = 0; c < 6; ++c) s += IA[i].a[r][c] * Sm[a][c];
      Um[a][r] = s; U[(size_t)(vs + a) * 6 + r] = s;
    }
    for (int a = 0; a < k; ++a) for (int b = 0; b < k; ++b) {
      T s = T(0);
      for (int r = 0; r < 6; ++r) s += Sm[a][r] * Um[b][r];
      D[a + b * k] = s;
    }
    T u[6];
    for (int a = 0; a < k; ++a) {
      T s = tau ? tau[vs + a] : T(0);
      for (int r = 0; r < 6; ++r) s -= Sm[a][r] * pa6[r];
      u[a] = s;
    }
    Lfac[i].assign((size_t)k * k, T(0));
    // Ia = IA - U D^-1 U^T ; pa = pA + Ia c + U D^-1 u
    T DinvUt[6][6];   // [a][r] = (D^-1 U^T)[a][r]
    for (int r = 0; r < 6; ++r) {
      T col[6];
      for (int a = 0; a < k; ++a) col[a] = Um[a][r];
      if (k > 0 && !cholesky_solve(k, D, Lfac[i].data(), col)) return false;
      for (int a = 0; a < k; ++a) DinvUt[a][r] = col[a];
    }
    T du[6];
    for (int a = 0; a < k; ++a) du[a] = u[a];
    if (k > 0 && !cholesky_solve(k, D, Lfac[i].data(), du)) return false;
    for (int a = 0; a < k; ++a) Dinv_u[vs + a] = du[a];
    int p = m.parent[i];
    if (p >= 0) {
      T Ia[6][6];
      for (int r = 0; r < 6; ++r) for (int c = 0; c < 6; ++c) {
        T s = IA[i].a[r][c];
        for (int a = 0; a < k; ++a) s -= Um[a][r] * DinvUt[a][c];
        Ia[r][c] = s;
      }
      T pa[6];
      for (int r = 0; r < 6; ++r) {
        T s = pa6[r];
        for (int c = 0; c < 6; ++c) s += Ia[r][c] * c6[c];
        for (int a = 0; a < k; ++a) s += Um[a][r] * du[a];
        pa[r] = s;
      }
      for (int r = 0; r < 6; ++r) for (int c = 0; c < 6; ++c) IA[p].a[r][c] += Ia[r][c];
      pA[p] = pA[p] + from6(pa);
    }
    // keep D^-1 U^T rows for the outward pass in U (overwrite): U <- D^-1 U^T
    for (int a = 0; a < k; ++a) for (int r = 0; r < 6; ++r) U[(size_t)(vs + a) * 6 + r] = DinvUt[a][r];
  }
  S6<T> root{V3<T>(), -w.g};
  for (int i = 0; i < nb; ++i) {
    int k = joint_nv(m.jtype[i]), vs = m.vstart[i], p = m.parent[i];
    S6<T> ap = (p < 0 ? root : w.accel[p]) + cb[i];
    T a6[6]; to6(ap, a6);
    S6<T> a = ap;
    for (int j = 0; j < k; ++j) {
      T s = Dinv_u[vs + j];
      for (int r = 0; r < 6; ++r) s -= U[(size_t)(vs + j) * 6 + r] * a6[r];
      vd[vs + j] = s;
      a.ang = a.ang + w.S[vs + j].ang * s;
      a.lin = a.lin + w.S[vs + j].lin * s;
    }
    w.accel[i] = a;
  }
  return true;
}


// ------------------------------------------------------------------------------------------------
// MuntheKaasIntegrator step with the RK4 tableau (ode_integrators.jl:48-55, 233-300) around dynamics(),
// local / global coordinates per joint type with the reference's own closed forms (no series expansions).
// ------------------------------------------------------------------------------------------------
inline void o_quat_mul(const double* a, const double* b, double* o) {
  o[0] = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  o[1] = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  o[2] = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
  o[3] = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
}
inline void o_rotvec_to_quat(const V3<double>& r, double* q) {
  double th = std::sqrt(dot(r, r));
  if (th < 1e-300) { q[0] = 1; q[1] = q[2] = q[3] = 0; return; }
  double s = std::sin(th / 2) / th;
  q[0] = std::cos(th / 2); q[1] = s * r.x; q[2] = s * r.y; q[3] = s * r.z;
}
inline V3<double> o_quat_to_rotvec(const double* qin, double& th) {      // angle in [0, pi]
  double q[4] = {qin[0], qin[1], qin[2], qin[3]};
  if (q[0] < 0) for (double& c : q) c = -c;
  double sn = std::sqrt(q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  th = 2 * std::atan2(sn, q[0]);
  if (sn < 1e-300) return V3<double>();
  double k = th / sn;
  return V3<double>(k * q[1], k * q[2], k * q[3]);
}
// exp(::Twist) spatialmotion.jl:306-326 -> (relative quaternion, translation)
inline void o_se3_exp(const V3<double>& pr, const V3<double>& pt, double* dq, V3<double>& tr) {
  double th = std::sqrt(dot(pr, pr));
  o_rotvec_to_quat(pr, dq);
  if (std::fabs(std::remainder(th, 2 * M_PI)) < 2.220446049250313e-16) { tr = pt; return; }
  V3<double> w = pr * (1 / th), v = pt * (1 / th);
  M3<double> R = rot_quat(dq[0], dq[1], dq[2], dq[3]);
  V3<double> t = cross(w, v);
  t = t - R * t;
  tr = t + w * (dot(w, v) * th);
}
// log_with_time_derivative spatialmotion.jl:262-300 (+ _log :226-252): rate of the exponential coordinates
inline void o_se3_log_rate(const double* dq, const V3<double>& p, const V3<double>& w, const V3<double>& v, double* rate) {
  double th;
  V3<double> psi = o_quat_to_rotvec(dq, th);
  double th2 = th * th, h = th / 2, sh = std::sin(h), ch = std::cos(h);
  V3<double> qq = p;
  bool small = std::fabs(std::remainder(th, 2 * M_PI)) < 2.220446049250313e-16;
  double alpha = 1;
  if (!small) {
    alpha = h * ch / sh;
    qq = p - cross(psi, p) * 0.5 + cross(psi, cross(psi, p)) * ((1 - alpha) / th2);
  }
  S6<double> X{psi, qq}, V{w, v}, Xd = V;
  if (!small) {
    double beta = h * h / (sh * sh);
    double A = (2 * (1 - alpha) + (alpha - beta) / 2) / th2;
    double B = ((1 - alpha) + (alpha - beta) / 2) / (th2 * th2);
    S6<double> a1 = se3_commutator(X, V), a2 = se3_commutator(X, a1), a3 = se3_commutator(X, a2), a4 = se3_commutator(X, a3);
    Xd.ang = V.ang + a1.ang * 0.5 + a2.ang * A + a4.ang * B;
    Xd.lin = V.lin + a1.lin * 0.5 + a2.lin * A + a4.lin * B;
  }
  rate[0] = Xd.ang.x; rate[1] = Xd.ang.y; rate[2] = Xd.ang.z; rate[3] = Xd.lin.x; rate[4] = Xd.lin.y; rate[5] = Xd.lin.z;
}

inline void o_global_coordinates(const Model& m, const double* q0, const double* phi, double* q) {
  for (int i = 0; i < m.nb; ++i) {
    const double* a = q0 + m.qstart[i];
    const double* f = phi + m.vstart[i];
    double* o = q + m.qstart[i];
    switch (m.jtype[i]) {
      case JT_QUAT_FLOATING: {                       // quaternion_floating.jl:233-249
        double dq[4]; V3<double> tr;
        o_se3_exp(V3<double>(f[0], f[1], f[2]), V3<double>(f[3], f[4], f[5]), dq, tr);
        o_quat_mul(a, dq, o);
        V3<double> t = rot_quat(a[0], a[1], a[2], a[3]) * tr;
        o[4] = a[4] + t.x; o[5] = a[5] + t.y; o[6] = a[6] + t.z;
        break;
      }
      case JT_QUAT_SPHERICAL: {                      // quaternion_spherical.jl:149-154
        double dq[4];
        o_rotvec_to_quat(V3<double>(f[0], f[1], f[2]), dq);
        o_quat_mul(a, dq, o);
        break;
      }
      case JT_SINCOS_REVOLUTE: {                     // sin_cos_revolute.jl:186-196
        double s = std::sin(f[0]), c = std::cos(f[0]);
        o[0] = a[0] * c + a[1] * s; o[1] = a[1] * c - a[0] * s;
        break;
      }
      default:                                       // joint_types.jl:16-18
        for (int k = 0; k < joint_nq(m.jtype[i]); ++k) o[k] = a[k] + f[k];
    }
  }
}
inline void o_local_rate(const Model& m, const double* q0, const double* q, const double* v, double* phid) {
  for (int i = 0; i < m.nb; ++i) {
    const double* a = q0 + m.qstart[i];
    const double* b = q + m.qstart[i];
    const double* w = v + m.vstart[i];
    double* o = phid + m.vstart[i];
    switch (m.jtype[i]) {
      case JT_QUAT_FLOATING: {                       // quaternion_floating.jl:205-231
        double ac[4] = {a[0], -a[1], -a[2], -a[3]}, dq[4];
        o_quat_mul(ac, b, dq);
        V3<double> dp = transpose(rot_quat(a[0], a[1], a[2], a[3])) * V3<double>(b[4] - a[4], b[5] - a[5], b[6] - a[6]);
        o_se3_log_rate(dq, dp, V3<double>(w[0], w[1], w[2]), V3<double>(w[3], w[4], w[5]), o);
        break;
      }
      case JT_QUAT_SPHERICAL: {                      // quaternion_spherical.jl:139-147, util.jl:83-101
        double ac[4] = {a[0], -a[1], -a[2], -a[3]}, dq[4], th;
        o_quat_mul(ac, b, dq);
        V3<double> phi = o_quat_to_rotvec(dq, th), om(w[0], w[1], w[2]);
        V3<double> r = om + cross(phi, om) * 0.5;
        if (th > 2.220446049250313e-16) {
          double s = std::sin(th), c = std::cos(th);
          r = r + cross(phi, cross(phi, om)) * (1 / (th * th) * (1 - (th * s) / (2 * (1 - c))));
        }
        o[0] = r.x; o[1] = r.y; o[2] = r.z;
        break;
      }
      case JT_SINCOS_REVOLUTE: o[0] = w[0]; break;   // sin_cos_revolute.jl:173-184
      default: qdot_joint(m.jtype[i], b, w, o);      // joint_types.jl:9-14: phi_dot = q̇ (nq == nv for these types)
    }
  }
}
// one RK4 Munthe-Kaas step with constant torques (zero-order hold); q, v updated in place
inline bool integrate_step(Workspace<double>& w, double* q, double* v, const double* tau, double dt) {
  const Model& m = *w.mdl;
  const double a[4] = {0, 0.5, 0.5, 1.0}, b[4] = {1.0 / 6, 1.0 / 3, 1.0 / 3, 1.0 / 6};
  std::vector<double> q0(q, q + m.nq), v0(v, v + m.nv), qs(m.nq), vs(m.nv), phi(m.nv);
  std::vector<std::vector<double>> phid(4, std::vector<double>(m.nv)), vd(4, std::vector<double>(m.nv));
  for (int i = 0; i < 4; ++i) {
    for (int k = 0; k < m.nv; ++k) {
      phi[k] = i ? dt * a[i] * phid[i - 1][k] : 0.0;
      vs[k] = v0[k] + (i ? dt * a[i] * vd[i - 1][k] : 0.0);
    }
    o_global_coordinates(m, q0.data(), phi.data(), qs.data());
    if (!dynamics(w, qs.data(), vs.data(), tau, (const double*)nullptr, vd[i].data(), (double*)nullptr)) return false;
    o_local_rate(m, q0.data(), qs.data(), vs.data(), phid[i].data());
  }
  for (int k = 0; k < m.nv; ++k) {
    phi[k] = 0; v[k] = v0[k];
    for (int i = 0; i < 4; ++i) { phi[k] += dt * b[i] * phid[i][k]; v[k] += dt * b[i] * vd[i][k]; }
  }
  o_global_coordinates(m, q0.data(), phi.data(), q);
  return true;
}

}  // namespace rbdo
