// Reverse mode of the whole-body kinematics (rbd_kinematics_vjp, DESIGN 4.23): for cotangents ȳ on any subset of the eight outputs
// of rbd_kinematics (rbd_kin.cuh), the product  L = Σ ȳ . y  differentiated w.r.t. q and v, one thread per sample, O(nb + size of
// the cotangents) -- no nv x nv object.  Every forward quantity is recomputed from (q, v).
//
// Derivation: the scheme of rbd_task_adjoint.cuh (DESIGN 4.20), every body a "named" body.  ROOT-frame quantities: X_i pose, S_k
// world-frame subspace column, v_i twist, a_i = a_p + v_p x (S v) the bias acceleration (v̇ = 0, no gravity: momentum_rate_bias's),
// I_i the body's inertia in the root frame, mc_i = R_i h_i + m_i p_i its mass moment.  L is pulled back onto the three covectors per
// body of that scheme (f_i pose, t_i twist, α_i acceleration), using that a rigid motion δ of body i alone changes
// I_i by  δ x* I_i - I_i δx  and the identities (a x b) . f = -b . (a x* f) = a . (b x* f):
//   transforms_to_root  (R̄, p̄) in the caller's body frame, Ro = R_i At_i the output rotation:
//                       f_i += (ax(G) + p_i x p̄, p̄),  G = R̄ Ro^T    (the transform term of rbd_task_adjoint.cuh with base = root)
//   center_of_mass c̄, gravitational_potential_energy ē:
//                       f_i += (mc_i x c, m_i c),  c = c̄ / m - ē g
//   kinetic_energy k̄:   t_i += k̄ I_i v_i,  f_i -= k̄ v_i x* I_i v_i
//   momentum h̄:         t_i += I_i h̄,      f_i -= h̄ x* I_i v_i + v_i x* I_i h̄
//   momentum_rate_bias m̄ (Σ I_i a_i + v_i x* I_i v_i), u = v_i x m̄:
//                       α_i += I_i m̄,  t_i += I_i (m̄ x v_i) - m̄ x* I_i v_i,
//                       f_i += u x* I_i v_i + v_i x* I_i u - m̄ x* I_i a_i - a_i x* I_i m̄
//   geometric_jacobian  J_k = s_k S_k (s the path sign, columns with s = 0 are not read): the column term S_k x* (s_k J̄_k) on the
//                       column's body (moving coordinate j rotates S_k with the subtree: δS_k = S_j x S_k)
//   momentum_matrix     A_k = Ic_{b(k)} S_k, Ic symmetric, so Ā_k . A_k = (Ic_{b(k)} Ā_k) . S_k = Σ_{i in sub(b(k))} Ā_k . I_i S_k:
//                       the column term S_k x* (Ic_{b(k)} Ā_k) on the column's body, and on every body i
//                       f_i -= Σ_{k on the path root -> i} (Ā_k x* I_i S_k + S_k x* I_i Ā_k) = Σ_c H_i[:, c] x* (I_i e_c),
//                       H_i = Σ_{k on the path} (Ā_k S_k^T + S_k Ā_k^T), symmetric 6 x 6, accumulated along the path
// The inward sweep is rbd_task_adjoint.cuh's: A_J = Σ α_i, T_J = Σ (t_i + v_i x* α_i), W_J = Σ (f_i + v_i x* t_i + a_i x* α_i) +
// Σ_columns S_k x* φ_k over the subtree, and task_joint_adjoint forms v̄_j = S_j . T_J + Sdp_j . A_J and q̄_j = S_j . W_J + Ψ̇_j . T_J +
// Ψ̈_j . A_J, q̄_cfg through cfg_adjoint.
//
// Work split: one thread per sample.  Outward sweep: pose, twist and bias acceleration of every body into its workspace rows; the
// body's covectors formed on the spot and folded into its sums A, T, W; with a momentum-matrix cotangent also I_i into the body's
// composite-inertia rows and H along the path (the parent's H is the carry row block for a first child, a pending slot otherwise, as
// the forward sweeps park the pose).  Inward sweep (reverse preorder): composite inertias completed as one more subtree sum, the
// momentum-matrix column terms, the coordinate adjoints, the sums handed to the parent.  Twists and bias accelerations are formed only
// with a kinetic_energy, momentum or momentum_rate_bias cotangent; H and composite inertias only with a momentum_matrix cotangent.
// Workspace per sample (kin_adjoint_rows): kTaskAdjRows rows per body, plus with a momentum-matrix cotangent kKinAdjIcRows per body and
// kKinAdjHRows for the carry and for each pending slot.
#pragma once
#include "rbd_task_adjoint.cuh"

namespace rbd {

constexpr int kKinAdjIcRows = 10;     // composite inertia m, h, J of a body
constexpr int kKinAdjHRows = 21;      // H: the upper triangle of a symmetric 6 x 6

inline int kin_adjoint_rows(int nb, int nslots, bool mm) {
  return kTaskAdjRows * nb + (mm ? kKinAdjIcRows * nb + kKinAdjHRows * (nslots + 1) : 0);
}

// row of entry (a, b) of a symmetric 6 x 6 in its upper-triangle layout
RBD_HD constexpr int sym6(int a, int b) { return a <= b ? a * (11 - a) / 2 + b : b * (11 - b) / 2 + a; }

template <class T> struct KinBarIO {
  Col<T> q, v;                           // v may be invalid when no velocity-dependent cotangent is given
  Col<T> tr, com, ke, pe, mom, mrb, A, J;   // cotangents in the layout of rbd_kinematics_out; invalid = zero
  ColOut<T> qt, qc, vb;                  // q̄_tan [nv], q̄_cfg [nq], v̄ [nv]; each may be invalid
  Scr<T> s;                              // this thread's workspace column
};

// component c (0..5 of [w; l]) of a motion vector, c a compile-time constant after unrolling
template <class T> RBD_HD T mot_comp(const Mot<T>& m, int c) { return c < 3 ? m.w[c] : m.l[c - 3]; }

template <class T>
RBD_HD void kin_vjp_sample(const ModelDev<T>& M, const KinDev<T>& K, const KinBarIO<T>& io) {
  const int nb = M.nb;
  const ScrStash<T> w{io.s};
  const bool want_vel = io.ke.valid() || io.mom.valid() || io.mrb.valid();
  const bool mm = io.A.valid();
  const bool want_q = io.qt.valid() || io.qc.valid();
  const int ic_base = kTaskAdjRows * nb, h_base = ic_base + kKinAdjIcRows * nb;   // composite inertias, H carry, H pending slots

  // ---- outward: pose, twist, bias acceleration; every body's covectors folded into its sums ----
  Pose<T> cur;
  Mot<T> vc, ac;
  for (int i = 0; i < nb; ++i) {
    const BodyDev<T>& bd = M.body[i];
    Pose<T> pp;
    Mot<T> vp, ap;
    if (bd.flags & F_ROOT_CHILD) {
      pose_identity(pp);
#pragma unroll
      for (int k = 0; k < 3; ++k) vp.w[k] = vp.l[k] = ap.w[k] = ap.l[k] = T(0);
    } else if (bd.flags & F_FIRST_CHILD) {
      pp = cur; vp = vc; ap = ac;
    } else {
      const int row = kTaskAdjRows * bd.parent;
#pragma unroll
      for (int k = 0; k < 9; ++k) pp.R[k] = w.ld(row + k);
#pragma unroll
      for (int k = 0; k < 3; ++k) pp.p[k] = w.ld(row + 9 + k);
      if (want_vel) { ld_mot(io.s, row + kTaV, vp); ld_mot(io.s, row + kTaA, ap); }
    }
    T R[9], r[3], t3[3];
    frame_any(bd, io.q, R, r);
    Pose<T> X;
    mat_mul3(pp.R, R, X.R);
    mat_vec(pp.R, r, t3);
    X.p[0] = pp.p[0] + t3[0]; X.p[1] = pp.p[1] + t3[1]; X.p[2] = pp.p[2] + t3[2];
    const int nvj = kind_nv_dev(bd.kind);
    Mot<T> v = vp, a = ap;
    if (want_vel) {
      Mot<T> jt, cm;
#pragma unroll
      for (int k = 0; k < 3; ++k) jt.w[k] = jt.l[k] = T(0);
      for (int k = 0; k < nvj; ++k) {
        Mot<T> S;
        world_subspace(X, sub_comp(bd.kind, k), S);
        const T x = io.v(bd.vrow + k);
#pragma unroll
        for (int c = 0; c < 3; ++c) { jt.w[c] += x * S.w[c]; jt.l[c] += x * S.l[c]; }
      }
      motion_cross(vp, jt, cm);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        v.w[k] = vp.w[k] + jt.w[k]; v.l[k] = vp.l[k] + jt.l[k];
        a.w[k] = ap.w[k] + cm.w[k]; a.l[k] = ap.l[k] + cm.l[k];
      }
    }
    const int row = kTaskAdjRows * i;
#pragma unroll
    for (int k = 0; k < 9; ++k) w.st(row + k, X.R[k]);
#pragma unroll
    for (int k = 0; k < 3; ++k) w.st(row + 9 + k, X.p[k]);
    if (want_vel) { st_mot(io.s, row + kTaV, v); st_mot(io.s, row + kTaA, a); }

    T fn[3] = {T(0), T(0), T(0)}, ff[3] = {T(0), T(0), T(0)};     // f_i
    T tn[3] = {T(0), T(0), T(0)}, tf[3] = {T(0), T(0), T(0)};     // t_i
    T an[3] = {T(0), T(0), T(0)}, af[3] = {T(0), T(0), T(0)};     // α_i
    if (io.tr.valid()) {
      T Ro[9], Rb[9], G[9], pb[3], x[3];
      mat_mul3(X.R, K.At[i], Ro);
      const int trow = 12 * bd.refidx;
#pragma unroll
      for (int k = 0; k < 9; ++k) Rb[k] = io.tr(trow + k);
#pragma unroll
      for (int k = 0; k < 3; ++k) pb[k] = io.tr(trow + 9 + k);
#pragma unroll
      for (int r0 = 0; r0 < 3; ++r0)
#pragma unroll
        for (int c0 = 0; c0 < 3; ++c0)
          G[3 * r0 + c0] = Rb[3 * r0] * Ro[3 * c0] + Rb[3 * r0 + 1] * Ro[3 * c0 + 1] + Rb[3 * r0 + 2] * Ro[3 * c0 + 2];
      cross3(X.p, pb, x);
      fn[0] += G[7] - G[5] + x[0]; fn[1] += G[2] - G[6] + x[1]; fn[2] += G[3] - G[1] + x[2];
#pragma unroll
      for (int k = 0; k < 3; ++k) ff[k] += pb[k];
    }
    if (io.com.valid() || io.pe.valid()) {
      T c[3] = {T(0), T(0), T(0)}, mc[3], Rh[3], x[3];
      if (io.com.valid()) {
#pragma unroll
        for (int k = 0; k < 3; ++k) c[k] = io.com(k) * K.inv_mass;
      }
      if (io.pe.valid()) {
        const T e = io.pe(0);
#pragma unroll
        for (int k = 0; k < 3; ++k) c[k] -= e * M.g[k];
      }
      mat_vec(X.R, bd.h, Rh);
#pragma unroll
      for (int k = 0; k < 3; ++k) mc[k] = Rh[k] + bd.m * X.p[k];
      cross3(mc, c, x);
#pragma unroll
      for (int k = 0; k < 3; ++k) { fn[k] += x[k]; ff[k] += bd.m * c[k]; }
    }
    Rbi<T> Iw;
    if (want_vel || mm) {
      Rbi<T> Ib;
      body_rbi(bd, Ib);
      rbi_to_parent(X.R, X.p, Ib, Iw);
    }
    if (want_vel) {
      T hn[3], hf[3];                    // I v
      rbi_mul(Iw, v, hn, hf);
      if (io.ke.valid()) {
        const T k_ = io.ke(0);
#pragma unroll
        for (int k = 0; k < 3; ++k) { tn[k] += k_ * hn[k]; tf[k] += k_ * hf[k]; }
        task_fcross_add(v, hn, hf, -k_, fn, ff);
      }
      if (io.mom.valid()) {
        Mot<T> hb;
        T yn[3], yf[3];                  // I h̄
#pragma unroll
        for (int k = 0; k < 3; ++k) { hb.w[k] = io.mom(k); hb.l[k] = io.mom(3 + k); }
        rbi_mul(Iw, hb, yn, yf);
#pragma unroll
        for (int k = 0; k < 3; ++k) { tn[k] += yn[k]; tf[k] += yf[k]; }
        task_fcross_add(hb, hn, hf, T(-1), fn, ff);
        task_fcross_add(v, yn, yf, T(-1), fn, ff);
      }
      if (io.mrb.valid()) {
        Mot<T> mb, u, mv;
        T yn[3], yf[3], zn[3], zf[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) { mb.w[k] = io.mrb(k); mb.l[k] = io.mrb(3 + k); }
        rbi_mul(Iw, mb, yn, yf);         // α += I m̄
#pragma unroll
        for (int k = 0; k < 3; ++k) { an[k] += yn[k]; af[k] += yf[k]; }
        task_fcross_add(a, yn, yf, T(-1), fn, ff);      // f -= a x* I m̄
        motion_cross(mb, v, mv);         // t += I (m̄ x v) - m̄ x* I v
        rbi_mul(Iw, mv, zn, zf);
#pragma unroll
        for (int k = 0; k < 3; ++k) { tn[k] += zn[k]; tf[k] += zf[k]; }
        task_fcross_add(mb, hn, hf, T(-1), tn, tf);
        motion_cross(v, mb, u);          // f += u x* I v + v x* I u,  u = v x m̄
        task_fcross_add(u, hn, hf, T(1), fn, ff);
        rbi_mul(Iw, u, zn, zf);
        task_fcross_add(v, zn, zf, T(1), fn, ff);
        rbi_mul(Iw, a, zn, zf);          // f -= m̄ x* I a
        task_fcross_add(mb, zn, zf, T(-1), fn, ff);
      }
    }
    // sums of this body: A = α, T = t + v x* α, W = f + v x* t + a x* α + column terms
    if (want_vel) {
      task_fcross_add(v, tn, tf, T(1), fn, ff);
      task_fcross_add(a, an, af, T(1), fn, ff);
      task_fcross_add(v, an, af, T(1), tn, tf);
    }
    if (io.J.valid() && K.sign[i] != 0) {                 // column terms S_k x* (s J̄_k)
      const T sg = T((int)K.sign[i]);
      for (int k = 0; k < nvj; ++k) {
        Mot<T> S;
        world_subspace(X, sub_comp(bd.kind, k), S);
        const int jrow = 6 * (bd.vrow + k);
        T jn[3], jf[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) { jn[c] = io.J(jrow + c); jf[c] = io.J(jrow + 3 + c); }
        task_fcross_add(S, jn, jf, sg, fn, ff);
      }
    }
    if (mm) {
      T H[21];
      if (bd.flags & F_ROOT_CHILD) {
#pragma unroll
        for (int k = 0; k < 21; ++k) H[k] = T(0);
      } else {
        const int prow = (bd.flags & F_FIRST_CHILD) ? h_base : h_base + kKinAdjHRows * (1 + bd.pslot);
#pragma unroll
        for (int k = 0; k < 21; ++k) H[k] = w.ld(prow + k);
      }
      for (int k = 0; k < nvj; ++k) {    // H += Ā_k S_k^T + S_k Ā_k^T
        Mot<T> S, Ab;
        world_subspace(X, sub_comp(bd.kind, k), S);
        const int arow = 6 * (bd.vrow + k);
#pragma unroll
        for (int c = 0; c < 3; ++c) { Ab.w[c] = io.A(arow + c); Ab.l[c] = io.A(arow + 3 + c); }
#pragma unroll
        for (int r0 = 0; r0 < 6; ++r0)
#pragma unroll
          for (int c0 = r0; c0 < 6; ++c0)
            H[sym6(r0, c0)] += mot_comp(Ab, r0) * mot_comp(S, c0) + mot_comp(S, r0) * mot_comp(Ab, c0);
      }
#pragma unroll
      for (int k = 0; k < 21; ++k) w.st(h_base + k, H[k]);
      if (bd.flags & F_HAS_PENDING) {
#pragma unroll
        for (int k = 0; k < 21; ++k) w.st(h_base + kKinAdjHRows * (1 + bd.oslot) + k, H[k]);
      }
#pragma unroll
      for (int c0 = 0; c0 < 6; ++c0) {   // f -= Σ_c H[:, c] x* (I e_c)
        Mot<T> e, hc;
        T yn[3], yf[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
          e.w[d] = c0 == d ? T(1) : T(0); e.l[d] = c0 == 3 + d ? T(1) : T(0);
          hc.w[d] = H[sym6(d, c0)]; hc.l[d] = H[sym6(3 + d, c0)];
        }
        rbi_mul(Iw, e, yn, yf);
        task_fcross_add(hc, yn, yf, T(-1), fn, ff);
      }
      const int irow = ic_base + kKinAdjIcRows * i;      // composite inertia: this body's, children add theirs inward
      w.st(irow, Iw.m);
#pragma unroll
      for (int k = 0; k < 3; ++k) w.st(irow + 1 + k, Iw.h[k]);
#pragma unroll
      for (int k = 0; k < 6; ++k) w.st(irow + 4 + k, Iw.J[k]);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      w.st(row + kTaSA + k, an[k]); w.st(row + kTaSA + 3 + k, af[k]);
      w.st(row + kTaST + k, tn[k]); w.st(row + kTaST + 3 + k, tf[k]);
      w.st(row + kTaSW + k, fn[k]); w.st(row + kTaSW + 3 + k, ff[k]);
    }
    cur = X; vc = v; ac = a;
  }

  // ---- inward: composite inertias, momentum-matrix column terms, coordinate adjoints, sums handed to the parent ----
  for (int i = nb - 1; i >= 0; --i) {
    const BodyDev<T>& bd = M.body[i];
    const int row = kTaskAdjRows * i;
    T A[6], Tt[6], W[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) { A[k] = w.ld(row + kTaSA + k); Tt[k] = w.ld(row + kTaST + k); W[k] = w.ld(row + kTaSW + k); }
    Mot<T> vi;
    if (want_vel) ld_mot(io.s, row + kTaV, vi);
    if (mm) {
      const int irow = ic_base + kKinAdjIcRows * i;
      Rbi<T> Ic;
      Ic.m = w.ld(irow);
#pragma unroll
      for (int k = 0; k < 3; ++k) Ic.h[k] = w.ld(irow + 1 + k);
#pragma unroll
      for (int k = 0; k < 6; ++k) Ic.J[k] = w.ld(irow + 4 + k);
      const int nvj = kind_nv_dev(bd.kind);
      if (nvj > 0) {
        Pose<T> X;
#pragma unroll
        for (int k = 0; k < 9; ++k) X.R[k] = w.ld(row + k);
#pragma unroll
        for (int k = 0; k < 3; ++k) X.p[k] = w.ld(row + 9 + k);
        for (int k = 0; k < nvj; ++k) {  // W += S_k x* (Ic Ā_k)
          Mot<T> S, Ab;
          world_subspace(X, sub_comp(bd.kind, k), S);
          const int arow = 6 * (bd.vrow + k);
#pragma unroll
          for (int c = 0; c < 3; ++c) { Ab.w[c] = io.A(arow + c); Ab.l[c] = io.A(arow + 3 + c); }
          T yn[3], yf[3];
          rbi_mul(Ic, Ab, yn, yf);
          task_fcross_add(S, yn, yf, T(1), W, W + 3);
        }
      }
      if (!(bd.flags & F_ROOT_CHILD)) {
        const int prow = ic_base + kKinAdjIcRows * bd.parent;
        w.add(prow, Ic.m);
#pragma unroll
        for (int k = 0; k < 3; ++k) w.add(prow + 1 + k, Ic.h[k]);
#pragma unroll
        for (int k = 0; k < 6; ++k) w.add(prow + 4 + k, Ic.J[k]);
      }
    }
    task_joint_adjoint(bd, io.s, row, A, Tt, W, vi, want_vel, want_vel, want_q, io.q, io.qt, io.qc, io.vb, ColOut<T>{nullptr, 0, false});
    if (bd.flags & F_ROOT_CHILD) continue;
    const int prow = kTaskAdjRows * bd.parent;
#pragma unroll
    for (int k = 0; k < 6; ++k) { w.add(prow + kTaSA + k, A[k]); w.add(prow + kTaST + k, Tt[k]); w.add(prow + kTaSW + k, W[k]); }
  }
}

// Host side: KinDev for rbd_kinematics' arguments (path_sign: nb entries in tree-joint order, or NULL)
template <class T> inline void build_kin_dev(const HostModel& hm, const int8_t* path_sign, KinDev<T>& K) {
  std::memset(&K, 0, sizeof(K));
  for (int p = 0; p < hm.nb; ++p) {
    for (int k = 0; k < 9; ++k) K.At[p][k] = (T)hm.alignT[9 * p + k];
    K.sign[p] = path_sign ? path_sign[hm.order[p]] : 0;
  }
  K.inv_mass = (T)(1.0 / hm.total_mass);
}

}  // namespace rbd
