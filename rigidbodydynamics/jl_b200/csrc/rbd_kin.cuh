// Per-sample kinematics by-products in the ROOT frame (SURVEY 8(f) rank 2), one thread per sample, same depth-first order,
// register hand-over and pending slots as the dynamics passes.  Reference (relative to the reference's src/):
//   transform_to_root               mechanism_state.jl:687-714      T_i = T_parent * joint_to_predecessor_i * J_i(q_i)
//   center_of_mass                  mechanism_algorithms.jl:30-49
//   kinetic_energy                  mechanism_state.jl:886-888, :989-994 ; spatial/motion_force_interaction.jl:337-346
//   gravitational_potential_energy  mechanism_state.jl:897-903, :996-1000
//   momentum, momentum_rate_bias    mechanism_state.jl:878-884, :975-987
//   momentum_matrix!                mechanism_algorithms.jl:313-327   A[:, k] = Ic_{body(k)} S_k
//   geometric_jacobian!             mechanism_algorithms.jl:80-100    J[:, k] = +-S_k for the joints on a tree path
// The kernels keep body frames canonicalised (rbd_model.cpp); every quantity written here is expressed in the root frame,
// which does not depend on that choice, except transform_to_root itself, which is mapped back to the caller's body frames
// with the per-body alignment rotation kept in KinDev.
#pragma once
#include <cmath>
#include <cstring>

#include "../../../include/rbd_b200.h"
#include "rbd_rnea_crba.cuh"

namespace rbd {

constexpr int kSlotRowsKin = 24;   // pose (12) + twist (6) + bias acceleration (6) of a branch node; 10 for the inward sweep

template <class T> struct KinDev {
  T At[kMaxBodies][9];         // preorder position -> A_i^T (canonical body frame <- caller's body frame), row-major
  T inv_mass;                  // 1 / total mass
  int8_t sign[kMaxBodies];     // preorder position -> +1 / -1 / 0: joint's direction on the jacobian path
};

template <class T> struct KinIO {
  Col<T> q, v;                 // v may be invalid when no velocity-dependent output is requested
  ColOut<T> tr, com, ke, pe, mom, mrb, A, J;
  Scr<T> poses;                // [12 nb] rows per resident thread, only for the momentum matrix
};

// column c (0..2) of a row-major 3x3 with a warp-uniform runtime c
template <class T> RBD_HD void mat_col(const T* R, int c, T* o) {
#pragma unroll
  for (int j = 0; j < 3; ++j) o[j] = c == 0 ? R[3 * j] : (c == 1 ? R[3 * j + 1] : R[3 * j + 2]);
}

// world-frame motion subspace column driven by one-hot body-frame component `comp` of [w; l]   (:749-763)
template <class T> RBD_HD void world_subspace(const Pose<T>& w, int comp, Mot<T>& S) {
  T ax[3];
  mat_col(w.R, comp < 3 ? comp : comp - 3, ax);
  if (comp < 3) {
    S.w[0] = ax[0]; S.w[1] = ax[1]; S.w[2] = ax[2];
    cross3(w.p, ax, S.l);
  } else {
    S.w[0] = S.w[1] = S.w[2] = T(0);
    S.l[0] = ax[0]; S.l[1] = ax[1]; S.l[2] = ax[2];
  }
}

template <class T> RBD_HD void body_rbi(const BodyDev<T>& bd, Rbi<T>& I) {
  I.m = bd.m;
#pragma unroll
  for (int k = 0; k < 3; ++k) I.h[k] = bd.h[k];
#pragma unroll
  for (int k = 0; k < 6; ++k) I.J[k] = bd.J[k];
}

template <class T, class ST>
RBD_HD void kin_sample(const ModelDev<T>& M, const KinDev<T>& K, const KinIO<T>& io, const ST& st) {
  const int nb = M.nb;
  const bool vel = io.v.valid();
  const bool want_mom = vel && (io.ke.valid() || io.mom.valid() || io.mrb.valid());
  Pose<T> cur;
  pose_identity(cur);
  Mot<T> twc, bc;
#pragma unroll
  for (int k = 0; k < 3; ++k) twc.w[k] = twc.l[k] = bc.w[k] = bc.l[k] = T(0);
  T mc[3] = {T(0), T(0), T(0)}, ke = T(0);
  T hn[3] = {T(0), T(0), T(0)}, hf[3] = {T(0), T(0), T(0)}, bn[3] = {T(0), T(0), T(0)}, bf[3] = {T(0), T(0), T(0)};

  // ---- outward sweep: poses, twists, bias accelerations, sums ----
  // software pipeline: the joint scalars of body i+1 are loaded while body i is processed (multi-DoF joints read theirs directly)
  T q0n = T(0), q1n = T(0), qdn = T(0);
  auto fetch = [&](int i, T& q0, T& q1, T& qd) {
    q0 = q1 = qd = T(0);
    if (i < nb) {
      const BodyDev<T>& b = M.body[i];
      if (b.kind == K_REV || b.kind == K_PRIS || b.kind == K_SINCOS) {
        q0 = io.q(b.qrow);
        if (b.kind == K_SINCOS) q1 = io.q(b.qrow + 1);
        if (vel) qd = io.v(b.vrow);
      }
    }
  };
  fetch(0, q0n, q1n, qdn);
  for (int i = 0; i < nb; ++i) {
    const BodyDev<T>& bd = M.body[i];
    const T q0c = q0n, q1c = q1n, qdc = qdn;
    fetch(i + 1, q0n, q1n, qdn);
    const bool one_dof = bd.kind == K_REV || bd.kind == K_PRIS || bd.kind == K_SINCOS;
    Pose<T> pp;
    Mot<T> twp, bp;
    if (bd.flags & F_ROOT_CHILD) {
      pose_identity(pp);
#pragma unroll
      for (int k = 0; k < 3; ++k) twp.w[k] = twp.l[k] = bp.w[k] = bp.l[k] = T(0);
    } else if (bd.flags & F_FIRST_CHILD) {
      pp = cur; twp = twc; bp = bc;
    } else {
      const int row = bd.pslot * kSlotRowsKin;
#pragma unroll
      for (int k = 0; k < 9; ++k) pp.R[k] = st.ld(row + k);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        pp.p[k] = st.ld(row + 9 + k);
        twp.w[k] = st.ld(row + 12 + k); twp.l[k] = st.ld(row + 15 + k);
        bp.w[k] = st.ld(row + 18 + k); bp.l[k] = st.ld(row + 21 + k);
      }
    }
    T R[9], r[3], t[3];
    if (one_dof || bd.kind == K_FIXED) {
      Pre<T> pre;
      pre.q0 = q0c; pre.q1 = q1c;
      T sn, cs, d;
      joint_scd(bd.kind, pre, sn, cs, d);
      frame_1dof(bd, sn, cs, d, R, r);
    } else {
      frame_multi(bd, io.q, R, r);
    }
    Pose<T> w;
    mat_mul3(pp.R, R, w.R);
    mat_vec(pp.R, r, t);
    w.p[0] = pp.p[0] + t[0]; w.p[1] = pp.p[1] + t[1]; w.p[2] = pp.p[2] + t[2];
    if (io.tr.valid()) {
      T Ro[9];
      mat_mul3(w.R, K.At[i], Ro);
      const int row = 12 * bd.refidx;
#pragma unroll
      for (int k = 0; k < 9; ++k) io.tr.st(row + k, Ro[k]);
#pragma unroll
      for (int k = 0; k < 3; ++k) io.tr.st(row + 9 + k, w.p[k]);
    }
    if (io.poses.valid()) {
#pragma unroll
      for (int k = 0; k < 9; ++k) io.poses.st(12 * i + k, w.R[k]);
#pragma unroll
      for (int k = 0; k < 3; ++k) io.poses.st(12 * i + 9 + k, w.p[k]);
    }
    // joint twist in the root frame, jacobian columns
    Mot<T> jt;
#pragma unroll
    for (int k = 0; k < 3; ++k) jt.w[k] = jt.l[k] = T(0);
    const int nvj = kind_nv_dev(bd.kind);
    if (vel || io.J.valid()) {
      const T sg = T((int)K.sign[i]);
      for (int k = 0; k < nvj; ++k) {
        Mot<T> S;
        world_subspace(w, sub_comp(bd.kind, k), S);
        if (io.J.valid()) {
          const int row = 6 * (bd.vrow + k);
#pragma unroll
          for (int c = 0; c < 3; ++c) { io.J.st(row + c, sg * S.w[c]); io.J.st(row + 3 + c, sg * S.l[c]); }
        }
        if (vel) {
          const T x = one_dof ? qdc : io.v(bd.vrow + k);
#pragma unroll
          for (int c = 0; c < 3; ++c) { jt.w[c] += x * S.w[c]; jt.l[c] += x * S.l[c]; }
        }
      }
    }
    Mot<T> tw, bias;
    {
      Mot<T> cm;
      motion_cross(twp, jt, cm);          // v_parent x (S v) == v_i x (S v): the world-frame velocity-product acceleration
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        tw.w[k] = twp.w[k] + jt.w[k]; tw.l[k] = twp.l[k] + jt.l[k];
        bias.w[k] = bp.w[k] + cm.w[k]; bias.l[k] = bp.l[k] + cm.l[k];
      }
    }
    // mass moment (for the centre of mass and the potential energy)
    {
      T Rh[3];
      mat_vec(w.R, bd.h, Rh);
#pragma unroll
      for (int k = 0; k < 3; ++k) mc[k] += Rh[k] + bd.m * w.p[k];
    }
    if (want_mom) {
      Rbi<T> Ib, Iw;
      body_rbi(bd, Ib);
      rbi_to_parent(w.R, w.p, Ib, Iw);     // body -> root frame (:836-846)
      T n[3], f[3];
      rbi_mul(Iw, tw, n, f);               // momentum of this body
      ke += T(0.5) * (tw.w[0] * n[0] + tw.w[1] * n[1] + tw.w[2] * n[2] + tw.l[0] * f[0] + tw.l[1] * f[1] + tw.l[2] * f[2]);
#pragma unroll
      for (int k = 0; k < 3; ++k) { hn[k] += n[k]; hf[k] += f[k]; }
      if (io.mrb.valid()) {                // newton_euler(I, bias, twist) = I b + v x* (I v)
        T an[3], af[3], c1[3], c2[3], c3[3];
        rbi_mul(Iw, bias, an, af);
        cross3(tw.w, n, c1);
        cross3(tw.l, f, c2);
        cross3(tw.w, f, c3);
#pragma unroll
        for (int k = 0; k < 3; ++k) { bn[k] += an[k] + c1[k] + c2[k]; bf[k] += af[k] + c3[k]; }
      }
    }
    if (bd.flags & F_HAS_PENDING) {
      const int row = bd.oslot * kSlotRowsKin;
#pragma unroll
      for (int k = 0; k < 9; ++k) st.st(row + k, w.R[k]);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        st.st(row + 9 + k, w.p[k]);
        st.st(row + 12 + k, tw.w[k]); st.st(row + 15 + k, tw.l[k]);
        st.st(row + 18 + k, bias.w[k]); st.st(row + 21 + k, bias.l[k]);
      }
    }
    cur = w; twc = tw; bc = bias;
  }
  if (io.com.valid()) {
#pragma unroll
    for (int k = 0; k < 3; ++k) io.com.st(k, mc[k] * K.inv_mass);
  }
  if (io.pe.valid()) io.pe.st(0, -(M.g[0] * mc[0] + M.g[1] * mc[1] + M.g[2] * mc[2]));
  if (vel) {
    if (io.ke.valid()) io.ke.st(0, ke);
    if (io.mom.valid()) {
#pragma unroll
      for (int k = 0; k < 3; ++k) { io.mom.st(k, hn[k]); io.mom.st(3 + k, hf[k]); }
    }
    if (io.mrb.valid()) {
#pragma unroll
      for (int k = 0; k < 3; ++k) { io.mrb.st(k, bn[k]); io.mrb.st(3 + k, bf[k]); }
    }
  }
  if (!io.A.valid()) return;

  // ---- inward sweep: composite inertias in the root frame (plain sums, :852-868) and A[:, k] = Ic S_k ----
  Rbi<T> carry;
  carry.m = T(0);
#pragma unroll
  for (int k = 0; k < 3; ++k) carry.h[k] = T(0);
#pragma unroll
  for (int k = 0; k < 6; ++k) carry.J[k] = T(0);
  for (int i = nb - 1; i >= 0; --i) {
    const BodyDev<T>& bd = M.body[i];
    Pose<T> w;
#pragma unroll
    for (int k = 0; k < 9; ++k) w.R[k] = io.poses.get(12 * i + k);
#pragma unroll
    for (int k = 0; k < 3; ++k) w.p[k] = io.poses.get(12 * i + 9 + k);
    Rbi<T> Ib, Ic;
    body_rbi(bd, Ib);
    rbi_to_parent(w.R, w.p, Ib, Ic);
    if (!(bd.flags & F_LEAF)) {
      Ic.m += carry.m;
#pragma unroll
      for (int k = 0; k < 3; ++k) Ic.h[k] += carry.h[k];
#pragma unroll
      for (int k = 0; k < 6; ++k) Ic.J[k] += carry.J[k];
    }
    if (bd.flags & F_HAS_PENDING) {
      const int row = bd.oslot * kSlotRowsKin;
      Ic.m += st.ld(row);
#pragma unroll
      for (int k = 0; k < 3; ++k) Ic.h[k] += st.ld(row + 1 + k);
#pragma unroll
      for (int k = 0; k < 6; ++k) Ic.J[k] += st.ld(row + 4 + k);
    }
    const int nvj = kind_nv_dev(bd.kind);
    for (int k = 0; k < nvj; ++k) {
      Mot<T> S;
      world_subspace(w, sub_comp(bd.kind, k), S);
      T n[3], f[3];
      rbi_mul(Ic, S, n, f);
      const int row = 6 * (bd.vrow + k);
#pragma unroll
      for (int c = 0; c < 3; ++c) { io.A.st(row + c, n[c]); io.A.st(row + 3 + c, f[c]); }
    }
    if (bd.flags & F_ROOT_CHILD) continue;
    if (bd.flags & F_FIRST_CHILD) {
      carry = Ic;
    } else {
      const int row = bd.pslot * kSlotRowsKin;
      if (bd.flags & F_SLOT_INIT) {
        st.st(row, Ic.m);
#pragma unroll
        for (int k = 0; k < 3; ++k) st.st(row + 1 + k, Ic.h[k]);
#pragma unroll
        for (int k = 0; k < 6; ++k) st.st(row + 4 + k, Ic.J[k]);
      } else {
        st.add(row, Ic.m);
#pragma unroll
        for (int k = 0; k < 3; ++k) st.add(row + 1 + k, Ic.h[k]);
#pragma unroll
        for (int k = 0; k < 6; ++k) st.add(row + 4 + k, Ic.J[k]);
      }
    }
  }
}

// ==================================================================================================================
// momentum_matrix! alone, in two BODY-FRAME sweeps (mechanism_algorithms.jl:313-327: A[:, k] = Ic_{body(k)} S_k).  kin_sample
// keeps every body's root-frame pose from its outward sweep for the return sweep (12 nb scalars per sample: a global scratch
// column in the generic kernel, spills in the traced one).  Here nothing but the result columns crosses the sweeps:
//   inward   composite inertias in body frames exactly like mass_matrix! (carry in registers, pending slots for branch nodes),
//            F_k = Ic e_k (one-hot subspaces) parked in the stash, 6 rows per velocity coordinate;
//   outward  root-frame pose carried in registers (pending slots for branch nodes), each parked column transformed to the root
//            frame (f = R f_b, n = R n_b + p x f) and written.
// Stash: 6 nv rows + 12 per pending slot.  Used by the model-specialised kernels when that fits one warp's stash.
// ==================================================================================================================
constexpr int kSlotRowsMomMat = 12;
template <class T, class ST>
RBD_HD void momentum_matrix_sample(const ModelDev<T>& M, const Col<T>& q, const ColOut<T>& A, const ST& st) {
  const int nb = M.nb;
  const int slot_base = 6 * M.nv;
  Rbi<T> carry;
  carry.m = T(0);
#pragma unroll
  for (int k = 0; k < 3; ++k) carry.h[k] = T(0);
#pragma unroll
  for (int k = 0; k < 6; ++k) carry.J[k] = T(0);
  for (int i = nb - 1; i >= 0; --i) {
    const BodyDev<T>& bd = M.body[i];
    Rbi<T> ic;
    body_rbi(bd, ic);
    if (!(bd.flags & F_LEAF)) {
      ic.m += carry.m;
#pragma unroll
      for (int k = 0; k < 3; ++k) ic.h[k] += carry.h[k];
#pragma unroll
      for (int k = 0; k < 6; ++k) ic.J[k] += carry.J[k];
    }
    if (bd.flags & F_HAS_PENDING) {
      const int row = slot_base + bd.oslot * kSlotRowsMomMat;
      st.fence_st();
      ic.m += st.ld(row);
#pragma unroll
      for (int k = 0; k < 3; ++k) ic.h[k] += st.ld(row + 1 + k);
#pragma unroll
      for (int k = 0; k < 6; ++k) ic.J[k] += st.ld(row + 4 + k);
    }
    const int nvj = kind_nv_dev(bd.kind);
    for (int k = 0; k < nvj; ++k) {
      const int c = sub_comp(bd.kind, k);
      Mot<T> e;
#pragma unroll
      for (int d = 0; d < 3; ++d) { e.w[d] = (c == d) ? T(1) : T(0); e.l[d] = (c == 3 + d) ? T(1) : T(0); }
      T n[3], f[3];
      rbi_mul(ic, e, n, f);
      const int row = 6 * (bd.vrow + k);
#pragma unroll
      for (int d = 0; d < 3; ++d) { st.st(row + d, n[d]); st.st(row + 3 + d, f[d]); }
    }
    if (bd.flags & F_ROOT_CHILD) continue;
    T R[9], r[3];
    frame_any(bd, q, R, r);
    Rbi<T> up;
    rbi_to_parent(R, r, ic, up);
    if (bd.flags & F_FIRST_CHILD) carry = up;
    else {
      const int row = slot_base + bd.pslot * kSlotRowsMomMat;
      if (bd.flags & F_SLOT_INIT) {
        st.st(row, up.m);
#pragma unroll
        for (int k = 0; k < 3; ++k) st.st(row + 1 + k, up.h[k]);
#pragma unroll
        for (int k = 0; k < 6; ++k) st.st(row + 4 + k, up.J[k]);
      } else {
        st.add(row, up.m);
#pragma unroll
        for (int k = 0; k < 3; ++k) st.add(row + 1 + k, up.h[k]);
#pragma unroll
        for (int k = 0; k < 6; ++k) st.add(row + 4 + k, up.J[k]);
      }
    }
  }
  st.fence_st();
  Pose<T> cur;
  pose_identity(cur);
  for (int i = 0; i < nb; ++i) {
    const BodyDev<T>& bd = M.body[i];
    Pose<T> pp;
    if (bd.flags & F_ROOT_CHILD) pose_identity(pp);
    else if (bd.flags & F_FIRST_CHILD) pp = cur;
    else {
      const int row = slot_base + bd.pslot * kSlotRowsMomMat;
      T t[12];
      st.fence_st();
      st.template ldv<12>(row, t);
#pragma unroll
      for (int k = 0; k < 9; ++k) pp.R[k] = t[k];
#pragma unroll
      for (int k = 0; k < 3; ++k) pp.p[k] = t[9 + k];
    }
    T R[9], r[3], t3[3];
    frame_any(bd, q, R, r);
    Pose<T> w;
    mat_mul3(pp.R, R, w.R);
    mat_vec(pp.R, r, t3);
    w.p[0] = pp.p[0] + t3[0]; w.p[1] = pp.p[1] + t3[1]; w.p[2] = pp.p[2] + t3[2];
    const int nvj = kind_nv_dev(bd.kind);
    for (int k = 0; k < nvj; ++k) {
      const int row = 6 * (bd.vrow + k);
      T c6[6], n[3], f[3], nw[3], fw[3], x[3];
      st.template ldv<6>(row, c6);
#pragma unroll
      for (int d = 0; d < 3; ++d) { n[d] = c6[d]; f[d] = c6[3 + d]; }
      mat_vec(w.R, f, fw);
      mat_vec(w.R, n, nw);
      cross3(w.p, fw, x);
#pragma unroll
      for (int d = 0; d < 3; ++d) { A.st(row + d, nw[d] + x[d]); A.st(row + 3 + d, fw[d]); }
    }
    if (bd.flags & F_HAS_PENDING) {
      const int row = slot_base + bd.oslot * kSlotRowsMomMat;
#pragma unroll
      for (int k = 0; k < 9; ++k) st.st(row + k, w.R[k]);
#pragma unroll
      for (int k = 0; k < 3; ++k) st.st(row + 9 + k, w.p[k]);
    }
    cur = w;
  }
}

// ==================================================================================================================
// Per-body outputs of inverse_dynamics!: the `accelerations` and `jointwrenchesout` arguments of
//   inverse_dynamics!(torquesout, jointwrenchesout, accelerations, state, v̇, externalwrenches)   mechanism_algorithms.jl:542-553
// in the reference's own terms -- ROOT-frame quantities per body:
//   spatial_accelerations!        :387-417   a_i = a_parent + v_parent x (S v)_i + S_i v̇_i ,  a_root = -g
//   newton_euler!                 :428-439   w_i = I_i a_i + v_i x* (I_i v_i) - w_ext,i      (net wrench)
//   joint_wrenches_and_torques!   :442-459   w_parent += w_i in reverse tree order            (joint wrench = subtree sum)
// Outward sweep exactly like kin_sample (pose, twist, acceleration in registers; branch nodes park theirs in a pending slot);
// net wrenches go straight into the output column and the inward accumulation is a read-modify-write on that column (a thread
// owns its column; reverse preorder guarantees a body's sum is complete before it is added to its parent).
// ==================================================================================================================
template <class T> struct BodiesIO {
  Col<T> q, v, vd, wext;       // vd / wext may be invalid (zero accelerations / no external wrenches)
  T* acc; T* jw;               // output columns (already offset by the sample), rows 6 * refidx + c; either may be NULL
  int64_t ld;
  bool active;
};

template <class T, class ST>
RBD_HD void bodies_sample(const ModelDev<T>& M, const BodiesIO<T>& io, const ST& st) {
  const int nb = M.nb;
  Pose<T> cur;
  pose_identity(cur);
  Mot<T> twc, ac;
#pragma unroll
  for (int k = 0; k < 3; ++k) twc.w[k] = twc.l[k] = ac.w[k] = ac.l[k] = T(0);
  for (int i = 0; i < nb; ++i) {
    const BodyDev<T>& bd = M.body[i];
    Pose<T> pp;
    Mot<T> twp, ap;
    if (bd.flags & F_ROOT_CHILD) {
      pose_identity(pp);
#pragma unroll
      for (int k = 0; k < 3; ++k) { twp.w[k] = twp.l[k] = ap.w[k] = T(0); ap.l[k] = -M.g[k]; }
    } else if (bd.flags & F_FIRST_CHILD) {
      pp = cur; twp = twc; ap = ac;
    } else {
      const int row = bd.pslot * kSlotRowsKin;
#pragma unroll
      for (int k = 0; k < 9; ++k) pp.R[k] = st.ld(row + k);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        pp.p[k] = st.ld(row + 9 + k);
        twp.w[k] = st.ld(row + 12 + k); twp.l[k] = st.ld(row + 15 + k);
        ap.w[k] = st.ld(row + 18 + k); ap.l[k] = st.ld(row + 21 + k);
      }
    }
    T R[9], r[3], t[3];
    frame_any(bd, io.q, R, r);
    Pose<T> w;
    mat_mul3(pp.R, R, w.R);
    mat_vec(pp.R, r, t);
    w.p[0] = pp.p[0] + t[0]; w.p[1] = pp.p[1] + t[1]; w.p[2] = pp.p[2] + t[2];
    Mot<T> jt, ja;                     // S v and S v̇ in the root frame
#pragma unroll
    for (int k = 0; k < 3; ++k) jt.w[k] = jt.l[k] = ja.w[k] = ja.l[k] = T(0);
    const int nvj = kind_nv_dev(bd.kind);
    for (int k = 0; k < nvj; ++k) {
      Mot<T> S;
      world_subspace(w, sub_comp(bd.kind, k), S);
      const T x = io.v(bd.vrow + k);
      const T xd = io.vd.valid() ? io.vd(bd.vrow + k) : T(0);
#pragma unroll
      for (int c = 0; c < 3; ++c) { jt.w[c] += x * S.w[c]; jt.l[c] += x * S.l[c]; ja.w[c] += xd * S.w[c]; ja.l[c] += xd * S.l[c]; }
    }
    Mot<T> tw, a, cm;
    motion_cross(twp, jt, cm);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      tw.w[k] = twp.w[k] + jt.w[k]; tw.l[k] = twp.l[k] + jt.l[k];
      a.w[k] = ap.w[k] + cm.w[k] + ja.w[k]; a.l[k] = ap.l[k] + cm.l[k] + ja.l[k];
    }
    const int64_t orow = (int64_t)6 * bd.refidx;
    if (io.acc && io.active) {
#pragma unroll
      for (int k = 0; k < 3; ++k) { io.acc[(orow + k) * io.ld] = a.w[k]; io.acc[(orow + 3 + k) * io.ld] = a.l[k]; }
    }
    if (io.jw) {                       // net wrench of this body, root frame
      Rbi<T> Ib, Iw;
      body_rbi(bd, Ib);
      rbi_to_parent(w.R, w.p, Ib, Iw);
      T n[3], f[3], hn[3], hf[3], c1[3], c2[3], c3[3];
      rbi_mul(Iw, a, n, f);
      rbi_mul(Iw, tw, hn, hf);
      cross3(tw.w, hn, c1);
      cross3(tw.l, hf, c2);
      cross3(tw.w, hf, c3);
#pragma unroll
      for (int k = 0; k < 3; ++k) { n[k] += c1[k] + c2[k]; f[k] += c3[k]; }
      if (io.wext.valid()) {
#pragma unroll
        for (int k = 0; k < 3; ++k) { n[k] -= io.wext((int)orow + k); f[k] -= io.wext((int)orow + 3 + k); }
      }
      if (io.active) {
#pragma unroll
        for (int k = 0; k < 3; ++k) { io.jw[(orow + k) * io.ld] = n[k]; io.jw[(orow + 3 + k) * io.ld] = f[k]; }
      }
    }
    if (bd.flags & F_HAS_PENDING) {
      const int row = bd.oslot * kSlotRowsKin;
#pragma unroll
      for (int k = 0; k < 9; ++k) st.st(row + k, w.R[k]);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        st.st(row + 9 + k, w.p[k]);
        st.st(row + 12 + k, tw.w[k]); st.st(row + 15 + k, tw.l[k]);
        st.st(row + 18 + k, a.w[k]); st.st(row + 21 + k, a.l[k]);
      }
    }
    cur = w; twc = tw; ac = a;
  }
  if (!io.jw || !io.active) return;
  // inward accumulation on the output column
  for (int i = nb - 1; i >= 0; --i) {
    const BodyDev<T>& bd = M.body[i];
    if (bd.flags & F_ROOT_CHILD) continue;
    const int64_t crow = (int64_t)6 * bd.refidx, prow = (int64_t)6 * M.body[bd.parent].refidx;
#pragma unroll
    for (int k = 0; k < 6; ++k) io.jw[(prow + k) * io.ld] += io.jw[(crow + k) * io.ld];
  }
}

// ==================================================================================================================
// Soft point contact with half-spaces (SURVEY 8(f) rank 4): the batched contact_dynamics!   mechanism_algorithms.jl:680-723
// with the reference's default models (src/contact.jl):
//   normal force   HuntCrossleyModel          f_n = max(lambda z^n zdot + k z^n, 0)                  contact.jl:130-146
//   friction       ViscoelasticCoulombModel   f_stick = -k x - b v_t, clipped to the cone mu f_n;    :152-206
//                                             state x = tangential displacement, xdot = (-k x - f_t) / b
// One thread per sample; outward sweep with root-frame pose and twist per body (as bodies_sample); for every contact point
// p of the body and every half-space h:  point = T_body p,  velocity = omega x point + v_lin  (point_velocity),
// separation = (point - h.point) . h.normal;  inside (<= 0): force as above, wrench += (point x force, force), xdot written;
// outside: the state is RESET to zero and its derivative zeroed, exactly like the reference does inside contact_dynamics!.
// ==================================================================================================================
constexpr int kMaxContactPoints = 32, kMaxHalfSpaces = 4;
template <class T> struct ContactDev {
  int32_t npoints, nhalf;
  int32_t first[kMaxBodies + 1];        // preorder body i owns points first[i] .. first[i + 1] - 1 (sorted by body)
  int32_t orig[kMaxContactPoints];      // sorted position -> caller's point index (rows of the state arrays)
  T loc[kMaxContactPoints][3];          // location in the CANONICAL body frame
  T hc[kMaxContactPoints][3];           // Hunt-Crossley k, lambda, n
  T fr[kMaxContactPoints][3];           // viscoelastic Coulomb mu, k, b
  T hp[kMaxHalfSpaces][3], hn[kMaxHalfSpaces][3];   // half-space point and unit outward normal, root frame
};
template <class T> struct ContactIO {
  Col<T> q, v;
  T* s;            // [3 * npoints * nhalf] rows of this sample's column: tangential displacements (in / out: reset when outside)
  T* sd;           // same shape, derivative out; may be NULL
  T* wr;           // [6 nb] contact wrench per body (root frame, rows 6 * refidx + c)
  int64_t ld;
  bool active;
};
RBD_HD float contact_pow(float z, float n) {
#if defined(__CUDA_ARCH__)
  return n == 1.5f ? z * sqrtf(z) : powf(z, n);
#else
  return n == 1.5f ? z * std::sqrt(z) : std::pow(z, n);
#endif
}
RBD_HD double contact_pow(double z, double n) {
#if defined(__CUDA_ARCH__)
  return n == 1.5 ? z * sqrt(z) : pow(z, n);
#else
  return n == 1.5 ? z * std::sqrt(z) : std::pow(z, n);
#endif
}
RBD_HD float contact_sqrt(float x) {
#if defined(__CUDA_ARCH__)
  return sqrtf(x);
#else
  return std::sqrt(x);
#endif
}
RBD_HD double contact_sqrt(double x) {
#if defined(__CUDA_ARCH__)
  return sqrt(x);
#else
  return std::sqrt(x);
#endif
}

// Host side: rbd_contact_desc -> ContactDev (points sorted by the preorder position of their body, stable; locations rotated into
// the canonical body frame; normals normalised like the HalfSpace3D constructor, contact.jl:225).  pos: reference joint index ->
// preorder position, alignT: preorder position -> A^T (HostModel).
template <class T>
inline void build_contact_dev(int nb, const int* pos, const double* alignT, const rbd_contact_desc& cd, ContactDev<T>& C) {
  std::memset(&C, 0, sizeof(C));
  C.npoints = cd.npoints; C.nhalf = cd.nhalfspaces;
  int cnt[kMaxBodies + 1] = {0};
  for (int p = 0; p < cd.npoints; ++p) cnt[pos[cd.body[p]] + 1] += 1;
  for (int i = 0; i < nb; ++i) cnt[i + 1] += cnt[i];
  for (int i = 0; i <= kMaxBodies; ++i) C.first[i] = cnt[i < nb ? i : nb];
  int fill[kMaxBodies] = {0};
  for (int p = 0; p < cd.npoints; ++p) {
    const int i = pos[cd.body[p]];
    const int k = C.first[i] + fill[i]++;
    C.orig[k] = p;
    const double* At = alignT + 9 * i;
    const double* l = cd.location + 3 * p;
    for (int r = 0; r < 3; ++r) C.loc[k][r] = (T)(At[3 * r] * l[0] + At[3 * r + 1] * l[1] + At[3 * r + 2] * l[2]);
    for (int r = 0; r < 3; ++r) { C.hc[k][r] = (T)cd.normal_model[3 * p + r]; C.fr[k][r] = (T)cd.friction_model[3 * p + r]; }
  }
  for (int h = 0; h < cd.nhalfspaces; ++h) {
    const double* hs = cd.halfspace + 6 * h;
    const double nn = std::sqrt(hs[3] * hs[3] + hs[4] * hs[4] + hs[5] * hs[5]);
    for (int r = 0; r < 3; ++r) { C.hp[h][r] = (T)hs[r]; C.hn[h][r] = (T)(hs[3 + r] / nn); }
  }
}

// The force law of one (point pi, half-space with unit normal n) pair in contact: penetration z >= 0, point velocity vel (root
// frame), tangential displacement xs(k), k = 0..2 (read inside, where the friction force needs it).  Out: the force on the body f
// (root frame) and the state derivative xd.  Shared by contact_sample, the rollout's contact pass (contact_stage_pass) and, with
// T = Dual1<P>, its adjoint (rbd_contact_adjoint.cuh): P is the scalar type of the descriptor.
template <class T, class P, class XS>
RBD_HD void contact_force(const ContactDev<P>& C, int pi, const P* n, T z, const T* vel, const XS& xs, T* f, T* xd) {
  const T zd = -(vel[0] * n[0] + vel[1] * n[1] + vel[2] * n[2]);
  const T zn = contact_pow(z, C.hc[pi][2]);
  T fn = C.hc[pi][1] * zn * zd + C.hc[pi][0] * zn;
  fn = fn > T(0) ? fn : T(0);
  const T mu = C.fr[pi][0], kf = C.fr[pi][1], bf = C.fr[pi][2];
  T x[3], ft[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    x[k] = xs(k);
    ft[k] = -kf * x[k] - bf * (vel[k] + zd * n[k]);          // f_stick; tangential velocity = velocity + zdot * normal
  }
  const T n2 = ft[0] * ft[0] + ft[1] * ft[1] + ft[2] * ft[2], m2 = (mu * fn) * (mu * fn);
  if (n2 > m2) {
    const T sc = contact_sqrt(m2 / n2);
    ft[0] *= sc; ft[1] *= sc; ft[2] *= sc;
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) { f[k] = fn * n[k] + ft[k]; xd[k] = (-kf * x[k] - ft[k]) / bf; }
}

template <class T, class ST>
RBD_HD void contact_sample(const ModelDev<T>& M, const ContactDev<T>& C, const ContactIO<T>& io, const ST& st) {
  const int nb = M.nb;
  Pose<T> cur;
  pose_identity(cur);
  Mot<T> twc;
#pragma unroll
  for (int k = 0; k < 3; ++k) twc.w[k] = twc.l[k] = T(0);
  for (int i = 0; i < nb; ++i) {
    const BodyDev<T>& bd = M.body[i];
    Pose<T> pp;
    Mot<T> twp;
    if (bd.flags & F_ROOT_CHILD) {
      pose_identity(pp);
#pragma unroll
      for (int k = 0; k < 3; ++k) twp.w[k] = twp.l[k] = T(0);
    } else if (bd.flags & F_FIRST_CHILD) {
      pp = cur; twp = twc;
    } else {
      const int row = bd.pslot * kSlotRowsKin;
#pragma unroll
      for (int k = 0; k < 9; ++k) pp.R[k] = st.ld(row + k);
#pragma unroll
      for (int k = 0; k < 3; ++k) { pp.p[k] = st.ld(row + 9 + k); twp.w[k] = st.ld(row + 12 + k); twp.l[k] = st.ld(row + 15 + k); }
    }
    T R[9], r[3], t[3];
    frame_any(bd, io.q, R, r);
    Pose<T> w;
    mat_mul3(pp.R, R, w.R);
    mat_vec(pp.R, r, t);
    w.p[0] = pp.p[0] + t[0]; w.p[1] = pp.p[1] + t[1]; w.p[2] = pp.p[2] + t[2];
    Mot<T> tw = twp;
    const int nvj = kind_nv_dev(bd.kind);
    for (int k = 0; k < nvj; ++k) {
      Mot<T> S;
      world_subspace(w, sub_comp(bd.kind, k), S);
      const T x = io.v(bd.vrow + k);
#pragma unroll
      for (int c = 0; c < 3; ++c) { tw.w[c] += x * S.w[c]; tw.l[c] += x * S.l[c]; }
    }
    T wn[3] = {T(0), T(0), T(0)}, wf[3] = {T(0), T(0), T(0)};
    for (int pi = C.first[i]; pi < C.first[i + 1]; ++pi) {
      T pt[3], vel[3], tmp[3];
      mat_vec(w.R, C.loc[pi], tmp);
      pt[0] = w.p[0] + tmp[0]; pt[1] = w.p[1] + tmp[1]; pt[2] = w.p[2] + tmp[2];
      cross3(tw.w, pt, vel);                                   // point_velocity(twist, point), spatialmotion.jl
      vel[0] += tw.l[0]; vel[1] += tw.l[1]; vel[2] += tw.l[2];
      for (int h = 0; h < C.nhalf; ++h) {
        const int64_t srow = (int64_t)3 * (C.orig[pi] * C.nhalf + h);
        const T* n = C.hn[h];
        const T sep = (pt[0] - C.hp[h][0]) * n[0] + (pt[1] - C.hp[h][1]) * n[1] + (pt[2] - C.hp[h][2]) * n[2];
        T xd[3] = {T(0), T(0), T(0)};
        if (sep <= T(0)) {
          T f[3];
          contact_force(C, pi, n, -sep, vel, [&](int k) { return io.s ? io.s[(srow + k) * io.ld] : T(0); }, f, xd);
          T m[3];
          cross3(pt, f, m);                                   // Wrench(point, force)
#pragma unroll
          for (int k = 0; k < 3; ++k) { wn[k] += m[k]; wf[k] += f[k]; }
        } else if (io.s && io.active) {                       // Contact.reset!(contact_state)
#pragma unroll
          for (int k = 0; k < 3; ++k) io.s[(srow + k) * io.ld] = T(0);
        }
        if (io.sd && io.active) {
#pragma unroll
          for (int k = 0; k < 3; ++k) io.sd[(srow + k) * io.ld] = xd[k];
        }
      }
    }
    if (io.active) {
      const int64_t orow = (int64_t)6 * bd.refidx;
#pragma unroll
      for (int k = 0; k < 3; ++k) { io.wr[(orow + k) * io.ld] = wn[k]; io.wr[(orow + 3 + k) * io.ld] = wf[k]; }
    }
    if (bd.flags & F_HAS_PENDING) {
      const int row = bd.oslot * kSlotRowsKin;
#pragma unroll
      for (int k = 0; k < 9; ++k) st.st(row + k, w.R[k]);
#pragma unroll
      for (int k = 0; k < 3; ++k) { st.st(row + 9 + k, w.p[k]); st.st(row + 12 + k, tw.w[k]); st.st(row + 15 + k, tw.l[k]); }
    }
    cur = w; twc = tw;
  }
}

// ==================================================================================================================
// The contact pass of the contact rollout (rbd_integrate_contact, DESIGN 4.14): contact_dynamics! at one RK4 stage, as the
// pre-pass of the forward-dynamics kernel.  It replaces ext_wrench_pass there: same outward sweep, with the twist tracked next to
// the pose (branch nodes park both, 18 rows, in the ABA stash's pending slots), and the same output -- every body's wrench in its
// own frame in the scratch rows aba_sample reads.  The stage's contact state  s_i = s0 + wa sd_prev  (wa = dt a_i, sd_prev = ṡ of
// the previous stage, NULL at stage 0) is formed from two loads per pair in contact and never stored.  ṡ_i is written for every
// pair, zero out of contact; nothing is reset: within the reference's integrator a reset does not survive the stage (DESIGN 4.14).
// Only the bodies that carry contact points have scratch rows (ContactScr): 2 x 6 rows per sample for a biped instead of 6 nb.
// ==================================================================================================================
template <class T> struct ContactStageIO {
  const T* s0; const T* sdp;    // [ns] rows of this sample's column (leading dimension ld)
  T* sd;                        // ṡ_i out, same shape
  T wa;
  int64_t ld;
  bool active;
};
static_assert(kSlotRowsAba >= 18, "the contact pass parks pose and twist in the ABA pending slots");

// The scratch column of the body-frame contact wrenches: rows 6 slot[i] .. + 5 for body i (preorder) if it carries contact points
// (slot[i] >= 0, in preorder), none otherwise.  get() is the view aba_sample reads, rows 6 i + k of every body: zero without rows.
template <class T> struct ContactScr {
  T* p;
  int64_t ld;
  const int8_t* slot;           // [nb]
  RBD_HD T get(int row) const {
    const int i = row / 6, c = slot[i];
    return c < 0 ? T(0) : p[(int64_t)(6 * c + row - 6 * i) * ld];
  }
};
// host side: slot[] of the bodies that carry points; returns their number
template <class T> inline int contact_wrench_slots(int nb, const ContactDev<T>& C, int8_t* slot) {
  int n = 0;
  for (int i = 0; i < nb; ++i) slot[i] = (int8_t)(C.first[i + 1] > C.first[i] ? n++ : -1);
  return n;
}
// aba_sample's IO for the contact rollout: AbaIO with the external wrenches read through ContactScr
template <class T, int KINDS> struct ContactAbaIO {
  static constexpr bool kExt = true;
  static constexpr int kKinds = KINDS;
  Col<T> q, v, tau;
  ColOut<T> vd, qd;
  ContactScr<T> ext;
};

template <class T, class ST>
RBD_HD void contact_stage_pass(const ModelDev<T>& M, const ContactDev<T>& C, const Col<T>& q, const Col<T>& v,
                               const ContactStageIO<T>& io, const ContactScr<T>& ext, const ST& st, int slot_base, int slot_rows) {
  Pose<T> cur;
  pose_identity(cur);
  Mot<T> twc;
#pragma unroll
  for (int k = 0; k < 3; ++k) twc.w[k] = twc.l[k] = T(0);
  for (int i = 0; i < M.nb; ++i) {
    const BodyDev<T>& bd = M.body[i];
    Pose<T> pp;
    Mot<T> twp;
    if (bd.flags & F_ROOT_CHILD) {
      pose_identity(pp);
#pragma unroll
      for (int k = 0; k < 3; ++k) twp.w[k] = twp.l[k] = T(0);
    } else if (bd.flags & F_FIRST_CHILD) {
      pp = cur; twp = twc;
    } else {
      const int row = slot_base + bd.pslot * slot_rows;
      T t[18];
      st.fence_st();
      st.template ldv<18>(row, t);
#pragma unroll
      for (int k = 0; k < 9; ++k) pp.R[k] = t[k];
#pragma unroll
      for (int k = 0; k < 3; ++k) { pp.p[k] = t[9 + k]; twp.w[k] = t[12 + k]; twp.l[k] = t[15 + k]; }
    }
    T R[9], r[3], t[3];
    frame_any(bd, q, R, r);
    Pose<T> w;
    mat_mul3(pp.R, R, w.R);
    mat_vec(pp.R, r, t);
    w.p[0] = pp.p[0] + t[0]; w.p[1] = pp.p[1] + t[1]; w.p[2] = pp.p[2] + t[2];
    Mot<T> tw = twp;
    const int nvj = kind_nv_dev(bd.kind);
    for (int k = 0; k < nvj; ++k) {
      Mot<T> S;
      world_subspace(w, sub_comp(bd.kind, k), S);
      const T x = v(bd.vrow + k);
#pragma unroll
      for (int c = 0; c < 3; ++c) { tw.w[c] += x * S.w[c]; tw.l[c] += x * S.l[c]; }
    }
    T wn[3] = {T(0), T(0), T(0)}, wf[3] = {T(0), T(0), T(0)};      // root frame, as contact_sample sums them
    for (int pi = C.first[i]; pi < C.first[i + 1]; ++pi) {
      T pt[3], vel[3], tmp[3];
      mat_vec(w.R, C.loc[pi], tmp);
      pt[0] = w.p[0] + tmp[0]; pt[1] = w.p[1] + tmp[1]; pt[2] = w.p[2] + tmp[2];
      cross3(tw.w, pt, vel);
      vel[0] += tw.l[0]; vel[1] += tw.l[1]; vel[2] += tw.l[2];
      for (int h = 0; h < C.nhalf; ++h) {
        const int64_t srow = (int64_t)3 * (C.orig[pi] * C.nhalf + h);
        const T* n = C.hn[h];
        const T sep = (pt[0] - C.hp[h][0]) * n[0] + (pt[1] - C.hp[h][1]) * n[1] + (pt[2] - C.hp[h][2]) * n[2];
        T xd[3] = {T(0), T(0), T(0)};
        if (sep <= T(0)) {
          T f[3], m[3];
          contact_force(C, pi, n, -sep, vel, [&](int k) {        // s_i = s0 + wa sd_prev
            const int64_t e = (srow + k) * io.ld;
            return io.sdp ? io.s0[e] + io.wa * io.sdp[e] : io.s0[e];
          }, f, xd);
          cross3(pt, f, m);
#pragma unroll
          for (int k = 0; k < 3; ++k) { wn[k] += m[k]; wf[k] += f[k]; }
        }
        if (io.active) {
#pragma unroll
          for (int k = 0; k < 3; ++k) io.sd[(srow + k) * io.ld] = xd[k];
        }
      }
    }
    const int c = ext.slot[i];
    if (c >= 0) {      // root frame -> body frame as ext_wrench_pass:  f_b = Rw^T f ,  n_b = Rw^T (n - pw x f)
      T m[3], nb_[3], fb[3];
      cross3(w.p, wf, m);
      m[0] = wn[0] - m[0]; m[1] = wn[1] - m[1]; m[2] = wn[2] - m[2];
      matT_vec(w.R, m, nb_);
      matT_vec(w.R, wf, fb);
      T* o = ext.p + (int64_t)6 * c * ext.ld;
#pragma unroll
      for (int k = 0; k < 3; ++k) { o[k * ext.ld] = nb_[k]; o[(3 + k) * ext.ld] = fb[k]; }
    }
    if (bd.flags & F_HAS_PENDING) {
      const int row = slot_base + bd.oslot * slot_rows;
#pragma unroll
      for (int k = 0; k < 9; ++k) st.st(row + k, w.R[k]);
#pragma unroll
      for (int k = 0; k < 3; ++k) { st.st(row + 9 + k, w.p[k]); st.st(row + 12 + k, tw.w[k]); st.st(row + 15 + k, tw.l[k]); }
    }
    cur = w; twc = tw;
  }
  st.fence_st();     // the slots are re-used by aba_sample
}

}  // namespace rbd
