// Per-sample recursive Newton-Euler (inverse_dynamics! / dynamics_bias!), composite-rigid-body algorithm (mass_matrix!)
// and the external-wrench preparation pass, in the same body-frame / one-hot-subspace / depth-first conventions as the
// Articulated-Body code in rbd_device.cuh.  Reference (relative to the reference's src/):
//   spatial_accelerations!        mechanism_algorithms.jl:387-417     a_i = a_parent + v_parent x S v + S v̇, a_root = -g
//   newton_euler!                 mechanism_algorithms.jl:428-439     w_i = I a + v x* I v - w_ext
//   joint_wrenches_and_torques!   mechanism_algorithms.jl:442-459     w_parent += w_i ; tau_k = S_k . w
//   mass_matrix!                  mechanism_algorithms.jl:248-272     M[i,j] = (Ic S_i) . S_j along the support path
//   _update_crb_inertias!         mechanism_state.jl:852-868
#pragma once
#include "rbd_device.cuh"

namespace rbd {

constexpr int kRneaRowsPerBody = 6;
constexpr int kCrbaRowsPerBody = 2;

// body -> world pose
template <class T> struct Pose { T R[9]; T p[3]; };

template <class T> RBD_HD void pose_identity(Pose<T>& w) {
#pragma unroll
  for (int k = 0; k < 9; ++k) w.R[k] = (k % 4 == 0) ? T(1) : T(0);
  w.p[0] = w.p[1] = w.p[2] = T(0);
}

// joint frame (child -> parent rotation R, child origin r in the parent) of any kind from directly-read q
template <class T> RBD_HD void frame_any(const BodyDev<T>& bd, const Col<T>& q, T* R, T* r) {
  const int kind = bd.kind;
  if (kind == K_REV || kind == K_PRIS || kind == K_SINCOS || kind == K_FIXED) {
    Pre<T> pre;
    pre.q0 = (kind != K_FIXED) ? q(bd.qrow) : T(0);
    pre.q1 = (kind == K_SINCOS) ? q(bd.qrow + 1) : T(0);
    T s, c, d;
    joint_scd(kind, pre, s, c, d);
    frame_1dof(bd, s, c, d, R, r);
  } else {
    frame_multi(bd, q, R, r);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// external wrenches: root frame (as the reference takes them, mechanism_algorithms.jl:437) -> body frames
// ------------------------------------------------------------------------------------------------------------------
// Outward sweep that tracks each body's world pose in registers (branch nodes park theirs in their pending slot) and
// writes  f_b = Rw^T f ,  n_b = Rw^T (n - pw x f)  for every body into the scratch column (rows 6 i .. 6 i + 5,
// i = preorder position).  Wrench loads for body i+1 are issued while body i is processed.
template <class T, class ST>
RBD_HD void ext_wrench_pass(const ModelDev<T>& M, const Col<T>& q, const Col<T>& wext, const Scr<T>& ext,
                            const ST& stash, int slot_base, int slot_rows) {
  const auto st = stash.slots();     // only the pending slots are used here (world poses of branch nodes)
  Pose<T> cur;
  pose_identity(cur);
  T wn[6], wc[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) wn[k] = wext(6 * M.body[0].refidx + k);
  for (int i = 0; i < M.nb; ++i) {
    const BodyDev<T>& bd = M.body[i];
#pragma unroll
    for (int k = 0; k < 6; ++k) wc[k] = wn[k];
    if (i + 1 < M.nb) {
      const int rn = 6 * M.body[i + 1].refidx;
#pragma unroll
      for (int k = 0; k < 6; ++k) wn[k] = wext(rn + k);
    }
    Pose<T> pp;
    if (bd.flags & F_ROOT_CHILD) pose_identity(pp);
    else if (bd.flags & F_FIRST_CHILD) pp = cur;
    else {
      const int row = slot_base + bd.pslot * slot_rows;
      T t[12];
      st.fence_st();
      st.template ldv<12>(row, t);
#pragma unroll
      for (int k = 0; k < 9; ++k) pp.R[k] = t[k];
#pragma unroll
      for (int k = 0; k < 3; ++k) pp.p[k] = t[9 + k];
    }
    T R[9], r[3], t[3];
    frame_any(bd, q, R, r);
    Pose<T> w;
    mat_mul3(pp.R, R, w.R);
    mat_vec(pp.R, r, t);
    w.p[0] = pp.p[0] + t[0]; w.p[1] = pp.p[1] + t[1]; w.p[2] = pp.p[2] + t[2];
    T m[3], nb_[3], fb[3];
    cross3(w.p, wc + 3, m);
    m[0] = wc[0] - m[0]; m[1] = wc[1] - m[1]; m[2] = wc[2] - m[2];
    matT_vec(w.R, m, nb_);
    matT_vec(w.R, wc + 3, fb);
#pragma unroll
    for (int k = 0; k < 3; ++k) { ext.st(6 * i + k, nb_[k]); ext.st(6 * i + 3 + k, fb[k]); }
    if (bd.flags & F_HAS_PENDING) {
      const int row = slot_base + bd.oslot * slot_rows;
#pragma unroll
      for (int k = 0; k < 9; ++k) st.st(row + k, w.R[k]);
#pragma unroll
      for (int k = 0; k < 3; ++k) st.st(row + 9 + k, w.p[k]);
    }
    cur = w;
  }
  st.fence_st();     // the slots are re-used by the passes that follow
}

// ==================================================================================================================
// Recursive Newton-Euler:  tau = M(q) v̇ + c(q, v, w_ext)      (vd invalid => v̇ = 0 => dynamics_bias)
// ==================================================================================================================
template <class T> struct RneaIO {
  Col<T> q, v, vd, wext;
  ColOut<T> tau;
  Scr<T> ext;
};

// ST: Stash<T, STRIDE> (shared memory) or the symbolic stash of the code generator (rbd_sym.h); fence_st()
// stands wherever a thread re-reads a word it wrote; it is a no-op for shared memory
template <class T, class ST>
RBD_HD void rnea_sample(const ModelDev<T>& M, const RneaIO<T>& io, const ST& st) {
  const int nb = M.nb;
  const int slot_base = nb * kRneaRowsPerBody;
  if (io.ext.valid()) ext_wrench_pass(M, io.q, io.wext, io.ext, st, slot_base, kSlotRowsRnea);
  // ---- pass 1 (outward): v, a, net wrench f_i = I a + v x* I v - w_ext ----
  Mot<T> vcur, acur;
#pragma unroll
  for (int k = 0; k < 3; ++k) { vcur.w[k] = vcur.l[k] = acur.w[k] = acur.l[k] = T(0); }
  // software pipeline: scalars of body i+1 are loaded while body i is processed
  T q0n = T(0), q1n = T(0), qdn = T(0), vdn = T(0), qon = T(0);
  int zfn = 0;                       // fast-class bits / angle offset of the next body, fetched ahead like the joint scalars
  auto fetch = [&](int i, bool vel, T& q0, T& q1, T& qd, T& vd) {
    q0 = q1 = qd = vd = T(0);
    zfn = 0; qon = T(0);
    if (i >= 0 && i < nb) {
      const BodyDev<T>& b = M.body[i];
      zfn = b.flags & (F_ZPAR | F_ZPERP);
      qon = b.qoff;
      if (b.kind == K_REV || b.kind == K_PRIS || b.kind == K_SINCOS) {
        q0 = io.q(b.qrow);
        if (b.kind == K_SINCOS) q1 = io.q(b.qrow + 1);
        if (vel) {
          qd = io.v(b.vrow);
          if (io.vd.valid()) vd = io.vd(b.vrow);
        }
      }
    }
  };
  fetch(0, true, q0n, q1n, qdn, vdn);
  for (int i = 0; i < nb; ++i) {
    const BodyDev<T>& bd = M.body[i];
    const int kind = bd.kind;
    const T q0 = q0n, q1 = q1n, qd = qdn, vdj = vdn, qoff = qon;
    const int zf = zfn;
    fetch(i + 1, true, q0n, q1n, qdn, vdn);
    Mot<T> vp, ap;
    if (bd.flags & F_ROOT_CHILD) {
#pragma unroll
      for (int k = 0; k < 3; ++k) { vp.w[k] = T(0); vp.l[k] = T(0); ap.w[k] = T(0); ap.l[k] = -M.g[k]; }
    } else if (bd.flags & F_FIRST_CHILD) {
      vp = vcur; ap = acur;
    } else {
      const int row = slot_base + bd.pslot * kSlotRowsRnea;
      T t[12];
      st.fence_st();
      st.template ldv<12>(row, t);
#pragma unroll
      for (int k = 0; k < 3; ++k) { vp.w[k] = t[k]; vp.l[k] = t[3 + k]; ap.w[k] = t[6 + k]; ap.l[k] = t[9 + k]; }
    }
    T R[9], r[3];
    Mot<T> v, a;
    if (zf) {                      // fast class (revolute, E = [P] Rz(q + qoff), rbd_types.h)
      T s, c;
      sincos_t(q0 + qoff, s, c);
      if (zf & F_ZPERP) { motion_to_child_z<T, 1>(s, c, bd.pt, vp, v); motion_to_child_z<T, 1>(s, c, bd.pt, ap, a); }
      else { motion_to_child_z<T, 0>(s, c, bd.pt, vp, v); motion_to_child_z<T, 0>(s, c, bd.pt, ap, a); }
      v.w[2] += qd;
      a.w[0] += qd * v.w[1]; a.w[1] -= qd * v.w[0]; a.w[2] += vdj;
      a.l[0] += qd * v.l[1]; a.l[1] -= qd * v.l[0];
    } else if (kind == K_REV || kind == K_PRIS || kind == K_SINCOS || kind == K_FIXED) {
      Pre<T> pre; pre.q0 = q0; pre.q1 = q1;
      T s, c, d;
      joint_scd(kind, pre, s, c, d);
      frame_1dof(bd, s, c, d, R, r);
      motion_to_child(R, r, vp, v);
      motion_to_child(R, r, ap, a);
      if (kind == K_PRIS) {
        v.l[2] += qd;
        a.l[0] += qd * v.w[1]; a.l[1] -= qd * v.w[0]; a.l[2] += vdj;
      } else if (kind != K_FIXED) {
        v.w[2] += qd;
        a.w[0] += qd * v.w[1]; a.w[1] -= qd * v.w[0]; a.w[2] += vdj;
        a.l[0] += qd * v.l[1]; a.l[1] -= qd * v.l[0];
      }
    } else {
      frame_multi(bd, io.q, R, r);
      motion_to_child(R, r, vp, v);
      motion_to_child(R, r, ap, a);
      const int K = (kind == K_QSPH || kind == K_PLANAR) ? 3 : 6;
      T x[6], xd[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        x[k] = k < K ? io.v(bd.vrow + k) : T(0);
        xd[k] = (k < K && io.vd.valid()) ? io.vd(bd.vrow + k) : T(0);
      }
      Mot<T> vj, sa, cm;
      if (kind == K_PLANAR) { joint_motion_multi<T, 3>(K_PLANAR, x, vj); joint_motion_multi<T, 3>(K_PLANAR, xd, sa); }
      else { joint_motion_multi<T, 6>(K_QFLOAT, x, vj); joint_motion_multi<T, 6>(K_QFLOAT, xd, sa); }
#pragma unroll
      for (int k = 0; k < 3; ++k) { v.w[k] += vj.w[k]; v.l[k] += vj.l[k]; }
      motion_cross(v, vj, cm);
#pragma unroll
      for (int k = 0; k < 3; ++k) { a.w[k] += cm.w[k] + sa.w[k]; a.l[k] += cm.l[k] + sa.l[k]; }
    }
    T n[3], f[3], bn[3], bf[3];
    inertia_mul(bd, a, n, f);
    bias_force(bd, v, bn, bf);
#pragma unroll
    for (int k = 0; k < 3; ++k) { n[k] += bn[k]; f[k] += bf[k]; }
    if (io.ext.valid()) {
#pragma unroll
      for (int k = 0; k < 3; ++k) { n[k] -= io.ext.get(6 * i + k); f[k] -= io.ext.get(6 * i + 3 + k); }
    }
    const int row0 = i * kRneaRowsPerBody;
#pragma unroll
    for (int k = 0; k < 3; ++k) { st.st(row0 + k, n[k]); st.st(row0 + 3 + k, f[k]); }
    if (bd.flags & F_HAS_PENDING) {
      const int row = slot_base + bd.oslot * kSlotRowsRnea;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        st.st(row + k, v.w[k]); st.st(row + 3 + k, v.l[k]);
        st.st(row + 6 + k, a.w[k]); st.st(row + 9 + k, a.l[k]);
      }
    }
    vcur = v; acur = a;
  }
  // ---- pass 2 (inward): joint wrenches and torques ----
  st.fence_st();
  T cn[3] = {T(0), T(0), T(0)}, cf[3] = {T(0), T(0), T(0)};   // contribution of the first child (registers)
  T q0c = T(0), q1c = T(0), dq = T(0), dv = T(0);
  fetch(nb - 1, false, q0n, q1n, dq, dv);
  for (int i = nb - 1; i >= 0; --i) {
    const BodyDev<T>& bd = M.body[i];
    const int kind = bd.kind;
    q0c = q0n; q1c = q1n;
    const int zf = zfn;
    const T qoff = qon;
    fetch(i - 1, false, q0n, q1n, dq, dv);
    const int row0 = i * kRneaRowsPerBody;
    T n[3], f[3];
    {
      T t[6];
      st.template ldv<6>(row0, t);
#pragma unroll
      for (int k = 0; k < 3; ++k) { n[k] = t[k]; f[k] = t[3 + k]; }
    }
    if (!(bd.flags & F_LEAF)) {
#pragma unroll
      for (int k = 0; k < 3; ++k) { n[k] += cn[k]; f[k] += cf[k]; }
    }
    if (bd.flags & F_HAS_PENDING) {
      const int row = slot_base + bd.oslot * kSlotRowsRnea;
      T t[6];
      st.fence_st();
      st.template ldv<6>(row, t);
#pragma unroll
      for (int k = 0; k < 3; ++k) { n[k] += t[k]; f[k] += t[3 + k]; }
    }
    // tau_k = S_k . w  (one-hot subspaces)
    if (kind == K_REV || kind == K_SINCOS) io.tau.st(bd.vrow, n[2]);
    else if (kind == K_PRIS) io.tau.st(bd.vrow, f[2]);
    else if (kind == K_PLANAR) { io.tau.st(bd.vrow, f[0]); io.tau.st(bd.vrow + 1, f[1]); io.tau.st(bd.vrow + 2, n[2]); }
    else if (kind == K_QSPH) { io.tau.st(bd.vrow, n[0]); io.tau.st(bd.vrow + 1, n[1]); io.tau.st(bd.vrow + 2, n[2]); }
    else if (kind == K_QFLOAT || kind == K_SPQFLOAT) {
#pragma unroll
      for (int k = 0; k < 3; ++k) { io.tau.st(bd.vrow + k, n[k]); io.tau.st(bd.vrow + 3 + k, f[k]); }
    }
    if (bd.flags & F_ROOT_CHILD) continue;
    T R[9], r[3], np[3], fp[3];
    if (zf) {
      T s, c;
      sincos_t(q0c + qoff, s, c);
      if (zf & F_ZPERP) force_to_parent_z<T, 1>(s, c, bd.pt, n, f, np, fp);
      else force_to_parent_z<T, 0>(s, c, bd.pt, n, f, np, fp);
    } else {
      if (kind == K_REV || kind == K_PRIS || kind == K_SINCOS || kind == K_FIXED) {
        Pre<T> pre; pre.q0 = q0c; pre.q1 = q1c;
        T s, c, d;
        joint_scd(kind, pre, s, c, d);
        frame_1dof(bd, s, c, d, R, r);
      } else {
        frame_multi(bd, io.q, R, r);
      }
      force_to_parent(R, r, n, f, np, fp);
    }
    if (bd.flags & F_FIRST_CHILD) {
#pragma unroll
      for (int k = 0; k < 3; ++k) { cn[k] = np[k]; cf[k] = fp[k]; }
    } else {
      const int row = slot_base + bd.pslot * kSlotRowsRnea;
      if (bd.flags & F_SLOT_INIT) {
#pragma unroll
        for (int k = 0; k < 3; ++k) { st.st(row + k, np[k]); st.st(row + 3 + k, fp[k]); }
      } else {
#pragma unroll
        for (int k = 0; k < 3; ++k) { st.add(row + k, np[k]); st.add(row + 3 + k, fp[k]); }
      }
    }
  }
}

// ==================================================================================================================
// Composite-rigid-body algorithm: M[i + j*nv] for both triangles
// ==================================================================================================================
template <class T> struct CrbaIO {
  Col<T> q;
  ColOut<T> M;
  bool lower;        // write only entries with row >= column (the triangle mass_matrix! fills, mechanism_algorithms.jl:248-272)
  // entry (r, c) of the column-major matrix; indices are warp-uniform, so the triangle test costs a uniform predicate
  RBD_HD void put(int r, int c, int nv, T val) const { if (!lower || r >= c) M.st(r + c * nv, val); }
};

// rigid-body inertia (m, h = m*com, J about the origin: xx xy xz yy yz zz)
template <class T> struct Rbi { T m; T h[3]; T J[6]; };

// child -> parent frame (motion_force_interaction.jl:160-176, same operation order)
template <class T> RBD_HD void rbi_to_parent(const T* R, const T* p, const Rbi<T>& c, Rbi<T>& o) {
  T Rmc[3], mp[3];
  mat_vec(R, c.h, Rmc);
  mp[0] = c.m * p[0]; mp[1] = c.m * p[1]; mp[2] = c.m * p[2];
  o.m = c.m;
  o.h[0] = Rmc[0] + mp[0]; o.h[1] = Rmc[1] + mp[1]; o.h[2] = Rmc[2] + mp[2];
  // Y = Rmc p^T + p Rmc^T + mp p^T (symmetric); Jnew = R J R^T - Y + tr(Y) 1
  T Y[6];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = i; j < 3; ++j) Y[sidx(i, j)] = Rmc[i] * p[j] + p[i] * Rmc[j] + mp[i] * p[j];
  const T trY = Y[0] + Y[3] + Y[5];
  T t[9];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int k = 0; k < 3; ++k)
      t[3 * i + k] = R[3 * i] * c.J[sidx(0, k)] + R[3 * i + 1] * c.J[sidx(1, k)] + R[3 * i + 2] * c.J[sidx(2, k)];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = i; j < 3; ++j) {
      T s = t[3 * i] * R[3 * j] + t[3 * i + 1] * R[3 * j + 1] + t[3 * i + 2] * R[3 * j + 2] - Y[sidx(i, j)];
      if (i == j) s += trY;
      o.J[sidx(i, j)] = s;
    }
}

// component `c` (0..5 of [n; f]) of a 6-vector; select chain, no runtime array indexing (registers stay registers)
template <class T> RBD_HD T comp6(const T* n, const T* f, int c) {
  return c == 0 ? n[0] : (c == 1 ? n[1] : (c == 2 ? n[2] : (c == 3 ? f[0] : (c == 4 ? f[1] : f[2]))));
}
RBD_HD int kind_nv_dev(int k) {
  return (k == K_REV || k == K_PRIS || k == K_SINCOS) ? 1 : (k == K_FIXED ? 0 : ((k == K_PLANAR || k == K_QSPH) ? 3 : 6));
}
RBD_HD int kind_nq_dev(int k) {
  return (k == K_REV || k == K_PRIS) ? 1 : (k == K_FIXED ? 0 : (k == K_SINCOS ? 2 : (k == K_PLANAR ? 3 : (k == K_QSPH ? 4 : (k == K_QFLOAT ? 7 : 6)))));
}
// one-hot component driven by velocity coordinate k of a joint of the given kind
RBD_HD int sub_comp(int kind, int k) {
  return (kind == K_REV || kind == K_SINCOS) ? 2 : (kind == K_PRIS ? 5 : sub_index(kind == K_PLANAR ? K_PLANAR : K_QFLOAT, k));
}
template <class T> RBD_HD void rbi_mul(const Rbi<T>& I, const Mot<T>& v, T* n, T* f) {
  const T* J = I.J; const T* h = I.h;
  n[0] = J[0] * v.w[0] + J[1] * v.w[1] + J[2] * v.w[2] + (h[1] * v.l[2] - h[2] * v.l[1]);
  n[1] = J[1] * v.w[0] + J[3] * v.w[1] + J[4] * v.w[2] + (h[2] * v.l[0] - h[0] * v.l[2]);
  n[2] = J[2] * v.w[0] + J[4] * v.w[1] + J[5] * v.w[2] + (h[0] * v.l[1] - h[1] * v.l[0]);
  f[0] = I.m * v.l[0] - (h[1] * v.w[2] - h[2] * v.w[1]);
  f[1] = I.m * v.l[1] - (h[2] * v.w[0] - h[0] * v.w[2]);
  f[2] = I.m * v.l[2] - (h[0] * v.w[1] - h[1] * v.w[0]);
}

// ST: Stash<T, STRIDE> on the device / host tier, SymStash when the algorithm is traced for a model-specialised kernel (rbd_sym.h)
template <class T, class ST, int KMAX>
RBD_HD void crba_sample(const ModelDev<T>& M, const CrbaIO<T>& io, const ST& st) {
  const int nb = M.nb, nv = M.nv;
  const int slot_base = nb * kCrbaRowsPerBody;
  // pass 0: sin / cos (or prismatic displacement) of every 1-DoF joint
  for (int i = 0; i < nb; ++i) {
    const BodyDev<T>& bd = M.body[i];
    const int kind = bd.kind;
    if (kind == K_REV || kind == K_PRIS || kind == K_SINCOS) {
      Pre<T> pre;
      pre.q0 = io.q(bd.qrow);
      pre.q1 = kind == K_SINCOS ? io.q(bd.qrow + 1) : T(0);
      T s, c, d;
      joint_scd(kind, pre, s, c, d, bd.qoff);        // fast classes (rbd_types.h): sin / cos of q + qoff, used with E = [P] Rz below
      st.st(2 * i, kind == K_PRIS ? d : s);
      st.st(2 * i + 1, c);
    }
  }
  auto frame_of = [&](int j, T* R, T* r) {
    const BodyDev<T>& b = M.body[j];
    const int kind = b.kind;
    if (b.flags & (F_ZPAR | F_ZPERP)) {             // R = [P] Rz(s, c) written out, r = pt
      const T sn = st.ld(2 * j), cs = st.ld(2 * j + 1);
      if (b.flags & F_ZPERP) {
        R[0] = T(0); R[1] = T(0); R[2] = T(1);  R[3] = cs; R[4] = -sn; R[5] = T(0);  R[6] = sn; R[7] = cs; R[8] = T(0);
      } else {
        R[0] = cs; R[1] = -sn; R[2] = T(0);  R[3] = sn; R[4] = cs; R[5] = T(0);  R[6] = T(0); R[7] = T(0); R[8] = T(1);
      }
      r[0] = b.pt[0]; r[1] = b.pt[1]; r[2] = b.pt[2];
    } else if (kind == K_REV || kind == K_SINCOS) frame_1dof(b, st.ld(2 * j), st.ld(2 * j + 1), T(0), R, r);
    else if (kind == K_PRIS) frame_1dof(b, T(0), T(1), st.ld(2 * j), R, r);
    else if (kind == K_FIXED) frame_1dof(b, T(0), T(1), T(0), R, r);
    else frame_multi(b, io.q, R, r);
  };
  Rbi<T> carry;
  carry.m = T(0);
#pragma unroll
  for (int k = 0; k < 3; ++k) carry.h[k] = T(0);
#pragma unroll
  for (int k = 0; k < 6; ++k) carry.J[k] = T(0);
  for (int i = nb - 1; i >= 0; --i) {
    const BodyDev<T>& bd = M.body[i];
    const int kind = bd.kind;
    Rbi<T> ic;
    ic.m = bd.m;
#pragma unroll
    for (int k = 0; k < 3; ++k) ic.h[k] = bd.h[k];
#pragma unroll
    for (int k = 0; k < 6; ++k) ic.J[k] = bd.J[k];
    if (!(bd.flags & F_LEAF)) {
      ic.m += carry.m;
#pragma unroll
      for (int k = 0; k < 3; ++k) ic.h[k] += carry.h[k];
#pragma unroll
      for (int k = 0; k < 6; ++k) ic.J[k] += carry.J[k];
    }
    if (bd.flags & F_HAS_PENDING) {
      const int row = slot_base + bd.oslot * kSlotRowsCrba;
      ic.m += st.ld(row);
#pragma unroll
      for (int k = 0; k < 3; ++k) ic.h[k] += st.ld(row + 1 + k);
#pragma unroll
      for (int k = 0; k < 6; ++k) ic.J[k] += st.ld(row + 4 + k);
    }
    // ---- columns of M owned by this joint: F_k = Ic S_k, walked up the support path ----
    const int K = kind_nv_dev(kind);
    if (K > 0) {
      T Fn[KMAX][3], Ff[KMAX][3];
#pragma unroll
      for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
          // S_k = unit vector e_c, c = sub_index: F = Ic e_c  (n = J e + h x e_lin ; f = m e_lin - h x e_ang)
          const int c = sub_comp(kind, k);
          Mot<T> e;
#pragma unroll
          for (int d = 0; d < 3; ++d) { e.w[d] = (c == d) ? T(1) : T(0); e.l[d] = (c == 3 + d) ? T(1) : T(0); }
          rbi_mul(ic, e, Fn[k], Ff[k]);
        }
      }
      // diagonal block
#pragma unroll
      for (int k = 0; k < KMAX; ++k)
#pragma unroll
        for (int l = 0; l < KMAX; ++l)
          if (k < K && l < K) {
            io.put(bd.vrow + l, bd.vrow + k, nv, comp6(Fn[k], Ff[k], sub_comp(kind, l)));
          }
      // ancestors (decreasing preorder index) and unrelated earlier bodies (zeros)
      int anc = bd.parent;
      int j = i;          // frame in which F currently lives
      for (int jj = i - 1; jj >= 0; --jj) {
        const BodyDev<T>& bj = M.body[jj];
        const int Kj = kind_nv_dev(bj.kind);
        if (jj == anc) {
          const BodyDev<T>& bs = M.body[j];
          if (bs.flags & (F_ZPAR | F_ZPERP)) {
            const T sn = st.ld(2 * j), cs = st.ld(2 * j + 1);
            const bool perp = (bs.flags & F_ZPERP) != 0;
#pragma unroll
            for (int k = 0; k < KMAX; ++k)
              if (k < K) {
                T np[3], fp[3];
                if (perp) force_to_parent_z<T, 1>(sn, cs, bs.pt, Fn[k], Ff[k], np, fp);
                else force_to_parent_z<T, 0>(sn, cs, bs.pt, Fn[k], Ff[k], np, fp);
#pragma unroll
                for (int d = 0; d < 3; ++d) { Fn[k][d] = np[d]; Ff[k][d] = fp[d]; }
              }
          } else {
            T R[9], r[3];
            frame_of(j, R, r);
#pragma unroll
            for (int k = 0; k < KMAX; ++k)
              if (k < K) {
                T np[3], fp[3];
                force_to_parent(R, r, Fn[k], Ff[k], np, fp);
#pragma unroll
                for (int d = 0; d < 3; ++d) { Fn[k][d] = np[d]; Ff[k][d] = fp[d]; }
              }
          }
          j = jj;
          anc = bj.parent;
          for (int l = 0; l < Kj; ++l) {
            const int cl = sub_comp(bj.kind, l);
#pragma unroll
            for (int k = 0; k < KMAX; ++k)
              if (k < K) {
                const T val = comp6(Fn[k], Ff[k], cl);
                io.put(bj.vrow + l, bd.vrow + k, nv, val);
                io.put(bd.vrow + k, bj.vrow + l, nv, val);
              }
          }
        } else {
          for (int l = 0; l < Kj; ++l)
#pragma unroll
            for (int k = 0; k < KMAX; ++k)
              if (k < K) {
                io.put(bj.vrow + l, bd.vrow + k, nv, T(0));
                io.put(bd.vrow + k, bj.vrow + l, nv, T(0));
              }
        }
      }
    }
    // ---- hand the composite inertia to the parent ----
    if (bd.flags & F_ROOT_CHILD) continue;
    T R[9], r[3];
    frame_of(i, R, r);
    Rbi<T> up;
    rbi_to_parent(R, r, ic, up);
    if (bd.flags & F_FIRST_CHILD) carry = up;
    else {
      const int row = slot_base + bd.pslot * kSlotRowsCrba;
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
}

}  // namespace rbd
