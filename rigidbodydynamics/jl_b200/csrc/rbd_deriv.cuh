// Analytic first derivatives of forward dynamics (SURVEY 8(f) rank 3):  dv̇/dq, dv̇/dv  of  v̇ = M(q)^-1 (tau - c(q, v))
// for a whole batch -- what the reference obtains by pushing ForwardDiff.Dual numbers through dynamics! one chunk of partials
// at a time (examples/5. Derivatives and gradients using ForwardDiff, test/test_mechanism_algorithms.jl:600-675).
//
//   dv̇/du = -M^-1 (d ID(q, v, v̇) / du) at fixed v̇ = FD(q, v, tau)              u = q (tangent space) or v
//
// The derivatives of inverse dynamics are taken in closed form from ROOT-frame quantities, the frame the reference keeps all
// its caches in (mechanism_state.jl:604-682).  Moving joint J along its velocity coordinate j moves the subtree of J rigidly
// by the twist S_j, so body-fixed vectors of the subtree change by S_j x (.) / S_j x* (.), and what is left over is
//   Psi_dot_j  = v_parent x S_j                        (the part of the subtree's velocities that does NOT follow)
//   Psi_ddot_j = a_parent x S_j + v_parent x Psi_dot_j
// (a includes the fictitious root acceleration -g, spatial_accelerations! mechanism_algorithms.jl:387-417).  With the
// subtree sums (plain additions in the root frame, like _update_crb_inertias! mechanism_state.jl:852-868)
//   Ic_K = sum I_i          G_K = sum [ x -> I_i (x x v_i) + x x* (I_i v_i) + v_i x* (I_i x) ]          F_K = sum f_i
// the entries are, for K a descendant-or-self of J (k a velocity coordinate of K, j of J):
//   d tau_k / d q_j = S_k . (Ic_K Psi_ddot_j + G_K Psi_dot_j)             d tau_j / d q_k = S_j . (S_k x* F_K + same with K's Psi)  [strict ancestor]
//   d tau_k / d v_j = S_k . (Ic_K Sdp_j + G_K S_j),  Sdp_j = (v_J + v_parent) x S_j
//   M_kj            = S_k . (Ic_K S_j)                                     (mass_matrix!, mechanism_algorithms.jl:248-272)
// and zero for unrelated pairs.  "d/dq_j" is the derivative along the joint's own velocity coordinate, i.e. along
// q̇ = velocity_to_configuration_derivative(e_j) (mechanism_state.jl:905-910): for 1-DoF joints that is d/dq itself; for
// quaternion joints it is the tangent-space derivative [dv̇/dq_raw] * velocity_to_configuration_derivative_jacobian.
//
// External wrenches W_i (root frame, fixed while the subtree moves) enter ID as f_i = I a + v x* I v - W_i.  Only the inertial part
// moves with a subtree, so with W_K = sum W_i over K's subtree the closed form gains one term, for K a descendant-or-self of J:
//   d tau_k / d q_j += S_k . (S_j x* W_K)          (from d S_k = S_j x S_k acting on -W_K)
// while the strict-ancestor rows keep S_j x* F_K with the INERTIAL F_K, and d tau / d v does not change.  tau itself is
// S_k . (F_K - W_K).
//
// M is then factored per sample as L^T D L with the tree's own sparsity (entry (k, i) only for i an ancestor of k in the
// chain of velocity coordinates) and every column of the right-hand sides is solved in place: d ID / dq, d ID / dv and, for
// d v̇ / d tau = M^-1, the constant columns -e_j.  The inverse-dynamics Jacobians are the pair entries themselves (no solve).
//
// Work split (rbd_deriv.cu): world pass = one thread per sample; subtree sums = one thread per (sample, component);
// pair entries = one thread per (sample, body); factor = one thread per sample; solves = one thread per (sample, column).
// Intermediates live in a global scratch, rows x chunk with the sample index fastest.
#pragma once
#include "rbd_kin.cuh"

namespace rbd {

constexpr int kMaxDofs = 128;
constexpr int kMaxNnz = 4096;    // stored entries of M (sum of depth + 1): a 89-coordinate serial chain, or any humanoid
constexpr int kDofRows = 24;     // S, Psi_dot, Psi_ddot, Sdp
constexpr int kBodyRows = 52;    // Ic (m, h, J: 10), G (36, row-major), F (6)

struct DerivDev {
  int32_t nb, nv, nnz;           // nnz: stored entries of M / its factor (row p holds depth[p] + 1 of them)
  int32_t dof_base, body_base, h_base, rows;   // scratch rows
  int32_t w_base;                // rows of W (6 per body, behind M's entries) when the call has external wrenches, else 0
  int16_t pdof0[kMaxBodies + 1]; // preorder body -> its first velocity coordinate in PREORDER numbering
  int16_t vrow[kMaxDofs];        // preorder coordinate -> row of v (reference order)
  int16_t pdof[kMaxDofs];        // row of v -> preorder coordinate
  int16_t lambda[kMaxDofs];      // parent coordinate in the chain expansion of the tree, -1 at the top
  int16_t depth[kMaxDofs];       // number of ancestors
  int16_t rowstart[kMaxDofs];    // entry (p, a) with a ancestor-or-self of p lives at h_base + rowstart[p] + depth[a]
  int16_t dsub[kMaxDofs];        // size of the coordinate's subtree: descendants-or-self are [p, p + dsub[p])
  int16_t comp[kMaxDofs];        // one-hot component of [w; l] in the canonical body frame
};
// anc[rowstart[p] + d] = the ancestor-or-self of coordinate p at depth d (d = 0 .. depth[p]; the last one is p itself): the same
// index as the entry (p, that ancestor) of M, so the walks up the tree are loops over consecutive table entries instead of
// pointer chases through lambda[]
struct DerivAnc { int16_t anc[kMaxNnz]; };

// Host side: tables from the flattened model (preorder bodies).
template <class T> inline bool build_deriv_dev(const ModelDev<T>& M, DerivDev& D, DerivAnc& A) {
  std::memset(&D, 0, sizeof(D));
  std::memset(&A, 0, sizeof(A));
  D.nb = M.nb; D.nv = M.nv;
  if (M.nv > kMaxDofs) return false;
  int p = 0;
  int last[kMaxBodies];          // last coordinate at or above body i (-1 = none)
  for (int i = 0; i < M.nb; ++i) {
    const BodyDev<T>& b = M.body[i];
    const int K = kind_nv(b.kind);
    D.pdof0[i] = (int16_t)p;
    int up = b.parent >= 0 ? last[b.parent] : -1;
    for (int k = 0; k < K; ++k, ++p) {
      D.vrow[p] = (int16_t)(b.vrow + k);
      D.pdof[b.vrow + k] = (int16_t)p;
      D.lambda[p] = (int16_t)up;
      D.depth[p] = (int16_t)(up >= 0 ? D.depth[up] + 1 : 0);
      D.comp[p] = (int16_t)((b.kind == K_REV || b.kind == K_SINCOS) ? 2 : (b.kind == K_PRIS ? 5 : sub_index(b.kind == K_PLANAR ? K_PLANAR : K_QFLOAT, k)));
      up = p;
    }
    last[i] = up;
  }
  D.pdof0[M.nb] = (int16_t)p;
  for (int i = M.nb + 1; i <= kMaxBodies; ++i) D.pdof0[i] = (int16_t)p;
  int nnz = 0;
  for (int k = 0; k < M.nv; ++k) { D.rowstart[k] = (int16_t)nnz; nnz += D.depth[k] + 1; D.dsub[k] = 1; }
  if (nnz > kMaxNnz) return false;
  for (int k = 0; k < M.nv; ++k)
    for (int a = k; a >= 0; a = D.lambda[a]) A.anc[D.rowstart[k] + D.depth[a]] = (int16_t)a;
  for (int k = M.nv - 1; k >= 0; --k) if (D.lambda[k] >= 0) D.dsub[D.lambda[k]] += D.dsub[k];
  D.nnz = nnz;
  D.dof_base = 0;
  D.body_base = kDofRows * M.nv;
  D.h_base = D.body_base + kBodyRows * M.nb;
  D.rows = D.h_base + nnz;
  return true;
}

// External wrenches: 6 more scratch rows per body (W_i, then the subtree sums W_K).  Without them the layout is unchanged.
inline void deriv_dev_add_wrenches(DerivDev& D) {
  D.w_base = D.rows;
  D.rows += 6 * D.nb;
}
// v x* f for a force vector (n, f)
template <class T> RBD_HD void force_cross(const Mot<T>& v, const T* n, const T* f, T* on, T* of) {
  T a[3], b[3];
  cross3(v.w, n, a);
  cross3(v.l, f, b);
  on[0] = a[0] + b[0]; on[1] = a[1] + b[1]; on[2] = a[2] + b[2];
  cross3(v.w, f, of);
}
template <class T> RBD_HD T dot6(const Mot<T>& S, const T* y) {
  return S.w[0] * y[0] + S.w[1] * y[1] + S.w[2] * y[2] + S.l[0] * y[3] + S.l[1] * y[4] + S.l[2] * y[5];
}
// rows row .. row + 5 of a scratch column; the address walks by ld (one 64-bit add per element instead of a multiply each)
template <class T> RBD_HD void load_mot(const T* s, int64_t ld, int row, Mot<T>& m) {
  const T* p = s + (int64_t)row * ld;
#pragma unroll
  for (int k = 0; k < 3; ++k) { m.w[k] = *p; p += ld; }
#pragma unroll
  for (int k = 0; k < 3; ++k) { m.l[k] = *p; p += ld; }
}
template <class T> RBD_HD void store_mot(T* s, int64_t ld, int row, const Mot<T>& m) {
  T* p = s + (int64_t)row * ld;
#pragma unroll
  for (int k = 0; k < 3; ++k) { *p = m.w[k]; p += ld; }
#pragma unroll
  for (int k = 0; k < 3; ++k) { *p = m.l[k]; p += ld; }
}

// ------------------------------------------------------------------------------------------------------------------
// 1. world pass: one thread per sample.  s = this sample's scratch column, sld its leading dimension.
// ------------------------------------------------------------------------------------------------------------------
template <class T> struct DerivIO {
  Col<T> q, v, vd;
  Col<T> wext{nullptr, 0};       // root-frame external wrenches (rows 6 refidx + c, as rbd_dynamics), read when EXT
  T* s;
  int64_t sld;
  bool active;
};

// EXT: also store each body's external wrench W_i in rows D.w_base + 6 i (deriv_dev_add_wrenches)
template <class T, class ST, bool EXT = false>
RBD_HD void deriv_world_sample(const ModelDev<T>& M, const DerivDev& D, const DerivIO<T>& io, const ST& st) {
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
    Mot<T> jt, ja;
#pragma unroll
    for (int k = 0; k < 3; ++k) jt.w[k] = jt.l[k] = ja.w[k] = ja.l[k] = T(0);
    const int nvj = kind_nv_dev(bd.kind);
    for (int k = 0; k < nvj; ++k) {
      Mot<T> S;
      world_subspace(w, sub_comp(bd.kind, k), S);
      const T x = io.v(bd.vrow + k), xd = io.vd(bd.vrow + k);
#pragma unroll
      for (int c = 0; c < 3; ++c) { jt.w[c] += x * S.w[c]; jt.l[c] += x * S.l[c]; ja.w[c] += xd * S.w[c]; ja.l[c] += xd * S.l[c]; }
    }
    Mot<T> tw, a, cm, tsum;
    motion_cross(twp, jt, cm);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      tw.w[k] = twp.w[k] + jt.w[k]; tw.l[k] = twp.l[k] + jt.l[k];
      a.w[k] = ap.w[k] + cm.w[k] + ja.w[k]; a.l[k] = ap.l[k] + cm.l[k] + ja.l[k];
      tsum.w[k] = tw.w[k] + twp.w[k]; tsum.l[k] = tw.l[k] + twp.l[k];
    }
    // per velocity coordinate: S, Psi_dot, Psi_ddot, Sdp
    for (int k = 0; k < nvj; ++k) {
      Mot<T> S, pd, pdd, t1, t2, sdp;
      world_subspace(w, sub_comp(bd.kind, k), S);
      motion_cross(twp, S, pd);
      motion_cross(ap, S, t1);
      motion_cross(twp, pd, t2);
#pragma unroll
      for (int c = 0; c < 3; ++c) { pdd.w[c] = t1.w[c] + t2.w[c]; pdd.l[c] = t1.l[c] + t2.l[c]; }
      motion_cross(tsum, S, sdp);
      if (io.active) {
        const int row = D.dof_base + kDofRows * (D.pdof0[i] + k);
        store_mot(io.s, io.sld, row, S);
        store_mot(io.s, io.sld, row + 6, pd);
        store_mot(io.s, io.sld, row + 12, pdd);
        store_mot(io.s, io.sld, row + 18, sdp);
      }
    }
    // body: root-frame inertia, net wrench, G
    Rbi<T> Ib, Iw;
    body_rbi(bd, Ib);
    rbi_to_parent(w.R, w.p, Ib, Iw);
    T hn[3], hf[3], fn[3], ff[3], bn[3], bf[3];
    rbi_mul(Iw, tw, hn, hf);
    rbi_mul(Iw, a, fn, ff);
    force_cross(tw, hn, hf, bn, bf);
    if (io.active) {
      const int row = D.body_base + kBodyRows * i;
      io.s[(int64_t)row * io.sld] = Iw.m;
#pragma unroll
      for (int k = 0; k < 3; ++k) io.s[(int64_t)(row + 1 + k) * io.sld] = Iw.h[k];
#pragma unroll
      for (int k = 0; k < 6; ++k) io.s[(int64_t)(row + 4 + k) * io.sld] = Iw.J[k];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        io.s[(int64_t)(row + 46 + k) * io.sld] = fn[k] + bn[k];
        io.s[(int64_t)(row + 49 + k) * io.sld] = ff[k] + bf[k];
      }
      if (EXT) {
#pragma unroll
        for (int k = 0; k < 6; ++k) io.s[(int64_t)(D.w_base + 6 * i + k) * io.sld] = io.wext(6 * bd.refidx + k);
      }
      // G e_c = I (e_c x v) + e_c x* (I v) + v x* (I e_c)
#pragma unroll
      for (int c = 0; c < 6; ++c) {
        Mot<T> e, ev;
#pragma unroll
        for (int d = 0; d < 3; ++d) { e.w[d] = (c == d) ? T(1) : T(0); e.l[d] = (c == 3 + d) ? T(1) : T(0); }
        motion_cross(e, tw, ev);
        T y1n[3], y1f[3], y2n[3], y2f[3], ien[3], ief[3], y3n[3], y3f[3];
        rbi_mul(Iw, ev, y1n, y1f);
        force_cross(e, hn, hf, y2n, y2f);
        rbi_mul(Iw, e, ien, ief);
        force_cross(tw, ien, ief, y3n, y3f);
#pragma unroll
        for (int d = 0; d < 3; ++d) {
          io.s[(int64_t)(row + 10 + 6 * d + c) * io.sld] = y1n[d] + y2n[d] + y3n[d];
          io.s[(int64_t)(row + 10 + 6 * (3 + d) + c) * io.sld] = y1f[d] + y2f[d] + y3f[d];
        }
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
}

// ------------------------------------------------------------------------------------------------------------------
// 2. subtree sums of (Ic, G, F): one thread per (sample, component c of the 52); of W: one per (sample, component c of the 6)
// ------------------------------------------------------------------------------------------------------------------
template <class T> RBD_HD void deriv_accumulate(const ModelDev<T>& M, const DerivDev& D, T* s, int64_t sld, int c) {
  for (int i = M.nb - 1; i > 0; --i) {
    const int par = M.body[i].parent;
    if (par < 0) continue;
    s[(int64_t)(D.body_base + kBodyRows * par + c) * sld] += s[(int64_t)(D.body_base + kBodyRows * i + c) * sld];
  }
}
template <class T> RBD_HD void deriv_accumulate_wrench(const ModelDev<T>& M, const DerivDev& D, T* s, int64_t sld, int c) {
  for (int i = M.nb - 1; i > 0; --i) {
    const int par = M.body[i].parent;
    if (par < 0) continue;
    s[(int64_t)(D.w_base + 6 * par + c) * sld] += s[(int64_t)(D.w_base + 6 * i + c) * sld];
  }
}

// ------------------------------------------------------------------------------------------------------------------
// 3. pair entries: one thread per (sample, body K).  Writes d tau / dq and d tau / dv into dq / dv (column-major nv x nv like
//    M.data, rows x batch) and the related entries of M into the scratch.  EXT: with the wrench term (W_K from the scratch).
//    TAU: also K's rows of tau = ID(q, v, v̇, W).
// ------------------------------------------------------------------------------------------------------------------
template <class T> RBD_HD void apply_IG(const Rbi<T>& I, const T* G, const Mot<T>& xi, const Mot<T>& xg, T* y) {
  T n[3], f[3];
  rbi_mul(I, xi, n, f);
  const T x[6] = {xg.w[0], xg.w[1], xg.w[2], xg.l[0], xg.l[1], xg.l[2]};
#pragma unroll
  for (int r = 0; r < 6; ++r) {
    T acc = r < 3 ? n[r] : f[r - 3];
#pragma unroll
    for (int c = 0; c < 6; ++c) acc += G[6 * r + c] * x[c];
    y[r] = acc;
  }
}

template <class T, bool EXT = false, bool TAU = false>
RBD_HD void deriv_pairs(const DerivDev& D, const DerivAnc& A, T* s, int64_t sld, T* dq, T* dv, int64_t ld, int K, bool active,
                        T* tau = nullptr) {
  const int nv = D.nv;
  const int pk0 = D.pdof0[K], nk = D.pdof0[K + 1] - pk0;
  if (nk == 0) return;
  Rbi<T> Ic;
  T G[36], Fn[3], Ff[3], Wn[3], Wf[3];
  {
    const T* p = s + (int64_t)(D.body_base + kBodyRows * K) * sld;
    Ic.m = *p; p += sld;
#pragma unroll
    for (int k = 0; k < 3; ++k) { Ic.h[k] = *p; p += sld; }
#pragma unroll
    for (int k = 0; k < 6; ++k) { Ic.J[k] = *p; p += sld; }
#pragma unroll
    for (int k = 0; k < 36; ++k) { G[k] = *p; p += sld; }
#pragma unroll
    for (int k = 0; k < 3; ++k) { Fn[k] = *p; p += sld; }
#pragma unroll
    for (int k = 0; k < 3; ++k) { Ff[k] = *p; p += sld; }
  }
  if (EXT) {
    const T* p = s + (int64_t)(D.w_base + 6 * K) * sld;
#pragma unroll
    for (int k = 0; k < 3; ++k) { Wn[k] = p[k * sld]; Wf[k] = p[(3 + k) * sld]; }
  }
  if (TAU) {
    T f[6];
#pragma unroll
    for (int k = 0; k < 3; ++k) { f[k] = EXT ? Fn[k] - Wn[k] : Fn[k]; f[3 + k] = EXT ? Ff[k] - Wf[k] : Ff[k]; }
    for (int kk = 0; kk < nk; ++kk) {
      Mot<T> Sk;
      load_mot(s, sld, D.dof_base + kDofRows * (pk0 + kk), Sk);
      if (active) tau[(int64_t)D.vrow[pk0 + kk] * ld] = dot6(Sk, f);
    }
  }
  // all coordinates at or above K, deepest first: the ancestor list of K's last coordinate
  const int plast = pk0 + nk - 1, rl = D.rowstart[plast];
  for (int dj = D.depth[plast]; dj >= 0; --dj) {
    const int pj = A.anc[rl + dj];
    const int rj = D.dof_base + kDofRows * pj;
    Mot<T> Sj, pd, pdd, sdp;
    {
      const T* p = s + (int64_t)rj * sld;
      T t[24];
#pragma unroll
      for (int k = 0; k < 24; ++k) { t[k] = *p; p += sld; }
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        Sj.w[k] = t[k]; Sj.l[k] = t[3 + k]; pd.w[k] = t[6 + k]; pd.l[k] = t[9 + k];
        pdd.w[k] = t[12 + k]; pdd.l[k] = t[15 + k]; sdp.w[k] = t[18 + k]; sdp.l[k] = t[21 + k];
      }
    }
    T yq[6], yv[6], ym[6], yw[6];
    apply_IG(Ic, G, pdd, pd, yq);
    apply_IG(Ic, G, sdp, Sj, yv);
    rbi_mul(Ic, Sj, ym, ym + 3);
    // K's own rows: yq + S_j x* W_K.  yq itself stays inertial for the strict-ancestor rows below.
#pragma unroll
    for (int c = 0; c < 6; ++c) yw[c] = yq[c];
    if (EXT) {
      T wn[3], wf[3];
      force_cross(Sj, Wn, Wf, wn, wf);
#pragma unroll
      for (int c = 0; c < 3; ++c) { yw[c] += wn[c]; yw[3 + c] += wf[c]; }
    }
    const int64_t colj = (int64_t)nv * D.vrow[pj];
    for (int kk = 0; kk < nk; ++kk) {
      const int pk = pk0 + kk;
      Mot<T> Sk;
      load_mot(s, sld, D.dof_base + kDofRows * pk, Sk);
      if (active) {
        dq[(colj + D.vrow[pk]) * ld] = dot6(Sk, yw);
        dv[(colj + D.vrow[pk]) * ld] = dot6(Sk, yv);
        if (pj <= pk) s[(int64_t)(D.h_base + D.rowstart[pk] + D.depth[pj]) * sld] = dot6(Sk, ym);
      }
    }
    if (pj >= pk0) {
      // j belongs to K itself: rows of the strict ancestors,  S_k' . (S_j x* F_K + y)
      T cn[3], cf[3];
      force_cross(Sj, Fn, Ff, cn, cf);
#pragma unroll
      for (int c = 0; c < 3; ++c) { yq[c] += cn[c]; yq[3 + c] += cf[c]; }
      for (int d2 = D.depth[pk0] - 1; d2 >= 0; --d2) {
        const int p2 = A.anc[D.rowstart[pk0] + d2];
        Mot<T> Sa;
        load_mot(s, sld, D.dof_base + kDofRows * p2, Sa);
        if (active) {
          dq[(colj + D.vrow[p2]) * ld] = dot6(Sa, yq);
          dv[(colj + D.vrow[p2]) * ld] = dot6(Sa, yv);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// 4. M = L^T D L in place on the scratch, one thread per sample; the diagonal is left INVERTED.
// ------------------------------------------------------------------------------------------------------------------
template <class T> RBD_HD void deriv_factor(const DerivDev& D, const DerivAnc& A, T* H, int64_t sld) {
  for (int k = D.nv - 1; k >= 0; --k) {
    const int rk = D.rowstart[k], dk = D.depth[k];
    const T inv = T(1) / H[(int64_t)(rk + dk) * sld];
    for (int di = dk - 1; di >= 0; --di) {
      const int ri = D.rowstart[A.anc[rk + di]];
      const T a = H[(int64_t)(rk + di) * sld] * inv;
      for (int d = di; d >= 0; --d) H[(int64_t)(ri + d) * sld] -= a * H[(int64_t)(rk + d) * sld];
    }
    for (int di = 0; di < dk; ++di) H[(int64_t)(rk + di) * sld] *= inv;
    H[(int64_t)(rk + dk) * sld] = inv;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// 5. one column of  X = -M^-1 R  in place.  x: per-thread vector of nv entries (shared memory, stride XS);
//    H(row) reads the factor; col: this sample's column of the nv x nv array, rows x batch.  unit: R = -e_vj (a column of
//    d v̇ / d tau = M^-1; nothing is read), whose only non-zero row is pj itself.
// ------------------------------------------------------------------------------------------------------------------
template <class T, class HF>
RBD_HD void deriv_solve_column(const DerivDev& D, const DerivAnc& A, const HF& H, T* x, int xs, T* col, int64_t ld, int vj, bool active,
                               bool unit = false) {
  const int nv = D.nv;
  const int pj = D.pdof[vj];
  const int lo = pj, hi = unit ? pj + 1 : pj + D.dsub[pj];
  // right-hand side: non-zero only on the subtree and the ancestors of pj
  for (int p = 0; p < nv; ++p) {
    const bool rel = (p >= lo && p < hi) || (pj >= p && pj < p + D.dsub[p]);
    x[p * xs] = unit ? (p == pj ? T(-1) : T(0)) : rel ? col[(int64_t)D.vrow[p] * ld] : T(0);
  }
  // L^-T: coordinates push to their ancestors; only the subtree and the ancestor chain of pj carry anything.  The ancestors of
  // one coordinate are distinct, so four read-modify-writes go out together (the compiler cannot know they do not alias).
  for (int i = hi - 1; i >= 0; i = (i > lo ? i - 1 : D.lambda[i])) {
    const T xi = x[i * xs];
    const int ri = D.rowstart[i];
    int d = D.depth[i] - 1;
    for (; d >= 3; d -= 4) {
      const int j0 = A.anc[ri + d], j1 = A.anc[ri + d - 1], j2 = A.anc[ri + d - 2], j3 = A.anc[ri + d - 3];
      const T h0 = H(ri + d), h1 = H(ri + d - 1), h2 = H(ri + d - 2), h3 = H(ri + d - 3);
      const T x0 = x[j0 * xs], x1 = x[j1 * xs], x2 = x[j2 * xs], x3 = x[j3 * xs];
      x[j0 * xs] = x0 - h0 * xi; x[j1 * xs] = x1 - h1 * xi; x[j2 * xs] = x2 - h2 * xi; x[j3 * xs] = x3 - h3 * xi;
    }
    for (; d >= 0; --d) { const int j = A.anc[ri + d]; x[j * xs] -= H(ri + d) * xi; }
  }
  for (int p = 0; p < nv; ++p) x[p * xs] *= H(D.rowstart[p] + D.depth[p]);
  // L^-1: coordinates pull from their ancestors
  for (int i = 0; i < nv; ++i) {
    T acc = x[i * xs];
    const int ri = D.rowstart[i];
    for (int d = D.depth[i] - 1; d >= 0; --d) acc -= H(ri + d) * x[A.anc[ri + d] * xs];
    x[i * xs] = acc;
    if (active) col[(int64_t)D.vrow[i] * ld] = -acc;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// 6. inverse-dynamics Jacobians: one thread per (sample, column vj).  Zeroes the rows of dq / dv that deriv_pairs leaves alone
//    (pairs unrelated in the tree) and, when Mo != NULL, writes column vj of M, both triangles, from the scratch entries.
// ------------------------------------------------------------------------------------------------------------------
template <class T>
RBD_HD void deriv_expand_column(const DerivDev& D, const T* H, int64_t sld, T* dq, T* dv, T* Mo, int64_t ld, int vj, bool active) {
  const int nv = D.nv;
  const int pj = D.pdof[vj];
  for (int vi = 0; vi < nv; ++vi) {
    const int p = D.pdof[vi];
    const int64_t o = ((int64_t)vj * nv + vi) * ld;
    const bool below = p >= pj && p < pj + D.dsub[pj], above = pj >= p && pj < p + D.dsub[p];
    if (!active) continue;
    if (!below && !above) {
      dq[o] = T(0);
      dv[o] = T(0);
      if (Mo) Mo[o] = T(0);
    } else if (Mo) {
      Mo[o] = below ? H[(int64_t)(D.rowstart[p] + D.depth[pj]) * sld] : H[(int64_t)(D.rowstart[pj] + D.depth[p]) * sld];
    }
  }
}

}  // namespace rbd
