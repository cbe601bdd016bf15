// dynamics! for mechanisms with kinematic loops (SURVEY 8(f) rank 4, second half): one thread per sample, one launch.
// Reference (relative to the reference's src/):
//   non-tree joint transform           mechanism_state.jl:703-711   inv(T_pred X_pred) (T_succ X_succ)
//   constraint wrench subspaces        mechanism_state.jl:786-793   basis (frame after the joint) -> root frame by T_succ X_succ
//   constraint_jacobian!               mechanism_algorithms.jl:574-598   K[c, v_k] = +-T_c . S_k along path(pred, succ)
//   constraint_bias!                   mechanism_algorithms.jl:630-673   k_c = T_c . (v_s x v_p + b_s - b_p - stab)
//   Baumgarte term (SE3 PD, linearised) pdcontrol.jl:35,109-122, spatial/util.jl:178-183
//   dynamics_solve! (BLAS branch)      mechanism_algorithms.jl:747-822
// Phases of loops_sample, all for the same sample in the same thread:
//   1. M (lower triangle) by crba_sample into the workspace column, c by rnea_sample (external wrenches included), q̇;
//   2. one outward sweep in the ROOT frame (pose, twist, velocity-product bias acceleration without gravity, like kin_sample):
//      the loop endpoints park pose / twist / bias in the workspace, the joints on a loop path park their world motion subspace;
//   3. per loop: root-frame wrench basis T_c, bias k_c, row c of K;
//   4. the solve: Cholesky of M, Y = K L^-T (overwrites K), z = L^-1 (tau - c), A = Y Y^T, b = Y z + k, diagonally pivoted
//      Cholesky of A with the rank rule of include/rbd_b200.h, lambda = P^T G (G^T G)^-2 G^T P b, v̇ = L^-T (z - Y^T lambda)
//      (= M^-1 (tau - c - K^T lambda)).
// The workspace is one column per RESIDENT thread (rows x resident threads, a persistent grid-stride kernel), not per sample.
#pragma once
#include <cmath>
#include <cstring>

#include "../../../include/rbd_b200.h"
#include "rbd_kin.cuh"
#include "rbd_model.h"

namespace rbd {

constexpr int kMaxLoops = RBD_MAX_LOOP_JOINTS, kMaxConstraints = RBD_MAX_CONSTRAINTS;
constexpr int kLoopEndRows = 24;     // pose (12) + twist (6) + bias acceleration (6) of a loop endpoint, root frame
// Rank rule of A (include/rbd_b200.h): fp64 = the reference's singular_value_zero_tolerance (mechanism_algorithms.jl:804); fp32 =
// about 100 fp32 epsilons, above the rounding that the Schur complement of a structurally zero constraint row carries.
constexpr double kLoopRcond64 = 1e-10, kLoopRcond32 = 1e-5;

template <class T> struct LoopDev {
  int32_t nl, nc;                          // loop joints, constraint rows
  int32_t stab;                            // Baumgarte stabilisation on
  int32_t body_end[kMaxBodies];            // preorder position -> endpoint slot, -1 = not an endpoint
  int32_t pred_end[kMaxLoops], succ_end[kMaxLoops];   // endpoint slot of the loop's predecessor / successor, -1 = root
  int32_t crow[kMaxLoops + 1];             // loop l owns constraint rows crow[l] .. crow[l + 1] - 1
  int8_t on_path[kMaxBodies];              // preorder position -> joint lies on some loop's path
  int8_t sign[kMaxLoops][kMaxBodies];      // preorder position -> -1 up / +1 down / 0 off the path
  T Xp[kMaxLoops][12], Xs[kMaxLoops][12];  // joint_to_predecessor / joint_to_successor in CANONICAL body frames: R row-major, p
  T basis[kMaxConstraints][6];             // [torque; force] in the frame after the joint
  T gains[kMaxLoops][4];                   // angular k, d, linear k, d
  T rcond;                                 // rank rule of the pivoted Cholesky factorisation of A
};

// Rows of the per-thread workspace column.
struct LoopRows {
  int M, z, K, A, b, x, E, S, ext, total;
};
inline LoopRows loop_rows(int nb, int nv, int nc, int nends, bool ext) {
  LoopRows r;
  int o = 0;
  r.M = o; o += nv * nv;              // mass matrix (lower triangle), then its Cholesky factor L
  r.z = o; o += nv;                   // c, then z = L^-1 (tau - c), then v̇
  r.K = o; o += nc * nv;              // K (row c + j * nc), then Y
  r.A = o; o += nc * nc;              // A = Y Y^T (full), then its pivoted factor G
  r.b = o; o += nc;                   // b, then G^T P b, then lambda (pivoted)
  r.x = o; o += nc;                   // k, then the solve vector
  r.E = o; o += kLoopEndRows * nends;
  r.S = o; o += 6 * nv;               // root-frame motion subspace of the path joints
  r.ext = o; o += ext ? 6 * nb : 0;   // body-frame external wrenches (rnea_sample)
  r.total = o;
  return r;
}

template <class T, class W = Col<T>> struct LoopsIO {
  Col<T> q, v, tau;
  W wext;                             // root-frame external wrenches (ext_wrench_pass)
  ColOut<T> vd, qd, lam, K, k;       // all but vd may be invalid (NULL = not wanted)
  Scr<T> w;                           // workspace column
  LoopRows r;
};

template <class T> RBD_HD T loop_sqrt(T x) { return contact_sqrt(x); }

template <class T> RBD_HD void mat_mul3_tn(const T* a, const T* b, T* o) {      // o = a^T b
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) o[3 * i + j] = a[i] * b[j] + a[3 + i] * b[3 + j] + a[6 + i] * b[6 + j];
}

// x_root = R x + p for a pose given as R (9) p (3); composition a * b
template <class T> RBD_HD void pose_mul(const T* Ra, const T* pa, const T* Rb, const T* pb, T* R, T* p) {
  mat_mul3(Ra, Rb, R);
  T t[3];
  mat_vec(Ra, pb, t);
  p[0] = pa[0] + t[0]; p[1] = pa[1] + t[1]; p[2] = pa[2] + t[2];
}

template <class T, class ST, int KMAX, class W>
RBD_HD void loops_sample(const ModelDev<T>& M, const LoopDev<T>& L, const LoopsIO<T, W>& io, const ST& st) {
  const int nb = M.nb, nv = M.nv, nc = L.nc;
  const Scr<T>& w = io.w;
  const LoopRows& r = io.r;
  // ---- 1. M, c, q̇ ----
  {
    CrbaIO<T> cio;
    cio.q = io.q;
    cio.M = {w.p + (int64_t)r.M * w.ld, w.ld, true};
    cio.lower = true;
    crba_sample<T, ST, KMAX>(M, cio, st);
  }
  {
    RneaIO<T, W> rio;
    rio.q = io.q; rio.v = io.v; rio.vd = {nullptr, io.q.ld}; rio.wext = io.wext;
    rio.tau = {w.p + (int64_t)r.z * w.ld, w.ld, true};
    rio.ext = {io.wext.valid() ? w.p + (int64_t)r.ext * w.ld : nullptr, w.ld};
    rnea_sample<T>(M, rio, st);
  }
  if (io.qd.valid())
    for (int i = 0; i < nb; ++i) qdot_joint<T>(M.body[i], io.q, io.v, io.qd);

  // ---- 2. outward sweep in the root frame (kin_sample's recursion; pending slots in the stash) ----
  if (nc > 0) {
    Pose<T> cur;
    pose_identity(cur);
    Mot<T> twc, bc;
#pragma unroll
    for (int k = 0; k < 3; ++k) twc.w[k] = twc.l[k] = bc.w[k] = bc.l[k] = T(0);
    for (int i = 0; i < nb; ++i) {
      const BodyDev<T>& bd = M.body[i];
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
      T R[9], rr[3];
      frame_any(bd, io.q, R, rr);
      Pose<T> wp;
      pose_mul(pp.R, pp.p, R, rr, wp.R, wp.p);
      Mot<T> jt;
#pragma unroll
      for (int k = 0; k < 3; ++k) jt.w[k] = jt.l[k] = T(0);
      const int nvj = kind_nv_dev(bd.kind);
      for (int k = 0; k < nvj; ++k) {
        Mot<T> S;
        world_subspace(wp, sub_comp(bd.kind, k), S);
        const T x = io.v(bd.vrow + k);
#pragma unroll
        for (int c = 0; c < 3; ++c) { jt.w[c] += x * S.w[c]; jt.l[c] += x * S.l[c]; }
        if (L.on_path[i]) {
          const int row = r.S + 6 * (bd.vrow + k);
#pragma unroll
          for (int c = 0; c < 3; ++c) { w.st(row + c, S.w[c]); w.st(row + 3 + c, S.l[c]); }
        }
      }
      Mot<T> tw, bias, cm;
      motion_cross(twp, jt, cm);          // v_parent x (S v): the joint's contribution to the bias acceleration wrt world
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        tw.w[k] = twp.w[k] + jt.w[k]; tw.l[k] = twp.l[k] + jt.l[k];
        bias.w[k] = bp.w[k] + cm.w[k]; bias.l[k] = bp.l[k] + cm.l[k];
      }
      const int e = L.body_end[i];
      if (e >= 0) {
        const int row = r.E + kLoopEndRows * e;
#pragma unroll
        for (int k = 0; k < 9; ++k) w.st(row + k, wp.R[k]);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          w.st(row + 9 + k, wp.p[k]);
          w.st(row + 12 + k, tw.w[k]); w.st(row + 15 + k, tw.l[k]);
          w.st(row + 18 + k, bias.w[k]); w.st(row + 21 + k, bias.l[k]);
        }
      }
      if (bd.flags & F_HAS_PENDING) {
        const int row = bd.oslot * kSlotRowsKin;
#pragma unroll
        for (int k = 0; k < 9; ++k) st.st(row + k, wp.R[k]);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          st.st(row + 9 + k, wp.p[k]);
          st.st(row + 12 + k, tw.w[k]); st.st(row + 15 + k, tw.l[k]);
          st.st(row + 18 + k, bias.w[k]); st.st(row + 21 + k, bias.l[k]);
        }
      }
      cur = wp; twc = tw; bc = bias;
    }
  }

  // ---- 3. per loop: root-frame wrench basis, constraint bias, constraint Jacobian rows ----
  for (int l = 0; l < L.nl; ++l) {
    T Rp[9], pp[3], Rs[9], ps[3];
    Mot<T> vp, vs, bpr, bsu;
    auto endpoint = [&](int e, T* R, T* p, Mot<T>& tw, Mot<T>& b) {
      if (e < 0) {
        Pose<T> id;
        pose_identity(id);
#pragma unroll
        for (int k = 0; k < 9; ++k) R[k] = id.R[k];
#pragma unroll
        for (int k = 0; k < 3; ++k) { p[k] = T(0); tw.w[k] = tw.l[k] = b.w[k] = b.l[k] = T(0); }
        return;
      }
      const int row = r.E + kLoopEndRows * e;
#pragma unroll
      for (int k = 0; k < 9; ++k) R[k] = w.get(row + k);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        p[k] = w.get(row + 9 + k);
        tw.w[k] = w.get(row + 12 + k); tw.l[k] = w.get(row + 15 + k);
        b.w[k] = w.get(row + 18 + k); b.l[k] = w.get(row + 21 + k);
      }
    };
    {
      T Rb[9], pb[3];
      endpoint(L.pred_end[l], Rb, pb, vp, bpr);
      pose_mul(Rb, pb, L.Xp[l], L.Xp[l] + 9, Rp, pp);        // frame before the joint -> root
      endpoint(L.succ_end[l], Rb, pb, vs, bsu);
      pose_mul(Rb, pb, L.Xs[l], L.Xs[l] + 9, Rs, ps);        // frame after the joint -> root
    }
    // bias acceleration: v_s x v_p + (b_s - b_p)          (:641-647)
    Mot<T> a;
    motion_cross(vs, vp, a);
#pragma unroll
    for (int k = 0; k < 3; ++k) { a.w[k] += bsu.w[k] - bpr.w[k]; a.l[k] += bsu.l[k] - bpr.l[k]; }
    if (L.stab) {                                             // (:649-663)
      // joint transform (after -> before) and joint twist in the frame after the joint
      T Re[9], pe[3], d[3];
      mat_mul3_tn(Rp, Rs, Re);
      d[0] = ps[0] - pp[0]; d[1] = ps[1] - pp[1]; d[2] = ps[2] - pp[2];
      matT_vec(Rp, d, pe);
      T jw[3], jl[3], t[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) { jw[k] = vs.w[k] - vp.w[k]; jl[k] = vs.l[k] - vp.l[k]; }
      cross3(ps, jw, t);
#pragma unroll
      for (int k = 0; k < 3; ++k) t[k] = jl[k] - t[k];
      T ew[3], el[3];
      matT_vec(Rs, jw, ew);
      matT_vec(Rs, t, el);
      // pd(gains, e, ė, SE3PDMethod{:Linearized}): psi = linearized_rodrigues_vec(R), lin error R^T p
      const T psi[3] = {(Re[7] - Re[5]) * T(0.5), (Re[2] - Re[6]) * T(0.5), (Re[3] - Re[1]) * T(0.5)};
      T rtp[3];
      matT_vec(Re, pe, rtp);
      const T ka = L.gains[l][0], da = L.gains[l][1], kl = L.gains[l][2], dl = L.gains[l][3];
      T sa[3], sl[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) { sa[k] = -ka * psi[k] - da * ew[k]; sl[k] = -kl * rtp[k] - dl * el[k]; }
      // back to the root frame (transform_spatial_motion) and subtracted
      T wa[3], wl[3], c3[3];
      mat_vec(Rs, sa, wa);
      mat_vec(Rs, sl, wl);
      cross3(ps, wa, c3);
#pragma unroll
      for (int k = 0; k < 3; ++k) { a.w[k] -= wa[k]; a.l[k] -= wl[k] + c3[k]; }
    }
    for (int c = L.crow[l]; c < L.crow[l + 1]; ++c) {
      // basis column to the root frame: f = R f_j, n = R n_j + p x f
      T n[3], f[3], x[3];
      mat_vec(Rs, L.basis[c] + 3, f);
      mat_vec(Rs, L.basis[c], n);
      cross3(ps, f, x);
#pragma unroll
      for (int k = 0; k < 3; ++k) n[k] += x[k];
      const T kc = n[0] * a.w[0] + n[1] * a.w[1] + n[2] * a.w[2] + f[0] * a.l[0] + f[1] * a.l[1] + f[2] * a.l[2];
      w.st(r.x + c, kc);
      if (io.k.valid()) io.k.st(c, kc);
      for (int i = 0; i < nb; ++i) {
        const BodyDev<T>& bd = M.body[i];
        const int sg = L.sign[l][i];
        const int nvj = kind_nv_dev(bd.kind);
        for (int k = 0; k < nvj; ++k) {
          const int j = bd.vrow + k;
          T val = T(0);
          if (sg != 0) {
            const int row = r.S + 6 * j;
            val = n[0] * w.get(row) + n[1] * w.get(row + 1) + n[2] * w.get(row + 2) +
                  f[0] * w.get(row + 3) + f[1] * w.get(row + 4) + f[2] * w.get(row + 5);
            if (sg < 0) val = -val;
          }
          w.st(r.K + c + j * nc, val);
          if (io.K.valid()) io.K.st(c + j * nc, val);
        }
      }
    }
  }

  // ---- 4. the solve ----
  // Cholesky M = L L^T in place (lower triangle, entry (i, j) at row i + j nv)
  auto Lm = [&](int i, int j) { return w.get(r.M + i + j * nv); };
  for (int j = 0; j < nv; ++j) {
    T d = Lm(j, j);
    for (int k = 0; k < j; ++k) { const T x = Lm(j, k); d -= x * x; }
    const T ljj = loop_sqrt(d);
    const T inv = T(1) / ljj;
    w.st(r.M + j + j * nv, ljj);
    for (int i = j + 1; i < nv; ++i) {
      T s = Lm(i, j);
      for (int k = 0; k < j; ++k) s -= Lm(i, k) * Lm(j, k);
      w.st(r.M + i + j * nv, s * inv);
    }
  }
  // z = L^-1 (tau - c)
  for (int i = 0; i < nv; ++i) {
    T s = (io.tau.valid() ? io.tau(i) : T(0)) - w.get(r.z + i);
    for (int k = 0; k < i; ++k) s -= Lm(i, k) * w.get(r.z + k);
    w.st(r.z + i, s / Lm(i, i));
  }
  if (nc > 0) {
    // Y = K L^-T: row c of Y solves L y = K[c, :]^T
    for (int c = 0; c < nc; ++c)
      for (int i = 0; i < nv; ++i) {
        T s = w.get(r.K + c + i * nc);
        for (int k = 0; k < i; ++k) s -= Lm(i, k) * w.get(r.K + c + k * nc);
        w.st(r.K + c + i * nc, s / Lm(i, i));
      }
    // A = Y Y^T (full), b = Y z + k
    for (int c = 0; c < nc; ++c) {
      T bc = w.get(r.x + c);
      for (int i = 0; i < nv; ++i) bc += w.get(r.K + c + i * nc) * w.get(r.z + i);
      w.st(r.b + c, bc);
      for (int e = 0; e <= c; ++e) {
        T s = T(0);
        for (int i = 0; i < nv; ++i) s += w.get(r.K + c + i * nc) * w.get(r.K + e + i * nc);
        w.st(r.A + c + e * nc, s);
        w.st(r.A + e + c * nc, s);
      }
    }
    // diagonally pivoted Cholesky A ~ P^T G G^T P (outer-product form, full symmetric storage, rows and columns swapped)
    int piv[kMaxConstraints];
    for (int c = 0; c < nc; ++c) piv[c] = c;
    auto Aa = [&](int i, int j) { return w.get(r.A + i + j * nc); };
    int rank = 0;
    T d0 = T(0);
    for (int j = 0; j < nc; ++j) {
      int p = j;
      T best = Aa(j, j);
      for (int i = j + 1; i < nc; ++i) { const T x = Aa(i, i); if (x > best) { best = x; p = i; } }
      if (j == 0) d0 = best;
      if (!(best > L.rcond * d0) || !(best > T(0))) break;
      if (p != j) {
        for (int k = 0; k < nc; ++k) { const T x = Aa(j, k); w.st(r.A + j + k * nc, Aa(p, k)); w.st(r.A + p + k * nc, x); }
        for (int k = 0; k < nc; ++k) { const T x = Aa(k, j); w.st(r.A + k + j * nc, Aa(k, p)); w.st(r.A + k + p * nc, x); }
        const int t = piv[j]; piv[j] = piv[p]; piv[p] = t;
      }
      const T gjj = loop_sqrt(best);
      const T inv = T(1) / gjj;
      w.st(r.A + j + j * nc, gjj);
      for (int i = j + 1; i < nc; ++i) w.st(r.A + i + j * nc, Aa(i, j) * inv);
      for (int e = j + 1; e < nc; ++e) {
        const T ge = Aa(e, j);
        for (int i = e; i < nc; ++i) {
          const T x = Aa(i, e) - Aa(i, j) * ge;
          w.st(r.A + i + e * nc, x);
          w.st(r.A + e + i * nc, x);
        }
      }
      rank = j + 1;
    }
    // y = G^T P b (r entries, into r.x), C = G^T G (r x r, upper triangle of the A block's columns is free: use rows < column)
    // C is kept in the strictly-upper part of A (rows e < c) plus a diagonal in r.b; G stays in the lower part.
    auto G = [&](int i, int j) { return w.get(r.A + i + j * nc); };
    for (int a = 0; a < rank; ++a) {
      T s = T(0);
      for (int i = a; i < nc; ++i) s += G(i, a) * w.get(r.b + piv[i]);
      w.st(r.x + a, s);
    }
    for (int a = 0; a < rank; ++a)
      for (int e = 0; e <= a; ++e) {
        T s = T(0);
        for (int i = a; i < nc; ++i) s += G(i, a) * G(i, e);   // G(i, a) = 0 for i < a
        if (e == a) w.st(r.b + a, s);
        else w.st(r.A + e + a * nc, s);                        // C(a, e) = C(e, a) at (row e, column a), e < a
      }
    // Cholesky of C in place: H (upper storage: H^T stored at (row e, column a), e < a; diagonal in r.b)
    auto Cu = [&](int e, int a) { return e == a ? w.get(r.b + a) : w.get(r.A + e + a * nc); };
    for (int a = 0; a < rank; ++a) {
      T d = Cu(a, a);
      for (int k = 0; k < a; ++k) { const T x = Cu(k, a); d -= x * x; }
      const T haa = loop_sqrt(d);
      w.st(r.b + a, haa);
      for (int e = a + 1; e < rank; ++e) {
        T s = Cu(a, e);
        for (int k = 0; k < a; ++k) s -= Cu(k, a) * Cu(k, e);
        w.st(r.A + a + e * nc, s / haa);
      }
    }
    // x = C^-1 C^-1 y  (two forward / backward substitution pairs with H, H(a, k) = Cu(k, a) for k < a)
    for (int rep = 0; rep < 2; ++rep) {
      for (int a = 0; a < rank; ++a) {
        T s = w.get(r.x + a);
        for (int k = 0; k < a; ++k) s -= Cu(k, a) * w.get(r.x + k);
        w.st(r.x + a, s / Cu(a, a));
      }
      for (int a = rank - 1; a >= 0; --a) {
        T s = w.get(r.x + a);
        for (int k = a + 1; k < rank; ++k) s -= Cu(a, k) * w.get(r.x + k);
        w.st(r.x + a, s / Cu(a, a));
      }
    }
    // lambda = P^T G x  (pivoted row i of G x is lambda[piv[i]])
    for (int i = 0; i < nc; ++i) {
      T s = T(0);
      const int amax = i < rank ? i + 1 : rank;
      for (int a = 0; a < amax; ++a) s += G(i, a) * w.get(r.x + a);
      w.st(r.b + piv[i], s);
    }
    if (io.lam.valid())
      for (int c = 0; c < nc; ++c) io.lam.st(c, w.get(r.b + c));
    // z <- z - Y^T lambda
    for (int i = 0; i < nv; ++i) {
      T s = w.get(r.z + i);
      for (int c = 0; c < nc; ++c) s -= w.get(r.K + c + i * nc) * w.get(r.b + c);
      w.st(r.z + i, s);
    }
  }
  // v̇ = L^-T z
  for (int i = nv - 1; i >= 0; --i) {
    T s = w.get(r.z + i);
    for (int k = i + 1; k < nv; ++k) s -= Lm(k, i) * w.get(r.z + k);
    s /= Lm(i, i);
    w.st(r.z + i, s);
    io.vd.st(i, s);
  }
}

// contact_dynamics! at one stage of the loop rollout (rbd_integrate_loops, DESIGN 4.16): contact_sample's sweep (root-frame pose and
// twist, pending slots in the kin layout of the stash) with the stage semantics of contact_stage_pass -- the stage state
// s_i = s0 + wa ṡ_{i-1} formed from two loads and never stored, ṡ_i written for every pair (zero out of contact), nothing reset --
// and every body's ROOT-frame wrench (rows 6 refidx + c, as contact_sample writes them) into `wr`, the thread's own workspace rows,
// by inactive lanes too.  A sibling rather than a variant of contact_sample, so that contact_kernel's code stays as it is.
template <class T, class ST>
RBD_HD void loops_contact_pass(const ModelDev<T>& M, const ContactDev<T>& C, const Col<T>& q, const Col<T>& v, const ContactStageIO<T>& io,
                               const Scr<T>& wr, const ST& st) {
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
      const int row = bd.pslot * kSlotRowsKin;
#pragma unroll
      for (int k = 0; k < 9; ++k) pp.R[k] = st.ld(row + k);
#pragma unroll
      for (int k = 0; k < 3; ++k) { pp.p[k] = st.ld(row + 9 + k); twp.w[k] = st.ld(row + 12 + k); twp.l[k] = st.ld(row + 15 + k); }
    }
    T R[9], r[3];
    frame_any(bd, q, R, r);
    Pose<T> w;
    pose_mul(pp.R, pp.p, R, r, w.R, w.p);
    Mot<T> tw = twp;
    const int nvj = kind_nv_dev(bd.kind);
    for (int k = 0; k < nvj; ++k) {
      Mot<T> S;
      world_subspace(w, sub_comp(bd.kind, k), S);
      const T x = v(bd.vrow + k);
#pragma unroll
      for (int c = 0; c < 3; ++c) { tw.w[c] += x * S.w[c]; tw.l[c] += x * S.l[c]; }
    }
    T wn[3] = {T(0), T(0), T(0)}, wf[3] = {T(0), T(0), T(0)};
    for (int pi = C.first[i]; pi < C.first[i + 1]; ++pi) {
      T pt[3], vel[3], tmp[3];
      mat_vec(w.R, C.loc[pi], tmp);
      pt[0] = w.p[0] + tmp[0]; pt[1] = w.p[1] + tmp[1]; pt[2] = w.p[2] + tmp[2];
      cross3(tw.w, pt, vel);                                   // point_velocity(twist, point)
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
          cross3(pt, f, m);                                     // Wrench(point, force)
#pragma unroll
          for (int k = 0; k < 3; ++k) { wn[k] += m[k]; wf[k] += f[k]; }
        }
        if (io.active) {
#pragma unroll
          for (int k = 0; k < 3; ++k) io.sd[(srow + k) * io.ld] = xd[k];
        }
      }
    }
    const int orow = 6 * bd.refidx;
#pragma unroll
    for (int k = 0; k < 3; ++k) { wr.st(orow + k, wn[k]); wr.st(orow + 3 + k, wf[k]); }
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

// One stage of the loop rollout with contact: dynamics! as mechanism_algorithms.jl:845-864 runs it -- loops_contact_pass into rows
// wrow .. wrow + 6 nb - 1 of the workspace column (behind LoopRows::total), then loops_sample with them as the external wrenches.
// io.r must be planned with ext = true.  The wrench rows are read back with plain loads (ColRW): the same thread wrote them in this
// kernel, and the column is reused by the next sample the thread takes.
template <class T, class ST, int KMAX>
RBD_HD void loops_contact_sample(const ModelDev<T>& M, const LoopDev<T>& L, const ContactDev<T>& C, const ContactStageIO<T>& cs,
                                 LoopsIO<T, ColRW<T>> io, int wrow, const ST& st) {
  const Scr<T> wr{io.w.p + (int64_t)wrow * io.w.ld, io.w.ld};
  loops_contact_pass(M, C, io.q, io.v, cs, wr, st);
  io.wext = {wr.p, wr.ld};
  loops_sample<T, ST, KMAX>(M, L, io, st);
}

// ------------------------------------------------------------------------------------------------------------------
// Host side: rbd_loop_desc -> LoopDev (validated by the caller).  pos: reference joint index -> preorder position, alignT:
// preorder position -> A^T (canonical body frame <- caller's body frame).  Paths follow the tree's parent links.
// ------------------------------------------------------------------------------------------------------------------
template <class T>
inline void build_loop_dev(const HostModel& hm, const rbd_loop_desc& ld, double rcond, LoopDev<T>& D) {
  std::memset(&D, 0, sizeof(D));
  D.nl = ld.nloops;
  D.stab = ld.gains != nullptr;
  D.rcond = (T)rcond;
  for (int i = 0; i < kMaxBodies; ++i) D.body_end[i] = -1;
  int nends = 0;
  auto end_of = [&](int ref) {
    if (ref < 0) return -1;
    const int p = hm.pos[ref];
    if (D.body_end[p] < 0) D.body_end[p] = nends++;
    return D.body_end[p];
  };
  int c = 0;
  for (int l = 0; l < ld.nloops; ++l) {
    const int P = ld.predecessor[l], S = ld.successor[l];
    D.pred_end[l] = end_of(P);
    D.succ_end[l] = end_of(S);
    D.crow[l] = c;
    // canonical attachment transforms: X' = (A^T R, A^T p) with A the body's alignment (identity for the root)
    auto canon = [&](int ref, const double* X, T* out) {
      double At[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
      if (ref >= 0) std::memcpy(At, hm.alignT.data() + 9 * hm.pos[ref], sizeof(At));
      for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) out[3 * i + j] = (T)(At[3 * i] * X[j] + At[3 * i + 1] * X[3 + j] + At[3 * i + 2] * X[6 + j]);
        out[9 + i] = (T)(At[3 * i] * X[9] + At[3 * i + 1] * X[10] + At[3 * i + 2] * X[11]);
      }
    };
    canon(P, ld.joint_to_predecessor + 12 * l, D.Xp[l]);
    canon(S, ld.joint_to_successor + 12 * l, D.Xs[l]);
    for (int k = 0; k < ld.nconstraints[l]; ++k, ++c)
      for (int m = 0; m < 6; ++m) D.basis[c][m] = (T)ld.wrench_basis[6 * c + m];
    if (ld.gains)
      for (int m = 0; m < 4; ++m) D.gains[l][m] = (T)ld.gains[4 * l + m];
    // path(predecessor, successor): up from the predecessor to the lowest common ancestor (-1), then down (+1)
    // (preorder positions; the parent links of the device model)
    int up[kMaxBodies], dn[kMaxBodies], nu = 0, nd = 0;
    for (int j = P < 0 ? -1 : hm.pos[P]; j >= 0; j = hm.dev64.body[j].parent) up[nu++] = j;
    for (int j = S < 0 ? -1 : hm.pos[S]; j >= 0; j = hm.dev64.body[j].parent) dn[nd++] = j;
    while (nu > 0 && nd > 0 && up[nu - 1] == dn[nd - 1]) { --nu; --nd; }
    for (int k = 0; k < nu; ++k) { D.sign[l][up[k]] = -1; D.on_path[up[k]] = 1; }
    for (int k = 0; k < nd; ++k) { D.sign[l][dn[k]] = 1; D.on_path[dn[k]] = 1; }
  }
  D.crow[ld.nloops] = c;
  D.nc = c;
}

// Descriptor checks of rbd_dynamics_loops: RBD_EINVAL for a malformed descriptor, RBD_EUNSUPPORTED beyond the limits.
inline int check_loop_desc(const HostModel& hm, const rbd_loop_desc* ld, std::string& err) {
  if (!ld) { err = "rbd_dynamics_loops: loops must not be NULL"; return RBD_EINVAL; }
  if (ld->nloops < 0) { err = "rbd_dynamics_loops: negative nloops"; return RBD_EINVAL; }
  if (ld->nloops == 0) return RBD_OK;
  if (!ld->predecessor || !ld->successor || !ld->joint_to_predecessor || !ld->joint_to_successor || !ld->nconstraints) {
    err = "rbd_dynamics_loops: descriptor arrays must not be NULL";
    return RBD_EINVAL;
  }
  int nc = 0;
  for (int l = 0; l < ld->nloops; ++l) {
    const int P = ld->predecessor[l], S = ld->successor[l], n = ld->nconstraints[l];
    if (P < -1 || P >= hm.nb || S < -1 || S >= hm.nb) { err = "rbd_dynamics_loops: body index out of range"; return RBD_EINVAL; }
    if (P == S) { err = "rbd_dynamics_loops: predecessor == successor"; return RBD_EINVAL; }
    if (n < 0 || n > 6) { err = "rbd_dynamics_loops: nconstraints outside 0..6"; return RBD_EINVAL; }
    nc += n;
  }
  if (nc > 0 && !ld->wrench_basis) { err = "rbd_dynamics_loops: wrench_basis must not be NULL"; return RBD_EINVAL; }
  if (ld->nloops > kMaxLoops || nc > kMaxConstraints) {
    err = "rbd_dynamics_loops: more than RBD_MAX_LOOP_JOINTS loop joints or RBD_MAX_CONSTRAINTS constraint rows";
    return RBD_EUNSUPPORTED;
  }
  return RBD_OK;
}

inline int loop_nends(const HostModel& hm, const rbd_loop_desc& ld) {
  int seen[kMaxBodies] = {0}, n = 0;
  for (int l = 0; l < ld.nloops; ++l)
    for (int ref : {ld.predecessor[l], ld.successor[l]})
      if (ref >= 0 && !seen[hm.pos[ref]]) { seen[hm.pos[ref]] = 1; ++n; }
  return n;
}

}  // namespace rbd
