// Reverse mode (SURVEY 8(f) rank 3, second half): vector-Jacobian products of inverse_dynamics! and dynamics! for a whole batch,
// O(n) per sample -- no nv x nv object anywhere.  What a reference user gets from ForwardDiff/ReverseDiff over
// inverse_dynamics! (mechanism_algorithms.jl:542-553) or dynamics! (:845-864) contracted with an adjoint.
//
// Both VJPs are the reverse sweep of  L = w . ID(q, v, v̇, w_ext)  for a weight vector w:
//   inverse dynamics   w = τ̄                 -> q̄, v̄, v̇̄ = M τ̄, w̄
//   forward dynamics   w = -μ, μ = M^-1 ν̄     -> q̄, v̄, τ̄ = μ, w̄        (v̇ = FD(q, v, τ, w_ext) held fixed: v̇ MUST be the
//                                                                    forward result for the same inputs, the VJP does not recompute it)
// μ is the Articulated-Body Algorithm with τ = ν̄, zero velocity, zero gravity and no wrenches (aba_sample, rbd_device.cuh).
//
// Derivation, ROOT-frame quantities as in rbd_deriv.cuh (the reference's caches, mechanism_state.jl:604-682):
//   X_i pose, S_k = Ad_{X_i} e_k, v_i = v_p + sum_k S_k v_k, a_i = a_p + v_p x (sum_k S_k v_k) + sum_k S_k v̇_k (a_root = -g,
//   spatial_accelerations! :387-417), I_i root-frame inertia, f_i = I_i a_i + v_i x* I_i v_i - w_i (newton_euler! :428-439),
//   F_i = sum_{sub(i)} f (joint_wrenches_and_torques! :442-459), τ_k = S_k . F_{body(k)}.
// Then L = sum_k w_k S_k . F = sum_i m_i . f_i  with the PATH sum  m_i = sum_{k on the path root..i} w_k S_k  (the root-frame
// twist of body i if the joint velocities were w).  Hence
//   ∂L/∂w_i = -m_i                                              (w̄ of the inverse-dynamics VJP; the forward one is +m_i(μ))
//   ∂L/∂v̇_j = S_j . P_J,             P_J = sum_{i in sub(J)} h_i,   h_i = I_i m_i
// Moving velocity coordinate j of joint J moves the subtree rigidly by the twist S_j (rbd_deriv.cuh): body-fixed quantities
// (S, I, and f_i + w_i) rotate with it, what does not follow is Psi_dot_j = v_p x S_j in v_i and, in f_i, I Psi_ddot_j + G_i Psi_dot_j,
// Psi_ddot_j = a_p x S_j + v_p x Psi_dot_j, G_i x = I_i (x x v_i) + x x* (I_i v_i) + v_i x* (I_i x) (rbd_deriv.cuh, p = parent of J).
// The root-frame external wrench w_i does NOT rotate with the subtree: f_i changes by  S_j x* (f_i + w_i) + ..., not S_j x* f_i.
// Contracting the closed forms of rbd_deriv.cuh (d τ_k / d q_j for K in sub(J), and for K a strict ancestor of J, extended by this
// wrench term) with w, the sums over K regroup per body i in sub(J) with weight (m_i - m_p) + m_p = m_i, and the wrench terms of
// the two cases cancel down to a subtree sum:
//   q̄_j = Psi_ddot_j . P_J + Psi_dot_j . Q_J + S_j . E_J + (m_p x S_j) . F_J
//   v̄_j = Sdp_j . P_J + S_j . Q_J,        Sdp_j = (v_J + v_p) x S_j           (d a_i / d v_j = Sdp_j + S_j x v_i)
// with the subtree sums of force vectors
//   Q_J = sum g_i,  g_i = G_i^T m_i = v_i x* h_i - m_i x* (I_i v_i) + I_i (m_i x v_i)
//   E_J = sum e_i,  e_i = -m_i x* w_i                 (the external-wrench term; absent from rbd_deriv.cuh's closed forms)
//   F_J = sum f_i                                    (the joint wrench, w_ext included)
// (identities used: (x x m) . f + m . (x x* f) = 0, and I symmetric).  "d/dq_j" is the tangent derivative along
// q̇ = velocity_to_configuration_derivative(e_j) (mechanism_state.jl:905-910), the convention of rbd_dynamics_derivatives' dvd_dq.
//
// Configuration covector (q̄_cfg): the tangent covector mapped like configuration_derivative_to_velocity_adjoint!
// (mechanism_state.jl:912-918, joint_types/*.jl) -- the minimal-norm c with N(q)^T c = q̄_tan (N = this library's q̇ = N(q) v),
// so  c . (N(q) u) = q̄_tan . u  for every u, also for non-unit quaternions:
//   revolute / prismatic: c = q̄_tan;  planar: c = N q̄_tan (N orthogonal, planar.jl:131-137);  sin/cos: c = (cos, -sin) f / |q|^2
//   (sin_cos_revolute.jl:153-158);  quaternion rotation: c = 2 Q(q) f / |q|^2 (quaternion_floating.jl:116-124; orthogonal to q);
//   MRP and every translation block: c = N_block^-T f.  The derivative of the unnormalised quaternion formula in the radial
//   direction is deliberately NOT part of c (SURVEY 8(c): parity unpinned).
//
// Work split: one thread per sample, two sweeps over the bodies.  Outward: pose, twist, acceleration, m in registers (a branch
// node's successors read them back from the workspace); every body parks X (12), v, a, m (18) and its own h, g, e, f (24) in a
// workspace column -- 54 rows per body.  Inward (reverse preorder): a body's four sums are complete when it is reached; its
// coordinates' adjoints are formed from the parked X, its own v and its parent's v, a, m; then its sums are added to the
// parent's rows.  The workspace is one column per RESIDENT thread (a persistent kernel, like rbd_loops.cuh), DESIGN 4.12.
#pragma once
#include <cmath>
#include <cstring>

#include "rbd_deriv.cuh"

namespace rbd {

constexpr int kAdjBodyRows = 54;   // pose 12, v 6, a 6, m 6, then the subtree sums P (h), Q (g), E (e), F (f)
constexpr int kAdjV = 12, kAdjA = 18, kAdjM = 24, kAdjP = 30, kAdjQ = 36, kAdjE = 42, kAdjF = 48;

// Workspace rows per sample: the bodies, then (forward VJP) μ in reference velocity order.
inline int adjoint_rows(int nb, int nv) { return kAdjBodyRows * nb + nv; }

template <class T> struct AdjIO {
  Col<T> q, v, vd, wext;           // wext may be invalid (no external wrenches)
  ColOut<T> qt, qc, vb, vdb, wb;   // q̄_tan [nv], q̄_cfg [nq], v̄ [nv], v̇̄ [nv], w̄ [6 nb]; each may be invalid (not wanted)
  Scr<T> s;                        // this thread's workspace column
};

template <class T> RBD_HD T dot_mf(const Mot<T>& m, const T* n, const T* f) {
  return m.w[0] * n[0] + m.w[1] * n[1] + m.w[2] * n[2] + m.l[0] * f[0] + m.l[1] * f[1] + m.l[2] * f[2];
}
template <class T> RBD_HD void ld_mot(const Scr<T>& s, int row, Mot<T>& m) {
#pragma unroll
  for (int k = 0; k < 3; ++k) { m.w[k] = s.get(row + k); m.l[k] = s.get(row + 3 + k); }
}
template <class T> RBD_HD void st_mot(const Scr<T>& s, int row, const Mot<T>& m) {
#pragma unroll
  for (int k = 0; k < 3; ++k) { s.st(row + k, m.w[k]); s.st(row + 3 + k, m.l[k]); }
}
template <class T> RBD_HD void st_force(const Scr<T>& s, int row, const T* n, const T* f) {
#pragma unroll
  for (int k = 0; k < 3; ++k) { s.st(row + k, n[k]); s.st(row + 3 + k, f[k]); }
}

// y = A^-T x for a 3x3 row-major A (columns a0, a1, a2):  A^-T x = (x0 a1 x a2 + x1 a2 x a0 + x2 a0 x a1) / det A
template <class T> RBD_HD void inv_t3(const T* A, const T* x, T* y) {
  const T a0[3] = {A[0], A[3], A[6]}, a1[3] = {A[1], A[4], A[7]}, a2[3] = {A[2], A[5], A[8]};
  T c0[3], c1[3], c2[3];
  cross3(a1, a2, c0);
  cross3(a2, a0, c1);
  cross3(a0, a1, c2);
  const T inv = T(1) / (a0[0] * c0[0] + a0[1] * c0[1] + a0[2] * c0[2]);
#pragma unroll
  for (int k = 0; k < 3; ++k) y[k] = (x[0] * c0[k] + x[1] * c1[k] + x[2] * c2[k]) * inv;
}

// Quaternion block of N: q̇ = 0.5 Q(q) ω  (quaternion_floating.jl:126-136);  Q(q) ω written out
template <class T> RBD_HD void quat_Q(T w, T x, T y, T z, const T* a, T* o) {
  o[0] = -x * a[0] - y * a[1] - z * a[2];
  o[1] = w * a[0] - z * a[1] + y * a[2];
  o[2] = z * a[0] + w * a[1] - x * a[2];
  o[3] = -y * a[0] + x * a[1] + w * a[2];
}

// configuration_derivative_to_velocity_adjoint! of one joint: f = q̄_tan of its velocity coordinates -> rows qrow.. of q̄_cfg
template <class T> RBD_HD void cfg_adjoint(const BodyDev<T>& bd, const Col<T>& q, const T* f, const ColOut<T>& out) {
  const int q0 = bd.qrow;
  switch (bd.kind) {
    case K_REV: case K_PRIS: out.st(q0, f[0]); break;
    case K_FIXED: break;
    case K_SINCOS: {
      const T s = q(q0), c = q(q0 + 1), inv = T(1) / (s * s + c * c);
      out.st(q0, c * f[0] * inv);
      out.st(q0 + 1, -s * f[0] * inv);
      break;
    }
    case K_PLANAR: {
      T s, c;
      sincos_t(q(q0 + 2), s, c);
      out.st(q0, c * f[0] - s * f[1]);
      out.st(q0 + 1, s * f[0] + c * f[1]);
      out.st(q0 + 2, f[2]);
      break;
    }
    case K_QFLOAT: case K_QSPH: {
      const T w = q(q0), x = q(q0 + 1), y = q(q0 + 2), z = q(q0 + 3);
      const T sc = T(2) / (w * w + x * x + y * y + z * z);
      T o[4];
      quat_Q(w, x, y, z, f, o);
#pragma unroll
      for (int k = 0; k < 4; ++k) out.st(q0 + k, sc * o[k]);
      if (bd.kind == K_QFLOAT) {
        T R[9], t[3];
        rot_quat(w, x, y, z, R);
        inv_t3(R, f + 3, t);
#pragma unroll
        for (int k = 0; k < 3; ++k) out.st(q0 + 4 + k, t[k]);
      }
      break;
    }
    case K_SPQFLOAT: {
      // rotation block of N: the MRP rate for ω = e_k (columns), as qdot_joint computes it; then its inverse transpose
      T qq[4];
      mrp_to_quat(q(q0), q(q0 + 1), q(q0 + 2), qq);
      const T d = T(1) + qq[0];
      T N[9];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const T e[3] = {T(k == 0), T(k == 1), T(k == 2)};
        T dq[4];
        quat_Q(qq[0], qq[1], qq[2], qq[3], e, dq);
#pragma unroll
        for (int r = 0; r < 3; ++r) N[3 * r + k] = T(0.5) * dq[1 + r] / d - qq[1 + r] * T(0.5) * dq[0] / (d * d);
      }
      T t[3], R[9];
      inv_t3(N, f, t);
#pragma unroll
      for (int k = 0; k < 3; ++k) out.st(q0 + k, t[k]);
      rot_quat(qq[0], qq[1], qq[2], qq[3], R);
      inv_t3(R, f + 3, t);
#pragma unroll
      for (int k = 0; k < 3; ++k) out.st(q0 + 3 + k, t[k]);
      break;
    }
  }
}

// The reverse sweep of L = wt . ID(q, v, v̇, w_ext); weight k = wsign * W(row k).  g: gravity (the model's own; M.g is not read,
// so the forward VJP can pass the zero-gravity copy of the model it solves with).
template <class T, class W>
RBD_HD void adjoint_sample(const ModelDev<T>& M, const T* g, const AdjIO<T>& io, const W& wt, T wsign) {
  const int nb = M.nb;
  const Scr<T>& s = io.s;
  // ---- outward: pose, twist, acceleration, m; the body's own h, g, e, f ----
  Pose<T> cur;
  Mot<T> vc, ac, mc;
  for (int i = 0; i < nb; ++i) {
    const BodyDev<T>& bd = M.body[i];
    Pose<T> pp;
    Mot<T> vp, ap, mp;
    if (bd.flags & F_ROOT_CHILD) {
      pose_identity(pp);
#pragma unroll
      for (int k = 0; k < 3; ++k) { vp.w[k] = vp.l[k] = ap.w[k] = mp.w[k] = mp.l[k] = T(0); ap.l[k] = -g[k]; }
    } else if (bd.flags & F_FIRST_CHILD) {
      pp = cur; vp = vc; ap = ac; mp = mc;
    } else {
      const int row = kAdjBodyRows * bd.parent;
#pragma unroll
      for (int k = 0; k < 9; ++k) pp.R[k] = s.get(row + k);
#pragma unroll
      for (int k = 0; k < 3; ++k) pp.p[k] = s.get(row + 9 + k);
      ld_mot(s, row + kAdjV, vp);
      ld_mot(s, row + kAdjA, ap);
      ld_mot(s, row + kAdjM, mp);
    }
    T R[9], r[3], t[3];
    frame_any(bd, io.q, R, r);
    Pose<T> X;
    mat_mul3(pp.R, R, X.R);
    mat_vec(pp.R, r, t);
    X.p[0] = pp.p[0] + t[0]; X.p[1] = pp.p[1] + t[1]; X.p[2] = pp.p[2] + t[2];
    Mot<T> jt, ja, v, a, m, cm;
#pragma unroll
    for (int k = 0; k < 3; ++k) jt.w[k] = jt.l[k] = ja.w[k] = ja.l[k] = T(0);
    m = mp;
    const int nvj = kind_nv_dev(bd.kind);
    for (int k = 0; k < nvj; ++k) {
      Mot<T> S;
      world_subspace(X, sub_comp(bd.kind, k), S);
      const T x = io.v(bd.vrow + k), xd = io.vd(bd.vrow + k), xw = wsign * wt(bd.vrow + k);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        jt.w[c] += x * S.w[c]; jt.l[c] += x * S.l[c];
        ja.w[c] += xd * S.w[c]; ja.l[c] += xd * S.l[c];
        m.w[c] += xw * S.w[c]; m.l[c] += xw * S.l[c];
      }
    }
    motion_cross(vp, jt, cm);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      v.w[k] = vp.w[k] + jt.w[k]; v.l[k] = vp.l[k] + jt.l[k];
      a.w[k] = ap.w[k] + cm.w[k] + ja.w[k]; a.l[k] = ap.l[k] + cm.l[k] + ja.l[k];
    }
    Rbi<T> Ib, I;
    body_rbi(bd, Ib);
    rbi_to_parent(X.R, X.p, Ib, I);
    T hn[3], hf[3], pn[3], pf[3], fn[3], ff[3], t1n[3], t1f[3], t2n[3], t2f[3], t3n[3], t3f[3];
    rbi_mul(I, m, hn, hf);                  // h = I m
    rbi_mul(I, v, pn, pf);                  // I v
    rbi_mul(I, a, fn, ff);
    force_cross(v, pn, pf, t1n, t1f);       // f = I a + v x* I v - w
#pragma unroll
    for (int k = 0; k < 3; ++k) { fn[k] += t1n[k]; ff[k] += t1f[k]; }
    // g = v x* h - m x* (I v) + I (m x v)
    Mot<T> mv;
    motion_cross(m, v, mv);
    force_cross(v, hn, hf, t1n, t1f);
    force_cross(m, pn, pf, t2n, t2f);
    rbi_mul(I, mv, t3n, t3f);
    T gn[3], gf[3], en[3] = {T(0), T(0), T(0)}, ef[3] = {T(0), T(0), T(0)};
#pragma unroll
    for (int k = 0; k < 3; ++k) { gn[k] = t1n[k] - t2n[k] + t3n[k]; gf[k] = t1f[k] - t2f[k] + t3f[k]; }
    const int orow = 6 * bd.refidx;
    if (io.wext.valid()) {                  // e = -m x* w_ext, and w_ext enters the net wrench
      T wn[3], wf[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) { wn[k] = io.wext(orow + k); wf[k] = io.wext(orow + 3 + k); }
      force_cross(m, wn, wf, en, ef);
#pragma unroll
      for (int k = 0; k < 3; ++k) { en[k] = -en[k]; ef[k] = -ef[k]; fn[k] -= wn[k]; ff[k] -= wf[k]; }
    }
    if (io.wb.valid()) {
#pragma unroll
      for (int k = 0; k < 3; ++k) { io.wb.st(orow + k, -m.w[k]); io.wb.st(orow + 3 + k, -m.l[k]); }
    }
    const int row = kAdjBodyRows * i;
#pragma unroll
    for (int k = 0; k < 9; ++k) s.st(row + k, X.R[k]);
#pragma unroll
    for (int k = 0; k < 3; ++k) s.st(row + 9 + k, X.p[k]);
    st_mot(s, row + kAdjV, v);
    st_mot(s, row + kAdjA, a);
    st_mot(s, row + kAdjM, m);
    st_force(s, row + kAdjP, hn, hf);
    st_force(s, row + kAdjQ, gn, gf);
    st_force(s, row + kAdjE, en, ef);
    st_force(s, row + kAdjF, fn, ff);
    cur = X; vc = v; ac = a; mc = m;
  }
  // ---- inward: subtree sums complete on arrival; coordinate adjoints; sums handed to the parent ----
  const bool want_q = io.qt.valid() || io.qc.valid();
  for (int i = nb - 1; i >= 0; --i) {
    const BodyDev<T>& bd = M.body[i];
    const int row = kAdjBodyRows * i;
    T P[6], Q[6], E[6], F[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      P[k] = s.get(row + kAdjP + k); Q[k] = s.get(row + kAdjQ + k);
      E[k] = s.get(row + kAdjE + k); F[k] = s.get(row + kAdjF + k);
    }
    const int nvj = kind_nv_dev(bd.kind);
    if (nvj > 0) {
      Pose<T> X;
#pragma unroll
      for (int k = 0; k < 9; ++k) X.R[k] = s.get(row + k);
#pragma unroll
      for (int k = 0; k < 3; ++k) X.p[k] = s.get(row + 9 + k);
      Mot<T> vp, ap, mp, vj, vs;
      if (bd.flags & F_ROOT_CHILD) {
#pragma unroll
        for (int k = 0; k < 3; ++k) { vp.w[k] = vp.l[k] = ap.w[k] = mp.w[k] = mp.l[k] = T(0); ap.l[k] = -g[k]; }
      } else {
        const int prow = kAdjBodyRows * bd.parent;
        ld_mot(s, prow + kAdjV, vp);
        ld_mot(s, prow + kAdjA, ap);
        ld_mot(s, prow + kAdjM, mp);
      }
      ld_mot(s, row + kAdjV, vj);
#pragma unroll
      for (int k = 0; k < 3; ++k) { vs.w[k] = vj.w[k] + vp.w[k]; vs.l[k] = vj.l[k] + vp.l[k]; }
      T ft[6] = {T(0), T(0), T(0), T(0), T(0), T(0)};
      for (int k = 0; k < nvj; ++k) {
        Mot<T> S, pd, pdd, t1, t2, sdp, ms;
        world_subspace(X, sub_comp(bd.kind, k), S);
        const T sp = dot_mf(S, P, P + 3);
        if (io.vdb.valid()) io.vdb.st(bd.vrow + k, sp);
        motion_cross(vp, S, pd);
        if (io.vb.valid()) {
          motion_cross(vs, S, sdp);
          io.vb.st(bd.vrow + k, dot_mf(sdp, P, P + 3) + dot_mf(S, Q, Q + 3));
        }
        if (want_q) {
          motion_cross(ap, S, t1);
          motion_cross(vp, pd, t2);
#pragma unroll
          for (int c = 0; c < 3; ++c) { pdd.w[c] = t1.w[c] + t2.w[c]; pdd.l[c] = t1.l[c] + t2.l[c]; }
          motion_cross(mp, S, ms);
          const T x = dot_mf(pdd, P, P + 3) + dot_mf(pd, Q, Q + 3) + dot_mf(S, E, E + 3) + dot_mf(ms, F, F + 3);
          if (io.qt.valid()) io.qt.st(bd.vrow + k, x);
          // ft[k] = x with a warp-uniform k: a select chain keeps ft in registers
#pragma unroll
          for (int c = 0; c < 6; ++c) if (c == k) ft[c] = x;
        }
      }
      if (io.qc.valid()) cfg_adjoint(bd, io.q, ft, io.qc);
    }
    if (bd.flags & F_ROOT_CHILD) continue;
    const int prow = kAdjBodyRows * bd.parent;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      s.st(prow + kAdjP + k, s.get(prow + kAdjP + k) + P[k]);
      s.st(prow + kAdjQ + k, s.get(prow + kAdjQ + k) + Q[k]);
      s.st(prow + kAdjE + k, s.get(prow + kAdjE + k) + E[k]);
      s.st(prow + kAdjF + k, s.get(prow + kAdjF + k) + F[k]);
    }
  }
}

// The solve's IO: aba_sample on (q, zero velocity, τ = ν̄), v̇ into the workspace's μ rows.
template <class T> using MinvIO = AbaIO<T, false, kAllKinds>;

// Forward-dynamics VJP of one sample.  Mz: the model with ZERO gravity (the solve), g: the model's gravity (the sweep).
// vd_bar: ν̄;  tau_bar: τ̄ = μ (may be invalid).  io.vdb must be invalid.  zero: one scalar 0 that is not written while the kernel
// runs (the solve's velocity column reads it for every row, leading dimension 0).
template <class T, class ST>
RBD_HD void dynamics_vjp_sample(const ModelDev<T>& Mz, const T* g, const AdjIO<T>& io, const Col<T>& vd_bar,
                                const ColOut<T>& tau_bar, const T* zero, const ST& st) {
  const int mu0 = kAdjBodyRows * Mz.nb;
  MinvIO<T> a;
  a.q = io.q;
  a.v = {zero, 0};
  a.tau = vd_bar;
  a.wext = {nullptr, 0};
  a.vd = {io.s.p + (int64_t)mu0 * io.s.ld, io.s.ld, true};
  a.qd = {nullptr, 0, false};
  a.ext = {nullptr, 0};
  aba_sample<T, ST, true>(Mz, a, st);
  const ColRW<T> mu{io.s.p + (int64_t)mu0 * io.s.ld, io.s.ld};
  adjoint_sample<T>(Mz, g, io, mu, T(-1));
  if (tau_bar.valid())
    for (int k = 0; k < Mz.nv; ++k) tau_bar.st(k, mu(k));
}

}  // namespace rbd
