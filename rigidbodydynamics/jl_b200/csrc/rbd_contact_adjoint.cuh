// Reverse mode through the contact rollout (rbd_integrate_contact_vjp, DESIGN 4.15): the adjoint of the contact pass and of the
// contact-state chain of the RK4 tableau, on top of the rollout adjoint of rbd_integrate_adjoint.cuh (DESIGN 4.13).
//
// Per stage i of a step the contact rollout (DESIGN 4.14) computes
//   s_i = s0 + dt a_i ṡ_{i-1},   (w_c, ṡ_i) = C(qs_i, vs_i, s_i),   v̇_i = FD(qs_i, vs_i, τ_i, w_c),   and at the end  s1 = s0 + dt Σ b_i ṡ_i
// with C the contact pass (contact_force per pair in contact; w_c the root-frame wrenches of the bodies that carry points).
// The backward step of rbd_integrate_adjoint.cuh is extended by
//   s-chain (Euclidean, elementwise):  finish  s̄0 = s̄1, ṡ̄_i = dt b_i s̄1;   stage i  s̄0 += s̄_i, ṡ̄_{i-1} += dt a_i s̄_i
//   contact adjoint at stage i, from w̄_b = -m_b (the forward-dynamics VJP's path sum, rbd_adjoint.cuh) and ṡ̄_i, per pair in contact:
//     wrench (pt x f, f):       f̄ = v̄_l + ω̄ x pt,  p̄t += f x ω̄                      (w̄_b = (ω̄, v̄_l))
//     contact_force adjoint:    (f̄, ṡ̄) -> (z̄, vēl, x̄),  s̄_i += x̄
//     z = -(pt - h.point) . n:  p̄t -= z̄ n
//     vel = ω x pt + v_l:       W_v += (pt x vēl, vēl)     (the body twist's covector)
//     pt = T_b loc:             W_p += (pt x p̄t, p̄t)     (the body pose's covector: pt moves by S_j when q_j moves)
//   and per joint coordinate j of joint J (p = parent of J), with the subtree sums over the contact bodies b of sub(J)
//     A_J = Σ W_v,b,   D_J = Σ (W_p,b + V_b x* W_v,b)      (V_b: root-frame twist of b)
//     v̄_j += S_j . A_J,   q̄_j += S_j . (D_J - V_p x* A_J)
//   The twist-through-q term comes from ∂S_k/∂q_j = S_j x S_k (k in sub(J)): ∂V_b/∂q_j = S_j x (V_b - V_p), and
//   W . (S x V) = S . (V x* W).  O(n) per sample; no nv x nv or point-Jacobian object is formed.
// A pair out of contact has ṡ = 0 and no wrench: its s̄ passes through unchanged (frozen, DESIGN 4.14).
//
// contact_force is differentiated AS IMPLEMENTED, on the branch it takes (in contact, max(f_n, 0), stick or slip), by forward-mode
// Dual1 through the same templated code (7 directions: z, vel, x).  At z = 0 (a point exactly on the surface) the derivative of
// z^n is its one-sided limit: 0 for n > 1, 1 for n = 1 (and 0 for n < 1, where the limit is infinite); sqrt at 0 has derivative 0
// (only reached by the slip clip when f_n = 0, with a zero direction).
//
// Work split: contact_vjp_sample, one thread per sample, replaces the forward-dynamics VJP of each stage: an outward wrench pass
// (pose and twist parked in the adjoint workspace rows, root-frame wrenches into 6 nb rows), dynamics_vjp_sample with those
// wrenches, then the contact adjoint, which reads pose, twist and m_b back from the rows adjoint_sample parked and sweeps inward
// once for the two subtree sums, the v̄ additions and the configuration covector.
#pragma once
#include "rbd_integrate_adjoint.cuh"

namespace rbd {

// products with the descriptor's plain scalars, z^n and sqrt on duals, for contact_force<Dual1<F>>
template <class F> RBD_HD Dual1<F> operator*(const Dual1<F>& a, F b) { return {a.v * b, a.d * b}; }
template <class F> RBD_HD Dual1<F> operator*(F a, const Dual1<F>& b) { return {a * b.v, a * b.d}; }
template <class F> RBD_HD Dual1<F> contact_pow(const Dual1<F>& z, F n) {
  const F zn = contact_pow(z.v, n);
  const F d = z.v > F(0) ? n * zn / z.v : (n == F(1) ? F(1) : F(0));
  return {zn, d * z.d};
}
template <class F> RBD_HD Dual1<F> contact_sqrt(const Dual1<F>& x) { return sqrt_t(x); }

// The adjoint of contact_force at one pair in contact: (f̄, ẋ̄) -> z̄, vēl, x̄; f: the force itself
template <class T>
RBD_HD void contact_force_adjoint(const ContactDev<T>& C, int pi, const T* n, T z, const T* vel, const T* x, const T* fb, const T* xdb,
                                  T* f, T& zb, T* velb, T* xb) {
  using D = Dual1<T>;
  for (int dir = 0; dir < 7; ++dir) {
    const D dz(z, dir == 0 ? T(1) : T(0));
    D dv[3], dx[3], df[3], dxd[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { dv[k] = D(vel[k], dir == 1 + k ? T(1) : T(0)); dx[k] = D(x[k], dir == 4 + k ? T(1) : T(0)); }
    contact_force(C, pi, n, dz, dv, [&](int k) { return dx[k]; }, df, dxd);
    T s = T(0);
#pragma unroll
    for (int k = 0; k < 3; ++k) s += fb[k] * df[k].d + xdb[k] * dxd[k].d;
    if (dir == 0) {
      zb = s;
#pragma unroll
      for (int k = 0; k < 3; ++k) f[k] = df[k].v;
    } else if (dir < 4) {
      velb[dir - 1] = s;
    } else {
      xb[dir - 4] = s;
    }
  }
}

// One stage of the contact rollout's backward step for one sample.  Every array column has leading dimension ld.
template <class T> struct ContactVjpIO {
  Col<T> q, v, vd, vdb;             // stage state (qs_l, vs_l), its recorded v̇_l, and ν̄ = v̇̄_l
  ColOut<T> qc, taub;               // q̄_cfg [nq] (written), τ̄ [nv] (written; may be invalid)
  T* vb;                            // v̄ [nv] (written)
  const T* s0; const T* sdp;        // contact state at the step's start, ṡ_{l-1} (NULL at stage 0): s_l = s0 + wa ṡ_{l-1}
  T* sb1; T* sacc; T* sdc;          // s̄1 of the step; the running s̄0; dt a_l s̄_l handed to stage l - 1
  const T* stb;                     // trajectory adjoint of the step's start state (read at stage 0), or NULL
  int64_t ld;
  T wa, wdb;                        // (T)(dt a_l), (T)dt * (T)b_l
  int l;
  Scr<T> s;                         // workspace column: adjoint_rows(nb, nv), then 6 nb wrench rows, then nv tangent rows
  bool active;
};

inline int contact_vjp_rows(int nb, int nv) { return adjoint_rows(nb, nv) + 6 * nb + nv; }

// pose and twist of body i from its parent's workspace rows (the outward sweeps of this file and of adjoint_sample park them there)
template <class T> RBD_HD void cv_pose_twist(const BodyDev<T>& bd, const Col<T>& q, const Col<T>& v, const Scr<T>& s, Pose<T>& X, Mot<T>& V) {
  Pose<T> pp;
  Mot<T> vp;
  if (bd.flags & F_ROOT_CHILD) {
    pose_identity(pp);
#pragma unroll
    for (int k = 0; k < 3; ++k) vp.w[k] = vp.l[k] = T(0);
  } else {
    const int row = kAdjBodyRows * bd.parent;
#pragma unroll
    for (int k = 0; k < 9; ++k) pp.R[k] = s.get(row + k);
#pragma unroll
    for (int k = 0; k < 3; ++k) pp.p[k] = s.get(row + 9 + k);
    ld_mot(s, row + kAdjV, vp);
  }
  T R[9], r[3], t[3];
  frame_any(bd, q, R, r);
  mat_mul3(pp.R, R, X.R);
  mat_vec(pp.R, r, t);
  X.p[0] = pp.p[0] + t[0]; X.p[1] = pp.p[1] + t[1]; X.p[2] = pp.p[2] + t[2];
  V = vp;
  const int nvj = kind_nv_dev(bd.kind);
  for (int k = 0; k < nvj; ++k) {
    Mot<T> S;
    world_subspace(X, sub_comp(bd.kind, k), S);
    const T x = v(bd.vrow + k);
#pragma unroll
    for (int c = 0; c < 3; ++c) { V.w[c] += x * S.w[c]; V.l[c] += x * S.l[c]; }
  }
}

template <class T> RBD_HD void cv_point(const Pose<T>& X, const Mot<T>& V, const T* loc, T* pt, T* vel) {
  T tmp[3];
  mat_vec(X.R, loc, tmp);
  pt[0] = X.p[0] + tmp[0]; pt[1] = X.p[1] + tmp[1]; pt[2] = X.p[2] + tmp[2];
  cross3(V.w, pt, vel);
  vel[0] += V.l[0]; vel[1] += V.l[1]; vel[2] += V.l[2];
}

template <class T> RBD_HD T cv_sep(const ContactDev<T>& C, int h, const T* pt) {
  const T* n = C.hn[h];
  return (pt[0] - C.hp[h][0]) * n[0] + (pt[1] - C.hp[h][1]) * n[1] + (pt[2] - C.hp[h][2]) * n[2];
}

// Mz: the model with ZERO gravity (the solve), g: the model's gravity (the sweeps), as dynamics_vjp_sample
template <class T, class ST>
RBD_HD void contact_vjp_sample(const ModelDev<T>& Mz, const T* g, const ContactDev<T>& C, const ContactVjpIO<T>& io, const T* zero,
                               const ST& st) {
  const int nb = Mz.nb;
  const Scr<T>& s = io.s;
  const int w0 = kAdjBodyRows * nb + Mz.nv, t0 = w0 + 6 * nb;     // adjoint_rows(nb, nv)
  auto state = [&](int64_t e) { return io.sdp ? io.s0[e * io.ld] + io.wa * io.sdp[e * io.ld] : io.s0[e * io.ld]; };
  // ---- the stage's contact wrenches, root frame, rows 6 refidx of the wrench block (contact_stage_pass's force law) ----
  for (int i = 0; i < nb; ++i) {
    const BodyDev<T>& bd = Mz.body[i];
    Pose<T> X;
    Mot<T> V;
    cv_pose_twist(bd, io.q, io.v, s, X, V);
    const int row = kAdjBodyRows * i;
#pragma unroll
    for (int k = 0; k < 9; ++k) s.st(row + k, X.R[k]);
#pragma unroll
    for (int k = 0; k < 3; ++k) s.st(row + 9 + k, X.p[k]);
    st_mot(s, row + kAdjV, V);
    T wn[3] = {T(0), T(0), T(0)}, wf[3] = {T(0), T(0), T(0)};
    for (int pi = C.first[i]; pi < C.first[i + 1]; ++pi) {
      T pt[3], vel[3];
      cv_point(X, V, C.loc[pi], pt, vel);
      for (int h = 0; h < C.nhalf; ++h) {
        const int64_t srow = (int64_t)3 * (C.orig[pi] * C.nhalf + h);
        const T sep = cv_sep(C, h, pt);
        if (sep <= T(0)) {
          T f[3], xd[3], m[3];
          contact_force(C, pi, C.hn[h], -sep, vel, [&](int k) { return state(srow + k); }, f, xd);
          cross3(pt, f, m);
#pragma unroll
          for (int k = 0; k < 3; ++k) { wn[k] += m[k]; wf[k] += f[k]; }
        }
      }
    }
    const int orow = w0 + 6 * bd.refidx;
    st_force(s, orow, wn, wf);
  }
  // ---- the forward-dynamics VJP with those wrenches; q̄ in tangent form into the workspace ----
  AdjIO<T, ColRW<T>> a;
  a.q = io.q; a.v = io.v; a.vd = io.vd;
  a.wext = {s.p + (int64_t)w0 * s.ld, s.ld};
  a.qt = {s.p + (int64_t)t0 * s.ld, s.ld, true};
  a.qc = {nullptr, 0, false};
  a.vb = {io.vb, io.ld, io.active};
  a.vdb = {nullptr, 0, false};
  a.wb = {nullptr, 0, false};
  a.s = s;
  dynamics_vjp_sample<T>(Mz, g, a, io.vdb, io.taub, zero, st);
  // ---- contact adjoint: per body W_v (rows kAdjP) and D = W_p + V x* W_v (rows kAdjQ); the s-chain of the pair rows ----
  for (int i = 0; i < nb; ++i) {
    const int row = kAdjBodyRows * i;
    T An[3] = {T(0), T(0), T(0)}, Af[3] = {T(0), T(0), T(0)}, Dn[3] = {T(0), T(0), T(0)}, Df[3] = {T(0), T(0), T(0)};
    if (C.first[i + 1] > C.first[i]) {
      Pose<T> X;
      Mot<T> V, m;
#pragma unroll
      for (int k = 0; k < 9; ++k) X.R[k] = s.get(row + k);
#pragma unroll
      for (int k = 0; k < 3; ++k) X.p[k] = s.get(row + 9 + k);
      ld_mot(s, row + kAdjV, V);
      ld_mot(s, row + kAdjM, m);
      const T wb[3] = {-m.w[0], -m.w[1], -m.w[2]}, lb[3] = {-m.l[0], -m.l[1], -m.l[2]};     // w̄_b = (ω̄, v̄_l) = -m_b
      for (int pi = C.first[i]; pi < C.first[i + 1]; ++pi) {
        T pt[3], vel[3];
        cv_point(X, V, C.loc[pi], pt, vel);
        for (int h = 0; h < C.nhalf; ++h) {
          const int64_t srow = (int64_t)3 * (C.orig[pi] * C.nhalf + h);
          const T sep = cv_sep(C, h, pt);
          T sdb[3], sb[3] = {T(0), T(0), T(0)};
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            const int64_t e = (srow + k) * io.ld;
            sdb[k] = io.wdb * io.sb1[e] + (io.l < 3 ? io.sdc[e] : T(0));
          }
          if (sep <= T(0)) {
            T x[3], fb[3], f[3], zb, velb[3], pb[3], t[3];
            for (int k = 0; k < 3; ++k) x[k] = state(srow + k);
            cross3(wb, pt, fb);
#pragma unroll
            for (int k = 0; k < 3; ++k) fb[k] += lb[k];
            contact_force_adjoint(C, pi, C.hn[h], -sep, vel, x, fb, sdb, f, zb, velb, sb);
            cross3(f, wb, pb);                     // wrench
            cross3(velb, V.w, t);                  // vel = ω x pt + v_l
#pragma unroll
            for (int k = 0; k < 3; ++k) pb[k] += t[k] - zb * C.hn[h][k];
            cross3(pt, velb, t);
#pragma unroll
            for (int k = 0; k < 3; ++k) { An[k] += t[k]; Af[k] += velb[k]; Df[k] += pb[k]; }
            cross3(pt, pb, t);
#pragma unroll
            for (int k = 0; k < 3; ++k) Dn[k] += t[k];
          }
          if (io.active) {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
              const int64_t e = (srow + k) * io.ld;
              if (io.l == 3) io.sacc[e] = io.sb1[e] + sb[k];
              else if (io.l > 0) io.sacc[e] += sb[k];
              else io.sb1[e] = io.sacc[e] + sb[k] + (io.stb ? io.stb[e] : T(0));
              if (io.l > 0) io.sdc[e] = io.wa * sb[k];
            }
          }
        }
      }
      T vn[3], vf[3];
      force_cross(V, An, Af, vn, vf);
#pragma unroll
      for (int k = 0; k < 3; ++k) { Dn[k] += vn[k]; Df[k] += vf[k]; }
    }
    st_force(s, row + kAdjP, An, Af);
    st_force(s, row + kAdjQ, Dn, Df);
  }
  // ---- inward: subtree sums complete on arrival; v̄ += S . A, q̄_tan += S . (D - V_p x* A), then the configuration covector ----
  for (int i = nb - 1; i >= 0; --i) {
    const BodyDev<T>& bd = Mz.body[i];
    const int row = kAdjBodyRows * i;
    T A[6], Dv[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) { A[k] = s.get(row + kAdjP + k); Dv[k] = s.get(row + kAdjQ + k); }
    const int nvj = kind_nv_dev(bd.kind);
    if (nvj > 0) {
      Pose<T> X;
#pragma unroll
      for (int k = 0; k < 9; ++k) X.R[k] = s.get(row + k);
#pragma unroll
      for (int k = 0; k < 3; ++k) X.p[k] = s.get(row + 9 + k);
      T Dq[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) Dq[k] = Dv[k];
      if (!(bd.flags & F_ROOT_CHILD)) {
        Mot<T> vp;
        ld_mot(s, kAdjBodyRows * bd.parent + kAdjV, vp);
        T tn[3], tf[3];
        force_cross(vp, A, A + 3, tn, tf);
#pragma unroll
        for (int k = 0; k < 3; ++k) { Dq[k] -= tn[k]; Dq[3 + k] -= tf[k]; }
      }
      T ft[6] = {T(0), T(0), T(0), T(0), T(0), T(0)};
      for (int k = 0; k < nvj; ++k) {
        Mot<T> S;
        world_subspace(X, sub_comp(bd.kind, k), S);
        const int r = bd.vrow + k;
        if (io.active) io.vb[(int64_t)r * io.ld] += dot_mf(S, A, A + 3);
        const T x = s.get(t0 + r) + dot_mf(S, Dq, Dq + 3);
#pragma unroll
        for (int c = 0; c < 6; ++c) if (c == k) ft[c] = x;
      }
      cfg_adjoint(bd, io.q, ft, io.qc);
    }
    if (bd.flags & F_ROOT_CHILD) continue;
    const int prow = kAdjBodyRows * bd.parent;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      s.st(prow + kAdjP + k, s.get(prow + kAdjP + k) + A[k]);
      s.st(prow + kAdjQ + k, s.get(prow + kAdjQ + k) + Dv[k]);
    }
  }
}

}  // namespace rbd
