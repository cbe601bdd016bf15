// Reverse mode of task-space kinematics (rbd_task_kinematics_vjp, DESIGN 4.20): for the tasks of rbd_task_kinematics (rbd_task.cuh)
// and cotangents ȳ on any subset of its eight outputs, the product  L = Σ ȳ . y  differentiated w.r.t. q, v and v̇, one thread per
// sample, O(nb + size of the cotangents) -- no nv x nv object.  Every forward quantity is recomputed from (q, v, v̇).
//
// Derivation, ROOT-frame quantities as in rbd_adjoint.cuh: X_i pose, S_k world-frame subspace column, v_i twist, a_i = a_p +
// v_p x (S v) + S v̇ (no gravity, a_root = 0).  Every output is a function of the poses, twists and accelerations of the bodies a
// task names (body b, base a, frame F), and the Jacobians also of the columns S_k on the task's path.  L is pulled back onto three
// root-frame covectors per named body n, all paired like wrenches with motion vectors:
//   f_n  pose:          dL = f_n . δ  when body n alone moves rigidly by the root-frame twist δ (R' = (I + ω^) R, p' = p + ω x p + ν)
//   t_n  twist:         dL = t_n . δv_n
//   α_n  acceleration:  dL = α_n . δa_n
// Epilogue adjoint of one task, with the F-frame cotangents gathered first (point_acceleration -> acceleration, point, twist and
// point_velocity; point_velocity -> twist and point), then mapped to the root by the wrench transform X_F^* (n = R_F c_w + p_F x
// R_F c_l, f = R_F c_l):
//   ψ = X_F^* (ā),  φ = X_F^* (t̄),  c = R_F p̄  (p the point in the root frame, rel = v_b - v_a, x = a_b - a_a, y = x - v_F x rel)
//   α_b += ψ, α_a -= ψ;  t_b += φ + v_F x* ψ, t_a -= the same;  t_F -= rel x* ψ        (af = Ad(T_F^-1)(x - v_F x rel))
//   f_b += (p x c, c);  f_F -= (p x c, c) + rel x* φ + y x* ψ                           (Ad(T_F^-1) m changes by Ad(T_F^-1)(m x δ))
//   transform:  f_b += (ax(G) + p_b x c_r, c_r),  f_a -= the same,  G = R_a R̄ R_b^T, c_r = R_a p̄_r, ax(G) = (G32 - G23, G13 - G31,
//               G21 - G12)
// Jacobian columns: with J̄, J̄p the cotangents of column k of a task (sign s folded in, S = s S_k), φ_k = X_F^* (J̄) + (p x c_k, c_k),
// c_k = R_F J̄p, so that the column contributes S . φ_k.  Moving coordinate j rotates S_k with the subtree (δS_k = S_j x S_k), which
// gives the per-column term  S_k x* φ_k  attached to the column's body; F's pose enters through -S x* X_F^*(J̄) and the angular
// c_k x (S_l + S_w x p); the point through b's pose as (p x y, y), y = Σ_k c_k x S_w.
// Inward sweep, the convention of rbd_adjoint.cuh: moving coordinate j of joint J moves sub(J) rigidly by S_j, so every body-fixed
// motion vector m of sub(J) changes by S_j x m, except for the parts that do not follow: Ψ̇_j = v_p x S_j in every v_i and
// Ψ̈_j + Ψ̇_j x v_i in every a_i, Ψ̈_j = a_p x S_j + v_p x Ψ̇_j (p = parent of J).  With the subtree sums over named bodies and columns
//   A_J = Σ α_n,   T_J = Σ (t_n + v_n x* α_n),   W_J = Σ (f_n + v_n x* t_n + a_n x* α_n) + Σ_columns S_k x* φ_k
// (identity used: (a x b) . f = -b . (a x* f)):
//   v̇̄_j = S_j . A_J
//   v̄_j = S_j . T_J + Sdp_j . A_J,                Sdp_j = (v_J + v_p) x S_j   (d a_n / d v_j = Sdp_j + S_j x v_n)
//   q̄_j = S_j . W_J + Ψ̇_j . T_J + Ψ̈_j . A_J      (tangent derivative along velocity_to_configuration_derivative(e_j))
// q̄_cfg is q̄_tan mapped by cfg_adjoint (rbd_adjoint.cuh).
//
// Work split: one thread per sample.  Outward sweep: pose, twist and acceleration of every body into its workspace rows, the sums
// zeroed; each named body's caller-frame pose, twist and acceleration into its named slot (the layout task_pose / task_mot read).
// Then the epilogue adjoint per task, the Jacobian columns per task (the task's F and point held in registers, the covectors of F
// and b accumulated in registers and added once), and the inward sweep (reverse preorder), which folds a named body's covectors into
// its sums on arrival, forms its coordinates' adjoints and hands its sums to the parent.  Workspace: kTaskAdjRows rows per body and
// kTaskAdjSlotRows per named slot, one column per resident thread (rbd_adjoint.cu).
#pragma once
#include "rbd_adjoint.cuh"
#include "rbd_task.cuh"

namespace rbd {

constexpr int kTaskAdjRows = 42;       // pose 12, v 6, a 6, then the subtree sums A, T, W
constexpr int kTaV = 12, kTaA = 18, kTaSA = 24, kTaST = 30, kTaSW = 36;
constexpr int kTaskAdjSlotRows = 42;   // named slot: caller-frame rotation 9, origin 3, v 6, a 6 (task_pose / task_mot), then f, t, α
constexpr int kTaF = 24, kTaT = 30, kTaAl = 36;

// Workspace rows per sample for nb bodies and nnamed named slots.
inline int task_adjoint_rows(int nb, int nnamed) { return kTaskAdjRows * nb + kTaskAdjSlotRows * nnamed; }

// The workspace column with the ld / st interface of a stash (task_pose, task_mot).
template <class T> struct ScrStash {
  Scr<T> s;
  RBD_HD T ld(int row) const { return s.get(row); }
  RBD_HD void st(int row, T v) const { s.st(row, v); }
  RBD_HD void add(int row, T v) const { s.st(row, s.get(row) + v); }
};

template <class T> struct TaskBarIO {
  Col<T> q, v, vd;                    // v may be invalid when no velocity-dependent cotangent is given; vd invalid = zero
  Col<T> tr, pt, tw, pv, J, Jp, acc, pacc;   // cotangents in the layout of the outputs; invalid = zero
  ColOut<T> qt, qc, vb, vdb;          // q̄_tan [nv], q̄_cfg [nq], v̄ [nv], v̇̄ [nv]; each may be invalid
  Scr<T> s;                           // this thread's workspace column
};

// rows row .. row + 5 += sg (n, f)
template <class T> RBD_HD void task_add6(const ScrStash<T>& w, int row, const T* n, const T* f, T sg) {
#pragma unroll
  for (int k = 0; k < 3; ++k) { w.add(row + k, sg * n[k]); w.add(row + 3 + k, sg * f[k]); }
}
// covector c = (cw, cl) given in frame F -> root-frame wrench X_F^* c:  f = R_F cl, n = R_F cw + p_F x f
template <class T> RBD_HD void task_force_to_root(const T* RF, const T* pF, const Mot<T>& c, T* n, T* f) {
  T x[3];
  mat_vec(RF, c.l, f);
  mat_vec(RF, c.w, n);
  cross3(pF, f, x);
#pragma unroll
  for (int k = 0; k < 3; ++k) n[k] += x[k];
}
// o = sg (m x* (n, f)) added to (on, of)
template <class T> RBD_HD void task_fcross_add(const Mot<T>& m, const T* n, const T* f, T sg, T* on, T* of) {
  T a[3], b[3];
  force_cross(m, n, f, a, b);
#pragma unroll
  for (int k = 0; k < 3; ++k) { on[k] += sg * a[k]; of[k] += sg * b[k]; }
}

template <class T>
RBD_HD void task_vjp_sample(const ModelDev<T>& M, const TaskDev<T>& D, const TaskBarIO<T>& io) {
  const int nb = M.nb, nv = M.nv, K = D.ntasks;
  const ScrStash<T> w{io.s};
  const bool jac = io.J.valid() || io.Jp.valid();
  const bool want_acc = io.acc.valid() || io.pacc.valid();
  const bool want_vel = want_acc || io.tw.valid() || io.pv.valid();
  const bool want_q = io.qt.valid() || io.qc.valid();

  // ---- outward: pose, twist, acceleration of every body; named slots; sums and covectors zeroed ----
  {
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
      T R[9], r[3], t[3];
      frame_any(bd, io.q, R, r);
      Pose<T> X;
      mat_mul3(pp.R, R, X.R);
      mat_vec(pp.R, r, t);
      X.p[0] = pp.p[0] + t[0]; X.p[1] = pp.p[1] + t[1]; X.p[2] = pp.p[2] + t[2];
      Mot<T> v = vp, a = ap;
      if (want_vel) {
        Mot<T> jt, ja, cm;
#pragma unroll
        for (int k = 0; k < 3; ++k) jt.w[k] = jt.l[k] = ja.w[k] = ja.l[k] = T(0);
        const int nvj = kind_nv_dev(bd.kind);
        for (int k = 0; k < nvj; ++k) {
          Mot<T> S;
          world_subspace(X, sub_comp(bd.kind, k), S);
          const T x = io.v(bd.vrow + k);
          const T xd = (want_acc && io.vd.valid()) ? io.vd(bd.vrow + k) : T(0);
#pragma unroll
          for (int c = 0; c < 3; ++c) { jt.w[c] += x * S.w[c]; jt.l[c] += x * S.l[c]; ja.w[c] += xd * S.w[c]; ja.l[c] += xd * S.l[c]; }
        }
        motion_cross(vp, jt, cm);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          v.w[k] = vp.w[k] + jt.w[k]; v.l[k] = vp.l[k] + jt.l[k];
          a.w[k] = ap.w[k] + cm.w[k] + ja.w[k]; a.l[k] = ap.l[k] + cm.l[k] + ja.l[k];
        }
      }
      const int row = kTaskAdjRows * i;
#pragma unroll
      for (int k = 0; k < 9; ++k) w.st(row + k, X.R[k]);
#pragma unroll
      for (int k = 0; k < 3; ++k) w.st(row + 9 + k, X.p[k]);
      if (want_vel) { st_mot(io.s, row + kTaV, v); st_mot(io.s, row + kTaA, a); }
#pragma unroll
      for (int k = 0; k < 18; ++k) w.st(row + kTaSA + k, T(0));
      const int s = D.named[i];
      if (s >= 0) {
        T Rc[9];
        mat_mul3(X.R, D.At[s], Rc);
        const int srow = D.named_base + s * D.slot_rows;
#pragma unroll
        for (int k = 0; k < 9; ++k) w.st(srow + k, Rc[k]);
#pragma unroll
        for (int k = 0; k < 3; ++k) w.st(srow + 9 + k, X.p[k]);
        if (want_vel) { st_mot(io.s, srow + kTaV, v); st_mot(io.s, srow + kTaA, a); }
#pragma unroll
        for (int k = 0; k < 18; ++k) w.st(srow + kTaF + k, T(0));
      }
      cur = X; vc = v; ac = a;
    }
  }

  // ---- epilogue adjoint, one task at a time: covectors of the named bodies ----
  const bool epi = want_vel || (want_q && (io.tr.valid() || io.pt.valid()));
  for (int tk = 0; epi && tk < K; ++tk) {
    const int bs = D.body_slot[tk], as = D.base_slot[tk], fs = D.frame_slot[tk];
    const int brow = D.named_base + bs * D.slot_rows, arow = D.named_base + as * D.slot_rows, frow = D.named_base + fs * D.slot_rows;
    T Rb[9], pb[3], Ra[9], pa[3], RF[9], pF[3];
    task_pose(D, w, bs, Rb, pb);
    task_pose(D, w, as, Ra, pa);
    task_pose(D, w, fs, RF, pF);
    if (io.tr.valid()) {                 // inv(T_base) T_body
      T Rbar[9], G[9], Y[9], pr[3], cr[3], n[3], x[3];
#pragma unroll
      for (int k = 0; k < 9; ++k) Rbar[k] = io.tr(12 * tk + k);
#pragma unroll
      for (int k = 0; k < 3; ++k) pr[k] = io.tr(12 * tk + 9 + k);
      mat_mul3(Ra, Rbar, Y);             // G = Ra R̄ Rb^T
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) G[3 * i + j] = Y[3 * i] * Rb[3 * j] + Y[3 * i + 1] * Rb[3 * j + 1] + Y[3 * i + 2] * Rb[3 * j + 2];
      mat_vec(Ra, pr, cr);
      cross3(pb, cr, x);
      n[0] = G[7] - G[5] + x[0]; n[1] = G[2] - G[6] + x[1]; n[2] = G[3] - G[1] + x[2];
      if (bs >= 0) task_add6(w, brow + kTaF, n, cr, T(1));
      if (as >= 0) task_add6(w, arow + kTaF, n, cr, T(-1));
    }
    T p[3], pf[3];                       // the point in the root frame and in F
    {
      T x[3], d[3];
      mat_vec(Rb, D.point[tk], x);
#pragma unroll
      for (int c = 0; c < 3; ++c) { p[c] = pb[c] + x[c]; d[c] = p[c] - pF[c]; }
      matT_vec(RF, d, pf);
    }
    // F-frame cotangents: point pbar, twist tbar, acceleration abar
    T pbar[3] = {T(0), T(0), T(0)};
    Mot<T> tbar, abar;
#pragma unroll
    for (int c = 0; c < 3; ++c) tbar.w[c] = tbar.l[c] = abar.w[c] = abar.l[c] = T(0);
    if (io.pt.valid()) {
#pragma unroll
      for (int c = 0; c < 3; ++c) pbar[c] = io.pt(3 * tk + c);
    }
    Mot<T> twb, twa, rel, twf, twF;
    if (want_vel) {
      task_mot(D, w, bs, kTaV, twb);
      task_mot(D, w, as, kTaV, twa);
      task_mot(D, w, fs, kTaV, twF);
#pragma unroll
      for (int c = 0; c < 3; ++c) { rel.w[c] = twb.w[c] - twa.w[c]; rel.l[c] = twb.l[c] - twa.l[c]; }
      task_to_frame(RF, pF, rel, twf);
      T upv[3] = {T(0), T(0), T(0)};     // point_velocity cotangent, point_acceleration's share included
      if (io.pacc.valid()) {             // pacc = af_w x pf + af_l + tw_w x pv
        T u[3], pv[3], x[3];
        Mot<T> ab, aa, y, af;
#pragma unroll
        for (int c = 0; c < 3; ++c) u[c] = io.pacc(3 * tk + c);
        cross3(twf.w, pf, x);
#pragma unroll
        for (int c = 0; c < 3; ++c) pv[c] = x[c] + twf.l[c];
        task_mot(D, w, bs, kTaA, ab);
        task_mot(D, w, as, kTaA, aa);
        Mot<T> cm;
        motion_cross(twF, rel, cm);
#pragma unroll
        for (int c = 0; c < 3; ++c) { y.w[c] = ab.w[c] - aa.w[c] - cm.w[c]; y.l[c] = ab.l[c] - aa.l[c] - cm.l[c]; }
        task_to_frame(RF, pF, y, af);
        T e[3];
        cross3(pf, u, e);                // abar += (pf x u, u)
#pragma unroll
        for (int c = 0; c < 3; ++c) { abar.w[c] += e[c]; abar.l[c] += u[c]; }
        cross3(u, af.w, e);              // pbar += u x af_w
#pragma unroll
        for (int c = 0; c < 3; ++c) pbar[c] += e[c];
        cross3(pv, u, e);                // tbar_w += pv x u
#pragma unroll
        for (int c = 0; c < 3; ++c) tbar.w[c] += e[c];
        cross3(u, twf.w, e);             // upv += u x tw_w
#pragma unroll
        for (int c = 0; c < 3; ++c) upv[c] += e[c];
      }
      if (io.acc.valid()) {
#pragma unroll
        for (int c = 0; c < 3; ++c) { abar.w[c] += io.acc(6 * tk + c); abar.l[c] += io.acc(6 * tk + 3 + c); }
      }
      if (io.pv.valid()) {
#pragma unroll
        for (int c = 0; c < 3; ++c) upv[c] += io.pv(3 * tk + c);
      }
      if (io.pv.valid() || io.pacc.valid()) {   // pv = tw_w x pf + tw_l
        T e[3];
        cross3(pf, upv, e);
#pragma unroll
        for (int c = 0; c < 3; ++c) { tbar.w[c] += e[c]; tbar.l[c] += upv[c]; }
        cross3(upv, twf.w, e);
#pragma unroll
        for (int c = 0; c < 3; ++c) pbar[c] += e[c];
      }
      if (io.tw.valid()) {
#pragma unroll
        for (int c = 0; c < 3; ++c) { tbar.w[c] += io.tw(6 * tk + c); tbar.l[c] += io.tw(6 * tk + 3 + c); }
      }
    }
    // to the root frame
    T c[3], fn[3], ff[3];                // f_b's share (p x c, c); f_F gets minus it and the frame terms
    mat_vec(RF, pbar, c);
    cross3(p, c, fn);
#pragma unroll
    for (int k = 0; k < 3; ++k) ff[k] = c[k];
    if (bs >= 0) task_add6(w, brow + kTaF, fn, ff, T(1));
    T Fn[3], Ff[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { Fn[k] = -fn[k]; Ff[k] = -ff[k]; }
    if (want_vel) {
      T phn[3], phf[3], psn[3], psf[3], tn[3], tf[3];
      task_force_to_root(RF, pF, tbar, phn, phf);
      task_force_to_root(RF, pF, abar, psn, psf);
#pragma unroll
      for (int k = 0; k < 3; ++k) { tn[k] = phn[k]; tf[k] = phf[k]; }
      task_fcross_add(twF, psn, psf, T(1), tn, tf);            // + v_F x* ψ
      if (bs >= 0) { task_add6(w, brow + kTaT, tn, tf, T(1)); task_add6(w, brow + kTaAl, psn, psf, T(1)); }
      if (as >= 0) { task_add6(w, arow + kTaT, tn, tf, T(-1)); task_add6(w, arow + kTaAl, psn, psf, T(-1)); }
      if (fs >= 0) {
        T un[3] = {T(0), T(0), T(0)}, uf[3] = {T(0), T(0), T(0)};
        task_fcross_add(rel, psn, psf, T(-1), un, uf);         // t_F -= rel x* ψ
        task_add6(w, frow + kTaT, un, uf, T(1));
        task_fcross_add(rel, phn, phf, T(-1), Fn, Ff);         // f_F -= rel x* φ + y x* ψ
        if (want_acc) {
          Mot<T> ab, aa, y, cm;
          task_mot(D, w, bs, kTaA, ab);
          task_mot(D, w, as, kTaA, aa);
          motion_cross(twF, rel, cm);
#pragma unroll
          for (int k = 0; k < 3; ++k) { y.w[k] = ab.w[k] - aa.w[k] - cm.w[k]; y.l[k] = ab.l[k] - aa.l[k] - cm.l[k]; }
          task_fcross_add(y, psn, psf, T(-1), Fn, Ff);
        }
      }
    }
    if (fs >= 0) task_add6(w, frow + kTaF, Fn, Ff, T(1));
  }

  // ---- Jacobian columns, one task at a time ----
  for (int tk = 0; jac && want_q && tk < K; ++tk) {
    const int bs = D.body_slot[tk], fs = D.frame_slot[tk];
    T RF[9], pF[3], Rb[9], pb[3], p[3], x[3];
    task_pose(D, w, fs, RF, pF);
    task_pose(D, w, bs, Rb, pb);
    mat_vec(Rb, D.point[tk], x);
#pragma unroll
    for (int c = 0; c < 3; ++c) p[c] = pb[c] + x[c];
    T Fn[3] = {T(0), T(0), T(0)}, Ff[3] = {T(0), T(0), T(0)}, y[3] = {T(0), T(0), T(0)};
    const int grow = tk * 6 * nv, prow = tk * 3 * nv;
    for (int i = 0; i < nb; ++i) {
      const int sg = task_bit(D.body_mask[tk], i) - task_bit(D.base_mask[tk], i);
      const BodyDev<T>& bd = M.body[i];
      const int nvj = kind_nv_dev(bd.kind);
      if (sg == 0 || nvj == 0) continue;
      const int row = kTaskAdjRows * i;
      Pose<T> X;
#pragma unroll
      for (int k = 0; k < 9; ++k) X.R[k] = w.ld(row + k);
#pragma unroll
      for (int k = 0; k < 3; ++k) X.p[k] = w.ld(row + 9 + k);
      T Wn[3] = {T(0), T(0), T(0)}, Wf[3] = {T(0), T(0), T(0)};
      for (int k = 0; k < nvj; ++k) {
        const int col = bd.vrow + k;
        Mot<T> S;
        world_subspace(X, sub_comp(bd.kind, k), S);
#pragma unroll
        for (int c = 0; c < 3; ++c) { S.w[c] *= T(sg); S.l[c] *= T(sg); }
        T phn[3] = {T(0), T(0), T(0)}, phf[3] = {T(0), T(0), T(0)};
        if (io.J.valid()) {
          Mot<T> jb;
#pragma unroll
          for (int c = 0; c < 3; ++c) { jb.w[c] = io.J(grow + 6 * col + c); jb.l[c] = io.J(grow + 6 * col + 3 + c); }
          task_force_to_root(RF, pF, jb, phn, phf);
          if (fs >= 0) task_fcross_add(S, phn, phf, T(-1), Fn, Ff);     // f_F -= S x* X_F^*(J̄)
        }
        if (io.Jp.valid()) {
          T jp[3], ck[3], e[3], u[3];
#pragma unroll
          for (int c = 0; c < 3; ++c) jp[c] = io.Jp(prow + 3 * col + c);
          mat_vec(RF, jp, ck);
          cross3(p, ck, e);
#pragma unroll
          for (int c = 0; c < 3; ++c) { phn[c] += e[c]; phf[c] += ck[c]; }
          cross3(ck, S.w, e);            // y += c x S_w
#pragma unroll
          for (int c = 0; c < 3; ++c) y[c] += e[c];
          if (fs >= 0) {                 // f_F angular += c x (S_l + S_w x p)
            cross3(S.w, p, e);
#pragma unroll
            for (int c = 0; c < 3; ++c) u[c] = S.l[c] + e[c];
            cross3(ck, u, e);
#pragma unroll
            for (int c = 0; c < 3; ++c) Fn[c] += e[c];
          }
        }
        task_fcross_add(S, phn, phf, T(1), Wn, Wf);
      }
      task_add6(w, row + kTaSW, Wn, Wf, T(1));
    }
    if (fs >= 0) task_add6(w, D.named_base + fs * D.slot_rows + kTaF, Fn, Ff, T(1));
    if (bs >= 0 && io.Jp.valid()) {
      T n[3];
      cross3(p, y, n);
      task_add6(w, D.named_base + bs * D.slot_rows + kTaF, n, y, T(1));
    }
  }

  // ---- inward: named covectors folded in on arrival; coordinate adjoints; sums handed to the parent ----
  for (int i = nb - 1; i >= 0; --i) {
    const BodyDev<T>& bd = M.body[i];
    const int row = kTaskAdjRows * i;
    T A[6], Tt[6], W[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) { A[k] = w.ld(row + kTaSA + k); Tt[k] = w.ld(row + kTaST + k); W[k] = w.ld(row + kTaSW + k); }
    Mot<T> vi, ai;
    if (want_vel) { ld_mot(io.s, row + kTaV, vi); ld_mot(io.s, row + kTaA, ai); }
    const int s = D.named[i];
    if (s >= 0) {
      const int srow = D.named_base + s * D.slot_rows;
      T f[6], t[6], al[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) { f[k] = w.ld(srow + kTaF + k); t[k] = w.ld(srow + kTaT + k); al[k] = w.ld(srow + kTaAl + k); }
#pragma unroll
      for (int k = 0; k < 6; ++k) { A[k] += al[k]; Tt[k] += t[k]; W[k] += f[k]; }
      if (want_vel) {
        task_fcross_add(vi, al, al + 3, T(1), Tt, Tt + 3);     // T += v x* α
        task_fcross_add(vi, t, t + 3, T(1), W, W + 3);          // W += v x* t + a x* α
        task_fcross_add(ai, al, al + 3, T(1), W, W + 3);
      }
    }
    const int nvj = kind_nv_dev(bd.kind);
    if (nvj > 0) {
      Pose<T> X;
#pragma unroll
      for (int k = 0; k < 9; ++k) X.R[k] = w.ld(row + k);
#pragma unroll
      for (int k = 0; k < 3; ++k) X.p[k] = w.ld(row + 9 + k);
      Mot<T> vp, ap;
#pragma unroll
      for (int k = 0; k < 3; ++k) vp.w[k] = vp.l[k] = ap.w[k] = ap.l[k] = T(0);
      if (want_vel && !(bd.flags & F_ROOT_CHILD)) {
        const int prow = kTaskAdjRows * bd.parent;
        ld_mot(io.s, prow + kTaV, vp);
        ld_mot(io.s, prow + kTaA, ap);
      }
      T ft[6] = {T(0), T(0), T(0), T(0), T(0), T(0)};
      for (int k = 0; k < nvj; ++k) {
        Mot<T> S;
        world_subspace(X, sub_comp(bd.kind, k), S);
        if (io.vdb.valid()) io.vdb.st(bd.vrow + k, want_acc ? dot_mf(S, A, A + 3) : T(0));
        if (io.vb.valid()) {
          T x = T(0);
          if (want_vel) {
            Mot<T> vs, sdp;
#pragma unroll
            for (int c = 0; c < 3; ++c) { vs.w[c] = vi.w[c] + vp.w[c]; vs.l[c] = vi.l[c] + vp.l[c]; }
            motion_cross(vs, S, sdp);
            x = dot_mf(S, Tt, Tt + 3) + dot_mf(sdp, A, A + 3);
          }
          io.vb.st(bd.vrow + k, x);
        }
        if (want_q) {
          T x = dot_mf(S, W, W + 3);
          if (want_vel) {
            Mot<T> pd, pdd, t1, t2;
            motion_cross(vp, S, pd);
            motion_cross(ap, S, t1);
            motion_cross(vp, pd, t2);
#pragma unroll
            for (int c = 0; c < 3; ++c) { pdd.w[c] = t1.w[c] + t2.w[c]; pdd.l[c] = t1.l[c] + t2.l[c]; }
            x += dot_mf(pd, Tt, Tt + 3) + dot_mf(pdd, A, A + 3);
          }
          if (io.qt.valid()) io.qt.st(bd.vrow + k, x);
          // ft[k] = x with a warp-uniform k: a select chain keeps ft in registers
#pragma unroll
          for (int c = 0; c < 6; ++c) if (c == k) ft[c] = x;
        }
      }
      if (io.qc.valid()) cfg_adjoint(bd, io.q, ft, io.qc);
    }
    if (bd.flags & F_ROOT_CHILD) continue;
    const int prow = kTaskAdjRows * bd.parent;
#pragma unroll
    for (int k = 0; k < 6; ++k) { w.add(prow + kTaSA + k, A[k]); w.add(prow + kTaST + k, Tt[k]); w.add(prow + kTaSW + k, W[k]); }
  }
}

// TaskDev for the VJP: build_task_dev's tasks and named slots, the slots placed behind the bodies' workspace rows.  Returns the
// number of named slots.
template <class T> inline int build_task_vjp_dev(const HostModel& hm, const rbd_task_desc& d, TaskDev<T>& D) {
  const int nnamed = build_task_dev<T>(hm, d, true, true, D);
  D.named_base = kTaskAdjRows * hm.nb;
  D.slot_rows = kTaskAdjSlotRows;
  return nnamed;
}

}  // namespace rbd
