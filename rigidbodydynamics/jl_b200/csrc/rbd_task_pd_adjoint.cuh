// Reverse mode of the task-space law (rbd_integrate_task_pd_vjp / rbd_task_pd_torques_vjp, DESIGN 4.22): for the law of
// rbd_task_pd.cuh, u = Σ_t J_t(q)^T f_t(q, v; Kp, Kd, x_ref, ẋ_ref), and a velocity-row cotangent w [nv] (the masked τ̄ in torque
// mode, v̇̄_des from the inverse-dynamics VJP in computed-torque mode), the product  L = w . u  differentiated w.r.t. q, v, the
// gains and the references, one thread per sample, O(nb + ntasks) -- no Jacobian is formed or read.
//
// Derivation, ROOT-frame quantities and covector conventions of rbd_task_adjoint.cuh (f_n pose, t_n twist covectors of the
// named bodies, paired like wrenches with motion vectors):
//   δL = Σ_t [ ξ_t . δf_t  +  Σ_k w_k f_t . δJ_{t,k} ],   ξ_t = J_t w
// ξ_t is the task velocity w produces: with V = Σ_k ±S_k w_k (the relative twist of body w.r.t. base in the velocity field w) and
// V_p = V_l + V_w x p (p the task's point), ξ = R_F^T V_p (point) or (R_b^T V_w, R_b^T V_p) (pose).  So every body carries two
// twists, v_i from v (the law's ė) and τ_i from w (ξ and the Jacobian term).  f̄_t = ξ_t is pulled back through the law:
//   point  e = R_F^T (d - R_a x_ref), ė = R_F^T (v_p - R_a ẋ_ref), f = -Kp e - Kd ė  (d = p - p_a, v_p the point's velocity in v):
//          K̄p -= ξ e, K̄d -= ξ ė;  d̄ = -R_F Kp ξ, ū = -R_F Kd ξ;  x̄_ref -= R_a^T d̄, ẋ̄_ref -= R_a^T ū;  p̄ = d̄ + ū x rel_w
//          f_b += (p x p̄, p̄);  f_a -= ((p_a + R_a x_ref) x d̄ + (R_a ẋ_ref) x ū, d̄);  f_F += (d̄ x (d - R_a x_ref) + ū x (v_p - R_a
//          ẋ_ref), 0);  t_b += (p x ū, ū), t_a -= the same
//   pose   R_e = R_ref^T R_a^T R_b, p_e = R_ref^T (R_a^T d - p_ref), ψ = log R_e (Shepperd quaternion, quat_from_rot ->
//          rotvec_from_quat), l = R_e^T p_e; ang = -Kω ψ - Dω (R_b^T rel_w - ω_ref), lin = -Kv l - Dv (R_b^T v_p - v_ref):
//          K̄p, K̄d, ẋ̄_ref as the point's, row by row;  ω̄ = -R_b Dω ξ_w, ū = -R_b Dv ξ_l;  t_b += (ω̄ + p x ū, ū), t_a -= the same;
//          f_b += (ω̄ x rel_w + ū x v_p, 0) + (p x p̄, p̄) with p̄ = ū x rel_w;
//          R̄_e = p_e l̄^T + (∂ψ/∂R_e)^T ψ̄ (Dual1 through quat_from_rot / rotvec_from_quat, nine directions, on the branch the forward
//          took: exact at ψ = 0 and near π), p̄_e = R_e l̄ (ψ̄ = -Kω ξ_w, l̄ = -Kv ξ_l);  x̄_ref: R̄_ref = R_a^T R_b R̄_e^T + y p̄_e^T
//          (all nine entries as given: the law does not re-orthonormalise), p̄_ref = -ȳ, ȳ = R_ref p̄_e, y = R_a^T d - p_ref;
//          d̄ = R_a ȳ, G = R_a R_ref R̄_e R_b^T:  f_b += (ax(G) + p x d̄, d̄),  f_a -= the same
// The Jacobian term is rbd_task_kinematics_vjp's column pass with the rank-one cotangent J̄_k = w_k f_t (the point Jacobian in F;
// for a pose task the geometric Jacobian of C, whose angular rows are the body-frame geometric Jacobian and linear rows the point
// Jacobian).  Summed over the columns in closed form it needs only the root-frame law wrench (n_t, c_t) and V:
//   column k (joint body i):  W_i += w_k S_k x* Σ_t ±(n_t, c_t)      (the aggregate wrench of the forward J^T pass)
//   per task:  f_b += (p x y, y), y = c_t x V_w;  f_F += (c_t x V_p, 0);  pose (F = b):  f_b -= V x* (R_b ang, 0)
// Inward sweep as rbd_task_adjoint.cuh's without accelerations: T_J = Σ t_n, W_J = Σ (f_n + v_n x* t_n) + column terms,
//   v̄_j = S_j . T_J,   q̄_j = S_j . W_J + (v_p x S_j) . T_J,   q̄_cfg by cfg_adjoint.
//
// Workspace (one column per resident thread): task_pose_sweep's pending slots, then kTpSlotRows per named slot, 6 per task (the law
// wrench), kTpBodyRows per body and nq rows for cfg_adjoint's output.
#pragma once
#include "rbd_integrate_adjoint.cuh"
#include "rbd_task_adjoint.cuh"
#include "rbd_task_pd.cuh"

namespace rbd {

constexpr int kTpSlotRows = 36;      // named slot: rotation 9, origin 3 (task_pose), v-twist 6 (kTaV), w-twist 6, f 6, t 6
constexpr int kTpW = 18, kTpF = 24, kTpT = 30;
constexpr int kTpBodyRows = 36;      // body: pose 12, v-twist 6 (kTaV), w-twist 6 (kTpW), subtree sums T, W
constexpr int kTpST = 24, kTpSW = 30;

// The law's descriptor with the VJP's slot layout (build_task_pd_dev's, slots widened to kTpSlotRows).  Returns the workspace rows
// per sample.
template <class T> inline int build_task_pd_vjp_dev(const HostModel& hm, const rbd_task_pd_desc& c, TaskPdDev<T>& D) {
  build_task_pd_dev<T>(hm, c, D);
  const int nnamed = (D.wrench_base - D.t.named_base) / D.t.slot_rows;
  D.t.slot_rows = kTpSlotRows;
  D.wrench_base = D.t.named_base + nnamed * kTpSlotRows;
  return D.wrench_base + 6 * D.t.ntasks + kTpBodyRows * hm.nb + hm.nq;
}

// One sample: the law's arrays (s, rbd_task_pd.cuh) and their adjoints, each pointer offset by the sample's column, row stride bld
// (NULL = not wanted); kpb / kdb are per sample even for shared gains.
template <class T> struct TaskPdBarIO {
  Col<T> q, v, w;
  TaskPdSample<T> s;
  T *kpb, *kdb, *xrefb, *xdrefb;
  int64_t bld;
  Scr<T> scr;
};

// o += sg x (3-vectors)
template <class T> RBD_HD void tp_add3(T* o, const T* x, T sg) {
#pragma unroll
  for (int k = 0; k < 3; ++k) o[k] += sg * x[k];
}

// The law's adjoint at one sample: q̄ (configuration coordinates) to out_qc(row, x), v̄ to out_v(row, x), each row once; the bars
// of io are added to.
template <class T, class FC, class FV>
RBD_HD void task_pd_vjp_sample(const ModelDev<T>& M, const TaskPdDev<T>& D, const TaskPdBarIO<T>& io, FC&& out_qc, FV&& out_v) {
  const TaskDev<T>& td = D.t;
  const int nb = M.nb, K = td.ntasks;
  const ScrStash<T> w{io.scr};
  const int bb = D.wrench_base + 6 * K, cb = bb + kTpBodyRows * nb;

  // ---- outward: pose, v-twist and w-twist of every body and named slot; sums and covectors zeroed ----
  task_pose_sweep(M, td, io.q, w, [&](int i, const BodyDev<T>& bd, const Pose<T>& X) {
    Mot<T> v, u;
    if (bd.flags & F_ROOT_CHILD) {
#pragma unroll
      for (int k = 0; k < 3; ++k) v.w[k] = v.l[k] = u.w[k] = u.l[k] = T(0);
    } else {
      ld_mot(io.scr, bb + kTpBodyRows * bd.parent + kTaV, v);
      ld_mot(io.scr, bb + kTpBodyRows * bd.parent + kTpW, u);
    }
    const int nvj = kind_nv_dev(bd.kind);
    for (int k = 0; k < nvj; ++k) {
      Mot<T> S;
      world_subspace(X, sub_comp(bd.kind, k), S);
      const T x = io.v(bd.vrow + k), y = io.w(bd.vrow + k);
#pragma unroll
      for (int c = 0; c < 3; ++c) { v.w[c] += x * S.w[c]; v.l[c] += x * S.l[c]; u.w[c] += y * S.w[c]; u.l[c] += y * S.l[c]; }
    }
    const int row = bb + kTpBodyRows * i;
#pragma unroll
    for (int k = 0; k < 9; ++k) w.st(row + k, X.R[k]);
#pragma unroll
    for (int k = 0; k < 3; ++k) w.st(row + 9 + k, X.p[k]);
    st_mot(io.scr, row + kTaV, v);
    st_mot(io.scr, row + kTpW, u);
#pragma unroll
    for (int k = 0; k < 12; ++k) w.st(row + kTpST + k, T(0));
    const int s = td.named[i];
    if (s >= 0) {
      const int srow = td.named_base + s * td.slot_rows;
      st_mot(io.scr, srow + kTaV, v);
      st_mot(io.scr, srow + kTpW, u);
#pragma unroll
      for (int k = 0; k < 12; ++k) w.st(srow + kTpF + k, T(0));
    }
  });

  // ---- the law and its adjoint, one task at a time ----
  for (int tk = 0; tk < K; ++tk) {
    const int bs = td.body_slot[tk], as = td.base_slot[tk], fs = td.frame_slot[tk];
    T Rb[9], pb[3], Ra[9], pa[3], p[3], d[3], x[3], vp[3], Vp[3];
    task_pose(td, w, bs, Rb, pb);
    task_pose(td, w, as, Ra, pa);
    Mot<T> tb, ta, ub, ua, rel, V;
    task_mot(td, w, bs, kTaV, tb);
    task_mot(td, w, as, kTaV, ta);
    task_mot(td, w, bs, kTpW, ub);
    task_mot(td, w, as, kTpW, ua);
    mat_vec(Rb, td.point[tk], x);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      p[c] = pb[c] + x[c];
      d[c] = p[c] - pa[c];
      rel.w[c] = tb.w[c] - ta.w[c]; rel.l[c] = tb.l[c] - ta.l[c];
      V.w[c] = ub.w[c] - ua.w[c]; V.l[c] = ub.l[c] - ua.l[c];
    }
    cross3(rel.w, p, x);
#pragma unroll
    for (int c = 0; c < 3; ++c) vp[c] = rel.l[c] + x[c];
    cross3(V.w, p, x);
#pragma unroll
    for (int c = 0; c < 3; ++c) Vp[c] = V.l[c] + x[c];
    const int r0 = D.row[tk], x0 = D.xrow[tk];
    const TaskPdSample<T>& s = io.s;
    auto kp = [&](int k) { return s.kp[(int64_t)(r0 + k) * s.gstride]; };
    auto kd = [&](int k) { return s.kd[(int64_t)(r0 + k) * s.gstride]; };
    auto xr = [&](int k) { return s.xref[(int64_t)(x0 + k) * s.ld]; };
    auto xd = [&](int k) { return s.xdref ? s.xdref[(int64_t)(r0 + k) * s.ld] : T(0); };
    auto bar = [&](T* a, int r, T val) { if (a) a[(int64_t)r * io.bld] += val; };
    // covector additions of this task: f_b, f_a, f_F (angular only), t_b (t_a = -t_b); the law wrench (n, c) and, for a pose task,
    // its angular part ar at C in root axes
    T fbn[3] = {T(0), T(0), T(0)}, fbf[3] = {T(0), T(0), T(0)}, fan[3] = {T(0), T(0), T(0)}, faf[3] = {T(0), T(0), T(0)};
    T fFn[3] = {T(0), T(0), T(0)}, tn[3], tf[3], n[3], c[3], pbar[3];
    if (D.kind[tk] == RBD_TASK_POINT) {
      T RF[9], pF[3], er[3], e[3], vr[3], ve[3], xi[3], eb[3], vb[3], dr[3], ub_[3], y[3];
      task_pose(td, w, fs, RF, pF);
      T xrv[3], xdv[3], axr[3], axd[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) { xrv[k] = xr(k); xdv[k] = xd(k); }
      mat_vec(Ra, xrv, axr);
      mat_vec(Ra, xdv, axd);
      {                                  // the forward law as task_pd_wrench evaluates it
        T xb[3], ebb[3];
        matT_vec(Ra, d, xb);
#pragma unroll
        for (int k = 0; k < 3; ++k) ebb[k] = xb[k] - xrv[k];
        mat_vec(Ra, ebb, er);
        matT_vec(RF, er, e);
#pragma unroll
        for (int k = 0; k < 3; ++k) vr[k] = vp[k] - axd[k];
        matT_vec(RF, vr, ve);
        T fF[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) fF[k] = -kp(k) * e[k] - kd(k) * ve[k];
        mat_vec(RF, fF, c);
        cross3(p, c, n);
      }
      matT_vec(RF, Vp, xi);              // ξ: the point velocity w produces, in F
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        bar(io.kpb, r0 + k, -xi[k] * e[k]);
        bar(io.kdb, r0 + k, -xi[k] * ve[k]);
        eb[k] = -kp(k) * xi[k];
        vb[k] = -kd(k) * xi[k];
      }
      mat_vec(RF, eb, dr);
      mat_vec(RF, vb, ub_);
      matT_vec(Ra, dr, y);
#pragma unroll
      for (int k = 0; k < 3; ++k) bar(io.xrefb, x0 + k, -y[k]);
      matT_vec(Ra, ub_, y);
#pragma unroll
      for (int k = 0; k < 3; ++k) bar(io.xdrefb, r0 + k, -y[k]);
      cross3(ub_, rel.w, y);
#pragma unroll
      for (int k = 0; k < 3; ++k) pbar[k] = dr[k] + y[k];
      T rp[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) rp[k] = pa[k] + axr[k];
      cross3(rp, dr, y); tp_add3(fan, y, T(-1));
      cross3(axd, ub_, y); tp_add3(fan, y, T(-1));
      tp_add3(faf, dr, T(-1));
      cross3(dr, er, y); tp_add3(fFn, y, T(1));
      cross3(ub_, vr, y); tp_add3(fFn, y, T(1));
      cross3(p, ub_, tn);
#pragma unroll
      for (int k = 0; k < 3; ++k) tf[k] = ub_[k];
      cross3(c, Vp, y); tp_add3(fFn, y, T(1));      // the Jacobian term: f_F += (c x V_p, 0)
    } else {
      T Rx[9], px[3], Rr[9], pr[3], Re[9], pe[3], y[3], qe[4], psi[3], th2, le[3], wc[3], vc[3], ang[3], lin[3];
      mat_tmul3(Ra, Rb, Rx);
      matT_vec(Ra, d, px);
#pragma unroll
      for (int k = 0; k < 9; ++k) Rr[k] = xr(k);
#pragma unroll
      for (int k = 0; k < 3; ++k) { pr[k] = xr(9 + k); y[k] = px[k] - pr[k]; }
      mat_tmul3(Rr, Rx, Re);
      matT_vec(Rr, y, pe);
      quat_from_rot(Re, qe);
      rotvec_from_quat(qe, psi, th2);
      matT_vec(Re, pe, le);
      matT_vec(Rb, rel.w, wc);
      matT_vec(Rb, vp, vc);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        ang[k] = -kp(k) * psi[k] - kd(k) * (wc[k] - xd(k));
        lin[k] = -kp(3 + k) * le[k] - kd(3 + k) * (vc[k] - xd(3 + k));
      }
      T ar[3];
      mat_vec(Rb, lin, c);
      mat_vec(Rb, ang, ar);
      cross3(p, c, x);
#pragma unroll
      for (int k = 0; k < 3; ++k) n[k] = ar[k] + x[k];
      T xia[3], xil[3], psib[3], lb[3], wb[3], vb[3], om[3], ub_[3];
      matT_vec(Rb, V.w, xia);            // ξ: the twist of C that w produces, in C
      matT_vec(Rb, Vp, xil);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        bar(io.kpb, r0 + k, -xia[k] * psi[k]);
        bar(io.kpb, r0 + 3 + k, -xil[k] * le[k]);
        bar(io.kdb, r0 + k, -xia[k] * (wc[k] - xd(k)));
        bar(io.kdb, r0 + 3 + k, -xil[k] * (vc[k] - xd(3 + k)));
        bar(io.xdrefb, r0 + k, kd(k) * xia[k]);
        bar(io.xdrefb, r0 + 3 + k, kd(3 + k) * xil[k]);
        psib[k] = -kp(k) * xia[k];
        lb[k] = -kp(3 + k) * xil[k];
        wb[k] = -kd(k) * xia[k];
        vb[k] = -kd(3 + k) * xil[k];
      }
      mat_vec(Rb, wb, om);
      mat_vec(Rb, vb, ub_);
      cross3(p, ub_, tn);
#pragma unroll
      for (int k = 0; k < 3; ++k) { tn[k] += om[k]; tf[k] = ub_[k]; }
      cross3(om, rel.w, x); tp_add3(fbn, x, T(1));
      cross3(ub_, vp, x); tp_add3(fbn, x, T(1));
      cross3(ub_, rel.w, pbar);
      // R̄_e: from l = R_e^T p_e, then from ψ through the quaternion (Dual1, one entry of R_e per pass)
      T Reb[9], peb[3];
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) Reb[3 * i + j] = pe[i] * lb[j];
      mat_vec(Re, lb, peb);
      using D1 = Dual1<T>;
      for (int dir = 0; dir < 9; ++dir) {
        D1 dR[9], dq[4], dpsi[3], dth;
#pragma unroll
        for (int k = 0; k < 9; ++k) dR[k] = D1(Re[k], dir == k ? T(1) : T(0));
        quat_from_rot(dR, dq);
        rotvec_from_quat(dq, dpsi, dth);
        Reb[dir] += psib[0] * dpsi[0].d + psib[1] * dpsi[1].d + psib[2] * dpsi[2].d;
      }
      // x̄_ref: R̄_ref = R_x R̄_e^T + y p̄_e^T, p̄_ref = -ȳ
      T yb[3];
      mat_vec(Rr, peb, yb);
#pragma unroll
      for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 3; ++j)
          bar(io.xrefb, x0 + 3 * i + j, Rx[3 * i] * Reb[3 * j] + Rx[3 * i + 1] * Reb[3 * j + 1] + Rx[3 * i + 2] * Reb[3 * j + 2] + y[i] * peb[j]);
        bar(io.xrefb, x0 + 9 + i, -yb[i]);
      }
      T db[3], G[9], Y[9], Z[9];
      mat_vec(Ra, yb, db);
      mat_mul3(Ra, Rr, Y);               // G = R_a R_ref R̄_e R_b^T
      mat_mul3(Y, Reb, Z);
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) G[3 * i + j] = Z[3 * i] * Rb[3 * j] + Z[3 * i + 1] * Rb[3 * j + 1] + Z[3 * i + 2] * Rb[3 * j + 2];
      T ag[3] = {G[7] - G[5], G[2] - G[6], G[3] - G[1]};
      cross3(p, db, x);
#pragma unroll
      for (int k = 0; k < 3; ++k) { fbn[k] += ag[k]; fan[k] -= ag[k] + x[k]; faf[k] -= db[k]; pbar[k] += db[k]; }
      // the Jacobian term (F = b): f_b += (c x V_p, 0) - V x* (ar, 0)
      cross3(c, Vp, x); tp_add3(fbn, x, T(1));
      cross3(V.w, ar, x); tp_add3(fbn, x, T(-1));
    }
    {                                    // the Jacobian term: f_b += (p x y, y), y = c x V_w
      T yv[3];
      cross3(c, V.w, yv);
      tp_add3(pbar, yv, T(1));
    }
    cross3(p, pbar, x);
    tp_add3(fbn, x, T(1));
    tp_add3(fbf, pbar, T(1));
    const int wrow = D.wrench_base + 6 * tk;
#pragma unroll
    for (int k = 0; k < 3; ++k) { w.st(wrow + k, n[k]); w.st(wrow + 3 + k, c[k]); }
    if (bs >= 0) {
      const int srow = td.named_base + bs * td.slot_rows;
      task_add6(w, srow + kTpF, fbn, fbf, T(1));
      task_add6(w, srow + kTpT, tn, tf, T(1));
    }
    if (as >= 0) {
      const int srow = td.named_base + as * td.slot_rows;
      task_add6(w, srow + kTpF, fan, faf, T(1));
      task_add6(w, srow + kTpT, tn, tf, T(-1));
    }
    if (D.kind[tk] == RBD_TASK_POINT && fs >= 0) {      // a pose task's F is its body: already in f_b
      const T z[3] = {T(0), T(0), T(0)};
      task_add6(w, td.named_base + fs * td.slot_rows + kTpF, fFn, z, T(1));
    }
  }

  // ---- inward: the column terms, named covectors folded in on arrival, coordinate adjoints, sums handed to the parent ----
  for (int i = nb - 1; i >= 0; --i) {
    const BodyDev<T>& bd = M.body[i];
    const int row = bb + kTpBodyRows * i;
    T Tt[6], W[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) { Tt[k] = w.ld(row + kTpST + k); W[k] = w.ld(row + kTpSW + k); }
    const int s = td.named[i];
    if (s >= 0) {
      const int srow = td.named_base + s * td.slot_rows;
      T f[6], t[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) { f[k] = w.ld(srow + kTpF + k); t[k] = w.ld(srow + kTpT + k); Tt[k] += t[k]; W[k] += f[k]; }
      Mot<T> vi;
      ld_mot(io.scr, row + kTaV, vi);
      task_fcross_add(vi, t, t + 3, T(1), W, W + 3);           // W += v x* t
    }
    const int nvj = kind_nv_dev(bd.kind);
    if (nvj > 0) {
      Pose<T> X;
#pragma unroll
      for (int k = 0; k < 9; ++k) X.R[k] = w.ld(row + k);
#pragma unroll
      for (int k = 0; k < 3; ++k) X.p[k] = w.ld(row + 9 + k);
      for (int k = 0; k < nvj; ++k) {    // W += w_k S_k x* Σ_t ±(n_t, c_t)
        Mot<T> S;
        world_subspace(X, sub_comp(bd.kind, k), S);
        T On[3] = {T(0), T(0), T(0)}, Of[3] = {T(0), T(0), T(0)};
        for (int tk = 0; tk < K; ++tk) {
          const int sg = task_bit(td.body_mask[tk], i) - task_bit(td.base_mask[tk], i);
          if (sg == 0) continue;
          const int wrow = D.wrench_base + 6 * tk;
#pragma unroll
          for (int c = 0; c < 3; ++c) { On[c] += T(sg) * w.ld(wrow + c); Of[c] += T(sg) * w.ld(wrow + 3 + c); }
        }
        task_fcross_add(S, On, Of, io.w(bd.vrow + k), W, W + 3);
      }
      Mot<T> vp;
      if (bd.flags & F_ROOT_CHILD) {
#pragma unroll
        for (int k = 0; k < 3; ++k) vp.w[k] = vp.l[k] = T(0);
      } else {
        ld_mot(io.scr, bb + kTpBodyRows * bd.parent + kTaV, vp);
      }
      T ft[6] = {T(0), T(0), T(0), T(0), T(0), T(0)};
      for (int k = 0; k < nvj; ++k) {
        Mot<T> S, pd;
        world_subspace(X, sub_comp(bd.kind, k), S);
        out_v(bd.vrow + k, dot_mf(S, Tt, Tt + 3));
        motion_cross(vp, S, pd);
        const T x = dot_mf(S, W, W + 3) + dot_mf(pd, Tt, Tt + 3);
        // ft[k] = x with a warp-uniform k: a select chain keeps ft in registers
#pragma unroll
        for (int c = 0; c < 6; ++c) if (c == k) ft[c] = x;
      }
      const int nqj = kind_nq_dev(bd.kind);
      cfg_adjoint(bd, io.q, ft, ColOut<T>{io.scr.p + (int64_t)cb * io.scr.ld, io.scr.ld, true});
      for (int k = 0; k < nqj; ++k) out_qc(bd.qrow + k, w.ld(cb + bd.qrow + k));
    }
    if (bd.flags & F_ROOT_CHILD) continue;
    const int prow = bb + kTpBodyRows * bd.parent;
#pragma unroll
    for (int k = 0; k < 6; ++k) { w.add(prow + kTpST + k, Tt[k]); w.add(prow + kTpSW + k, W[k]); }
  }
}

// ---- one sample of rbd_integrate_task_pd_vjp's / rbd_task_pd_torques_vjp's kernel ------------------------------------------
// Every array is [rows x B] (dense).  w: the cotangent of the law's output rows.  qacc / vacc receive += q̄ (configuration
// coordinates) / v̄ of the law, plus qfold / vfold when set (computed-torque mode without a joint term: the inverse-dynamics VJP's
// q̄ / v̄, which no phase kernel reads otherwise).  has_joint: the joint term's adjoint (pd_adj_joint) in the same pass, with
// joint.idq / idv / idvd set in computed-torque mode (rbd_task_pd_torques_vjp; the rollout's phase kernels do it there).
template <class T> struct TaskPdVjpArgs {
  const T *q, *v, *w;
  const T *xref, *xdref, *kp, *kd; int64_t gain_ld;    // the task references of the step, the gains
  T *kpb, *kdb, *xrefb, *xdrefb;                       // added to; NULL = not wanted
  T *qacc, *vacc;
  const T *qfold, *vfold;
  PdAdjArgs<T> joint; bool has_joint;
  T* work;                                             // [rows][resident threads]
  int64_t B;
};

template <class T>
RBD_HD void task_pd_vjp_column(const ModelDev<T>& M, const TaskPdDev<T>& D, const TaskPdVjpArgs<T>& a, int64_t b, bool active,
                               const Scr<T>& scr) {
  const int64_t B = a.B;
  if (a.has_joint && active) {
    AdjStepArgs<T> st{};
    st.qs[0] = a.q; st.vs[0] = a.v; st.taub = a.w; st.ld = B; st.g = 0;
    for (int i = 0; i < M.nb; ++i) {
      const BodyDev<T>& bd = M.body[i];
      const int nq = kind_nq_dev(bd.kind), nv = kind_nv_dev(bd.kind);
      if (nv == 0) continue;
      T cq[7], cv[6], m[6];
      pd_adj_joint(bd, st, a.joint, b, cq, cv, m);
      for (int k = 0; k < nq; ++k) a.qacc[(int64_t)(bd.qrow + k) * B + b] += cq[k];
      for (int k = 0; k < nv; ++k) a.vacc[(int64_t)(bd.vrow + k) * B + b] += cv[k];
    }
  }
  const int64_t gc = a.gain_ld ? b : 0;
  TaskPdBarIO<T> io;
  io.q = {a.q + b, B}; io.v = {a.v + b, B}; io.w = {a.w + b, B};
  io.s = TaskPdSample<T>{a.xref + b, a.xdref ? a.xdref + b : nullptr, B, a.kp + gc, a.kd + gc, a.gain_ld ? a.gain_ld : 1};
  auto o = [&](T* p) { return (p && active) ? p + b : nullptr; };
  io.kpb = o(a.kpb); io.kdb = o(a.kdb); io.xrefb = o(a.xrefb); io.xdrefb = o(a.xdrefb); io.bld = B;
  io.scr = scr;
  task_pd_vjp_sample<T>(M, D, io,
      [&](int r, T x) {
        if (!active) return;
        const int64_t e = (int64_t)r * B + b;
        a.qacc[e] += (a.qfold ? a.qfold[e] : T(0)) + x;
      },
      [&](int r, T x) {
        if (!active) return;
        const int64_t e = (int64_t)r * B + b;
        a.vacc[e] += (a.vfold ? a.vfold[e] : T(0)) + x;
      });
}

}  // namespace rbd
