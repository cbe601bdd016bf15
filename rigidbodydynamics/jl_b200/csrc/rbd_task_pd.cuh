// Task-space feedback (rbd_integrate_task_pd / rbd_task_pd_torques, DESIGN 4.21): the per-task law and the per-joint J^T
// accumulation, shared by task_pd_kernel (rbd_b200.cu) and, compiled for the host, by tests/hostsim/hostsim_task_pd.cpp.
//
// Each task of an rbd_task_desc yields a 3- or 6-vector f_t in its task frame, and the controller adds u = Σ_t J_t^T f_t to the
// joint-space command.  Signs follow the reference's pd(gains, e, ė) = -k e - d ė (src/pdcontrol.jl:35); gains are diagonal.
//   point (RBD_TASK_POINT, 3 rows)  x = the point relative to base, in base coordinates; F = the task's frame:
//       e = R_F<-base (x - x_ref),  ė = point_velocity_F - R_F<-base ẋ_ref,  f = -Kp e - Kd ė  (FramePDGains: F rotates the gains),
//       J_t = the point Jacobian in F
//   pose (RBD_TASK_POSE, 6 rows)  the controlled frame C has its origin at the task's point and the body's axes; x = C -> base,
//       T = twist of C w.r.t. base in C, x_ref [12] (rotation row-major, translation) and T_ref [6] the targets; with e = inv(x_ref) x,
//       ψ the rotation vector of R_e and p_e its translation (SE3PDMethod{:DoubleGeodesic}, src/pdcontrol.jl:83-107):
//       ang = -Kω ψ - Dω (ω - ω_ref),  lin = -Kv R_e^T p_e - Dv (v - v_ref),  J_t = the geometric Jacobian of C in C
// J is never formed: f_t becomes a root-frame wrench w_t = [n; f] (moment about the root origin, force), and every joint on the
// task's path adds ±S_k . w_t with S_k its root-frame subspace column (the path signs of rbd_task_kinematics: +1 down, -1 up).
// task_pd_sample runs task_sample's sweeps A and B (the named bodies' poses and twists), the law per task, then the pose sweep
// again with the J^T pass.
#pragma once
#include "rbd_pd.cuh"
#include "rbd_task.cuh"

namespace rbd {

template <class T> struct TaskPdDev {
  TaskDev<T> t;
  int32_t wrench_base;                 // first stash row of the per-task wrenches (6 rows each), behind the named slots
  int32_t R, X;                        // rows of kp / kd / ẋ_ref (Σ 3 | 6) and of x_ref (Σ 3 | 12)
  int32_t pad_;
  int8_t kind[kMaxTasks];
  int16_t row[kMaxTasks], xrow[kMaxTasks];   // first row of task t in kp / kd / ẋ_ref and in x_ref
};

// One sample's view of the law's caller arrays, each pointer already offset by the sample's column:
//   xref [X], xdref [R] (NULL = 0): leading dimension ld;  kp, kd [R]: row stride gstride (1: shared by the batch; ld: per sample)
template <class T> struct TaskPdSample {
  const T* xref; const T* xdref; int64_t ld;
  const T* kp; const T* kd; int64_t gstride;
};

// stash rows [row, ...) of one sample as an output column (task_sample's outputs parked in the stash)
template <class T, int S> RBD_HD ColOut<T> stash_rows(const Stash<T, S>& st, int row) { return ColOut<T>{st.p + row * S, S, true}; }

// unit quaternion [w x y z] of a rotation matrix (row-major), pivoting on the largest of w, x, y, z (Shepperd): accurate at
// every angle, 0 and pi included
template <class T> RBD_HD void quat_from_rot(const T* R, T* q) {
  const T tr = R[0] + R[4] + R[8];
  if (tr >= R[0] && tr >= R[4] && tr >= R[8]) {
    const T s = T(2) * sqrt_t(T(1) + tr);
    q[0] = T(0.25) * s; q[1] = (R[7] - R[5]) / s; q[2] = (R[2] - R[6]) / s; q[3] = (R[3] - R[1]) / s;
  } else if (R[0] >= R[4] && R[0] >= R[8]) {
    const T s = T(2) * sqrt_t(T(1) + R[0] - R[4] - R[8]);
    q[0] = (R[7] - R[5]) / s; q[1] = T(0.25) * s; q[2] = (R[1] + R[3]) / s; q[3] = (R[2] + R[6]) / s;
  } else if (R[4] >= R[8]) {
    const T s = T(2) * sqrt_t(T(1) + R[4] - R[0] - R[8]);
    q[0] = (R[2] - R[6]) / s; q[1] = (R[1] + R[3]) / s; q[2] = T(0.25) * s; q[3] = (R[5] + R[7]) / s;
  } else {
    const T s = T(2) * sqrt_t(T(1) + R[8] - R[0] - R[4]);
    q[0] = (R[3] - R[1]) / s; q[1] = (R[2] + R[6]) / s; q[2] = (R[5] + R[7]) / s; q[3] = T(0.25) * s;
  }
}

// o = a^T b (row-major 3x3)
template <class T> RBD_HD void mat_tmul3(const T* a, const T* b, T* o) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) o[3 * i + j] = a[i] * b[j] + a[3 + i] * b[3 + j] + a[6 + i] * b[6 + j];
}

// The law of task tk at one sample, from the named slots sweeps A and B left in the stash: the root-frame wrench [n; f] with
// J_t^T f_t = Σ_k ±S_k . [n; f].
template <class T, class ST>
RBD_HD void task_pd_wrench(const TaskPdDev<T>& D, const TaskPdSample<T>& s, int tk, const ST& st, T* n, T* f) {
  const TaskDev<T>& td = D.t;
  const int vel_off = 12;
  T Rb[9], pb[3], Ra[9], pa[3], p[3], x[3], d[3], vp[3];
  task_pose(td, st, td.body_slot[tk], Rb, pb);
  task_pose(td, st, td.base_slot[tk], Ra, pa);
  Mot<T> twb, twa, rel;
  task_mot(td, st, td.body_slot[tk], vel_off, twb);
  task_mot(td, st, td.base_slot[tk], vel_off, twa);
  mat_vec(Rb, td.point[tk], x);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    p[c] = pb[c] + x[c];                 // the point in the root frame
    d[c] = p[c] - pa[c];
    rel.w[c] = twb.w[c] - twa.w[c]; rel.l[c] = twb.l[c] - twa.l[c];
  }
  cross3(rel.w, p, x);
#pragma unroll
  for (int c = 0; c < 3; ++c) vp[c] = rel.l[c] + x[c];     // velocity of the point w.r.t. base, root frame
  const int r0 = D.row[tk], x0 = D.xrow[tk];
  auto kp = [&](int k) { return s.kp[(int64_t)(r0 + k) * s.gstride]; };
  auto kd = [&](int k) { return s.kd[(int64_t)(r0 + k) * s.gstride]; };
  auto xr = [&](int k) { return s.xref[(int64_t)(x0 + k) * s.ld]; };
  auto xd = [&](int k) { return s.xdref ? s.xdref[(int64_t)(r0 + k) * s.ld] : T(0); };
  if (D.kind[tk] == RBD_TASK_POINT) {
    T RF[9], pF[3], xb[3], eb[3], er[3], e[3], vr[3], ve[3], fF[3];
    task_pose(td, st, td.frame_slot[tk], RF, pF);
    matT_vec(Ra, d, xb);                 // x: the point relative to base, in base coordinates
#pragma unroll
    for (int c = 0; c < 3; ++c) { eb[c] = xb[c] - xr(c); x[c] = xd(c); }
    mat_vec(Ra, eb, er);                 // R_F<-base = R_F^T R_base
    matT_vec(RF, er, e);
    mat_vec(Ra, x, vr);
#pragma unroll
    for (int c = 0; c < 3; ++c) vr[c] = vp[c] - vr[c];
    matT_vec(RF, vr, ve);
#pragma unroll
    for (int c = 0; c < 3; ++c) fF[c] = -kp(c) * e[c] - kd(c) * ve[c];
    mat_vec(RF, fF, f);
    cross3(p, f, n);
    return;
  }
  T Rx[9], px[3], Rr[9], pr[3], Re[9], pe[3], qe[4], psi[3], th2, le[3], w[3], v[3], ang[3], lin[3], y[3];
  mat_tmul3(Ra, Rb, Rx);                 // x = C -> base
  matT_vec(Ra, d, px);
#pragma unroll
  for (int k = 0; k < 9; ++k) Rr[k] = xr(k);
#pragma unroll
  for (int c = 0; c < 3; ++c) { pr[c] = xr(9 + c); y[c] = px[c] - pr[c]; }
  mat_tmul3(Rr, Rx, Re);                 // e = inv(x_ref) x
  matT_vec(Rr, y, pe);
  quat_from_rot(Re, qe);
  rotvec_from_quat(qe, psi, th2);        // RotationVec(R_e), angle in [0, pi]
  matT_vec(Re, pe, le);
  matT_vec(Rb, rel.w, w);                // T: the twist of C w.r.t. base, in C
  matT_vec(Rb, vp, v);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    ang[c] = -kp(c) * psi[c] - kd(c) * (w[c] - xd(c));
    lin[c] = -kp(3 + c) * le[c] - kd(3 + c) * (v[c] - xd(3 + c));
  }
  mat_vec(Rb, lin, f);                   // the wrench [ang; lin] at C, in C, to the root frame
  mat_vec(Rb, ang, n);
  cross3(p, f, x);
#pragma unroll
  for (int c = 0; c < 3; ++c) n[c] += x[c];
}

// The law at one sample: u_k = Σ_t J_t^T f_t for every velocity row k, handed to emit(k, u_k) joint by joint in preorder.
// q, v: the state; the stash needs task_pd_rows rows.
template <class T, class ST, class F>
RBD_HD void task_pd_sample(const ModelDev<T>& M, const TaskPdDev<T>& D, const Col<T>& q, const Col<T>& v, const TaskPdSample<T>& s,
                           const ST& st, F&& emit) {
  const TaskDev<T>& td = D.t;
  {                                      // sweeps A and B; the twist output is parked in the wrench rows, overwritten below
    TaskIO<T> io;
    io.q = q; io.v = v; io.vd = {nullptr, 0};
    const ColOut<T> none{nullptr, 0, false};
    io.tr = none; io.pt = none; io.pv = none; io.J = none; io.Jp = none; io.acc = none; io.pacc = none;
    io.tw = stash_rows(st, D.wrench_base);
    task_sample<T>(M, td, io, st);
  }
  for (int tk = 0; tk < td.ntasks; ++tk) {
    T n[3], f[3];
    task_pd_wrench(D, s, tk, st, n, f);
    const int row = D.wrench_base + 6 * tk;
#pragma unroll
    for (int c = 0; c < 3; ++c) { st.st(row + c, n[c]); st.st(row + 3 + c, f[c]); }
  }
  task_pose_sweep(M, td, q, st, [&](int i, const BodyDev<T>& bd, const Pose<T>& w) {
    const int nvj = kind_nv_dev(bd.kind);
    for (int k = 0; k < nvj; ++k) {
      Mot<T> S;
      world_subspace(w, sub_comp(bd.kind, k), S);
      T u = T(0);
      for (int tk = 0; tk < td.ntasks; ++tk) {
        const int sg = task_bit(td.body_mask[tk], i) - task_bit(td.base_mask[tk], i);
        if (sg == 0) continue;
        const int row = D.wrench_base + 6 * tk;
        T x = T(0);
#pragma unroll
        for (int c = 0; c < 3; ++c) x += S.w[c] * st.ld(row + c) + S.l[c] * st.ld(row + 3 + c);
        u += sg > 0 ? x : -x;
      }
      emit(bd.vrow + k, u);
    }
  });
}

// ---- host side ------------------------------------------------------------------------------------------------------------
// rbd_task_pd_desc -> TaskPdDev (descriptor checked by check_task_pd).  Returns the stash rows per sample.
template <class T> inline int build_task_pd_dev(const HostModel& hm, const rbd_task_pd_desc& c, TaskPdDev<T>& D) {
  std::memset(&D, 0, sizeof(D));
  const int nnamed = build_task_dev<T>(hm, c.tasks, true, false, D.t);
  D.wrench_base = D.t.named_base + nnamed * D.t.slot_rows;
  for (int t = 0; t < c.tasks.ntasks; ++t) {
    D.kind[t] = (int8_t)c.kind[t];
    D.row[t] = (int16_t)D.R;
    D.xrow[t] = (int16_t)D.X;
    D.R += c.kind[t] == RBD_TASK_POINT ? 3 : 6;
    D.X += c.kind[t] == RBD_TASK_POINT ? 3 : 12;
  }
  return D.wrench_base + 6 * c.tasks.ntasks;
}

// The controller's own checks (the joint term's JointPD checks are the caller's): RBD_OK or a status with a message in `err`.
inline int check_task_pd(int nb, int nv, int64_t ld, const rbd_task_pd_desc* c, std::string& err) {
  if (!c) { err = "ctrl must not be NULL"; return RBD_EINVAL; }
  if (c->mode != RBD_PD_TORQUE && c->mode != RBD_PD_COMPUTED_TORQUE) { err = "unknown mode"; return RBD_EINVAL; }
  if (int rc = check_task_desc(nb, &c->tasks, err)) return rc;
  const int K = c->tasks.ntasks;
  if (K && !c->kind) { err = "kind must not be NULL"; return RBD_EINVAL; }
  for (int t = 0; t < K; ++t) {
    if (c->kind[t] != RBD_TASK_POINT && c->kind[t] != RBD_TASK_POSE) { err = "unknown task kind"; return RBD_EINVAL; }
    if (c->kind[t] == RBD_TASK_POSE && (c->tasks.frame ? c->tasks.frame[t] : -1) != c->tasks.body[t]) {
      err = "a pose task is expressed in its own body's frame (frame[t] == body[t])"; return RBD_EINVAL;
    }
  }
  if (K && (!c->kp || !c->kd || !c->x_ref)) { err = "kp, kd and x_ref must not be NULL"; return RBD_EINVAL; }
  if (c->gain_ld != 0 && c->gain_ld != ld) { err = "gain_ld must be 0 or ld"; return RBD_EINVAL; }
  if (c->x_ref_step_stride < 0 || c->xd_ref_step_stride < 0) { err = "reference strides must be >= 0"; return RBD_EINVAL; }
  if (c->joint && c->joint->mode != c->mode) { err = "the joint term must have the controller's mode"; return RBD_EINVAL; }
  if (c->joint && (c->joint->effort_lo || c->joint->effort_hi)) {
    err = "the joint term's effort bounds must be NULL (the controller's bounds clamp the sum)"; return RBD_EINVAL;
  }
  if (!c->effort_lo != !c->effort_hi) { err = "effort_lo and effort_hi must be both NULL or both set"; return RBD_EINVAL; }
  if (c->effort_lo)
    for (int k = 0; k < nv; ++k)
      if (!(c->effort_lo[k] <= c->effort_hi[k])) { err = "effort bounds need lo <= hi"; return RBD_EINVAL; }
  return RBD_OK;
}

}  // namespace rbd
