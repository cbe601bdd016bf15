// Task-space kinematics (rbd_task_kinematics, DESIGN 4.17): for a set of tasks -- a body, a base body, a point fixed in the body
// and a frame to express results in -- the reference's
//   relative_transform(state, from, to)                 mechanism_state.jl:1011-1014
//   relative_twist(state, body, base)                   mechanism_state.jl:1016-1038
//   geometric_jacobian!(J, state, path), J.frame != root mechanism_algorithms.jl:101-132
//   point_jacobian!(Jp, state, path, point)             mechanism_algorithms.jl:154-224
//   point_velocity(twist, point)                        spatial/spatialmotion.jl:346-349
//   relative_acceleration(accels, body, base)           mechanism_algorithms.jl:421-426
//   transform(state, accel, frame)                      mechanism_state.jl:1049-1056 -> spatialmotion.jl:375-401
//   point_acceleration(twist, accel, point)             spatialmotion.jl:351-363
// One thread per sample, preorder walk and pending slots as kin_sample (rbd_kin.cuh):
//   sweep A  poses only; the pose of every body a task names (body, base, frame) is parked in its "named slot" of the stash, with
//            its rotation mapped back to the CALLER's body frame (R A^T), so that everything after it works in the caller's frames;
//   sweep B  pose, twist and (when asked for) spatial acceleration of every body, all in the root frame; the named bodies' twists
//            and accelerations go to their slots; every joint's world-frame subspace columns S_k are mapped once per task into the
//            geometric column Ad(T_F^-1) (±S_k) and the point column R_F^T (±(v_S + w_S x p)), zero columns off the task's path;
//   epilogue per task, from the named slots.
// Sweep B runs only when a Jacobian or a velocity-dependent output is requested.  Gravity is left out of the accelerations (the
// root's -g is common to body and base and cancels in every relative acceleration).  Every output element is written exactly once
// and none is read back; each output's arithmetic does not depend on which other outputs are requested.
#pragma once
#include <cstdint>
#include <cstring>
#include <string>

#include "../../../include/rbd_b200.h"
#include "rbd_kin.cuh"
#include "rbd_model.h"

namespace rbd {

constexpr int kMaxTasks = RBD_MAX_TASKS;

template <class T> struct TaskDev {
  int32_t ntasks;
  int32_t named_base;                 // first stash row of named slot 0 (behind the pending slots of the outward sweep)
  int32_t slot_rows;                  // rows per named slot: pose 12, + twist 6 when velocities are needed, + acceleration 6
  int32_t pad_;
  uint64_t body_mask[kMaxTasks];      // preorder positions of the body's ancestors-or-self (0 for the root body)
  uint64_t base_mask[kMaxTasks];      // same for the base: the joint at position i is on the path with sign bit(body) - bit(base)
  int8_t body_slot[kMaxTasks], base_slot[kMaxTasks], frame_slot[kMaxTasks];   // named slot, -1 = root body / root frame
  int8_t named[kMaxBodies];           // preorder position -> named slot, -1 = not named by any task
  T point[kMaxTasks][3];              // point fixed in the body, in the caller's body frame
  T At[kMaxBodies][9];                // named slot -> A^T of its body (canonical body frame <- caller's body frame), row-major
};

template <class T> struct TaskIO {
  Col<T> q, v, vd;                    // v may be invalid when nothing velocity-dependent is requested; vd invalid = zero
  ColOut<T> tr, pt, tw, pv, J, Jp, acc, pacc;
};

// bit i of m as 0 / 1
RBD_HD int task_bit(uint64_t m, int i) { return (int)((m >> i) & 1ull); }

// pose (caller-frame rotation, origin) of named slot s, identity for the root (s < 0)
template <class T, class ST> RBD_HD void task_pose(const TaskDev<T>& D, const ST& st, int s, T* R, T* p) {
  if (s < 0) {
#pragma unroll
    for (int k = 0; k < 9; ++k) R[k] = (k % 4 == 0) ? T(1) : T(0);
#pragma unroll
    for (int k = 0; k < 3; ++k) p[k] = T(0);
    return;
  }
  const int row = D.named_base + s * D.slot_rows;
#pragma unroll
  for (int k = 0; k < 9; ++k) R[k] = st.ld(row + k);
#pragma unroll
  for (int k = 0; k < 3; ++k) p[k] = st.ld(row + 9 + k);
}
// root-frame motion vector kept at rows `off` .. off + 5 of named slot s, zero for the root
template <class T, class ST> RBD_HD void task_mot(const TaskDev<T>& D, const ST& st, int s, int off, Mot<T>& m) {
  if (s < 0) {
#pragma unroll
    for (int k = 0; k < 3; ++k) m.w[k] = m.l[k] = T(0);
    return;
  }
  const int row = D.named_base + s * D.slot_rows + off;
#pragma unroll
  for (int k = 0; k < 3; ++k) { m.w[k] = st.ld(row + k); m.l[k] = st.ld(row + 3 + k); }
}
// root-frame motion vector -> frame F (rotation RF, origin pF):  w' = RF^T w,  l' = RF^T (l + w x pF)   (Ad(T_F^-1))
template <class T> RBD_HD void task_to_frame(const T* RF, const T* pF, const Mot<T>& m, Mot<T>& o) {
  T x[3], l[3];
  cross3(m.w, pF, x);
#pragma unroll
  for (int k = 0; k < 3; ++k) l[k] = m.l[k] + x[k];
  matT_vec(RF, m.w, o.w);
  matT_vec(RF, l, o.l);
}

// Sweep A: the root-frame pose w of every body in preorder; the named bodies' poses are parked in their slots, and body_fn(bd, w)
// runs for every body (rbd_task_pd.cuh's J^T pass walks the joints with it).
template <class T, class ST, class F>
RBD_HD void task_pose_sweep(const ModelDev<T>& M, const TaskDev<T>& D, const Col<T>& q, const ST& st, F&& body_fn) {
  Pose<T> cur;
  pose_identity(cur);
  for (int i = 0; i < M.nb; ++i) {
    const BodyDev<T>& bd = M.body[i];
    Pose<T> pp;
    if (bd.flags & F_ROOT_CHILD) pose_identity(pp);
    else if (bd.flags & F_FIRST_CHILD) pp = cur;
    else {
      const int row = bd.pslot * kSlotRowsKin;
#pragma unroll
      for (int k = 0; k < 9; ++k) pp.R[k] = st.ld(row + k);
#pragma unroll
      for (int k = 0; k < 3; ++k) pp.p[k] = st.ld(row + 9 + k);
    }
    T R[9], r[3], t[3];
    frame_any(bd, q, R, r);
    Pose<T> w;
    mat_mul3(pp.R, R, w.R);
    mat_vec(pp.R, r, t);
    w.p[0] = pp.p[0] + t[0]; w.p[1] = pp.p[1] + t[1]; w.p[2] = pp.p[2] + t[2];
    const int s = D.named[i];
    if (s >= 0) {
      T Rc[9];
      mat_mul3(w.R, D.At[s], Rc);
      const int row = D.named_base + s * D.slot_rows;
#pragma unroll
      for (int k = 0; k < 9; ++k) st.st(row + k, Rc[k]);
#pragma unroll
      for (int k = 0; k < 3; ++k) st.st(row + 9 + k, w.p[k]);
    }
    body_fn(i, bd, w);
    if (bd.flags & F_HAS_PENDING) {
      const int row = bd.oslot * kSlotRowsKin;
#pragma unroll
      for (int k = 0; k < 9; ++k) st.st(row + k, w.R[k]);
#pragma unroll
      for (int k = 0; k < 3; ++k) st.st(row + 9 + k, w.p[k]);
    }
    cur = w;
  }
}

template <class T, class ST>
RBD_HD void task_sample(const ModelDev<T>& M, const TaskDev<T>& D, const TaskIO<T>& io, const ST& st) {
  const int nb = M.nb, nv = M.nv, K = D.ntasks;
  const bool jac = io.J.valid() || io.Jp.valid();
  const bool want_acc = io.acc.valid() || io.pacc.valid();
  const bool want_vel = want_acc || io.tw.valid() || io.pv.valid();
  const int vel_off = 12, acc_off = 18;

  // ---- sweep A: poses of the named bodies ----
  task_pose_sweep(M, D, io.q, st, [](int, const BodyDev<T>&, const Pose<T>&) {});

  // ---- sweep B: twists, accelerations, Jacobian columns ----
  if (jac || want_vel) {
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
        for (int k = 0; k < 3; ++k) twp.w[k] = twp.l[k] = ap.w[k] = ap.l[k] = T(0);
      } else if (bd.flags & F_FIRST_CHILD) {
        pp = cur; twp = twc; ap = ac;
      } else {
        const int row = bd.pslot * kSlotRowsKin;
#pragma unroll
        for (int k = 0; k < 9; ++k) pp.R[k] = st.ld(row + k);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          pp.p[k] = st.ld(row + 9 + k);
          twp.w[k] = want_vel ? st.ld(row + 12 + k) : T(0); twp.l[k] = want_vel ? st.ld(row + 15 + k) : T(0);
          ap.w[k] = want_acc ? st.ld(row + 18 + k) : T(0); ap.l[k] = want_acc ? st.ld(row + 21 + k) : T(0);
        }
      }
      T R[9], r[3], t[3];
      frame_any(bd, io.q, R, r);
      Pose<T> w;
      mat_mul3(pp.R, R, w.R);
      mat_vec(pp.R, r, t);
      w.p[0] = pp.p[0] + t[0]; w.p[1] = pp.p[1] + t[1]; w.p[2] = pp.p[2] + t[2];
      const int nvj = kind_nv_dev(bd.kind);
      Mot<T> tw = twp, a = ap;
      if (want_vel) {
        Mot<T> jt, ja;                   // S v and S v̇ in the root frame
#pragma unroll
        for (int k = 0; k < 3; ++k) jt.w[k] = jt.l[k] = ja.w[k] = ja.l[k] = T(0);
        for (int k = 0; k < nvj; ++k) {
          Mot<T> S;
          world_subspace(w, sub_comp(bd.kind, k), S);
          const T x = io.v(bd.vrow + k);
          const T xd = (want_acc && io.vd.valid()) ? io.vd(bd.vrow + k) : T(0);
#pragma unroll
          for (int c = 0; c < 3; ++c) { jt.w[c] += x * S.w[c]; jt.l[c] += x * S.l[c]; ja.w[c] += xd * S.w[c]; ja.l[c] += xd * S.l[c]; }
        }
        Mot<T> cm;
        motion_cross(twp, jt, cm);       // spatial_accelerations!: a_i = a_parent + v_parent x (S v) + S v̇   (:387-417)
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          tw.w[k] = twp.w[k] + jt.w[k]; tw.l[k] = twp.l[k] + jt.l[k];
          a.w[k] = ap.w[k] + cm.w[k] + ja.w[k]; a.l[k] = ap.l[k] + cm.l[k] + ja.l[k];
        }
      }
      if (jac) {
        for (int tk = 0; tk < K; ++tk) {
          const int sg = task_bit(D.body_mask[tk], i) - task_bit(D.base_mask[tk], i);
          const int grow = tk * 6 * nv, prow = tk * 3 * nv;
          if (sg == 0) {                 // joint off this task's path: zero columns
            for (int k = 0; k < nvj; ++k) {
              const int col = bd.vrow + k;
              if (io.J.valid()) {
#pragma unroll
                for (int c = 0; c < 6; ++c) io.J.st(grow + 6 * col + c, T(0));
              }
              if (io.Jp.valid()) {
#pragma unroll
                for (int c = 0; c < 3; ++c) io.Jp.st(prow + 3 * col + c, T(0));
              }
            }
            continue;
          }
          const int fs = D.frame_slot[tk];
          T RF[9], pF[3], Rb[9], pb[3], p[3], x[3];
          task_pose(D, st, fs, RF, pF);
          task_pose(D, st, D.body_slot[tk], Rb, pb);
          mat_vec(Rb, D.point[tk], x);
#pragma unroll
          for (int c = 0; c < 3; ++c) p[c] = pb[c] + x[c];      // the point in the root frame
          const T s = T(sg);
          for (int k = 0; k < nvj; ++k) {
            const int col = bd.vrow + k;
            Mot<T> S;
            world_subspace(w, sub_comp(bd.kind, k), S);
#pragma unroll
            for (int c = 0; c < 3; ++c) { S.w[c] *= s; S.l[c] *= s; }
            if (io.J.valid()) {
              Mot<T> G;
              if (fs < 0) G = S;
              else task_to_frame(RF, pF, S, G);
#pragma unroll
              for (int c = 0; c < 3; ++c) { io.J.st(grow + 6 * col + c, G.w[c]); io.J.st(grow + 6 * col + 3 + c, G.l[c]); }
            }
            if (io.Jp.valid()) {         // -p̂ w_S + v_S = v_S + w_S x p   (:170-171)
              T y[3], l[3];
              cross3(S.w, p, y);
#pragma unroll
              for (int c = 0; c < 3; ++c) l[c] = S.l[c] + y[c];
              if (fs >= 0) { T lf[3]; matT_vec(RF, l, lf); l[0] = lf[0]; l[1] = lf[1]; l[2] = lf[2]; }
#pragma unroll
              for (int c = 0; c < 3; ++c) io.Jp.st(prow + 3 * col + c, l[c]);
            }
          }
        }
      }
      const int s = D.named[i];
      if (s >= 0 && want_vel) {
        const int row = D.named_base + s * D.slot_rows;
#pragma unroll
        for (int k = 0; k < 3; ++k) { st.st(row + vel_off + k, tw.w[k]); st.st(row + vel_off + 3 + k, tw.l[k]); }
        if (want_acc) {
#pragma unroll
          for (int k = 0; k < 3; ++k) { st.st(row + acc_off + k, a.w[k]); st.st(row + acc_off + 3 + k, a.l[k]); }
        }
      }
      if (bd.flags & F_HAS_PENDING) {
        const int row = bd.oslot * kSlotRowsKin;
#pragma unroll
        for (int k = 0; k < 9; ++k) st.st(row + k, w.R[k]);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          st.st(row + 9 + k, w.p[k]);
          if (want_vel) { st.st(row + 12 + k, tw.w[k]); st.st(row + 15 + k, tw.l[k]); }
          if (want_acc) { st.st(row + 18 + k, a.w[k]); st.st(row + 21 + k, a.l[k]); }
        }
      }
      cur = w; twc = tw; ac = a;
    }
  }

  // ---- epilogue: one task at a time, from the named slots ----
  for (int tk = 0; tk < K; ++tk) {
    const int bs = D.body_slot[tk], as = D.base_slot[tk], fs = D.frame_slot[tk];
    T Rb[9], pb[3], Ra[9], pa[3], RF[9], pF[3];
    task_pose(D, st, bs, Rb, pb);
    task_pose(D, st, as, Ra, pa);
    task_pose(D, st, fs, RF, pF);
    if (io.tr.valid()) {                 // inv(T_base) T_body
      T Rr[9], d[3], pr[3];
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) Rr[3 * i + j] = Ra[i] * Rb[j] + Ra[3 + i] * Rb[3 + j] + Ra[6 + i] * Rb[6 + j];
#pragma unroll
      for (int c = 0; c < 3; ++c) d[c] = pb[c] - pa[c];
      matT_vec(Ra, d, pr);
#pragma unroll
      for (int k = 0; k < 9; ++k) io.tr.st(12 * tk + k, Rr[k]);
#pragma unroll
      for (int k = 0; k < 3; ++k) io.tr.st(12 * tk + 9 + k, pr[k]);
    }
    T pf[3];                             // the point in F
    {
      T x[3], p[3];
      mat_vec(Rb, D.point[tk], x);
#pragma unroll
      for (int c = 0; c < 3; ++c) p[c] = pb[c] + x[c];
      if (fs < 0) { pf[0] = p[0]; pf[1] = p[1]; pf[2] = p[2]; }
      else {
        T d[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) d[c] = p[c] - pF[c];
        matT_vec(RF, d, pf);
      }
    }
    if (io.pt.valid()) {
#pragma unroll
      for (int c = 0; c < 3; ++c) io.pt.st(3 * tk + c, pf[c]);
    }
    if (!want_vel) continue;
    Mot<T> twb, twa, rel, twf;
    task_mot(D, st, bs, vel_off, twb);
    task_mot(D, st, as, vel_off, twa);
#pragma unroll
    for (int c = 0; c < 3; ++c) { rel.w[c] = twb.w[c] - twa.w[c]; rel.l[c] = twb.l[c] - twa.l[c]; }
    if (fs < 0) twf = rel;
    else task_to_frame(RF, pF, rel, twf);
    if (io.tw.valid()) {
#pragma unroll
      for (int c = 0; c < 3; ++c) { io.tw.st(6 * tk + c, twf.w[c]); io.tw.st(6 * tk + 3 + c, twf.l[c]); }
    }
    T pv[3];                             // point_velocity(twist, point) = w x p + v, all in F
    {
      T x[3];
      cross3(twf.w, pf, x);
#pragma unroll
      for (int c = 0; c < 3; ++c) pv[c] = x[c] + twf.l[c];
    }
    if (io.pv.valid()) {
#pragma unroll
      for (int c = 0; c < 3; ++c) io.pv.st(3 * tk + c, pv[c]);
    }
    if (!want_acc) continue;
    Mot<T> ab, aa, x, af;
    task_mot(D, st, bs, acc_off, ab);
    task_mot(D, st, as, acc_off, aa);
#pragma unroll
    for (int c = 0; c < 3; ++c) { x.w[c] = ab.w[c] - aa.w[c]; x.l[c] = ab.l[c] - aa.l[c]; }
    if (fs < 0) af = x;
    else {                               // transform(accel, root_to_F, twist of root wrt F, twist of body wrt base)
      Mot<T> twF, cm, y;                 //   = Ad(T_F^-1) (a - v_F x v_rel), root-frame twists   (spatialmotion.jl:375-401)
      task_mot(D, st, fs, vel_off, twF);
      motion_cross(twF, rel, cm);
#pragma unroll
      for (int c = 0; c < 3; ++c) { y.w[c] = x.w[c] - cm.w[c]; y.l[c] = x.l[c] - cm.l[c]; }
      task_to_frame(RF, pF, y, af);
    }
    if (io.acc.valid()) {
#pragma unroll
      for (int c = 0; c < 3; ++c) { io.acc.st(6 * tk + c, af.w[c]); io.acc.st(6 * tk + 3 + c, af.l[c]); }
    }
    if (io.pacc.valid()) {               // w' x p + a_lin + w x (w x p + v_lin)   (spatialmotion.jl:358-363)
      T u[3], z[3];
      cross3(af.w, pf, u);
      cross3(twf.w, pv, z);
#pragma unroll
      for (int c = 0; c < 3; ++c) io.pacc.st(3 * tk + c, u[c] + af.l[c] + z[c]);
    }
  }
}

// ---- host side ------------------------------------------------------------------------------------------------------------
// The descriptor checks of rbd_task_kinematics (also used by the CPU harness): RBD_OK or a status with a message in `err`.
inline int check_task_desc(int nb, const rbd_task_desc* d, std::string& err) {
  if (!d) { err = "tasks must not be NULL"; return RBD_EINVAL; }
  if (d->ntasks < 0) { err = "ntasks must be >= 0"; return RBD_EINVAL; }
  if (d->ntasks > kMaxTasks) { err = "at most RBD_MAX_TASKS (32) tasks per call"; return RBD_EUNSUPPORTED; }
  if (d->ntasks && (!d->body || !d->base)) { err = "body and base must not be NULL"; return RBD_EINVAL; }
  for (int t = 0; t < d->ntasks; ++t) {
    const int idx[3] = {d->body[t], d->base[t], d->frame ? d->frame[t] : -1};
    for (int k = 0; k < 3; ++k)
      if (idx[k] < -1 || idx[k] >= nb) { err = "body / base / frame index outside -1 .. nb-1"; return RBD_EINVAL; }
  }
  return RBD_OK;
}

// rbd_task_desc -> TaskDev (checked by check_task_desc).  named_base: first stash row behind the outward sweep's pending slots.
// Returns the number of named slots.
template <class T>
inline int build_task_dev(const HostModel& hm, const rbd_task_desc& d, bool want_vel, bool want_acc, TaskDev<T>& D) {
  std::memset(&D, 0, sizeof(D));
  D.ntasks = d.ntasks;
  D.named_base = kin_rows(hm);
  D.slot_rows = 12 + (want_vel ? 6 : 0) + (want_acc ? 6 : 0);
  std::memset(D.named, -1, sizeof(D.named));
  int nnamed = 0;
  auto slot = [&](int ref) -> int8_t {
    if (ref < 0) return -1;
    const int p = hm.pos[ref];
    if (D.named[p] < 0) {
      D.named[p] = (int8_t)nnamed;
      for (int k = 0; k < 9; ++k) D.At[nnamed][k] = (T)hm.alignT[9 * p + k];
      ++nnamed;
    }
    return D.named[p];
  };
  auto mask = [&](int ref) {
    uint64_t m = 0;
    for (int p = ref < 0 ? -1 : hm.pos[ref]; p >= 0; p = hm.dev64.body[p].parent) m |= 1ull << p;
    return m;
  };
  for (int t = 0; t < d.ntasks; ++t) {
    D.body_mask[t] = mask(d.body[t]);
    D.base_mask[t] = mask(d.base[t]);
    D.body_slot[t] = slot(d.body[t]);
    D.base_slot[t] = slot(d.base[t]);
    D.frame_slot[t] = slot(d.frame ? d.frame[t] : -1);
    for (int k = 0; k < 3; ++k) D.point[t][k] = d.point ? (T)d.point[3 * t + k] : T(0);
  }
  return nnamed;
}

}  // namespace rbd
