// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
// The law of rbd_integrate_task_pd / rbd_task_pd_torques ON THE CPU: task_pd_sample (csrc/rbd_task_pd.cuh) one sample at a time
// with a stash of one row per scalar, plus the joint term pd_joint (csrc/rbd_pd.cuh), combined as task_pd_kernel combines them.
#include <string>
#include <vector>

#include "../../rigidbodydynamics/jl_b200/csrc/rbd_task_pd.cuh"

using namespace rbd;

namespace {
template <class T>
void run(const HostModel& hm, const rbd_task_pd_desc& c, int64_t B, const T* q, const T* v, const T* ff, T* out) {
  const ModelDev<T>& M = dev_model<T>(hm);
  const bool ct = c.mode == RBD_PD_COMPUTED_TORQUE;
  std::vector<TaskPdDev<T>> Dv(1);
  TaskPdDev<T>& D = Dv[0];
  std::vector<T> stash(build_task_pd_dev<T>(hm, c, D) + 1);
  std::vector<T> lh(2 * hm.nv);
  for (int k = 0; c.effort_lo && k < hm.nv; ++k) { lh[k] = (T)c.effort_lo[k]; lh[hm.nv + k] = (T)c.effort_hi[k]; }
  const rbd_pd_desc* j = c.joint;
  for (int64_t b = 0; b < B; ++b) {
    const Col<T> qc{q + b, B}, vc{v + b, B};
    const int64_t gc = c.gain_ld ? b : 0;
    const TaskPdSample<T> s{c.x_ref ? (const T*)c.x_ref + b : nullptr, c.xd_ref ? (const T*)c.xd_ref + b : nullptr, B,
                            c.kp ? (const T*)c.kp + gc : nullptr, c.kd ? (const T*)c.kd + gc : nullptr, c.gain_ld ? c.gain_ld : 1};
    const ColOut<T> o{out + b, B, true};
    if (j) {
      const int64_t jc = j->gain_ld ? b : 0;
      const T* jff = ct ? (const T*)j->vd_ref : ff;
      const PdSample<T> js{q + b, v + b, B, (const T*)j->q_ref + b, j->v_ref ? (const T*)j->v_ref + b : nullptr, jff ? jff + b : nullptr,
                           B, (const T*)j->kp + jc, (const T*)j->kd + jc, j->gain_ld ? j->gain_ld : 1, nullptr, nullptr};
      for (int i = 0; i < hm.nb; ++i) pd_joint(M.body[i], js, o);
    }
    task_pd_sample<T>(M, D, qc, vc, s, Stash<T, 1>{stash.data()}, [&](int row, T u) {
      T x = j ? out[b + (int64_t)row * B] : (ff && !ct ? ff[b + (int64_t)row * B] : T(0));
      x += u;
      if (c.effort_lo && !ct) x = clamp_t(x, lh[row], lh[hm.nv + row]);
      o.st(row, x);
    });
  }
}
}  // namespace

extern "C" {
// out [nv x B]: the torques (RBD_PD_TORQUE) or v̇_des (RBD_PD_COMPUTED_TORQUE, before the inverse dynamics) of the controller at
// (q, v), every array on the host with leading dimension B (the descriptor's "device" arrays too, gain_ld 0 or B; step 0).
// Returns an rbd_status (the controller checks of rbd_integrate_task_pd without the joint term's).
int hostsim_task_pd_law(const rbd_model_desc* d, const rbd_task_pd_desc* c, int dtype, int64_t B, const void* q, const void* v,
                        const void* ff, void* out) {
  HostModel hm; std::string err;
  int rc = build_host_model(d, hm, err);
  if (rc) return rc;
  if ((rc = check_task_pd(hm.nb, hm.nv, B, c, err))) return rc;
  if (dtype == 0) run<float>(hm, *c, B, (const float*)q, (const float*)v, (const float*)ff, (float*)out);
  else run<double>(hm, *c, B, (const double*)q, (const double*)v, (const double*)ff, (double*)out);
  return 0;
}
}
