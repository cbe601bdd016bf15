// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
// The adjoint of the task-space law ON THE CPU: task_pd_vjp_column (csrc/rbd_task_pd_adjoint.cuh) one sample at a time with a
// workspace column of one row per scalar -- the per-sample code task_pd_vjp_kernel runs, the joint term's adjoint included.
#include <string>
#include <vector>

#include "../../rigidbodydynamics/jl_b200/csrc/rbd_task_pd_adjoint.cuh"

using namespace rbd;

namespace {
template <class T>
void run(const HostModel& hm, const rbd_task_pd_desc& c, int64_t B, const T* q, const T* v, const T* w, T* qc, T* qt, T* vb,
         T* const* bars) {
  const ModelDev<T>& M = dev_model<T>(hm);
  const bool ct = c.mode == RBD_PD_COMPUTED_TORQUE;
  std::vector<TaskPdDev<T>> Dv(1);
  TaskPdDev<T>& D = Dv[0];
  std::vector<T> work(build_task_pd_vjp_dev<T>(hm, c, D) + 1);
  std::vector<T> zero((size_t)(hm.nq + hm.nv) * B, T(0));
  for (int64_t e = 0; e < (int64_t)hm.nq * B; ++e) qc[e] = T(0);
  for (int64_t e = 0; e < (int64_t)hm.nv * B; ++e) vb[e] = T(0);
  TaskPdVjpArgs<T> a{};
  a.q = q; a.v = v; a.w = w;
  a.xref = (const T*)c.x_ref; a.xdref = (const T*)c.xd_ref; a.kp = (const T*)c.kp; a.kd = (const T*)c.kd; a.gain_ld = c.gain_ld;
  a.kpb = bars[0]; a.kdb = bars[1]; a.xrefb = bars[2]; a.xdrefb = bars[3];
  a.qacc = qc; a.vacc = vb; a.B = B;
  if (const rbd_pd_desc* j = c.joint) {
    a.has_joint = true;
    PdAdjArgs<T>& p = a.joint;
    p.qref = (const T*)j->q_ref; p.vref = (const T*)j->v_ref; p.kp = (const T*)j->kp; p.kd = (const T*)j->kd; p.g_ld = j->gain_ld;
    if (ct) { p.idvd = w; p.idv = zero.data(); }      // the law alone: the inverse-dynamics VJP's q̄ / v̄ are zero here
    p.kpb = bars[4]; p.kdb = bars[5]; p.qrefb = bars[6]; p.vrefb = bars[7]; p.vdrefb = bars[8];
  }
  for (int64_t b = 0; b < B; ++b) task_pd_vjp_column<T>(M, D, a, b, true, Scr<T>{work.data(), 1});
  for (int64_t b = 0; b < B; ++b)
    for (int i = 0; i < hm.nb; ++i) {
      const BodyDev<T>& bd = M.body[i];
      const int nq = kind_nq_dev(bd.kind), nv = kind_nv_dev(bd.kind);
      if (nv == 0) continue;
      T qq[7], g[7], f[6];
      for (int k = 0; k < nq; ++k) { qq[k] = q[(bd.qrow + k) * B + b]; g[k] = qc[(bd.qrow + k) * B + b]; }
      cfg_to_tan(bd.kind, qq, g, f);
      for (int k = 0; k < nv; ++k) qt[(bd.vrow + k) * B + b] = f[k];
    }
}
}  // namespace

extern "C" {
// The adjoint of hostsim_task_pd_law (without effort bounds): for the cotangent w [nv x B] of its output, q̄_cfg [nq x B], q̄_tan
// [nv x B] and v̄ [nv x B] (written), and bars[9] = kp, kd, x_ref, xd_ref, then the joint term's kp, kd, q_ref, v_ref, vd_ref
// (added to, NULL = not wanted; the gains' bars per sample).  Arrays as hostsim_task_pd_law's.  Returns an rbd_status.
int hostsim_task_pd_law_vjp(const rbd_model_desc* d, const rbd_task_pd_desc* c, int dtype, int64_t B, const void* q, const void* v,
                            const void* w, void* qc, void* qt, void* vb, void* const* bars) {
  HostModel hm; std::string err;
  int rc = build_host_model(d, hm, err);
  if (rc) return rc;
  if ((rc = check_task_pd(hm.nb, hm.nv, B, c, err))) return rc;
  if (dtype == 0) run<float>(hm, *c, B, (const float*)q, (const float*)v, (const float*)w, (float*)qc, (float*)qt, (float*)vb, (float* const*)bars);
  else run<double>(hm, *c, B, (const double*)q, (const double*)v, (const double*)w, (double*)qc, (double*)qt, (double*)vb, (double* const*)bars);
  return 0;
}
}
