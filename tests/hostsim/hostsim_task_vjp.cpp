// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
// Runs task_vjp_sample (csrc/rbd_task_adjoint.cuh), the per-sample function of rbd_task_kinematics_vjp, ON THE CPU: one sample at a
// time with a workspace column of one row per scalar, so the mathematics of the kernel can be checked without a GPU.
#include <string>
#include <vector>

#include "../../rigidbodydynamics/jl_b200/csrc/rbd_task_adjoint.cuh"

using namespace rbd;

namespace {
template <class T>
void run_task_vjp(const HostModel& hm, const rbd_task_desc& d, int64_t B, const T* q, const T* v, const T* vd, const T* const* bar,
                  T* const* o) {
  const ModelDev<T>& M = dev_model<T>(hm);
  std::vector<TaskDev<T>> Dv(1);
  TaskDev<T>& D = Dv[0];
  const int nnamed = build_task_vjp_dev<T>(hm, d, D);
  std::vector<T> work(task_adjoint_rows(hm.nb, nnamed) + 1);
  for (int64_t b = 0; b < B; ++b) {
    TaskBarIO<T> io;
    auto in = [&](const T* p) { return Col<T>{p ? p + b : nullptr, B}; };
    auto out = [&](T* p) { return ColOut<T>{p ? p + b : nullptr, B, true}; };
    io.q = in(q); io.v = in(v); io.vd = in(vd);
    io.tr = in(bar[0]); io.pt = in(bar[1]); io.tw = in(bar[2]); io.pv = in(bar[3]);
    io.J = in(bar[4]); io.Jp = in(bar[5]); io.acc = in(bar[6]); io.pacc = in(bar[7]);
    io.qt = out(o[0]); io.qc = out(o[1]); io.vb = out(o[2]); io.vdb = out(o[3]);
    io.s = {work.data(), 1};
    task_vjp_sample<T>(M, D, io);
  }
}
}  // namespace

extern "C" {
// bars: the eight cotangents in rbd_task_out's order, each NULL or [rows x B]; outs: q̄_tan, q̄_cfg, v̄, v̇̄, each NULL or [rows x B].
// Returns an rbd_status (descriptor checks as rbd_task_kinematics_vjp).
int hostsim_task_kinematics_vjp(const rbd_model_desc* d, const rbd_task_desc* td, int dtype, int64_t B, const void* q, const void* v,
                                const void* vd, const void* const* bars, void* const* outs) {
  HostModel hm; std::string err;
  int rc = build_host_model(d, hm, err);
  if (rc) return rc;
  if ((rc = check_task_desc(hm.nb, td, err))) return rc;
  if (dtype == 0) {
    const float* b[8]; float* o[4];
    for (int k = 0; k < 8; ++k) b[k] = (const float*)bars[k];
    for (int k = 0; k < 4; ++k) o[k] = (float*)outs[k];
    run_task_vjp<float>(hm, *td, B, (const float*)q, (const float*)v, (const float*)vd, b, o);
  } else {
    const double* b[8]; double* o[4];
    for (int k = 0; k < 8; ++k) b[k] = (const double*)bars[k];
    for (int k = 0; k < 4; ++k) o[k] = (double*)outs[k];
    run_task_vjp<double>(hm, *td, B, (const double*)q, (const double*)v, (const double*)vd, b, o);
  }
  return 0;
}
}
