// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
// Runs task_sample (csrc/rbd_task.cuh), the per-sample function of rbd_task_kinematics, ON THE CPU: one sample at a time with a
// stash of one row per scalar, so the mathematics of the kernel can be checked against the oracle without a GPU.
#include <string>
#include <vector>

#include "../../rigidbodydynamics/jl_b200/csrc/rbd_task.cuh"

using namespace rbd;

namespace {
template <class T>
void run_task(const HostModel& hm, const rbd_task_desc& d, int64_t B, const T* q, const T* v, const T* vd, T* const* o) {
  const ModelDev<T>& M = dev_model<T>(hm);
  const bool want_acc = o[6] || o[7];
  const bool want_vel = want_acc || o[2] || o[3];
  std::vector<TaskDev<T>> Dv(1);
  TaskDev<T>& D = Dv[0];
  const int nnamed = build_task_dev<T>(hm, d, want_vel, want_acc, D);
  std::vector<T> stash(D.named_base + nnamed * D.slot_rows + 1);
  for (int64_t b = 0; b < B; ++b) {
    TaskIO<T> io;
    io.q = {q + b, B}; io.v = {v ? v + b : nullptr, B}; io.vd = {vd ? vd + b : nullptr, B};
    auto out = [&](T* p) { return ColOut<T>{p ? p + b : nullptr, B, true}; };
    io.tr = out(o[0]); io.pt = out(o[1]); io.tw = out(o[2]); io.pv = out(o[3]);
    io.J = out(o[4]); io.Jp = out(o[5]); io.acc = out(o[6]); io.pacc = out(o[7]);
    task_sample<T>(M, D, io, Stash<T, 1>{stash.data()});
  }
}
}  // namespace

extern "C" {
// outs: the eight arrays of rbd_task_out in its order, each NULL or [rows x B].  Returns an rbd_status (descriptor checks as
// rbd_task_kinematics).
int hostsim_task_kinematics(const rbd_model_desc* d, const rbd_task_desc* td, int dtype, int64_t B, const void* q, const void* v,
                            const void* vd, void* const* outs) {
  HostModel hm; std::string err;
  int rc = build_host_model(d, hm, err);
  if (rc) return rc;
  if ((rc = check_task_desc(hm.nb, td, err))) return rc;
  if (dtype == 0) {
    float* o[8];
    for (int k = 0; k < 8; ++k) o[k] = (float*)outs[k];
    run_task<float>(hm, *td, B, (const float*)q, (const float*)v, (const float*)vd, o);
  } else {
    double* o[8];
    for (int k = 0; k < 8; ++k) o[k] = (double*)outs[k];
    run_task<double>(hm, *td, B, (const double*)q, (const double*)v, (const double*)vd, o);
  }
  return 0;
}
}
