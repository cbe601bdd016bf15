// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
// Runs kin_vjp_sample (csrc/rbd_kin_adjoint.cuh), the per-sample function of rbd_kinematics_vjp, ON THE CPU: one sample at a time
// with a workspace column of one row per scalar, so the mathematics of the kernel can be checked without a GPU.
#include <string>
#include <vector>

#include "../../rigidbodydynamics/jl_b200/csrc/rbd_kin_adjoint.cuh"

using namespace rbd;

namespace {
template <class T>
void run_kin_vjp(const HostModel& hm, const int8_t* sign, int64_t B, const T* q, const T* v, const T* const* bar, T* const* o) {
  const ModelDev<T>& M = dev_model<T>(hm);
  std::vector<KinDev<T>> Kv(1);
  KinDev<T>& K = Kv[0];
  build_kin_dev<T>(hm, sign, K);
  std::vector<T> work(kin_adjoint_rows(hm.nb, M.nslots, bar[6] != nullptr) + 1);
  for (int64_t b = 0; b < B; ++b) {
    KinBarIO<T> io;
    auto in = [&](const T* p) { return Col<T>{p ? p + b : nullptr, B}; };
    auto out = [&](T* p) { return ColOut<T>{p ? p + b : nullptr, B, true}; };
    io.q = in(q); io.v = in(v);
    io.tr = in(bar[0]); io.com = in(bar[1]); io.ke = in(bar[2]); io.pe = in(bar[3]);
    io.mom = in(bar[4]); io.mrb = in(bar[5]); io.A = in(bar[6]); io.J = in(bar[7]);
    io.qt = out(o[0]); io.qc = out(o[1]); io.vb = out(o[2]);
    io.s = {work.data(), 1};
    kin_vjp_sample<T>(M, K, io);
  }
}
}  // namespace

extern "C" {
// sign: the path's nb signs in tree-joint order or NULL; bars: the eight cotangents in rbd_kinematics_out's order, each NULL or
// [rows x B]; outs: q̄_tan, q̄_cfg, v̄, each NULL or [rows x B].  Returns an rbd_status.
int hostsim_kinematics_vjp(const rbd_model_desc* d, const int8_t* sign, int dtype, int64_t B, const void* q, const void* v,
                           const void* const* bars, void* const* outs) {
  HostModel hm; std::string err;
  const int rc = build_host_model(d, hm, err);
  if (rc) return rc;
  if (dtype == 0) {
    const float* b[8]; float* o[3];
    for (int k = 0; k < 8; ++k) b[k] = (const float*)bars[k];
    for (int k = 0; k < 3; ++k) o[k] = (float*)outs[k];
    run_kin_vjp<float>(hm, sign, B, (const float*)q, (const float*)v, b, o);
  } else {
    const double* b[8]; double* o[3];
    for (int k = 0; k < 8; ++k) b[k] = (const double*)bars[k];
    for (int k = 0; k < 3; ++k) o[k] = (double*)outs[k];
    run_kin_vjp<double>(hm, sign, B, (const double*)q, (const double*)v, b, o);
  }
  return 0;
}
}
