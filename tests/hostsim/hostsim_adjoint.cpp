// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
// Runs adjoint_sample / dynamics_vjp_sample (csrc/rbd_adjoint.cuh), the per-sample functions of rbd_inverse_dynamics_vjp /
// rbd_dynamics_vjp, ON THE CPU: one sample at a time with a workspace column of one row per scalar, so the mathematics of the kernels
// can be checked against the oracle without a GPU.
#include <string>
#include <vector>

#include "../../rigidbodydynamics/jl_b200/csrc/rbd_adjoint.cuh"
#include "../../rigidbodydynamics/jl_b200/csrc/rbd_model.h"

using namespace rbd;

namespace {
template <class T> const ModelDev<T>& dev(const HostModel& m);
template <> const ModelDev<float>& dev<float>(const HostModel& m) { return m.dev32; }
template <> const ModelDev<double>& dev<double>(const HostModel& m) { return m.dev64; }

// fd = 1: dynamics VJP (wbar = ν̄, taub = τ̄); fd = 0: inverse-dynamics VJP (wbar = τ̄, vdb = M τ̄)
template <class T>
void run(const HostModel& hm, int fd, int64_t B, const T* q, const T* v, const T* vd, const T* wext, const T* wbar, T* qt, T* qc,
         T* vb, T* vdb, T* taub, T* wb) {
  ModelDev<T> M = dev<T>(hm);
  const T g[3] = {M.g[0], M.g[1], M.g[2]};
  if (fd) M.g[0] = M.g[1] = M.g[2] = T(0);
  std::vector<T> work(adjoint_rows(hm.nb, hm.nv)), stash(M.nrows + 64);
  const T zero = T(0);
  for (int64_t b = 0; b < B; ++b) {
    AdjIO<T> io;
    io.q = {q + b, B}; io.v = {v + b, B}; io.vd = {vd + b, B}; io.wext = {wext ? wext + b : nullptr, B};
    auto out = [&](T* p) { return ColOut<T>{p ? p + b : nullptr, B, true}; };
    io.qt = out(qt); io.qc = out(qc); io.vb = out(vb); io.vdb = out(vdb); io.wb = out(wb);
    io.s = {work.data(), 1};
    if (fd) dynamics_vjp_sample<T>(M, g, io, Col<T>{wbar + b, B}, out(taub), &zero, Stash<T, 1>{stash.data()});
    else adjoint_sample<T>(M, g, io, Col<T>{wbar + b, B}, T(1));
  }
}
}  // namespace

extern "C" {
int hostsim_vjp(const rbd_model_desc* d, int fd, int dtype, int64_t B, const void* q, const void* v, const void* vd, const void* wext,
                const void* wbar, void* qt, void* qc, void* vb, void* vdb, void* taub, void* wb) {
  HostModel hm; std::string err;
  int rc = build_host_model(d, hm, err);
  if (rc) return rc;
  if (dtype == 0)
    run<float>(hm, fd, B, (const float*)q, (const float*)v, (const float*)vd, (const float*)wext, (const float*)wbar, (float*)qt,
               (float*)qc, (float*)vb, (float*)vdb, (float*)taub, (float*)wb);
  else
    run<double>(hm, fd, B, (const double*)q, (const double*)v, (const double*)vd, (const double*)wext, (const double*)wbar,
                (double*)qt, (double*)qc, (double*)vb, (double*)vdb, (double*)taub, (double*)wb);
  return 0;
}
}
