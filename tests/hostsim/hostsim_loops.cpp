// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
// Runs loops_sample (csrc/rbd_loops.cuh), the per-sample function of rbd_dynamics_loops, ON THE CPU: one sample at a time with a
// workspace column of one row per scalar, so the mathematics of the kernel can be checked against the oracle without a GPU.
#include <algorithm>
#include <string>
#include <vector>

#include "../../rigidbodydynamics/jl_b200/csrc/rbd_loops.cuh"

using namespace rbd;

namespace {
template <class T> const ModelDev<T>& dev(const HostModel& m);
template <> const ModelDev<float>& dev<float>(const HostModel& m) { return m.dev32; }
template <> const ModelDev<double>& dev<double>(const HostModel& m) { return m.dev64; }

template <class T>
void run_loops(const HostModel& hm, const rbd_loop_desc& ld, int64_t B, const T* q, const T* v, const T* tau, const T* wext, T* vd,
               T* qd, T* lam, T* K, T* k) {
  const ModelDev<T>& M = dev<T>(hm);
  std::vector<LoopDev<T>> Lv(1);
  LoopDev<T>& L = Lv[0];
  build_loop_dev<T>(hm, ld, sizeof(T) == 8 ? kLoopRcond64 : kLoopRcond32, L);
  const LoopRows rows = loop_rows(hm.nb, hm.nv, L.nc, loop_nends(hm, ld), wext != nullptr);
  std::vector<T> work(rows.total + 1), stash(std::max({crba_rows(hm), rnea_rows(hm), kin_rows(hm)}) + 64);
  bool multi = false;
  for (int i = 0; i < hm.nb; ++i) multi |= kind_nv(M.body[i].kind) > 1;
  for (int64_t b = 0; b < B; ++b) {
    LoopsIO<T> io;
    io.q = {q + b, B}; io.v = {v + b, B};
    io.tau = {tau ? tau + b : nullptr, B}; io.wext = {wext ? wext + b : nullptr, B};
    auto out = [&](T* p) { return ColOut<T>{p ? p + b : nullptr, B, true}; };
    io.vd = out(vd); io.qd = out(qd); io.lam = out(lam); io.K = out(K); io.k = out(k);
    io.w = {work.data(), 1};
    io.r = rows;
    if (multi) loops_sample<T, Stash<T, 1>, 6>(M, L, io, Stash<T, 1>{stash.data()});
    else loops_sample<T, Stash<T, 1>, 1>(M, L, io, Stash<T, 1>{stash.data()});
  }
}
}  // namespace

extern "C" {
// Returns an rbd_status: the descriptor is checked exactly like rbd_dynamics_loops does.
int hostsim_dynamics_loops(const rbd_model_desc* d, const rbd_loop_desc* ld, int dtype, int64_t B, const void* q, const void* v,
                           const void* tau, const void* wext, void* vd, void* qd, void* lam, void* K, void* k) {
  HostModel hm; std::string err;
  int rc = build_host_model(d, hm, err);
  if (rc) return rc;
  if ((rc = check_loop_desc(hm, ld, err))) return rc;
  if (dtype == 0)
    run_loops<float>(hm, *ld, B, (const float*)q, (const float*)v, (const float*)tau, (const float*)wext, (float*)vd, (float*)qd,
                     (float*)lam, (float*)K, (float*)k);
  else
    run_loops<double>(hm, *ld, B, (const double*)q, (const double*)v, (const double*)tau, (const double*)wext, (double*)vd,
                      (double*)qd, (double*)lam, (double*)K, (double*)k);
  return 0;
}
}
