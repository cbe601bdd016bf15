// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
// The feedback law of rbd_integrate_pd ON THE CPU: pd_joint (csrc/rbd_pd.cuh) for every joint and sample exactly as
// integrate_stage_kernel evaluates it on the stage state, on [rows][B] arrays (leading dimension B).
#include <string>
#include <vector>

#include "../../rigidbodydynamics/jl_b200/csrc/rbd_model.h"
#include "../../rigidbodydynamics/jl_b200/csrc/rbd_pd.cuh"

using namespace rbd;

namespace {
template <class T> const ModelDev<T>& dev(const HostModel& m);
template <> const ModelDev<float>& dev<float>(const HostModel& m) { return m.dev32; }
template <> const ModelDev<double>& dev<double>(const HostModel& m) { return m.dev64; }

template <class T>
void run(const HostModel& hm, int64_t B, const T* q, const T* v, const T* qref, const T* vref, const T* ff, const T* kp, const T* kd,
         bool per_sample, const double* lo, const double* hi, T* out) {
  const ModelDev<T>& M = dev<T>(hm);
  std::vector<T> lh(2 * hm.nv);
  for (int k = 0; lo && k < hm.nv; ++k) { lh[k] = (T)lo[k]; lh[hm.nv + k] = (T)hi[k]; }
  for (int64_t b = 0; b < B; ++b) {
    const int64_t gc = per_sample ? b : 0;
    const PdSample<T> s{q + b, v + b, B, qref + b, vref ? vref + b : nullptr, ff ? ff + b : nullptr, B, kp + gc, kd + gc,
                        per_sample ? B : 1, lo ? lh.data() : nullptr, lo ? lh.data() + hm.nv : nullptr};
    for (int i = 0; i < hm.nb; ++i) pd_joint(M.body[i], s, ColOut<T>{out + b, B, true});
  }
}
}  // namespace

extern "C" {
// out [nv x B] = the law at (q, v); dtype 0 = fp32, 1 = fp64; kp / kd [nv] (per_sample 0) or [nv x B]; lo / hi host [nv] or NULL.
int hostsim_pd_law(const rbd_model_desc* d, int dtype, int64_t B, const void* q, const void* v, const void* qref, const void* vref,
                   const void* ff, const void* kp, const void* kd, int per_sample, const double* lo, const double* hi, void* out) {
  HostModel hm; std::string err;
  if (int rc = build_host_model(d, hm, err)) return rc;
  if (dtype == 0)
    run<float>(hm, B, (const float*)q, (const float*)v, (const float*)qref, (const float*)vref, (const float*)ff, (const float*)kp,
               (const float*)kd, per_sample != 0, lo, hi, (float*)out);
  else
    run<double>(hm, B, (const double*)q, (const double*)v, (const double*)qref, (const double*)vref, (const double*)ff,
                (const double*)kp, (const double*)kd, per_sample != 0, lo, hi, (double*)out);
  return 0;
}
}
