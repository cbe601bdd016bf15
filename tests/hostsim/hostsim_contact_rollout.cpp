// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
// One stage of rbd_integrate_contact's forward dynamics ON THE CPU, one sample at a time: contact_stage_pass (csrc/rbd_kin.cuh) and
// aba_sample (csrc/rbd_device.cuh) exactly as aba_contact_kernel runs them, compact wrench scratch included, on [rows][B] arrays
// (leading dimension B).
#include <string>
#include <vector>

#include "../../rigidbodydynamics/jl_b200/csrc/rbd_rnea_crba.cuh"
#include "../../rigidbodydynamics/jl_b200/csrc/rbd_kin.cuh"
#include "../../rigidbodydynamics/jl_b200/csrc/rbd_model.h"

using namespace rbd;

namespace {
template <class T> const ModelDev<T>& dev(const HostModel& m);
template <> const ModelDev<float>& dev<float>(const HostModel& m) { return m.dev32; }
template <> const ModelDev<double>& dev<double>(const HostModel& m) { return m.dev64; }

template <class T>
void run_stage(const HostModel& hm, int64_t B, const T* q, const T* v, const T* tau, const rbd_contact_desc& cd, const T* s0, const T* sdp,
               double wa, T* vd, T* sd) {
  const ModelDev<T>& M = dev<T>(hm);
  std::vector<ContactDev<T>> C(1);
  build_contact_dev<T>(hm.nb, hm.pos.data(), hm.alignT.data(), cd, C[0]);
  int8_t slot[kMaxBodies];
  const int nw = contact_wrench_slots(hm.nb, C[0], slot);
  std::vector<T> stash(M.nrows + 64), scratch(6 * nw + 1);
  for (int64_t b = 0; b < B; ++b) {
    ContactAbaIO<T, kAllKinds> io;
    io.q = {q + b, B}; io.v = {v + b, B};
    io.tau = {tau ? tau + b : nullptr, B};
    io.vd = {vd + b, B, true}; io.qd = {nullptr, 1, true};
    io.ext = {scratch.data(), 1, slot};
    const ContactStageIO<T> cs{s0 ? s0 + b : nullptr, sdp ? sdp + b : nullptr, sd ? sd + b : nullptr, (T)wa, B, true};
    Stash<T, 1> st{stash.data()};
    contact_stage_pass(M, C[0], io.q, io.v, cs, io.ext, st, M.slot_base, kSlotRowsAba);
    if (hm.general) aba_sample<T, Stash<T, 1>, true>(M, io, st);
    else aba_sample<T, Stash<T, 1>, false>(M, io, st);
  }
}
}  // namespace

extern "C" {
// v̇ and ṡ of stage state (q, v, s0 + wa sdp) -- sdp NULL: s0 itself.  dtype 0 = fp32, 1 = fp64.
int hostsim_contact_stage(const rbd_model_desc* d, int dtype, int64_t B, const void* q, const void* v, const void* tau,
                          const rbd_contact_desc* cd, const void* s0, const void* sdp, double wa, void* vd, void* sd) {
  HostModel hm; std::string err;
  int rc = build_host_model(d, hm, err);
  if (rc) return rc;
  if (dtype == 0)
    run_stage<float>(hm, B, (const float*)q, (const float*)v, (const float*)tau, *cd, (const float*)s0, (const float*)sdp, wa, (float*)vd,
                     (float*)sd);
  else
    run_stage<double>(hm, B, (const double*)q, (const double*)v, (const double*)tau, *cd, (const double*)s0, (const double*)sdp, wa,
                      (double*)vd, (double*)sd);
  return 0;
}
}
