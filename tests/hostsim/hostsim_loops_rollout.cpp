// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
// One stage of rbd_integrate_loops' dynamics with contact ON THE CPU, one sample at a time: loops_contact_sample (csrc/rbd_loops.cuh)
// exactly as loops_contact_kernel runs it -- the contact pass at the stage state s0 + wa ṡ_prev, its root-frame wrenches in the
// rows behind LoopRows::total of the workspace column, then loops_sample on them -- on [rows][B] arrays (leading dimension B).
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
void run_stage(const HostModel& hm, const rbd_loop_desc& ld, const rbd_contact_desc& cd, int64_t B, const T* q, const T* v, const T* tau,
               const T* s0, const T* sdp, double wa, T* vd, T* sd) {
  const ModelDev<T>& M = dev<T>(hm);
  std::vector<LoopDev<T>> L(1);
  build_loop_dev<T>(hm, ld, sizeof(T) == 8 ? kLoopRcond64 : kLoopRcond32, L[0]);
  std::vector<ContactDev<T>> C(1);
  build_contact_dev<T>(hm.nb, hm.pos.data(), hm.alignT.data(), cd, C[0]);
  const LoopRows rows = loop_rows(hm.nb, hm.nv, L[0].nc, loop_nends(hm, ld), true);
  std::vector<T> work(rows.total + 6 * hm.nb + 1), stash(std::max({crba_rows(hm), rnea_rows(hm), kin_rows(hm)}) + 64);
  bool multi = false;
  for (int i = 0; i < hm.nb; ++i) multi |= kind_nv(M.body[i].kind) > 1;
  for (int64_t b = 0; b < B; ++b) {
    LoopsIO<T, ColRW<T>> io;
    io.q = {q + b, B}; io.v = {v + b, B};
    io.tau = {tau ? tau + b : nullptr, B};
    io.vd = {vd + b, B, true};
    io.qd = io.lam = io.K = io.k = {nullptr, B, true};
    io.w = {work.data(), 1};
    io.r = rows;
    const ContactStageIO<T> cs{s0 + b, sdp ? sdp + b : nullptr, sd + b, (T)wa, B, true};
    if (multi) loops_contact_sample<T, Stash<T, 1>, 6>(M, L[0], C[0], cs, io, rows.total, Stash<T, 1>{stash.data()});
    else loops_contact_sample<T, Stash<T, 1>, 1>(M, L[0], C[0], cs, io, rows.total, Stash<T, 1>{stash.data()});
  }
}
}  // namespace

extern "C" {
// v̇ and ṡ at stage state (q, v, s0 + wa sdp) -- sdp NULL: s0 itself.  dtype 0 = fp32, 1 = fp64.  Returns an rbd_status (the loop
// descriptor is checked as rbd_integrate_loops checks it).
int hostsim_loops_contact_stage(const rbd_model_desc* d, const rbd_loop_desc* ld, const rbd_contact_desc* cd, int dtype, int64_t B,
                                const void* q, const void* v, const void* tau, const void* s0, const void* sdp, double wa, void* vd,
                                void* sd) {
  HostModel hm; std::string err;
  int rc = build_host_model(d, hm, err);
  if (rc) return rc;
  if ((rc = check_loop_desc(hm, ld, err))) return rc;
  if (dtype == 0)
    run_stage<float>(hm, *ld, *cd, B, (const float*)q, (const float*)v, (const float*)tau, (const float*)s0, (const float*)sdp, wa,
                     (float*)vd, (float*)sd);
  else
    run_stage<double>(hm, *ld, *cd, B, (const double*)q, (const double*)v, (const double*)tau, (const double*)s0, (const double*)sdp,
                      wa, (double*)vd, (double*)sd);
  return 0;
}
}
