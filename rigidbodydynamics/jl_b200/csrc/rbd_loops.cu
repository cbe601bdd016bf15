// rbd_dynamics_loops: dynamics! for mechanisms with kinematic loops (csrc/rbd_loops.cuh has the mathematics), and the stage
// dynamics of the loop rollout rbd_integrate_loops (its RK4 driver and entry point are in rbd_b200.cu).
//
// One generic persistent kernel, one thread per sample, one launch per call: CRBA, RNEA bias, q̇, the constraint Jacobian / bias
// sweep and the KKT solve run back to back in the same thread, so no intermediate crosses a launch boundary.  The per-sample
// working set (M, K / Y, A, ...) lives in the stream-ordered workspace of plan_persistent (rbd_handle.h): LoopRows::total rows x
// RESIDENT threads (blocks of one warp looping over groups of 32 samples), laid out [row][thread] so a warp's access to a row is
// one coalesced line; the pending slots of the tree sweeps live in shared memory as in the other kernels.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <memory>
#include <string>

#include "../../../include/rbd_b200.h"
// rbd_sincos.cuh defines one out-of-line __device__ function with external linkage; this translation unit gets its own copy
#define sincos_slow sincos_slow_loops_tu
#include "rbd_loops.cuh"
#include "rbd_handle.h"

using namespace rbd;

namespace {

constexpr int kNT = 32;     // one warp per block; warps never synchronise

template <class T> struct LoopArgs {
  const T *q, *v, *tau, *wext;
  T *vd, *qd, *lam, *K, *k;
  T* work;                  // [rows][grid * NT]
  LoopRows r;
  int64_t ld, B;
};

template <class T, int NT, int KMAX>
__global__ void __launch_bounds__(NT, 1)
loops_kernel(const __grid_constant__ ModelDev<T> M, const __grid_constant__ LoopDev<T> L, const LoopArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const Stash<T, NT> st{reinterpret_cast<T*>(smem_raw) + threadIdx.x};
  const int64_t tid = (int64_t)blockIdx.x * NT + threadIdx.x;
  const int64_t ngroups = (a.B + NT - 1) / NT;
  for (int64_t g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const int64_t b = g * NT + threadIdx.x;
    const bool active = b < a.B;
    const int64_t bl = active ? b : a.B - 1;      // inactive lanes recompute the last sample, stores are masked
    LoopsIO<T> io;
    io.q = {a.q + bl, a.ld};
    io.v = {a.v + bl, a.ld};
    io.tau = {a.tau ? a.tau + bl : nullptr, a.ld};
    io.wext = {a.wext ? a.wext + bl : nullptr, a.ld};
    io.vd = {a.vd + bl, a.ld, active};
    io.qd = {a.qd ? a.qd + bl : nullptr, a.ld, active};
    io.lam = {a.lam ? a.lam + bl : nullptr, a.ld, active};
    io.K = {a.K ? a.K + bl : nullptr, a.ld, active};
    io.k = {a.k ? a.k + bl : nullptr, a.ld, active};
    io.w = {a.work + tid, (int64_t)gridDim.x * NT};     // workspace column of this resident thread
    io.r = a.r;
    loops_sample<T, Stash<T, NT>, KMAX>(M, L, io, st);
  }
}

// One RK4 stage of the loop rollout with contact (loops_contact_sample): the arrays of `a` are the rollout's dense stage buffers
// (ld = B; q, v, tau, vd only), the contact state as in aba_contact_kernel, and the root-frame contact wrenches in workspace rows
// wrow .. wrow + 6 nb - 1, behind the LoopRows::total rows of the solve.
template <class T> struct LoopContactArgs {
  LoopArgs<T> a;
  const T* s0; const T* sdp;      // contact state at the start of the step, ṡ of the previous stage (NULL at stage 0)
  T* sd;                          // ṡ_i
  T wa;                           // dt a_i
  int wrow;
};
// The three descriptors travel in the parameter space (32,764 B on sm_90 since CUDA 12.1): in fp64 14,392 + 9,752 + 2,896 B.
static_assert(sizeof(ModelDev<double>) + sizeof(LoopDev<double>) + sizeof(ContactDev<double>) + sizeof(LoopContactArgs<double>) <= 32764,
              "loops_contact_kernel's parameters exceed the kernel-parameter limit");

template <class T, int NT, int KMAX>
__global__ void __launch_bounds__(NT, 1)
loops_contact_kernel(const __grid_constant__ ModelDev<T> M, const __grid_constant__ LoopDev<T> L,
                     const __grid_constant__ ContactDev<T> C, const __grid_constant__ LoopContactArgs<T> c) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const Stash<T, NT> st{reinterpret_cast<T*>(smem_raw) + threadIdx.x};
  const LoopArgs<T>& a = c.a;
  const int64_t tid = (int64_t)blockIdx.x * NT + threadIdx.x;
  const int64_t ngroups = (a.B + NT - 1) / NT;
  for (int64_t g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const int64_t b = g * NT + threadIdx.x;
    const bool active = b < a.B;
    const int64_t bl = active ? b : a.B - 1;      // inactive lanes recompute the last sample, stores are masked
    LoopsIO<T, ColRW<T>> io;
    io.q = {a.q + bl, a.ld};
    io.v = {a.v + bl, a.ld};
    io.tau = {a.tau ? a.tau + bl : nullptr, a.ld};
    io.vd = {a.vd + bl, a.ld, active};
    io.qd = io.lam = io.K = io.k = {nullptr, a.ld, active};
    io.w = {a.work + tid, (int64_t)gridDim.x * NT};
    io.r = a.r;
    const ContactStageIO<T> cs{c.s0 + bl, c.sdp ? c.sdp + bl : nullptr, c.sd + bl, c.wa, a.ld, active};
    loops_contact_sample<T, Stash<T, NT>, KMAX>(M, L, C, cs, io, c.wrow, st);
  }
}

}  // namespace

// Everything the loop kernels need beyond the model, planned once per call: rbd_dynamics_loops uses it for its one launch, the
// rollout keeps it for all 4 nsteps stages (rbd_handle.h, loop_stage_launch).
struct rbd::LoopStagePlan {
  virtual ~LoopStagePlan() = default;
};

namespace {

template <class T> struct LoopPlan : LoopStagePlan {
  LoopDev<T> L;
  ContactDev<T> C;          // built with contact only
  LoopRows rows;
  bool multi = false;       // some joint has nv > 1 (KMAX = 6)
  bool contact = false;
  LaunchPlan pl;
};

// Descriptors, workspace rows, grid and workspace (rows.total per resident thread, plus 6 nb contact-wrench rows with contact) for
// a batch of B samples.  `wext`: caller-supplied external wrenches; the contact kernel plans with them too (its wrenches go through
// rnea_sample's conversion rows).
template <class T>
int loop_plan(const HostModel& hm, const rbd_loop_desc& desc, const rbd_contact_desc* contact, bool wext, int64_t B, cudaStream_t stream,
              LoopPlan<T>& p) {
  const ModelDev<T>& M = dev_model<T>(hm);
  build_loop_dev<T>(hm, desc, sizeof(T) == 8 ? kLoopRcond64 : kLoopRcond32, p.L);
  p.contact = contact != nullptr;
  if (contact) build_contact_dev<T>(hm.nb, hm.pos.data(), hm.alignT.data(), *contact, p.C);
  p.rows = loop_rows(hm.nb, hm.nv, p.L.nc, loop_nends(hm, desc), wext || p.contact);
  for (int i = 0; i < hm.nb; ++i) p.multi |= kind_nv(M.body[i].kind) > 1;
  const void* kernel = p.contact ? (p.multi ? (const void*)loops_contact_kernel<T, kNT, 6> : (const void*)loops_contact_kernel<T, kNT, 1>)
                                 : (p.multi ? (const void*)loops_kernel<T, kNT, 6> : (const void*)loops_kernel<T, kNT, 1>);
  const int stash = std::max({1, crba_rows(hm), rnea_rows(hm), kin_rows(hm)});
  const size_t rows = (size_t)p.rows.total + (p.contact ? (size_t)6 * hm.nb : 0);
  return plan_persistent(kernel, kNT, (size_t)stash * kNT * sizeof(T), (B + kNT - 1) / kNT, stream, p.pl, rows * sizeof(T));
}

template <class T>
int launch_loops(const ModelDev<T>& M, const LoopPlan<T>& p, const LoopArgs<T>& a, cudaStream_t stream) {
  if (p.multi) loops_kernel<T, kNT, 6><<<p.pl.grid, p.pl.block, p.pl.smem, stream>>>(M, p.L, a);
  else loops_kernel<T, kNT, 1><<<p.pl.grid, p.pl.block, p.pl.smem, stream>>>(M, p.L, a);
  return api_launched(&p.pl);
}

template <class T>
int loops_t(const rbd_model* model, int64_t B, int64_t ld, const void* q, const void* v, const void* tau, const void* wext,
            const rbd_loop_desc& desc, void* vd, void* qd, void* lam, void* K, void* k, cudaStream_t stream) {
  const ModelDev<T>& M = dev_model<T>(model->hm);
  std::unique_ptr<LoopPlan<T>> p(new LoopPlan<T>());
  if (int rc = loop_plan<T>(model->hm, desc, nullptr, wext != nullptr, B, stream, *p)) return rc;
  const LoopArgs<T> a{(const T*)q, (const T*)v, (const T*)tau, (const T*)wext, (T*)vd, (T*)qd, (T*)lam, (T*)K, (T*)k,
                      (T*)p->pl.work.p, p->rows, ld, B};
  return launch_loops<T>(M, *p, a, stream);
}

template <class T>
int loop_stage_t(const rbd_model* model, const rbd_loop_desc& loops, const rbd_contact_desc* contact, const LoopStageArgs& s,
                 std::shared_ptr<LoopStagePlan>& plan, cudaStream_t stream) {
  const ModelDev<T>& M = dev_model<T>(model->hm);
  if (!plan) {
    std::shared_ptr<LoopPlan<T>> p(new LoopPlan<T>());
    if (int rc = loop_plan<T>(model->hm, loops, contact, false, s.B, stream, *p)) return rc;
    plan = p;
  }
  const LoopPlan<T>& p = static_cast<const LoopPlan<T>&>(*plan);
  const LoopArgs<T> a{(const T*)s.q, (const T*)s.v, (const T*)s.tau, nullptr, (T*)s.vd, nullptr, nullptr, nullptr, nullptr,
                      (T*)p.pl.work.p, p.rows, s.B, s.B};
  if (!p.contact) return launch_loops<T>(M, p, a, stream);
  const LoopContactArgs<T> c{a, (const T*)s.s0, (const T*)s.sdp, (T*)s.sd, (T)s.wa, p.rows.total};
  if (p.multi) loops_contact_kernel<T, kNT, 6><<<p.pl.grid, p.pl.block, p.pl.smem, stream>>>(M, p.L, p.C, c);
  else loops_contact_kernel<T, kNT, 1><<<p.pl.grid, p.pl.block, p.pl.smem, stream>>>(M, p.L, p.C, c);
  return api_launched(&p.pl);
}

}  // namespace

namespace rbd {
int api_check_loops(const rbd_model* model, const rbd_loop_desc* loops) {
  std::string err;
  if (int rc = check_loop_desc(model->hm, loops, err)) return api_fail(rc, err);
  return RBD_OK;
}
int loop_stage_launch(const rbd_model* model, int32_t dtype, const rbd_loop_desc& loops, const rbd_contact_desc* contact,
                      const LoopStageArgs& a, std::shared_ptr<LoopStagePlan>& plan, cudaStream_t stream) {
  return dtype == RBD_F32 ? loop_stage_t<float>(model, loops, contact, a, plan, stream)
                          : loop_stage_t<double>(model, loops, contact, a, plan, stream);
}
}  // namespace rbd

extern "C" int32_t rbd_dynamics_loops(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                                      const void* tau, const void* wext, const rbd_loop_desc* loops, void* vd_out, void* qd_out,
                                      void* lambda_out, void* K_out, void* k_out, void* stream) {
  if (int rc = api_check(model, dtype, B, ld)) return rc;
  const ApiCall call;
  std::string err;
  if (int rc = check_loop_desc(model->hm, loops, err)) return api_fail(rc, err);
  if (!q || !v || !vd_out) return api_fail(RBD_EINVAL, "rbd_dynamics_loops: q, v and vd_out must not be NULL");
  if (B == 0) return RBD_OK;
  cudaStream_t s = (cudaStream_t)stream;
  return dtype == RBD_F32 ? loops_t<float>(model, B, ld, q, v, tau, wext, *loops, vd_out, qd_out, lambda_out, K_out, k_out, s)
                          : loops_t<double>(model, B, ld, q, v, tau, wext, *loops, vd_out, qd_out, lambda_out, K_out, k_out, s);
}
