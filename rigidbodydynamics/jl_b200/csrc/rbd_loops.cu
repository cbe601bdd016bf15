// rbd_dynamics_loops: dynamics! for mechanisms with kinematic loops (csrc/rbd_loops.cuh has the mathematics).
//
// One generic persistent kernel, one thread per sample, one launch per call: CRBA, RNEA bias, q̇, the constraint Jacobian / bias
// sweep and the KKT solve run back to back in the same thread, so no intermediate crosses a launch boundary.  The per-sample
// working set (M, K / Y, A, ...) lives in the stream-ordered workspace of plan_persistent (rbd_handle.h): LoopRows::total rows x
// RESIDENT threads (blocks of one warp looping over groups of 32 samples), laid out [row][thread] so a warp's access to a row is
// one coalesced line; the pending slots of the tree sweeps live in shared memory as in the other kernels.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
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

template <class T>
int loops_t(const rbd_model* model, int64_t B, int64_t ld, const void* q, const void* v, const void* tau, const void* wext,
            const rbd_loop_desc& desc, void* vd, void* qd, void* lam, void* K, void* k, cudaStream_t stream) {
  const HostModel& hm = model->hm;
  const ModelDev<T>& M = dev_model<T>(hm);
  LoopDev<T> L;
  build_loop_dev<T>(hm, desc, sizeof(T) == 8 ? kLoopRcond64 : kLoopRcond32, L);
  const LoopRows rows = loop_rows(hm.nb, hm.nv, L.nc, loop_nends(hm, desc), wext != nullptr);
  bool multi = false;
  for (int i = 0; i < hm.nb; ++i) multi |= kind_nv(M.body[i].kind) > 1;
  const void* kernel = multi ? (const void*)loops_kernel<T, kNT, 6> : (const void*)loops_kernel<T, kNT, 1>;
  const int stash = std::max({1, crba_rows(hm), rnea_rows(hm), kin_rows(hm)});
  LaunchPlan pl;
  if (int rc = plan_persistent(kernel, kNT, (size_t)stash * kNT * sizeof(T), (B + kNT - 1) / kNT, stream, pl,
                               (size_t)rows.total * sizeof(T))) return rc;
  const LoopArgs<T> a{(const T*)q, (const T*)v, (const T*)tau, (const T*)wext, (T*)vd, (T*)qd, (T*)lam, (T*)K, (T*)k,
                      (T*)pl.work.p, rows, ld, B};
  if (multi) loops_kernel<T, kNT, 6><<<pl.grid, pl.block, pl.smem, stream>>>(M, L, a);
  else loops_kernel<T, kNT, 1><<<pl.grid, pl.block, pl.smem, stream>>>(M, L, a);
  return api_launched(&pl);
}

}  // namespace

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
