// librbd_b200.so -- C ABI (include/rbd_b200.h) over the sm_90a kernels.
//
// Kernel design (DESIGN.md has the long version):
//   * one THREAD owns one sample; a block is one or more independent warps; there are no block-level barriers;
//   * the grid is persistent: blocks_per_SM x SM_count blocks loop over groups of NT consecutive samples;
//   * inputs / outputs are rows x batch with the batch index fastest, so lane l of a warp touches element b0 + l of a
//     row: every global access of a warp is one fully-used 128-byte line (fp32) / two lines (fp64);
//   * the per-sample working set that must survive between the three passes lives in shared memory, laid out
//     [row][lane] so a warp's access to a row hits 32 distinct banks;
//   * the flattened mechanism is a __grid_constant__ kernel parameter: it is read through the constant bank with a
//     warp-uniform index, i.e. as uniform-register operands, not as per-thread loads.
// The host side of every launch (device properties, kernel configuration, persistent grid and workspace, error mapping, launch
// record) is the shared plumbing declared in rbd_handle.h and implemented below, used by the library's other units as well.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <new>
#include <optional>
#include <set>
#include <string>
#include <type_traits>

#include "../../../include/rbd_b200.h"
#include "rbd_rnea_crba.cuh"
#include "rbd_kin.cuh"
#include "rbd_dual.cuh"
#include "rbd_integrate.cuh"
#include "rbd_model.h"

using namespace rbd;

// ------------------------------------------------------------------------------------------------------------------
// handle, errors
// ------------------------------------------------------------------------------------------------------------------
#include "rbd_handle.h"

namespace {

thread_local std::string g_err;
thread_local rbd_launch_info g_launch = {0, 0, 0, 0, 0, 0.f, 0};
thread_local int g_call_depth = 0;     // C-ABI calls in progress on this thread (ApiCall)

int fail(int status, const std::string& msg) { g_err = msg; return status; }

}  // namespace

// ---- the host plumbing of rbd_handle.h, shared by the library's translation units ----------------------------------------
namespace rbd {

int api_fail(int status, const std::string& msg) { return fail(status, msg); }
int api_fail_cuda(cudaError_t e, const std::string& what) {
  cudaGetLastError();      // a non-sticky error must not be reported again by the next launch check
  return fail(e == cudaErrorMemoryAllocation ? RBD_ENOMEM : RBD_ECUDA, what + ": " + cudaGetErrorString(e));
}

cudaError_t device_props(DeviceProps& p) {
  static std::mutex mu;
  static DeviceProps cache[64];
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lk(mu);
  if (dev >= 0 && dev < 64 && cache[dev].sms) { p = cache[dev]; return cudaSuccess; }
  DeviceProps q;
  q.dev = dev;
  cudaMemPool_t pool;
  uint64_t keep = ~0ull;
  e = cudaDeviceGetAttribute(&q.sms, cudaDevAttrMultiProcessorCount, dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&q.max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&q.smem_per_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&q.l2_bytes, cudaDevAttrL2CacheSize, dev);
  if (e == cudaSuccess) e = cudaDeviceGetDefaultMemPool(&pool, dev);
  if (e == cudaSuccess) e = cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
  if (e != cudaSuccess) return e;
  if (dev >= 0 && dev < 64) cache[dev] = q;
  p = q;
  return cudaSuccess;
}

int kernel_config(const void* kernel, int block, size_t smem, const DeviceProps& p, int& blocks_per_sm) {
  if (smem > (size_t)p.max_smem_optin) return fail(RBD_EUNSUPPORTED, "model working set exceeds shared memory per block");
  if (smem > 0) {
    static std::mutex mu;
    static std::set<std::pair<const void*, int>> done;
    std::lock_guard<std::mutex> lk(mu);
    if (!done.count({kernel, p.dev})) {
      cudaFuncAttributes fa{};
      RBD_CUDA_TRY(cudaFuncGetAttributes(&fa, kernel));
      RBD_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, p.max_smem_optin - (int)fa.sharedSizeBytes));
      RBD_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
      done.insert({kernel, p.dev});
    }
  }
  RBD_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, kernel, block, smem));
  if (blocks_per_sm < 1) return fail(RBD_EUNSUPPORTED, "kernel does not fit on an SM");
  return RBD_OK;
}

int plan_persistent(const void* kernel, int block, size_t smem, int64_t ngroups, cudaStream_t stream, LaunchPlan& plan,
                    size_t work_per_thread, size_t work_extra, size_t work_cap) {
  DeviceProps p;
  RBD_CUDA_TRY(device_props(p));
  if (int rc = kernel_config(kernel, block, smem, p, plan.blocks_per_sm)) return rc;
  int64_t grid = std::min<int64_t>(ngroups, (int64_t)plan.blocks_per_sm * p.sms);
  if (work_cap) grid = std::min<int64_t>(grid, std::max<int64_t>(1, (int64_t)(work_cap / (work_per_thread * block))));
  plan.grid = (int)grid;
  plan.block = block;
  plan.smem = (int)smem;
  if (work_per_thread) RBD_CUDA_TRY(plan.work.alloc(work_per_thread * grid * block + work_extra, stream));
  return RBD_OK;
}

ApiCall::ApiCall() { if (g_call_depth++ == 0) g_launch = {0, 0, 0, 0, 0, 0.f, 0}; }
ApiCall::~ApiCall() { --g_call_depth; }

void api_note_launch(const LaunchShape* shape, bool specialised) {
  g_launch.kernels_launched += 1;
  if (shape) {
    g_launch.grid = shape->grid; g_launch.block = shape->block; g_launch.smem_bytes = shape->smem;
    g_launch.blocks_per_sm = shape->blocks_per_sm;
  }
  if (specialised) g_launch.specialised = 1;
}
int api_launched(const LaunchShape* shape) {
  RBD_CUDA_TRY(cudaGetLastError());
  api_note_launch(shape);
  return RBD_OK;
}

KeepLaunchRecord::KeepLaunchRecord() : saved(g_launch) {}
KeepLaunchRecord::~KeepLaunchRecord() {
  const int n = g_launch.kernels_launched;
  g_launch = saved;
  g_launch.kernels_launched = n;
}

}  // namespace rbd

namespace {

// ------------------------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// Pull the NEXT group's input lines into L2 while this group is being computed (one 128-byte line per row and warp).
template <class T>
__device__ __forceinline__ void prefetch_rows(const T* base, int rows, int64_t ld, int64_t b0) {
  if (!base) return;
  for (int r = threadIdx.x & 31; r < rows; r += 32) prefetch_l2(base + (int64_t)r * ld + b0);
}

template <class T> struct AbaArgs {
  const T* q; const T* v; const T* tau; const T* wext;
  T* vd; T* qd;
  T* scratch;            // [6 * nb][grid threads] body-frame external wrenches (EXT only), one column per resident thread
  int64_t ld, B;
  const int* gate;               // non-NULL: run only if *gate != 0 (fallback behind the model-specialised kernels, rbd_spec.cpp)
  // mixed CTA (launch_mix): work-queue counter, stash of the warps beyond `sw` in L2, stash rows, columns of `scratch`
  unsigned long long* counter; T* l2; int sw, rows; int64_t scratch_ld;
};

// KINDS: compile-time promise about the 1-DoF kinds present (kAllKinds, or 0 = revolute / sin-cos-revolute only).
template <class T, int NT, bool GENERAL, bool EXT, int KINDS>
__global__ void __launch_bounds__(NT, (sizeof(T) == 4 && !GENERAL && !EXT) ? 20 : 1)
aba_kernel(const __grid_constant__ ModelDev<T> M, const AbaArgs<T> a) {
  if (a.gate && *a.gate == 0) return;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* sh = reinterpret_cast<T*>(smem_raw);
  using ST = Stash<T, NT>;
  const int64_t nthreads = (int64_t)gridDim.x * NT;
  const int64_t tid = (int64_t)blockIdx.x * NT + threadIdx.x;
  const ST st{sh + threadIdx.x};
  const int64_t ngroups = (a.B + NT - 1) / NT;
  for (int64_t g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const int64_t gn = g + gridDim.x;
    if (gn < ngroups) {
      const int64_t bn = gn * NT + (threadIdx.x & ~31);
      prefetch_rows(a.q, M.nq, a.ld, bn);
      prefetch_rows(a.v, M.nv, a.ld, bn);
      prefetch_rows(a.tau, M.nv, a.ld, bn);
      if (EXT) prefetch_rows(a.wext, 6 * M.nb, a.ld, bn);
    }
    const int64_t b = g * NT + threadIdx.x;
    const bool active = b < a.B;
    const int64_t bl = active ? b : a.B - 1;     // inactive lanes recompute the last sample, stores are masked
    AbaIO<T, EXT, KINDS> io;
    io.q = {a.q + bl, a.ld};
    io.v = {a.v + bl, a.ld};
    io.tau = {a.tau ? a.tau + bl : nullptr, a.ld};
    io.wext = {EXT ? a.wext + bl : nullptr, a.ld};
    io.vd = {a.vd + bl, a.ld, active};
    io.qd = {a.qd ? a.qd + bl : nullptr, a.ld, active};
    io.ext = {EXT ? a.scratch + tid : nullptr, nthreads};
    if (EXT) ext_wrench_pass(M, io.q, io.wext, io.ext, st, M.slot_base, kSlotRowsAba);
    aba_sample<T, ST, GENERAL>(M, io, st);
  }
}

// dynamics! on Dual{Float64,6} arrays: thread t of the launch owns (sample t / 6, partial direction t % 6).
struct DualArgs {
  const double* q; const double* v; const double* tau;
  double* vd;
  int64_t ld, B;
  unsigned long long* counter; Dual64* l2; int sw, rows;     // mixed CTA (launch_mix), see AbaArgs
  double* scratch; int64_t scratch_ld;                         // unused: no external wrenches on this path
};
template <int NT, bool GENERAL>
__global__ void __launch_bounds__(NT) aba_dual_kernel(const __grid_constant__ ModelDev<Dual64> M, const DualArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Dual64* sh = reinterpret_cast<Dual64*>(smem_raw);
  const Stash<Dual64, NT> st{sh + threadIdx.x};
  const int64_t total = a.B * 6;
  const int64_t ngroups = (total + NT - 1) / NT;
  for (int64_t g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const int64_t t = g * NT + threadIdx.x;
    const bool active = t < total;
    const int64_t tl = active ? t : total - 1;
    const int64_t b = tl / 6;
    const int dir = (int)(tl - b * 6);
    AbaIO<Dual64, false> io;
    io.q = {a.q + b * kDualWidth, a.ld, dir};
    io.v = {a.v + b * kDualWidth, a.ld, dir};
    io.tau = {a.tau ? a.tau + b * kDualWidth : nullptr, a.ld, dir};
    io.wext = {nullptr, a.ld, dir};
    io.vd = {a.vd + b * kDualWidth, a.ld, dir, active};
    io.qd = {nullptr, a.ld, dir, active};
    io.ext = {nullptr, 0};
    aba_sample<Dual64, Stash<Dual64, NT>, GENERAL>(M, io, st);
  }
}

template <class T> struct RneaArgs {
  const T* q; const T* v; const T* vd; const T* wext;
  T* tau;
  T* scratch;
  int64_t ld, B;
  const int* gate;               // see AbaArgs
  // mixed CTA (launch_mix): work-queue counter, stash of the warps beyond `sw` in L2, stash rows, columns of `scratch`
  unsigned long long* counter; T* l2; int sw, rows; int64_t scratch_ld;
};

template <class T, int NT, bool EXT>
__global__ void __launch_bounds__(NT, sizeof(T) == 4 ? 32 : 1) rnea_kernel(const __grid_constant__ ModelDev<T> M, const RneaArgs<T> a) {
  if (a.gate && *a.gate == 0) return;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* sh = reinterpret_cast<T*>(smem_raw);
  const Stash<T, NT> st{sh + threadIdx.x};
  const int64_t ngroups = (a.B + NT - 1) / NT;
  for (int64_t g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const int64_t gn = g + gridDim.x;
    if (gn < ngroups) {
      const int64_t bn = gn * NT + (threadIdx.x & ~31);
      prefetch_rows(a.q, M.nq, a.ld, bn);
      prefetch_rows(a.v, M.nv, a.ld, bn);
      prefetch_rows(a.vd, M.nv, a.ld, bn);
      if (EXT) prefetch_rows(a.wext, 6 * M.nb, a.ld, bn);
    }
    const int64_t b = g * NT + threadIdx.x;
    const bool active = b < a.B;
    const int64_t bl = active ? b : a.B - 1;
    RneaIO<T> io;
    io.q = {a.q + bl, a.ld};
    io.v = {a.v + bl, a.ld};
    io.vd = {a.vd ? a.vd + bl : nullptr, a.ld};
    io.wext = {EXT ? a.wext + bl : nullptr, a.ld};
    io.tau = {a.tau + bl, a.ld, active};
    io.ext = {EXT ? a.scratch + (int64_t)blockIdx.x * NT + threadIdx.x : nullptr, (int64_t)gridDim.x * NT};
    rnea_sample<T>(M, io, st);
  }
}

// ---- mixed CTA: a second home for the stash in L2 -------------------------------------------------------------------------
// One CTA of up to kMixWarps<T> warps per SM (launch_mix).  Warps 0 .. sw-1 keep their stash in the CTA's shared memory, the
// others in a pool-allocated global scratch [block][warp][row][lane] small enough to stay resident in L2.  On H100 shared
// memory holds 8 Atlas fp32 stashes (4 in fp64, 2 of Dual<6>) while the register file has room for twice as many warps; the
// L2 warps fill it.  Warps claim groups of 32 samples from one counter, so the slower L2 warps simply take fewer groups.
template <class T> constexpr int kMixWarps = sizeof(T) == 4 ? 16 : 8;     // x 32 threads x 128 / 255 registers: the register file
template <class E>
__device__ __forceinline__ E* mix_stash(E* smem, E* l2, int sw, int rows) {
  const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  E* base = w < sw ? smem + (size_t)w * rows * 32 : l2 + ((size_t)blockIdx.x * (nw - sw) + (w - sw)) * rows * 32;
  return base + (threadIdx.x & 31);
}
__device__ __forceinline__ int64_t claim_group(unsigned long long* counter) {
  unsigned long long g = 0;
  if ((threadIdx.x & 31) == 0) g = atomicAdd(counter, 1ull);
  return (int64_t)__shfl_sync(0xffffffffu, g, 0);
}
// (No external wrenches: with them the mixed CTA measured slower on H100 than the shared-memory kernel, DESIGN.md 4.1.)
template <class T, int KINDS>
__global__ void __launch_bounds__(32 * kMixWarps<T>, 1) aba_kernel_mix(const __grid_constant__ ModelDev<T> M, const AbaArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const Stash<T, 32> st{mix_stash(reinterpret_cast<T*>(smem_raw), a.l2, a.sw, a.rows)};
  const int lane = threadIdx.x & 31;
  const int64_t ngroups = (a.B + 31) / 32;
  int64_t g = claim_group(a.counter);
  while (g < ngroups) {
    const int64_t gn = claim_group(a.counter);
    if (gn < ngroups) {
      const int64_t bn = gn * 32;
      prefetch_rows(a.q, M.nq, a.ld, bn);
      prefetch_rows(a.v, M.nv, a.ld, bn);
      prefetch_rows(a.tau, M.nv, a.ld, bn);
    }
    const int64_t b = g * 32 + lane;
    const bool active = b < a.B;
    const int64_t bl = active ? b : a.B - 1;
    AbaIO<T, false, KINDS> io;
    io.q = {a.q + bl, a.ld};
    io.v = {a.v + bl, a.ld};
    io.tau = {a.tau ? a.tau + bl : nullptr, a.ld};
    io.wext = {nullptr, a.ld};
    io.vd = {a.vd + bl, a.ld, active};
    io.qd = {a.qd ? a.qd + bl : nullptr, a.ld, active};
    io.ext = {nullptr, 0};
    aba_sample<T, Stash<T, 32>, false>(M, io, st);
    g = gn;
  }
}
template <class T, bool EXT>
__global__ void __launch_bounds__(32 * kMixWarps<T>, 1) rnea_kernel_mix(const __grid_constant__ ModelDev<T> M, const RneaArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const Stash<T, 32> st{mix_stash(reinterpret_cast<T*>(smem_raw), a.l2, a.sw, a.rows)};
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const int64_t ngroups = (a.B + 31) / 32;
  int64_t g = claim_group(a.counter);
  while (g < ngroups) {
    const int64_t gn = claim_group(a.counter);
    if (gn < ngroups) {
      const int64_t bn = gn * 32;
      prefetch_rows(a.q, M.nq, a.ld, bn);
      prefetch_rows(a.v, M.nv, a.ld, bn);
      prefetch_rows(a.vd, M.nv, a.ld, bn);
      if (EXT) prefetch_rows(a.wext, 6 * M.nb, a.ld, bn);
    }
    const int64_t b = g * 32 + lane;
    const bool active = b < a.B;
    const int64_t bl = active ? b : a.B - 1;
    RneaIO<T> io;
    io.q = {a.q + bl, a.ld};
    io.v = {a.v + bl, a.ld};
    io.vd = {a.vd ? a.vd + bl : nullptr, a.ld};
    io.wext = {EXT ? a.wext + bl : nullptr, a.ld};
    io.tau = {a.tau + bl, a.ld, active};
    io.ext = {EXT ? a.scratch + tid : nullptr, a.scratch_ld};
    rnea_sample<T>(M, io, st);
    g = gn;
  }
}
__global__ void __launch_bounds__(32 * kMixWarps<double>, 1) aba_dual_kernel_mix(const __grid_constant__ ModelDev<Dual64> M, const DualArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const Stash<Dual64, 32> st{mix_stash(reinterpret_cast<Dual64*>(smem_raw), a.l2, a.sw, a.rows)};
  const int64_t total = a.B * 6;
  const int64_t ngroups = (total + 31) / 32;
  for (int64_t g = claim_group(a.counter); g < ngroups; g = claim_group(a.counter)) {
    const int64_t t = g * 32 + (threadIdx.x & 31);
    const bool active = t < total;
    const int64_t tl = active ? t : total - 1;
    const int64_t b = tl / 6;
    const int dir = (int)(tl - b * 6);
    AbaIO<Dual64, false> io;
    io.q = {a.q + b * kDualWidth, a.ld, dir};
    io.v = {a.v + b * kDualWidth, a.ld, dir};
    io.tau = {a.tau ? a.tau + b * kDualWidth : nullptr, a.ld, dir};
    io.wext = {nullptr, a.ld, dir};
    io.vd = {a.vd + b * kDualWidth, a.ld, dir, active};
    io.qd = {nullptr, a.ld, dir, active};
    io.ext = {nullptr, 0};
    aba_sample<Dual64, Stash<Dual64, 32>, false>(M, io, st);
  }
}

template <class T> struct CrbaArgs {
  const T* q;
  T* M;
  int64_t ld, B;
  bool lower;
  const int* gate;       // non-NULL: run only if *gate != 0 (fallback behind the model-specialised kernel, see AbaArgs)
};

template <class T, int NT, int KMAX>
__global__ void __launch_bounds__(NT, sizeof(T) == 4 ? (KMAX == 1 ? 28 : 20) : 1) crba_kernel(const __grid_constant__ ModelDev<T> M, const CrbaArgs<T> a) {
  if (a.gate && *a.gate == 0) return;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* sh = reinterpret_cast<T*>(smem_raw);
  const Stash<T, NT> st{sh + threadIdx.x};
  const int64_t ngroups = (a.B + NT - 1) / NT;
  for (int64_t g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const int64_t gn = g + gridDim.x;
    if (gn < ngroups) prefetch_rows(a.q, M.nq, a.ld, gn * NT + (threadIdx.x & ~31));
    const int64_t b = g * NT + threadIdx.x;
    const bool active = b < a.B;
    const int64_t bl = active ? b : a.B - 1;
    CrbaIO<T> io;
    io.q = {a.q + bl, a.ld};
    io.M = {a.M + bl, a.ld, active};
    io.lower = a.lower;
    crba_sample<T, Stash<T, NT>, KMAX>(M, io, st);
  }
}

template <class T> struct KinArgs {
  const T* q; const T* v;
  T* tr; T* com; T* ke; T* pe; T* mom; T* mrb; T* A; T* J;
  T* scratch;
  int64_t ld, B;
  const int* gate;       // non-NULL: run only if *gate != 0 (fallback behind the model-specialised kernel, see AbaArgs)
};

template <class T, int NT>
__global__ void __launch_bounds__(NT, sizeof(T) == 4 ? 28 : 12) kin_kernel(const __grid_constant__ ModelDev<T> M, const KinArgs<T> a,
                                                  const __grid_constant__ KinDev<T> K) {
  if (a.gate && *a.gate == 0) return;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* sh = reinterpret_cast<T*>(smem_raw);
  const Stash<T, NT> st{sh + threadIdx.x};
  const int64_t ngroups = (a.B + NT - 1) / NT;
  for (int64_t g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const int64_t gn = g + gridDim.x;
    if (gn < ngroups) {
      const int64_t bn = gn * NT + (threadIdx.x & ~31);
      prefetch_rows(a.q, M.nq, a.ld, bn);
      if (a.v) prefetch_rows(a.v, M.nv, a.ld, bn);
    }
    const int64_t b = g * NT + threadIdx.x;
    const bool active = b < a.B;
    const int64_t bl = active ? b : a.B - 1;
    KinIO<T> io;
    io.q = {a.q + bl, a.ld};
    io.v = {a.v ? a.v + bl : nullptr, a.ld};
    auto out = [&](T* p) { return ColOut<T>{p ? p + bl : nullptr, a.ld, active}; };
    io.tr = out(a.tr); io.com = out(a.com); io.ke = out(a.ke); io.pe = out(a.pe);
    io.mom = out(a.mom); io.mrb = out(a.mrb); io.A = out(a.A); io.J = out(a.J);
    io.poses = {a.scratch ? a.scratch + (int64_t)blockIdx.x * NT + threadIdx.x : nullptr, (int64_t)gridDim.x * NT};
    kin_sample<T>(M, K, io, st);
  }
}

template <class T> struct BodiesArgs {
  const T* q; const T* v; const T* vd; const T* wext;
  T* acc; T* jw;
  int64_t ld, B;
};
template <class T, int NT>
__global__ void __launch_bounds__(NT, sizeof(T) == 4 ? 16 : 8) bodies_kernel(const __grid_constant__ ModelDev<T> M, const BodiesArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const Stash<T, NT> st{reinterpret_cast<T*>(smem_raw) + threadIdx.x};
  const int64_t ngroups = (a.B + NT - 1) / NT;
  for (int64_t g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const int64_t b = g * NT + threadIdx.x;
    const bool active = b < a.B;
    const int64_t bl = active ? b : a.B - 1;
    BodiesIO<T> io;
    io.q = {a.q + bl, a.ld};
    io.v = {a.v + bl, a.ld};
    io.vd = {a.vd ? a.vd + bl : nullptr, a.ld};
    io.wext = {a.wext ? a.wext + bl : nullptr, a.ld};
    io.acc = a.acc ? a.acc + bl : nullptr;
    io.jw = a.jw ? a.jw + bl : nullptr;
    io.ld = a.ld;
    io.active = active;
    bodies_sample<T>(M, io, st);
  }
}

// Soft contact (contact_sample, rbd_kin.cuh): one thread per sample, stash = pending poses + twists.
template <class T> struct ContactArgs {
  const T *q, *v;
  T *s, *sd, *wr;
  int64_t ld, B;
};
template <class T, int NT>
__global__ void __launch_bounds__(NT, sizeof(T) == 4 ? 16 : 8)
contact_kernel(const __grid_constant__ ModelDev<T> M, const __grid_constant__ ContactDev<T> C, const ContactArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const Stash<T, NT> st{reinterpret_cast<T*>(smem_raw) + threadIdx.x};
  const int64_t ngroups = (a.B + NT - 1) / NT;
  for (int64_t g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const int64_t b = g * NT + threadIdx.x;
    const bool active = b < a.B;
    const int64_t bl = active ? b : a.B - 1;
    ContactIO<T> io;
    io.q = {a.q + bl, a.ld};
    io.v = {a.v + bl, a.ld};
    io.s = a.s ? a.s + bl : nullptr;
    io.sd = a.sd ? a.sd + bl : nullptr;
    io.wr = a.wr + bl;
    io.ld = a.ld;
    io.active = active;
    contact_sample<T>(M, C, io, st);
  }
}

constexpr int kNT = 32;   // threads per block: one warp; warps never synchronise with each other

// Launch `kernel` persistently with a stash of `rows` rows per thread in shared memory (plan_persistent).  `scratch_rows` > 0
// gives the kernel's `scratch` member a workspace of that many rows per resident thread (the external-wrench path).
template <class T, class Kern, class Args>
int launch(Kern kernel, const ModelDev<T>& M, Args a, int rows, cudaStream_t stream, T* Args::*scratch = nullptr, int scratch_rows = 0) {
  LaunchPlan pl;
  if (int rc = plan_persistent((const void*)kernel, kNT, (size_t)rows * kNT * sizeof(T), (a.B + kNT - 1) / kNT, stream, pl,
                               (size_t)scratch_rows * sizeof(T))) return rc;
  if (scratch) a.*scratch = (T*)pl.work.p;
  kernel<<<pl.grid, pl.block, pl.smem, stream>>>(M, a);
  return api_launched(&pl);
}

// The mixed CTA (see aba_kernel_mix) in place of the shared-memory kernel `ks`: one CTA of up to `nw` warps per SM, as many
// as the registers allow, `sw` of them with their stash in shared memory and the rest in an L2 scratch of at most 60 % of
// the L2.  `used` = false (nothing launched) when that does not put at least 15 % more warps on the SM than `ks` gets, when
// the batch has fewer groups of 32 than the CTAs have warps, or with RBD_JIT_VARIANT=1 (shared-memory kernels only).
template <class KS, class KM, class Dev, class Args>
int launch_mix(const rbd_model* model, KS ks, KM km, int nw, const Dev& M, Args a, size_t warp_bytes, int64_t ngroups,
               int scratch_rows, cudaStream_t stream, bool& used) {
  used = false;
  if (jit_variant() == 1) return RBD_OK;
  DeviceProps p;
  RBD_CUDA_TRY(device_props(p));
  int bps = 0, bps_mix = 0;
  if (int rc = kernel_config((const void*)ks, kNT, warp_bytes, p, bps)) return rc;
  cudaFuncAttributes fa{};
  RBD_CUDA_TRY(cudaFuncGetAttributes(&fa, km));
  const int fit = std::min(nw, 65536 / (((fa.numRegs + 7) / 8) * 8 * 32));
  const int sw = std::min<int>(fit, (int)((p.max_smem_optin - (int)fa.sharedSizeBytes) / warp_bytes));
  const int gw = (int)std::min<int64_t>(fit - sw, (int64_t)(0.6 * p.l2_bytes) / ((int64_t)p.sms * (int64_t)warp_bytes));
  const int total = sw + std::max(0, gw);
  if (sw < 1 || total * 100 < bps * 115 || ngroups < (int64_t)total * p.sms) return RBD_OK;
  const LaunchShape shape{p.sms, 32 * total, (int)(sw * warp_bytes), 1};
  if (int rc = kernel_config((const void*)km, shape.block, shape.smem, p, bps_mix)) return rc;
  QueueCtx ctx;      // zeroed work-queue counter, cached in the handle
  RBD_CUDA_TRY(queue_begin(const_cast<rbd_model*>(model), stream, ctx));
  a.counter = ctx.counter;
  a.sw = sw;
  StreamAlloc l2s, scratch;
  if (gw > 0) RBD_CUDA_TRY(l2s.alloc((size_t)gw * p.sms * warp_bytes, stream));
  a.l2 = static_cast<decltype(a.l2)>(l2s.p);
  if (scratch_rows > 0) {       // external wrenches in body frames: one column per resident thread
    a.scratch_ld = (int64_t)p.sms * total * 32;
    RBD_CUDA_TRY(scratch.alloc((size_t)scratch_rows * a.scratch_ld * sizeof(*a.scratch), stream));
    a.scratch = static_cast<decltype(a.scratch)>(scratch.p);
  }
  km<<<shape.grid, shape.block, shape.smem, stream>>>(M, a);
  if (int rc = api_launched(&shape)) return rc;
  used = true;
  return RBD_OK;
}

template <class T>
int dynamics_t(const rbd_model* model, int64_t B, int64_t ld, const void* q, const void* v, const void* tau,
               const void* wext, void* vd, void* qd, cudaStream_t stream) {
  const HostModel& hm = model->hm;
  const ModelDev<T>& M = dev_model<T>(hm);
  AbaArgs<T> a{(const T*)q, (const T*)v, (const T*)tau, (const T*)wext, (T*)vd, (T*)qd, nullptr, ld, B};
  const int rows = M.nrows;
  const int sr = wext ? 6 * hm.nb : 0;
  bool other_kinds = false;          // prismatic / fixed joints anywhere -> kernels with those code paths
  for (int i = 0; i < hm.nb; ++i) other_kinds |= (M.body[i].kind == K_PRIS || M.body[i].kind == K_FIXED);
#define RBD_ABA(G, E, K) launch<T>(aba_kernel<T, kNT, G, E, K>, M, a, rows, stream, &AbaArgs<T>::scratch, sr)
  if (!wext) {      // model-specialised kernels (rbd_spec.cpp): straight-line code generated for this mechanism
    SpecKey key; key.algo = SPEC_ABA; key.f64 = sizeof(T) == 8; key.has_in2 = tau != nullptr; key.has_out1 = qd != nullptr;
    bool used = false;
    const int* gate = nullptr;
    if (int rc = spec_try_launch(const_cast<rbd_model*>(model), key, {q, v, tau, vd, qd, ld, B}, stream, used, &gate)) return rc;
    if (used) {
      if (!gate) return RBD_OK;
      // fp32: the specialised program has no slow sin / cos path; if any sample met an angle beyond 1e4 rad (flag raised on the
      // device) this generic launch redoes the batch with the library path, otherwise it exits at once
      const KeepLaunchRecord keep;
      a.gate = gate;
      return hm.general ? RBD_ABA(true, false, kAllKinds) : (other_kinds ? RBD_ABA(false, false, kAllKinds) : RBD_ABA(false, false, 0));
    }
  }
  if (!wext && !hm.general && !other_kinds && rows <= 256) {   // all-revolute trees (floating root allowed): the mixed CTA, see launch_mix
    bool used = false;
    a.rows = rows;
    const int rc = launch_mix(model, aba_kernel<T, kNT, false, false, 0>, aba_kernel_mix<T, 0>, kMixWarps<T>, M, a,
                              (size_t)rows * kNT * sizeof(T), (B + kNT - 1) / kNT, 0, stream, used);
    if (rc) return rc;
    if (used) return RBD_OK;
  }
  if (hm.general) return wext ? RBD_ABA(true, true, kAllKinds) : RBD_ABA(true, false, kAllKinds);
  if (other_kinds) return wext ? RBD_ABA(false, true, kAllKinds) : RBD_ABA(false, false, kAllKinds);
  return wext ? RBD_ABA(false, true, 0) : RBD_ABA(false, false, 0);
#undef RBD_ABA
}

template <class T>
int inverse_dynamics_t(const rbd_model* model, int64_t B, int64_t ld, const void* q, const void* v, const void* vd,
                       const void* wext, void* tau, cudaStream_t stream) {
  const HostModel& hm = model->hm;
  const ModelDev<T>& M = dev_model<T>(hm);
  RneaArgs<T> a{(const T*)q, (const T*)v, (const T*)vd, (const T*)wext, (T*)tau, nullptr, ld, B};
  const int rows = rnea_rows(hm);
  if (!wext) {
    SpecKey key; key.algo = SPEC_RNEA; key.f64 = sizeof(T) == 8; key.has_in2 = vd != nullptr;
    bool used = false;
    const int* gate = nullptr;
    if (int rc = spec_try_launch(const_cast<rbd_model*>(model), key, {q, v, vd, tau, nullptr, ld, B}, stream, used, &gate)) return rc;
    if (used) {
      if (!gate) return RBD_OK;
      const KeepLaunchRecord keep;      // gated generic fallback, see dynamics_t
      a.gate = gate;
      return launch<T>(rnea_kernel<T, kNT, false>, M, a, rows, stream);
    }
  }
  if (rows <= 256) {             // the mixed CTA, see launch_mix
    bool used = false;
    a.rows = rows;
    const int64_t ng = (B + kNT - 1) / kNT;
    const int rc = wext ? launch_mix(model, rnea_kernel<T, kNT, true>, rnea_kernel_mix<T, true>, kMixWarps<T>, M, a,
                                     (size_t)rows * kNT * sizeof(T), ng, 6 * hm.nb, stream, used)
                        : launch_mix(model, rnea_kernel<T, kNT, false>, rnea_kernel_mix<T, false>, kMixWarps<T>, M, a,
                                     (size_t)rows * kNT * sizeof(T), ng, 0, stream, used);
    if (rc) return rc;
    if (used) return RBD_OK;
  }
  return wext ? launch<T>(rnea_kernel<T, kNT, true>, M, a, rows, stream, &RneaArgs<T>::scratch, 6 * hm.nb)
              : launch<T>(rnea_kernel<T, kNT, false>, M, a, rows, stream);
}

template <class T>
int mass_matrix_t(const rbd_model* model, int64_t B, int64_t ld, const void* q, void* Mout, cudaStream_t stream, bool lower = false) {
  const HostModel& hm = model->hm;
  const ModelDev<T>& M = dev_model<T>(hm);
  CrbaArgs<T> a{(const T*)q, (T*)Mout, ld, B, lower, nullptr};
  const int rows = std::max(1, crba_rows(hm));
  bool multi = false;
  for (int i = 0; i < hm.nb; ++i) multi |= kind_nv(M.body[i].kind) > 1;
  {      // model-specialised kernel: the composite-rigid-body algorithm traced on this mechanism (rbd_codegen.cpp)
    SpecKey key; key.algo = SPEC_CRBA; key.f64 = sizeof(T) == 8; key.has_in2 = false; key.lower = lower;
    bool used = false;
    const int* gate = nullptr;
    if (int rc = spec_try_launch(const_cast<rbd_model*>(model), key, {q, nullptr, nullptr, Mout, nullptr, ld, B}, stream, used, &gate))
      return rc;
    if (used) {
      if (!gate) return RBD_OK;
      const KeepLaunchRecord keep;      // gated generic fallback, see dynamics_t
      a.gate = gate;
      return multi ? launch<T>(crba_kernel<T, kNT, 6>, M, a, rows, stream) : launch<T>(crba_kernel<T, kNT, 1>, M, a, rows, stream);
    }
  }
  return multi ? launch<T>(crba_kernel<T, kNT, 6>, M, a, rows, stream) : launch<T>(crba_kernel<T, kNT, 1>, M, a, rows, stream);
}

// Kinematics by-products (SURVEY 8(f) rank 2).  One launch; the momentum matrix additionally parks the 12 nb pose rows of
// every resident thread in a stream-ordered scratch between its outward and inward sweeps.
template <class T>
int kinematics_t(const rbd_model* model, int64_t B, int64_t ld, const void* q, const void* v, const int8_t* path_sign,
                 const rbd_kinematics_out& o, cudaStream_t stream) {
  const HostModel& hm = model->hm;
  const ModelDev<T>& M = dev_model<T>(hm);
  KinDev<T> K;
  std::memset(&K, 0, sizeof(K));
  for (int p = 0; p < hm.nb; ++p) {
    for (int k = 0; k < 9; ++k) K.At[p][k] = (T)hm.alignT[9 * p + k];
    K.sign[p] = path_sign ? path_sign[hm.order[p]] : 0;
  }
  K.inv_mass = (T)(1.0 / hm.total_mass);
  KinArgs<T> a{(const T*)q, (const T*)v, (T*)o.transforms_to_root, (T*)o.center_of_mass, (T*)o.kinetic_energy,
               (T*)o.gravitational_potential_energy, (T*)o.momentum, (T*)o.momentum_rate_bias, (T*)o.momentum_matrix,
               (T*)o.geometric_jacobian, nullptr, ld, B, nullptr};
  std::optional<KeepLaunchRecord> keep;
  {                              // model-specialised kernel for this output subset (and this jacobian path)
    SpecKey key;
    key.algo = SPEC_KIN; key.f64 = sizeof(T) == 8; key.has_in2 = v != nullptr;
    void* const outs[8] = {o.transforms_to_root, o.center_of_mass, o.kinetic_energy, o.gravitational_potential_energy, o.momentum,
                           o.momentum_rate_bias, o.momentum_matrix, o.geometric_jacobian};
    SpecLaunchArgs sa{q, v, nullptr, nullptr, nullptr, ld, B};
    for (int k = 0; k < 8; ++k) { if (outs[k]) key.kin_mask |= 1 << k; sa.ko[k] = outs[k]; }
    for (int i = 0; i < hm.nb; ++i) key.kin_sign[i] = K.sign[i];
    bool used = false;
    const int* gate = nullptr;
    if (key.kin_mask)
      if (int rc = spec_try_launch(const_cast<rbd_model*>(model), key, sa, stream, used, &gate)) return rc;
    if (used) {
      if (!gate) return RBD_OK;
      keep.emplace();
      a.gate = gate;               // gated generic fallback (angles beyond the fast sin / cos range), see dynamics_t
    }
  }
  auto kernel = kin_kernel<T, kNT>;
  LaunchPlan pl;
  if (int rc = plan_persistent((const void*)kernel, kNT, (size_t)std::max(1, kin_rows(hm)) * kNT * sizeof(T), (B + kNT - 1) / kNT,
                               stream, pl, o.momentum_matrix ? (size_t)12 * hm.nb * sizeof(T) : 0)) return rc;
  a.scratch = (T*)pl.work.p;
  kernel<<<pl.grid, pl.block, pl.smem, stream>>>(M, a, K);
  return api_launched(&pl);
}

// dynamics! on Dual{Float64,6} arrays (config 4).  The Dual model (constants with zero partials, 25 KB) is built per call
// from the fp64 one; this path is not the hot one.
int dynamics_dual(const rbd_model* model, int64_t B, int64_t ld, const void* q, const void* v, const void* tau, void* vd,
                  cudaStream_t stream) {
  const HostModel& hm = model->hm;
  const ModelDev<double>& S = hm.dev64;
  std::unique_ptr<ModelDev<Dual64>> Mp(new ModelDev<Dual64>());
  Mp->nb = S.nb; Mp->nq = S.nq; Mp->nv = S.nv; Mp->nrows = S.nrows; Mp->slot_base = S.slot_base; Mp->nslots = S.nslots;
  for (int k = 0; k < 3; ++k) Mp->g[k] = Dual64(S.g[k]);
  for (int i = 0; i < S.nb; ++i) {
    const BodyDev<double>& s = S.body[i];
    BodyDev<Dual64>& d = Mp->body[i];
    for (int k = 0; k < 9; ++k) d.Rt[k] = Dual64(s.Rt[k]);
    for (int k = 0; k < 3; ++k) { d.pt[k] = Dual64(s.pt[k]); d.h[k] = Dual64(s.h[k]); }
    for (int k = 0; k < 6; ++k) d.J[k] = Dual64(s.J[k]);
    d.m = Dual64(s.m);
    d.qoff = Dual64(s.qoff);
    d.kind = s.kind; d.parent = s.parent; d.qrow = s.qrow; d.vrow = s.vrow; d.row0 = s.row0;
    d.oslot = s.oslot; d.pslot = s.pslot; d.flags = s.flags; d.refidx = s.refidx;
  }
  DualArgs a{(const double*)q, (const double*)v, (const double*)tau, (double*)vd, ld, B};
  const int64_t ngroups = (B * 6 + kNT - 1) / kNT;      // one thread per (sample, partial direction)
  if (!hm.general && S.nrows <= 256) {      // the mixed CTA, see launch_mix
    bool used = false;
    a.rows = S.nrows;
    if (int rc = launch_mix(model, aba_dual_kernel<kNT, false>, aba_dual_kernel_mix, kMixWarps<double>, *Mp, a,
                            (size_t)S.nrows * kNT * sizeof(Dual64), ngroups, 0, stream, used)) return rc;
    if (used) return RBD_OK;
  }
  const auto kernel = hm.general ? aba_dual_kernel<kNT, true> : aba_dual_kernel<kNT, false>;
  LaunchPlan pl;
  if (int rc = plan_persistent((const void*)kernel, kNT, (size_t)S.nrows * kNT * sizeof(Dual64), ngroups, stream, pl)) return rc;
  kernel<<<pl.grid, pl.block, pl.smem, stream>>>(*Mp, a);
  return api_launched(&pl);
}

// ---- Munthe-Kaas RK4 (rbd_integrate): elementwise stage kernels around the dynamics kernels -----------------------------
// Stage i of a step, one thread per (sample, joint) -- every joint's coordinate map is independent of the others (blockIdx.y =
// body).  The local coordinates of the stage and the stage velocity are functions of the previous stage's rates,
//   phi = dt a_i phid_{i-1} ,  v_s = v0 + dt a_i vd_{i-1} ,
// evaluated on the fly by the two accessors below (nothing but the kernel's real outputs is written):
//   q_s = global(q0, phi) ,  v_s  -> inputs of the dynamics kernels ;  phid_i = d/dt local(q0, q_s, v_s) -> kept for the next stage
// and for the final combination.  The four (phid_i, vd_i) pairs are stored separately; the finishing kernel forms the weighted sums.
template <class T> struct ScaledRow {      // wa * p[row]  (zero when there is no previous stage)
  const T* p; int64_t ld; T wa;
  RBD_HD T operator()(int row) const { return p ? wa * p[(int64_t)row * ld] : T(0); }
};
template <class T> struct OffsetRow {      // base[row] + wa * p[row]
  const T* base; const T* p; int64_t ld; T wa;
  RBD_HD T operator()(int row) const {
    const T b = base[(int64_t)row * ld];
    return p ? b + wa * p[(int64_t)row * ld] : b;
  }
};
template <class T> struct StageArgs {
  const T* q0; const T* v0;               // state at the start of the step
  const T* phid_prev; const T* vd_prev;   // rates of the previous stage (NULL for stage 0)
  T* phid; T* qs; T* vs;                  // outputs
  T wa;                                   // dt * a_i
  int64_t B;
  bool skip_linear;                       // revolute / prismatic joints are done by the vectorised kernel below
};
template <class T>
__global__ void __launch_bounds__(128) integrate_stage_kernel(const __grid_constant__ ModelDev<T> M, const StageArgs<T> a) {
  const BodyDev<T>& bd = M.body[blockIdx.y];
  const int k0 = bd.vrow, k1 = bd.vrow + kind_nv_dev(bd.kind);
  if (k1 == k0) return;                                    // fixed joint: no coordinates
  if (a.skip_linear && (bd.kind == K_REV || bd.kind == K_PRIS)) return;
  for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < a.B; b += (int64_t)gridDim.x * blockDim.x) {
    const Col<T> q0{a.q0 + b, a.B};
    const ScaledRow<T> phi{a.phid_prev ? a.phid_prev + b : nullptr, a.B, a.wa};
    const OffsetRow<T> vs{a.v0 + b, a.vd_prev ? a.vd_prev + b : nullptr, a.B, a.wa};
    for (int k = k0; k < k1; ++k) a.vs[(int64_t)k * a.B + b] = vs(k);
    const ColOut<T> qs{a.qs + b, a.B, true}, phid{a.phid + b, a.B, true};
    joint_stage(bd, q0, phi, vs, qs, phid);
  }
}
// Revolute / prismatic joints (the bulk of a robot): q_s = q0 + wa phid_prev, v_s = v0 + wa vd_prev, phid = v_s -- plain row
// arithmetic, done VEC samples per thread with 16-byte accesses so that enough loads are in flight to approach the HBM rate (the
// per-(sample, joint) kernel above is latency-bound: too few loads in flight per thread).
template <class T> __device__ __forceinline__ void vec_axpy(const typename VecOf<T>::type& a, T w, const typename VecOf<T>::type& x,
                                                            typename VecOf<T>::type& o);
template <> __device__ __forceinline__ void vec_axpy<float>(const float4& a, float w, const float4& x, float4& o) {
  o.x = a.x + w * x.x; o.y = a.y + w * x.y; o.z = a.z + w * x.z; o.w = a.w + w * x.w;
}
template <> __device__ __forceinline__ void vec_axpy<double>(const double2& a, double w, const double2& x, double2& o) {
  o.x = a.x + w * x.x; o.y = a.y + w * x.y;
}
template <class T> __device__ __forceinline__ typename VecOf<T>::type vec_comb4(const typename VecOf<T>::type& base, T dt, const T* w,
                                                                                const typename VecOf<T>::type* x);
template <> __device__ __forceinline__ float4 vec_comb4<float>(const float4& b, float dt, const float* w, const float4* x) {
  float4 o;
  o.x = b.x + dt * (w[0] * x[0].x + w[1] * x[1].x + w[2] * x[2].x + w[3] * x[3].x);
  o.y = b.y + dt * (w[0] * x[0].y + w[1] * x[1].y + w[2] * x[2].y + w[3] * x[3].y);
  o.z = b.z + dt * (w[0] * x[0].z + w[1] * x[1].z + w[2] * x[2].z + w[3] * x[3].z);
  o.w = b.w + dt * (w[0] * x[0].w + w[1] * x[1].w + w[2] * x[2].w + w[3] * x[3].w);
  return o;
}
template <> __device__ __forceinline__ double2 vec_comb4<double>(const double2& b, double dt, const double* w, const double2* x) {
  double2 o;
  o.x = b.x + dt * (w[0] * x[0].x + w[1] * x[1].x + w[2] * x[2].x + w[3] * x[3].x);
  o.y = b.y + dt * (w[0] * x[0].y + w[1] * x[1].y + w[2] * x[2].y + w[3] * x[3].y);
  return o;
}

template <class T>
__global__ void __launch_bounds__(256) integrate_stage_linear_kernel(const __grid_constant__ ModelDev<T> M, const StageArgs<T> a) {
  using V = typename VecOf<T>::type;
  constexpr int N = VecOf<T>::N;
  const BodyDev<T>& bd = M.body[blockIdx.y];
  if (bd.kind != K_REV && bd.kind != K_PRIS) return;
  const int64_t qo = (int64_t)bd.qrow * a.B, vo = (int64_t)bd.vrow * a.B, nvec = a.B / N;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    const V q0 = reinterpret_cast<const V*>(a.q0 + qo)[i];
    const V v0 = reinterpret_cast<const V*>(a.v0 + vo)[i];
    V qs = q0, vs = v0;
    if (a.phid_prev) {
      const V pp = reinterpret_cast<const V*>(a.phid_prev + vo)[i];
      const V vp = reinterpret_cast<const V*>(a.vd_prev + vo)[i];
      vec_axpy<T>(q0, a.wa, pp, qs);
      vec_axpy<T>(v0, a.wa, vp, vs);
    }
    reinterpret_cast<V*>(a.qs + qo)[i] = qs;
    reinterpret_cast<V*>(a.vs + vo)[i] = vs;
    reinterpret_cast<V*>(a.phid + vo)[i] = vs;
  }
}
// v = v0 + dt sum_i b_i vd_i ,  q = global(q0, dt sum_i b_i phid_i)        (ode_integrators.jl:283-296)
template <class T> struct SumRow4 {        // [base[row] +] dt * sum_i w_i p_i[row]
  const T* base; const T* p[4]; int64_t ld; T w[4]; T dt;
  RBD_HD T operator()(int row) const {
    const int64_t e = (int64_t)row * ld;
    const T s = dt * (w[0] * p[0][e] + w[1] * p[1][e] + w[2] * p[2][e] + w[3] * p[3][e]);
    return base ? base[e] + s : s;
  }
};
template <class T> struct FinishArgs {
  const T* q0; const T* v0;
  const T* phid[4]; const T* vd[4];
  T* q; T* v;                              // user arrays (leading dimension ld)
  T w[4]; T dt;
  int64_t B, ld;
  bool refresh;                            // also write the new state into (q0, v0) for the next step (each thread owns its joint's rows)
  bool skip_linear;                        // revolute / prismatic joints are done by integrate_finish_linear_kernel
};
// finishing step of the revolute / prismatic rows, vectorised like integrate_stage_linear_kernel
template <class T>
__global__ void __launch_bounds__(256) integrate_finish_linear_kernel(const __grid_constant__ ModelDev<T> M, const FinishArgs<T> a) {
  using V = typename VecOf<T>::type;
  constexpr int N = VecOf<T>::N;
  const BodyDev<T>& bd = M.body[blockIdx.y];
  if (bd.kind != K_REV && bd.kind != K_PRIS) return;
  const int64_t qo = (int64_t)bd.qrow * a.B, vo = (int64_t)bd.vrow * a.B, nvec = a.B / N;
  V* qu = reinterpret_cast<V*>(a.q + (int64_t)bd.qrow * a.ld);
  V* vu = reinterpret_cast<V*>(a.v + (int64_t)bd.vrow * a.ld);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    V ph[4], vd[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) { ph[k] = reinterpret_cast<const V*>(a.phid[k] + vo)[i]; vd[k] = reinterpret_cast<const V*>(a.vd[k] + vo)[i]; }
    const V qn = vec_comb4<T>(reinterpret_cast<const V*>(a.q0 + qo)[i], a.dt, a.w, ph);
    const V vn = vec_comb4<T>(reinterpret_cast<const V*>(a.v0 + vo)[i], a.dt, a.w, vd);
    qu[i] = qn; vu[i] = vn;
    if (a.refresh) {
      reinterpret_cast<V*>(const_cast<T*>(a.q0) + qo)[i] = qn;
      reinterpret_cast<V*>(const_cast<T*>(a.v0) + vo)[i] = vn;
    }
  }
}
template <class T>
__global__ void __launch_bounds__(128) integrate_finish_kernel(const __grid_constant__ ModelDev<T> M, const FinishArgs<T> a) {
  const BodyDev<T>& bd = M.body[blockIdx.y];
  const int k0 = bd.vrow, k1 = bd.vrow + kind_nv_dev(bd.kind);
  if (k1 == k0) return;
  if (a.skip_linear && (bd.kind == K_REV || bd.kind == K_PRIS)) return;
  for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < a.B; b += (int64_t)gridDim.x * blockDim.x) {
    const Col<T> q0{a.q0 + b, a.B};
    const SumRow4<T> phi{nullptr, {a.phid[0] + b, a.phid[1] + b, a.phid[2] + b, a.phid[3] + b}, a.B, {a.w[0], a.w[1], a.w[2], a.w[3]}, a.dt};
    const SumRow4<T> vn{a.v0 + b, {a.vd[0] + b, a.vd[1] + b, a.vd[2] + b, a.vd[3] + b}, a.B, {a.w[0], a.w[1], a.w[2], a.w[3]}, a.dt};
    T vnew[6];
    for (int k = k0; k < k1; ++k) { vnew[k - k0] = vn(k); a.v[(int64_t)k * a.ld + b] = vnew[k - k0]; }
    const ColOut<T> q{a.q + b, a.ld, true}, dump{nullptr, a.B, false};
    joint_stage(bd, q0, phi, vn, q, dump);
    if (a.refresh) {                       // after every read of this joint's (q0, v0) rows above
      const int nqj = kind_nq_dev(bd.kind);
      for (int k = 0; k < nqj; ++k) const_cast<T*>(a.q0)[(int64_t)(bd.qrow + k) * a.B + b] = a.q[(int64_t)(bd.qrow + k) * a.ld + b];
      for (int k = k0; k < k1; ++k) const_cast<T*>(a.v0)[(int64_t)k * a.B + b] = vnew[k - k0];
    }
  }
}

// traj_q / traj_v (rbd_integrate_trajectory): [(nsteps + 1) x rows x B] -- block 0 the initial state, block s + 1 written by the
// finishing kernels of step s; q / v receive the final state as without them.  stages (rbd_integrate_vjp's recompute, nsteps = 1):
// the four stages' (qs_i, vs_i, φ̇_i, v̇_i) are kept in [4 nq + 12 nv] x B rows (stage_rows) and the finishing step is skipped.
template <class T>
int integrate_t(const rbd_model* model, int64_t B, int64_t ld, void* q, void* v, const void* tau, int64_t step_stride,
                int64_t stage_stride, double dt, int nsteps, cudaStream_t stream, T* traj_q = nullptr, T* traj_v = nullptr,
                T* stages = nullptr) {
  const HostModel& hm = model->hm;
  const ModelDev<T>& M = dev_model<T>(hm);
  DeviceProps p;
  RBD_CUDA_TRY(device_props(p));
  const size_t nq = hm.nq, nv = hm.nv;
  const size_t rows = 2 * nq + 10 * nv + (tau && ld != B ? nv : 0);
  StreamAlloc work;
  RBD_CUDA_TRY(work.alloc(rows * (size_t)B * sizeof(T), stream));
  T* q0 = (T*)work.p; T* qs = q0 + nq * B; T* v0 = qs + nq * B; T* vs = v0 + nv * B;
  T* phid[4]; T* vd[4];
  for (int i = 0; i < 4; ++i) { phid[i] = vs + (size_t)(1 + i) * nv * B; vd[i] = vs + (size_t)(5 + i) * nv * B; }
  T* taud = vs + (size_t)9 * nv * B;
  T* qsi[4] = {qs, qs, qs, qs};
  T* vsi[4] = {vs, vs, vs, vs};
  if (stages)
    for (int i = 0; i < 4; ++i) {
      qsi[i] = stages + (size_t)i * nq * B; vsi[i] = stages + (4 * nq + (size_t)i * nv) * B;
      phid[i] = stages + (4 * nq + (4 + (size_t)i) * nv) * B; vd[i] = stages + (4 * nq + (8 + (size_t)i) * nv) * B;
    }
  T* qout = traj_q ? traj_q : (T*)q;       // the finishing kernels' target (block s + 1 of a trajectory)
  T* vout = traj_v ? traj_v : (T*)v;
  const int64_t ldo = traj_q ? B : ld;
  // torques of (step s, stage i): tau + s * step_stride + i * stage_stride (both 0: one array held over the whole call); the
  // dynamics kernels want leading dimension B, so arrays with ld != B are densified per use
  const bool varying = step_stride != 0 || stage_stride != 0;
  auto tau_at = [&](int s_, int i_) -> const T* { return tau ? (const T*)tau + (size_t)s_ * step_stride + (size_t)i_ * stage_stride : nullptr; };
  const T* tau_dense = (const T*)tau;
  if (tau && ld != B && !varying) {
    RBD_CUDA_TRY(cudaMemcpy2DAsync(taud, B * sizeof(T), tau, ld * sizeof(T), B * sizeof(T), nv, cudaMemcpyDeviceToDevice, stream));
    tau_dense = taud;
  }
  const int grid = (int)std::min<int64_t>((B + 127) / 128, (int64_t)p.sms * 8);
  // the vectorised kernel needs whole vectors per row (workspace rows are B long and 256-byte aligned)
  const bool vec_ok = B % VecOf<T>::N == 0 && B >= 1024;
  const int grid_lin = (int)std::min<int64_t>((B / VecOf<T>::N + 255) / 256, (int64_t)p.sms * 4);
  // ... and, for the finishing kernel, vector-aligned rows of the caller's arrays too
  const bool vec_user = vec_ok && ldo % VecOf<T>::N == 0 && ((uintptr_t)qout % sizeof(typename VecOf<T>::type)) == 0 &&
                        ((uintptr_t)vout % sizeof(typename VecOf<T>::type)) == 0;
  bool has_other = false;
  for (int i = 0; i < hm.nb; ++i) has_other |= (M.body[i].kind != K_REV && M.body[i].kind != K_PRIS && M.body[i].kind != K_FIXED);
  const double a[4] = {0.0, 0.5, 0.5, 1.0}, bw[4] = {1.0 / 6, 1.0 / 3, 1.0 / 3, 1.0 / 6};   // runge_kutta_4, ode_integrators.jl:48-55
  // (q0, v0): dense copies of the state at the start of the step; the finishing kernel of step s refreshes them for step s + 1
  RBD_CUDA_TRY(cudaMemcpy2DAsync(q0, B * sizeof(T), q, ld * sizeof(T), B * sizeof(T), nq, cudaMemcpyDeviceToDevice, stream));
  RBD_CUDA_TRY(cudaMemcpy2DAsync(v0, B * sizeof(T), v, ld * sizeof(T), B * sizeof(T), nv, cudaMemcpyDeviceToDevice, stream));
  if (traj_q) {
    RBD_CUDA_TRY(cudaMemcpyAsync(traj_q, q0, nq * B * sizeof(T), cudaMemcpyDeviceToDevice, stream));
    RBD_CUDA_TRY(cudaMemcpyAsync(traj_v, v0, nv * B * sizeof(T), cudaMemcpyDeviceToDevice, stream));
  }
  for (int s = 0; s < nsteps; ++s) {
    for (int i = 0; i < 4; ++i) {
      if (varying) {
        tau_dense = tau_at(s, i);
        if (tau && ld != B) {
          RBD_CUDA_TRY(cudaMemcpy2DAsync(taud, B * sizeof(T), tau_dense, ld * sizeof(T), B * sizeof(T), nv, cudaMemcpyDeviceToDevice, stream));
          tau_dense = taud;
        }
      }
      StageArgs<T> sa{q0, v0, i ? phid[i - 1] : nullptr, i ? vd[i - 1] : nullptr, phid[i], qsi[i], vsi[i], (T)(dt * a[i]), B, vec_ok};
      if (vec_ok) {        // revolute / prismatic rows, VEC samples per thread
        integrate_stage_linear_kernel<T><<<dim3(grid_lin, hm.nb), 256, 0, stream>>>(M, sa);
        if (int rc = api_launched()) return rc;
      }
      if (!vec_ok || has_other) {
        integrate_stage_kernel<T><<<dim3(grid, hm.nb), 128, 0, stream>>>(M, sa);
        if (int rc = api_launched()) return rc;
      }
      if (int rc = dynamics_t<T>(model, B, B, qsi[i], vsi[i], tau_dense, nullptr, vd[i], nullptr, stream)) return rc;
    }
    if (stages) return RBD_OK;
    T* qo = traj_q ? traj_q + (size_t)(s + 1) * nq * B : (T*)q;
    T* vo = traj_v ? traj_v + (size_t)(s + 1) * nv * B : (T*)v;
    FinishArgs<T> fa{q0, v0, {phid[0], phid[1], phid[2], phid[3]}, {vd[0], vd[1], vd[2], vd[3]}, qo, vo,
                     {(T)bw[0], (T)bw[1], (T)bw[2], (T)bw[3]}, (T)dt, B, ldo, s + 1 < nsteps, vec_user};
    if (vec_user) {
      integrate_finish_linear_kernel<T><<<dim3(grid_lin, hm.nb), 256, 0, stream>>>(M, fa);
      if (int rc = api_launched()) return rc;
    }
    if (!vec_user || has_other) {
      integrate_finish_kernel<T><<<dim3(grid, hm.nb), 128, 0, stream>>>(M, fa);
      if (int rc = api_launched()) return rc;
    }
  }
  if (traj_q && nsteps > 0) {      // the final state into the caller's q / v, as rbd_integrate leaves it
    RBD_CUDA_TRY(cudaMemcpy2DAsync(q, ld * sizeof(T), traj_q + (size_t)nsteps * nq * B, B * sizeof(T), B * sizeof(T), nq,
                                   cudaMemcpyDeviceToDevice, stream));
    RBD_CUDA_TRY(cudaMemcpy2DAsync(v, ld * sizeof(T), traj_v + (size_t)nsteps * nv * B, B * sizeof(T), B * sizeof(T), nv,
                                   cudaMemcpyDeviceToDevice, stream));
  }
  return RBD_OK;
}

// rbd_dynamics_gather.  Fast path: the model-specialised kernels store v̇ straight into every GPU's gathered array (peer-mapped
// memory, posted writes over NVLink) -- the output store IS the gather.  Fallback (no specialised kernel for this model / dtype,
// or -- gated on their flag -- a sample beyond their fast sin / cos range): the generic kernels evaluate into a dense scratch
// and this kernel scatters it to the peers.
template <class T> struct ScatterArgs {
  const T* src; int64_t src_ld;
  T* dst[8]; int64_t dst_ld;
  int ndst, rows;
  int64_t B;
  const int* gate;
};
template <class T> __global__ void __launch_bounds__(256) gather_scatter_kernel(const ScatterArgs<T> a) {
  if (a.gate && *a.gate == 0) return;
  const int64_t total = (int64_t)a.rows * a.B;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = e / a.B, b = e - k * a.B;
    const T x = a.src[k * a.src_ld + b];
#pragma unroll
    for (int p = 0; p < 8; ++p)
      if (p < a.ndst) a.dst[p][k * a.dst_ld + b] = x;
  }
}

template <class T>
int dynamics_gather_t(const rbd_model* model, int64_t B, int64_t ld, const void* q, const void* v, const void* tau, int npeers,
                      void* const* peers, void* mc, int64_t peer_ld, int64_t col0, cudaStream_t stream) {
  const HostModel& hm = model->hm;
  const ModelDev<T>& M = dev_model<T>(hm);
  const int* gate = nullptr;
  bool used = false;
  {
    SpecKey key; key.algo = SPEC_ABA; key.f64 = sizeof(T) == 8; key.has_in2 = tau != nullptr; key.peers = true;
    SpecLaunchArgs sa{q, v, tau, nullptr, nullptr, ld, B};
    sa.peers = peers; sa.npeers = npeers; sa.peer_ld = peer_ld; sa.peer_col0 = col0; sa.mc = mc;
    if (int rc = spec_try_launch(const_cast<rbd_model*>(model), key, sa, stream, used, &gate)) return rc;
    if (used && !gate) return RBD_OK;
  }
  // the generic kernels use ONE leading dimension for inputs and outputs, so the scratch is [nv x ld]
  StreamAlloc scratch_;
  RBD_CUDA_TRY(scratch_.alloc((size_t)hm.nv * (size_t)ld * sizeof(T), stream));
  T* scratch = (T*)scratch_.p;
  std::optional<KeepLaunchRecord> keep;      // behind the specialised kernel: gated generic fallback, see dynamics_t
  if (!used) {
    if (int rc = dynamics_t<T>(model, B, ld, q, v, tau, nullptr, scratch, nullptr, stream)) return rc;
  } else {
    keep.emplace();
    AbaArgs<T> a{(const T*)q, (const T*)v, (const T*)tau, nullptr, scratch, nullptr, nullptr, ld, B};
    a.gate = gate;
    bool other_kinds = false;
    for (int i = 0; i < hm.nb; ++i) other_kinds |= (M.body[i].kind == K_PRIS || M.body[i].kind == K_FIXED);
    const int rows = M.nrows;
#define RBD_ABA_G(G, K) launch<T>(aba_kernel<T, kNT, G, false, K>, M, a, rows, stream)
    if (int rc = hm.general ? RBD_ABA_G(true, kAllKinds) : (other_kinds ? RBD_ABA_G(false, kAllKinds) : RBD_ABA_G(false, 0))) return rc;
#undef RBD_ABA_G
  }
  ScatterArgs<T> sc{};
  sc.src = scratch; sc.src_ld = ld; sc.dst_ld = peer_ld; sc.ndst = npeers; sc.rows = hm.nv; sc.B = B; sc.gate = gate;
  for (int p = 0; p < npeers; ++p) sc.dst[p] = (T*)peers[p] + col0;
  DeviceProps p;
  RBD_CUDA_TRY(device_props(p));
  gather_scatter_kernel<T><<<p.sms * 8, 256, 0, stream>>>(sc);
  return api_launched();
}

template <class T>
int bodies_t(const rbd_model* model, int64_t B, int64_t ld, const void* q, const void* v, const void* vd, const void* wext, void* acc,
             void* jw, cudaStream_t stream) {
  const HostModel& hm = model->hm;
  const ModelDev<T>& M = dev_model<T>(hm);
  BodiesArgs<T> a{(const T*)q, (const T*)v, (const T*)vd, (const T*)wext, (T*)acc, (T*)jw, ld, B};
  auto kernel = bodies_kernel<T, kNT>;
  LaunchPlan pl;
  if (int rc = plan_persistent((const void*)kernel, kNT, (size_t)std::max(1, kin_rows(hm)) * kNT * sizeof(T), (B + kNT - 1) / kNT,
                               stream, pl)) return rc;
  kernel<<<pl.grid, pl.block, pl.smem, stream>>>(M, a);
  return api_launched(&pl);
}

template <class T>
int contact_t(const rbd_model* model, int64_t B, int64_t ld, const void* q, const void* v, const rbd_contact_desc& cd, void* sx,
              void* sd, void* wr, cudaStream_t stream) {
  const HostModel& hm = model->hm;
  const ModelDev<T>& M = dev_model<T>(hm);
  ContactDev<T> C;
  build_contact_dev<T>(hm.nb, hm.pos.data(), hm.alignT.data(), cd, C);
  ContactArgs<T> a{(const T*)q, (const T*)v, (T*)sx, (T*)sd, (T*)wr, ld, B};
  auto kernel = contact_kernel<T, kNT>;
  LaunchPlan pl;
  if (int rc = plan_persistent((const void*)kernel, kNT, (size_t)std::max(1, kin_rows(hm)) * kNT * sizeof(T), (B + kNT - 1) / kNT,
                               stream, pl)) return rc;
  kernel<<<pl.grid, pl.block, pl.smem, stream>>>(M, C, a);
  return api_launched(&pl);
}

int check_common(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, bool allow_dual = false) {
  if (!model) return fail(RBD_EINVAL, "model handle is NULL");
  if (dtype != RBD_F32 && dtype != RBD_F64 && dtype != RBD_DUAL64X6)
    return fail(RBD_EINVAL, "dtype must be RBD_F32, RBD_F64 or RBD_DUAL64X6");
  if (dtype == RBD_DUAL64X6 && !allow_dual)
    return fail(RBD_EUNSUPPORTED, "RBD_DUAL64X6 is supported by rbd_dynamics only; use the reference's generic path");
  if (B < 0 || ld < B) return fail(RBD_EDIM, "batch size / leading dimension mismatch (need ld >= B >= 0)");
  return RBD_OK;
}

}  // namespace

// hooks for the other translation units of the library: argument checks, the RK4 driver
namespace rbd {
int api_check(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld) { return check_common(model, dtype, B, ld); }
int integrate_record(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, void* q, void* v, const void* tau, int64_t step_stride,
                     int64_t stage_stride, double dt, int nsteps, void* q_traj, void* v_traj, void* stages, cudaStream_t stream) {
  return dtype == RBD_F32 ? integrate_t<float>(model, B, ld, q, v, tau, step_stride, stage_stride, dt, nsteps, stream, (float*)q_traj,
                                               (float*)v_traj, (float*)stages)
                          : integrate_t<double>(model, B, ld, q, v, tau, step_stride, stage_stride, dt, nsteps, stream, (double*)q_traj,
                                                (double*)v_traj, (double*)stages);
}
}  // namespace rbd

// ------------------------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------------------------
int32_t rbd_kinematics(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                       const int8_t* path_sign, const rbd_kinematics_out* out, void* stream) {
  if (int rc = check_common(model, dtype, B, ld)) return rc;
  const ApiCall call;
  if (dtype != RBD_F32 && dtype != RBD_F64) return fail(RBD_EUNSUPPORTED, "rbd_kinematics: fp32 and fp64 only");
  if (!out) return fail(RBD_EINVAL, "rbd_kinematics: out must not be NULL");
  if (B == 0) return RBD_OK;      // empty batch: nothing to read or write, pointers may be NULL
  if (!q) return fail(RBD_EINVAL, "rbd_kinematics: q must not be NULL");
  if (!v && (out->kinetic_energy || out->momentum || out->momentum_rate_bias))
    return fail(RBD_EINVAL, "rbd_kinematics: kinetic_energy / momentum / momentum_rate_bias need v");
  if ((out->geometric_jacobian != nullptr) != (path_sign != nullptr))
    return fail(RBD_EINVAL, "rbd_kinematics: path_sign must be given iff geometric_jacobian is requested");
  if (path_sign)
    for (int i = 0; i < model->hm.nb; ++i)
      if (path_sign[i] < -1 || path_sign[i] > 1) return fail(RBD_EINVAL, "rbd_kinematics: path_sign entries must be -1, 0 or +1");
  if (model->hm.total_mass <= 0 && out->center_of_mass) return fail(RBD_EINVAL, "rbd_kinematics: mechanism has no mass");
  cudaStream_t s = (cudaStream_t)stream;
  return dtype == RBD_F32 ? kinematics_t<float>(model, B, ld, q, v, path_sign, *out, s)
                          : kinematics_t<double>(model, B, ld, q, v, path_sign, *out, s);
}

// ---- host-pointer variants: chunked H2D -> kernel -> D2H pipeline over three internal streams ----
namespace {
constexpr int64_t kChunk = 1 << 16;

int ensure_staging(rbd_model* m, size_t bytes_per_stream) {
  for (int i = 0; i < 3; ++i)
    if (!m->streams[i]) RBD_CUDA_TRY(cudaStreamCreateWithFlags(&m->streams[i], cudaStreamNonBlocking));
  if (!m->ev0) { RBD_CUDA_TRY(cudaEventCreate(&m->ev0)); RBD_CUDA_TRY(cudaEventCreate(&m->ev1)); }
  if (m->stage_bytes >= bytes_per_stream) return RBD_OK;
  m->stage_bytes = 0;               // a failed reallocation must not leave a stale size behind
  for (int i = 0; i < 3; ++i) {
    if (m->d_stage[i]) { cudaFree(m->d_stage[i]); m->d_stage[i] = nullptr; }
    RBD_CUDA_TRY(cudaMalloc(&m->d_stage[i], bytes_per_stream));
  }
  m->stage_bytes = bytes_per_stream;
  return RBD_OK;
}

// copy rows x C block between a host array with leading dimension ld and a dense device tile (leading dimension C)
int copy_rows(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, int rows, cudaMemcpyKind kind,
              cudaStream_t s) {
  RBD_CUDA_TRY(cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, rows, kind, s));
  return RBD_OK;
}
}  // namespace

namespace {
struct HostArr { const void* in; void* out; int rows; };

// Chunked host pipeline: chunk c uses stream c % 3 and that stream's staging buffer; H2D copies, the kernel and the D2H
// copies of one chunk are stream-ordered, chunks on different streams overlap (copy engines in both directions + SMs).
template <class Launch>
int host_pipeline_impl(rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const HostArr* ins, int nin, const HostArr* outs,
                       int nout, Launch launch_chunk);
template <class Launch>
int host_pipeline(rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const HostArr* ins, int nin, const HostArr* outs,
                  int nout, Launch launch_chunk) {
  std::lock_guard<std::mutex> lk(model->host_mu);
  const int rc = host_pipeline_impl(model, dtype, B, ld, ins, nin, outs, nout, launch_chunk);
  if (rc != RBD_OK)                 // never return with copies into the caller's host buffers still in flight
    for (int i = 0; i < 3; ++i) if (model->streams[i]) cudaStreamSynchronize(model->streams[i]);
  return rc;
}
template <class Launch>
int host_pipeline_impl(rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const HostArr* ins, int nin, const HostArr* outs,
                       int nout, Launch launch_chunk) {
  const size_t es = dtype == RBD_F32 ? 4 : 8;
  const int64_t C = std::min<int64_t>(kChunk, B);
  size_t rows_total = 0;
  for (int i = 0; i < nin; ++i) rows_total += ins[i].in ? ins[i].rows : 0;
  for (int i = 0; i < nout; ++i) rows_total += outs[i].out ? outs[i].rows : 0;
  if (int rc = ensure_staging(model, rows_total * C * es)) return rc;
  int nchunk = 0;
  for (int64_t b0 = 0; b0 < B; b0 += C, ++nchunk) {
    const int64_t n = std::min<int64_t>(C, B - b0);
    const int si = nchunk % 3;
    cudaStream_t s = model->streams[si];
    char* cur = (char*)model->d_stage[si];
    const size_t off = (size_t)b0 * es;
    const void* din[8] = {nullptr};
    void* dout[8] = {nullptr};
    for (int i = 0; i < nin; ++i) {
      if (!ins[i].in) continue;
      din[i] = cur;
      if (int rc = copy_rows(cur, C * es, (const char*)ins[i].in + off, ld * es, n * es, ins[i].rows, cudaMemcpyHostToDevice, s)) return rc;
      cur += (size_t)ins[i].rows * C * es;
    }
    for (int i = 0; i < nout; ++i) {
      if (!outs[i].out) continue;
      dout[i] = cur;
      cur += (size_t)outs[i].rows * C * es;
    }
    if (int rc = launch_chunk(n, C, din, dout, s)) return rc;
    for (int i = 0; i < nout; ++i) {
      if (!outs[i].out) continue;
      if (int rc = copy_rows((char*)outs[i].out + off, ld * es, dout[i], C * es, n * es, outs[i].rows, cudaMemcpyDeviceToHost, s)) return rc;
    }
  }
  for (int i = 0; i < 3; ++i) RBD_CUDA_TRY(cudaStreamSynchronize(model->streams[i]));
  return RBD_OK;
}
}  // namespace

extern "C" {

int32_t rbd_version(void) { return RBD_B200_VERSION; }
const char* rbd_last_error(void) { return g_err.c_str(); }
const char* rbd_status_string(int32_t s) {
  switch (s) {
    case RBD_OK: return "RBD_OK";
    case RBD_EINVAL: return "RBD_EINVAL";
    case RBD_EDIM: return "RBD_EDIM";
    case RBD_ELOOP: return "RBD_ELOOP";
    case RBD_ESTALE: return "RBD_ESTALE";
    case RBD_ECUDA: return "RBD_ECUDA";
    case RBD_EUNSUPPORTED: return "RBD_EUNSUPPORTED";
    case RBD_ENOMEM: return "RBD_ENOMEM";
  }
  return "RBD_?";
}

int32_t rbd_model_create(const rbd_model_desc* desc, rbd_model** out) {
  if (!out) return fail(RBD_EINVAL, "rbd_model_create: out is NULL");
  *out = nullptr;
  rbd_model* m = new (std::nothrow) rbd_model();
  if (!m) return fail(RBD_ENOMEM, "out of memory");
  std::string err;
  int rc = build_host_model(desc, m->hm, err);
  if (rc != RBD_OK) { delete m; return fail(rc, err); }
  *out = m;
  return RBD_OK;
}

int32_t rbd_model_destroy(rbd_model* m) {
  if (!m) return RBD_OK;
  for (int i = 0; i < 3; ++i) {
    if (m->d_stage[i]) cudaFree(m->d_stage[i]);
    if (m->streams[i]) cudaStreamDestroy(m->streams[i]);
  }
  spec_release(m);
  if (m->counters) cudaFree(m->counters);
  if (m->ev0) cudaEventDestroy(m->ev0);
  if (m->ev1) cudaEventDestroy(m->ev1);
  delete m;
  return RBD_OK;
}

int32_t rbd_model_get_info(const rbd_model* m, rbd_model_info* info) {
  if (!m || !info) return fail(RBD_EINVAL, "rbd_model_get_info: NULL argument");
  std::memset(info, 0, sizeof(*info));
  info->nb = m->hm.nb; info->nq = m->hm.nq; info->nv = m->hm.nv;
  info->stash_rows = m->hm.dev64.nrows;
  info->max_branch_depth = m->hm.nslots;
  info->general_path = m->hm.general ? 1 : 0;
  info->modcount = m->hm.modcount;
  for (int i = 0; i < m->hm.nb; ++i) {
    info->qstart[i] = m->hm.qstart[i];
    info->vstart[i] = m->hm.vstart[i];
    info->eval_order[i] = m->hm.order[i];
  }
  return RBD_OK;
}

int32_t rbd_model_check_modcount(const rbd_model* m, int64_t modcount) {
  if (!m) return fail(RBD_EINVAL, "model handle is NULL");
  if (m->hm.modcount != modcount)
    return fail(RBD_ESTALE, "ModificationCountMismatch: the Mechanism was modified after the model handle was created");
  return RBD_OK;
}

int32_t rbd_get_launch_info(rbd_launch_info* info) {
  if (!info) return fail(RBD_EINVAL, "rbd_get_launch_info: NULL argument");
  *info = g_launch;
  return RBD_OK;
}

int32_t rbd_model_precompile(rbd_model* model, int32_t dtype, int32_t what, int32_t load) {
  if (!model) return fail(RBD_EINVAL, "model handle is NULL");
  if (dtype != RBD_F32 && dtype != RBD_F64) return fail(RBD_EUNSUPPORTED, "rbd_model_precompile: fp32 / fp64 only");
  int rc_all = RBD_OK;
  std::string err;
  auto one = [&](int algo, bool in2, bool out1) {
    SpecKey key; key.algo = algo; key.f64 = dtype == RBD_F64; key.has_in2 = in2; key.has_out1 = out1;
    std::string e;
    const int rc = spec_prepare(model, key, load != 0, e);
    if (rc != RBD_OK) { rc_all = rc; err = e; }
  };
  if (what & RBD_SPEC_DYNAMICS) one(SPEC_ABA, true, false);
  if (what & RBD_SPEC_DYNAMICS_QDOT) one(SPEC_ABA, true, true);
  if (what & RBD_SPEC_DYNAMICS_NOTAU) { one(SPEC_ABA, false, false); one(SPEC_ABA, false, true); }
  if (what & RBD_SPEC_INVERSE_DYNAMICS) one(SPEC_RNEA, true, false);
  if (what & RBD_SPEC_DYNAMICS_BIAS) one(SPEC_RNEA, false, false);
  if (what & (RBD_SPEC_MASS_MATRIX | RBD_SPEC_MASS_MATRIX_LOWER)) {
    for (int lower = 0; lower < 2; ++lower) {
      if (!(what & (lower ? RBD_SPEC_MASS_MATRIX_LOWER : RBD_SPEC_MASS_MATRIX))) continue;
      SpecKey key; key.algo = SPEC_CRBA; key.f64 = dtype == RBD_F64; key.has_in2 = false; key.lower = lower != 0;
      std::string e;
      const int rc = spec_prepare(model, key, load != 0, e);
      if (rc != RBD_OK) { rc_all = rc; err = e; }
    }
  }
  if (what & RBD_SPEC_DYNAMICS_GATHER) {
    SpecKey key; key.algo = SPEC_ABA; key.f64 = dtype == RBD_F64; key.has_in2 = true; key.peers = true;
    std::string e;
    const int rc = spec_prepare(model, key, load != 0, e);
    if (rc != RBD_OK) { rc_all = rc; err = e; }
  }
  return rc_all == RBD_OK ? RBD_OK : fail(rc_all, err);
}

int32_t rbd_dynamics(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                     const void* tau, const void* wext, void* vd_out, void* qd_out, void* stream) {
  if (int rc = check_common(model, dtype, B, ld, true)) return rc;
  const ApiCall call;
  if (B == 0) return RBD_OK;      // empty batch: nothing to read or write, pointers may be NULL
  if (!q || !v || !vd_out) return fail(RBD_EINVAL, "rbd_dynamics: q, v and vd_out must not be NULL");
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype == RBD_DUAL64X6) {
    if (wext || qd_out) return fail(RBD_EUNSUPPORTED, "RBD_DUAL64X6: external wrenches / q̇ output are not implemented");
    return dynamics_dual(model, B, ld, q, v, tau, vd_out, s);
  }
  return dtype == RBD_F32 ? dynamics_t<float>(model, B, ld, q, v, tau, wext, vd_out, qd_out, s)
                          : dynamics_t<double>(model, B, ld, q, v, tau, wext, vd_out, qd_out, s);
}

int32_t rbd_dynamics_gather(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                            const void* tau, int32_t npeers, void* const* vd_peers, void* vd_multicast, int64_t peer_ld, int64_t col0,
                            void* stream) {
  if (int rc = check_common(model, dtype, B, ld)) return rc;
  const ApiCall call;
  if (npeers < 1 || npeers > 8 || !vd_peers) return fail(RBD_EINVAL, "rbd_dynamics_gather: need 1..8 peer arrays");
  for (int p = 0; p < npeers; ++p) if (!vd_peers[p]) return fail(RBD_EINVAL, "rbd_dynamics_gather: NULL peer array");
  if (col0 < 0 || peer_ld < col0 + B) return fail(RBD_EDIM, "rbd_dynamics_gather: columns [col0, col0 + B) exceed the gathered array");
  if (B == 0) return RBD_OK;
  if (!q || !v) return fail(RBD_EINVAL, "rbd_dynamics_gather: q and v must not be NULL");
  cudaStream_t s = (cudaStream_t)stream;
  return dtype == RBD_F32 ? dynamics_gather_t<float>(model, B, ld, q, v, tau, npeers, vd_peers, vd_multicast, peer_ld, col0, s)
                          : dynamics_gather_t<double>(model, B, ld, q, v, tau, npeers, vd_peers, vd_multicast, peer_ld, col0, s);
}

int32_t rbd_integrate_schedule(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, void* q, void* v, const void* tau,
                               int64_t tau_step_stride, int64_t tau_stage_stride, double dt, int32_t nsteps, void* stream) {
  if (int rc = check_common(model, dtype, B, ld)) return rc;
  if (nsteps < 0 || !(dt > 0)) return fail(RBD_EINVAL, "rbd_integrate: need dt > 0 and nsteps >= 0");
  if (tau_step_stride < 0 || tau_stage_stride < 0) return fail(RBD_EINVAL, "rbd_integrate: torque strides must be >= 0");
  const ApiCall call;
  if (B == 0 || nsteps == 0) return RBD_OK;
  if (!q || !v) return fail(RBD_EINVAL, "rbd_integrate: q and v must not be NULL");
  cudaStream_t s = (cudaStream_t)stream;
  return dtype == RBD_F32 ? integrate_t<float>(model, B, ld, q, v, tau, tau_step_stride, tau_stage_stride, dt, nsteps, s)
                          : integrate_t<double>(model, B, ld, q, v, tau, tau_step_stride, tau_stage_stride, dt, nsteps, s);
}

int32_t rbd_integrate(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, void* q, void* v, const void* tau,
                      double dt, int32_t nsteps, void* stream) {
  return rbd_integrate_schedule(model, dtype, B, ld, q, v, tau, 0, 0, dt, nsteps, stream);
}

int32_t rbd_integrate_trajectory(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, void* q, void* v, const void* tau,
                                 int64_t tau_step_stride, int64_t tau_stage_stride, double dt, int32_t nsteps, void* q_traj,
                                 void* v_traj, void* stream) {
  if (int rc = check_common(model, dtype, B, ld)) return rc;
  if (nsteps < 0 || !(dt > 0)) return fail(RBD_EINVAL, "rbd_integrate_trajectory: need dt > 0 and nsteps >= 0");
  if (tau_step_stride < 0 || tau_stage_stride < 0) return fail(RBD_EINVAL, "rbd_integrate_trajectory: torque strides must be >= 0");
  const ApiCall call;
  if (B == 0) return RBD_OK;
  if (!q || !v || !q_traj || !v_traj) return fail(RBD_EINVAL, "rbd_integrate_trajectory: q, v, q_traj and v_traj must not be NULL");
  return rbd::integrate_record(model, dtype, B, ld, q, v, tau, tau_step_stride, tau_stage_stride, dt, nsteps, q_traj, v_traj, nullptr,
                               (cudaStream_t)stream);
}

int32_t rbd_inverse_dynamics(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q,
                             const void* v, const void* vd, const void* wext, void* tau_out, void* stream) {
  if (int rc = check_common(model, dtype, B, ld)) return rc;
  const ApiCall call;
  if (B == 0) return RBD_OK;      // empty batch: nothing to read or write, pointers may be NULL
  if (!q || !v || !vd || !tau_out) return fail(RBD_EINVAL, "rbd_inverse_dynamics: q, v, vd and tau_out must not be NULL");
  cudaStream_t s = (cudaStream_t)stream;
  return dtype == RBD_F32 ? inverse_dynamics_t<float>(model, B, ld, q, v, vd, wext, tau_out, s)
                          : inverse_dynamics_t<double>(model, B, ld, q, v, vd, wext, tau_out, s);
}

int32_t rbd_inverse_dynamics_bodies(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                                    const void* vd, const void* wext, void* accelerations_out, void* jointwrenches_out, void* stream) {
  if (int rc = check_common(model, dtype, B, ld)) return rc;
  const ApiCall call;
  if (B == 0 || (!accelerations_out && !jointwrenches_out)) return RBD_OK;
  if (!q || !v) return fail(RBD_EINVAL, "rbd_inverse_dynamics_bodies: q and v must not be NULL");
  cudaStream_t s = (cudaStream_t)stream;
  return dtype == RBD_F32 ? bodies_t<float>(model, B, ld, q, v, vd, wext, accelerations_out, jointwrenches_out, s)
                          : bodies_t<double>(model, B, ld, q, v, vd, wext, accelerations_out, jointwrenches_out, s);
}

int32_t rbd_contact_dynamics(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                             const rbd_contact_desc* contact, void* state, void* state_deriv_out, void* wrenches_out, void* stream) {
  if (int rc = check_common(model, dtype, B, ld)) return rc;
  const ApiCall call;
  if (!contact) return fail(RBD_EINVAL, "rbd_contact_dynamics: contact must not be NULL");
  if (contact->npoints < 0 || contact->nhalfspaces < 0) return fail(RBD_EINVAL, "rbd_contact_dynamics: negative counts");
  if (contact->npoints > kMaxContactPoints || contact->nhalfspaces > kMaxHalfSpaces)
    return fail(RBD_EUNSUPPORTED, "rbd_contact_dynamics: at most 32 contact points and 4 half-spaces");
  if (contact->npoints && (!contact->body || !contact->location || !contact->normal_model || !contact->friction_model))
    return fail(RBD_EINVAL, "rbd_contact_dynamics: point arrays must not be NULL");
  if (contact->nhalfspaces && !contact->halfspace) return fail(RBD_EINVAL, "rbd_contact_dynamics: halfspace must not be NULL");
  for (int p = 0; p < contact->npoints; ++p) {
    if (contact->body[p] < 0 || contact->body[p] >= model->hm.nb) return fail(RBD_EINVAL, "rbd_contact_dynamics: body index out of range");
    if (!(contact->friction_model[3 * p + 2] > 0)) return fail(RBD_EINVAL, "rbd_contact_dynamics: friction damping b must be > 0");
  }
  for (int h = 0; h < contact->nhalfspaces; ++h) {
    const double* n = contact->halfspace + 6 * h + 3;
    if (!(n[0] * n[0] + n[1] * n[1] + n[2] * n[2] > 0)) return fail(RBD_EINVAL, "rbd_contact_dynamics: zero half-space normal");
  }
  if (B == 0) return RBD_OK;
  if (!q || !v || !wrenches_out) return fail(RBD_EINVAL, "rbd_contact_dynamics: q, v and wrenches_out must not be NULL");
  cudaStream_t s = (cudaStream_t)stream;
  return dtype == RBD_F32 ? contact_t<float>(model, B, ld, q, v, *contact, state, state_deriv_out, wrenches_out, s)
                          : contact_t<double>(model, B, ld, q, v, *contact, state, state_deriv_out, wrenches_out, s);
}

int32_t rbd_dynamics_result(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                            const void* tau, const void* wext, void* vd_out, void* qd_out, void* M_out, void* c_out,
                            void* accelerations_out, void* jointwrenches_out, void* stream) {
  const ApiCall call;
  int rc = rbd_dynamics(model, dtype, B, ld, q, v, tau, wext, vd_out, qd_out, stream);
  if (rc != RBD_OK || B == 0) return rc;
  if (dtype == RBD_DUAL64X6 && (M_out || c_out || accelerations_out || jointwrenches_out))
    return fail(RBD_EUNSUPPORTED, "rbd_dynamics_result: by-products are fp32 / fp64 only");
  const KeepLaunchRecord keep;      // the record describes the dynamics kernel; the by-products add their launches
  if (c_out && (rc = rbd_dynamics_bias(model, dtype, B, ld, q, v, wext, c_out, stream)) != RBD_OK) return rc;
  if (M_out && (rc = rbd_mass_matrix(model, dtype, B, ld, q, M_out, stream)) != RBD_OK) return rc;
  if (accelerations_out || jointwrenches_out)
    return rbd_inverse_dynamics_bodies(model, dtype, B, ld, q, v, vd_out, wext, accelerations_out, jointwrenches_out, stream);
  return RBD_OK;
}

int32_t rbd_dynamics_bias(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q,
                          const void* v, const void* wext, void* c_out, void* stream) {
  if (int rc = check_common(model, dtype, B, ld)) return rc;
  const ApiCall call;
  if (B == 0) return RBD_OK;      // empty batch: nothing to read or write, pointers may be NULL
  if (!q || !v || !c_out) return fail(RBD_EINVAL, "rbd_dynamics_bias: q, v and c_out must not be NULL");
  cudaStream_t s = (cudaStream_t)stream;
  return dtype == RBD_F32 ? inverse_dynamics_t<float>(model, B, ld, q, v, nullptr, wext, c_out, s)
                          : inverse_dynamics_t<double>(model, B, ld, q, v, nullptr, wext, c_out, s);
}

int32_t rbd_mass_matrix_uplo(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, void* M_out,
                             int32_t uplo, void* stream) {
  if (int rc = check_common(model, dtype, B, ld)) return rc;
  const ApiCall call;
  if (uplo != RBD_UPLO_FULL && uplo != RBD_UPLO_LOWER) return fail(RBD_EINVAL, "rbd_mass_matrix: uplo must be RBD_UPLO_FULL or RBD_UPLO_LOWER");
  if (B == 0) return RBD_OK;      // empty batch: nothing to read or write, pointers may be NULL
  if (!q || !M_out) return fail(RBD_EINVAL, "rbd_mass_matrix: q and M_out must not be NULL");
  cudaStream_t s = (cudaStream_t)stream;
  const bool lower = uplo == RBD_UPLO_LOWER;
  return dtype == RBD_F32 ? mass_matrix_t<float>(model, B, ld, q, M_out, s, lower) : mass_matrix_t<double>(model, B, ld, q, M_out, s, lower);
}

int32_t rbd_mass_matrix(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, void* M_out,
                        void* stream) {
  return rbd_mass_matrix_uplo(model, dtype, B, ld, q, M_out, RBD_UPLO_FULL, stream);
}

// ---- host-pointer variants: chunked H2D -> kernel -> D2H pipeline over three internal streams -----------------------


int32_t rbd_dynamics_host(rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                          const void* tau, const void* wext, void* vd_out, void* qd_out) {
  if (int rc = check_common(model, dtype, B, ld)) return rc;
  const ApiCall call;
  if (B == 0) return RBD_OK;      // empty batch: nothing to read or write, pointers may be NULL
  if (!q || !v || !vd_out) return fail(RBD_EINVAL, "rbd_dynamics_host: q, v and vd_out must not be NULL");
  const HostModel& hm = model->hm;
  const HostArr ins[4] = {{q, nullptr, hm.nq}, {v, nullptr, hm.nv}, {tau, nullptr, hm.nv}, {wext, nullptr, 6 * hm.nb}};
  const HostArr outs[2] = {{nullptr, vd_out, hm.nv}, {nullptr, qd_out, hm.nq}};
  return host_pipeline(model, dtype, B, ld, ins, 4, outs, 2,
                       [&](int64_t n, int64_t C, const void** di, void** dq, cudaStream_t s) {
                         return dtype == RBD_F32 ? dynamics_t<float>(model, n, C, di[0], di[1], di[2], di[3], dq[0], dq[1], s)
                                                 : dynamics_t<double>(model, n, C, di[0], di[1], di[2], di[3], dq[0], dq[1], s);
                       });
}

int32_t rbd_inverse_dynamics_host(rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q,
                                  const void* v, const void* vd, const void* wext, void* tau_out) {
  if (int rc = check_common(model, dtype, B, ld)) return rc;
  const ApiCall call;
  if (B == 0) return RBD_OK;      // empty batch: nothing to read or write, pointers may be NULL
  if (!q || !v || !vd || !tau_out) return fail(RBD_EINVAL, "rbd_inverse_dynamics_host: q, v, vd and tau_out must not be NULL");
  const HostModel& hm = model->hm;
  const HostArr ins[4] = {{q, nullptr, hm.nq}, {v, nullptr, hm.nv}, {vd, nullptr, hm.nv}, {wext, nullptr, 6 * hm.nb}};
  const HostArr outs[1] = {{nullptr, tau_out, hm.nv}};
  return host_pipeline(model, dtype, B, ld, ins, 4, outs, 1,
                       [&](int64_t n, int64_t C, const void** di, void** dq, cudaStream_t s) {
                         return dtype == RBD_F32 ? inverse_dynamics_t<float>(model, n, C, di[0], di[1], di[2], di[3], dq[0], s)
                                                 : inverse_dynamics_t<double>(model, n, C, di[0], di[1], di[2], di[3], dq[0], s);
                       });
}

int32_t rbd_dynamics_bias_host(rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q,
                               const void* v, const void* wext, void* c_out) {
  if (int rc = check_common(model, dtype, B, ld)) return rc;
  const ApiCall call;
  if (B == 0) return RBD_OK;      // empty batch: nothing to read or write, pointers may be NULL
  if (!q || !v || !c_out) return fail(RBD_EINVAL, "rbd_dynamics_bias_host: q, v and c_out must not be NULL");
  const HostModel& hm = model->hm;
  const HostArr ins[3] = {{q, nullptr, hm.nq}, {v, nullptr, hm.nv}, {wext, nullptr, 6 * hm.nb}};
  const HostArr outs[1] = {{nullptr, c_out, hm.nv}};
  return host_pipeline(model, dtype, B, ld, ins, 3, outs, 1,
                       [&](int64_t n, int64_t C, const void** di, void** dq, cudaStream_t s) {
                         return dtype == RBD_F32 ? inverse_dynamics_t<float>(model, n, C, di[0], di[1], nullptr, di[2], dq[0], s)
                                                 : inverse_dynamics_t<double>(model, n, C, di[0], di[1], nullptr, di[2], dq[0], s);
                       });
}

int32_t rbd_mass_matrix_host(rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, void* M_out) {
  if (int rc = check_common(model, dtype, B, ld)) return rc;
  const ApiCall call;
  if (B == 0) return RBD_OK;      // empty batch: nothing to read or write, pointers may be NULL
  if (!q || !M_out) return fail(RBD_EINVAL, "rbd_mass_matrix_host: q and M_out must not be NULL");
  const HostModel& hm = model->hm;
  const HostArr ins[1] = {{q, nullptr, hm.nq}};
  const HostArr outs[1] = {{nullptr, M_out, hm.nv * hm.nv}};
  return host_pipeline(model, dtype, B, ld, ins, 1, outs, 1,
                       [&](int64_t n, int64_t C, const void** di, void** dq, cudaStream_t s) {
                         return dtype == RBD_F32 ? mass_matrix_t<float>(model, n, C, di[0], dq[0], s)
                                                 : mass_matrix_t<double>(model, n, C, di[0], dq[0], s);
                       });
}

}  // extern "C"
