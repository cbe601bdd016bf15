// rbd_dynamics_derivatives(_ext): batched analytic dv̇/dq, dv̇/dv, dv̇/dtau; rbd_inverse_dynamics_derivatives: d tau/dq, d tau/dv, M
// (csrc/rbd_deriv.cuh has the mathematics and the work split).
//
// Four kernels (after the forward dynamics itself) per chunk of the batch, all with the sample index fastest (lane l of a warp = sample b0 + l, so every global
// access of a warp is one fully used line) and warp-uniform control flow (the tree walk depends on the model only):
//   deriv_world_kernel   one thread per sample            root-frame S, Psi_dot, Psi_ddot, Sdp per coordinate; I, G, f per body
//   deriv_accum_kernel   one thread per (sample, 1 of 52) subtree sums of (I, G, f)
//   deriv_pairs_kernel   one thread per (sample, body)    d tau/dq, d tau/dv (into the output arrays) and M (into the scratch)
//   deriv_solve_kernel   one CTA per 32 samples (lane = sample), W warps: M of the 32 samples is staged in shared memory, factored
//                        there as L^T D L (tree sparsity) by the W warps together, then each warp solves its share of the 2 nv
//                        columns (3 nv with d v̇ / d tau) in place with its right-hand side in shared memory, [row][lane]
//   (deriv_factor_kernel one thread per sample, on the scratch: only when M does not fit into shared memory)
// The inverse-dynamics Jacobians run world, accum and pairs at the caller's v̇ and then deriv_expand_kernel (one thread per
// (sample, column): the zeros of unrelated pairs and the dense M) instead of the forward dynamics, the factor and the solve.
// Intermediates: a global scratch of DerivDev::rows rows per sample, allocated from the stream-ordered pool per call and
// bounded by RBD_DERIV_SCRATCH_MB (default 2048): larger batches are processed in chunks on the same stream.  The launch record
// (rbd_handle.h) counts the kernels of every chunk, the forward dynamics included.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "../../../include/rbd_b200.h"
// rbd_sincos.cuh defines one out-of-line __device__ function with external linkage (its text is also compiled by NVRTC, where
// `static` would be noise); this second translation unit of the library gets its own copy under another name
#define sincos_slow sincos_slow_deriv_tu
#include "rbd_deriv.cuh"
#include "rbd_deriv_jit.h"
#include "rbd_handle.h"
#include "rbd_jit_text.h"

using namespace rbd;

namespace {

constexpr int kNT = 128;

template <class T> struct DerivArgs {
  const T* q; const T* v; const T* vd;
  T* dq; T* dv;
  T* s;                 // scratch [rows][sld]
  int64_t ld, sld, C;   // C: samples in this chunk (all pointers already offset to the chunk's first sample)
  const T* wext;        // external wrenches or NULL (then D.w_base == 0)
  T* dtau;              // forward: d v̇ / d tau (the solve's third block) or NULL
  T* tau;               // inverse: tau or NULL
  T* Mo;                // inverse: M or NULL
};

// EXT (here and below): the call has external wrenches (D.w_base != 0, a.wext != NULL)
template <class T, int NT, bool EXT>
__global__ void __launch_bounds__(NT) deriv_world_kernel(const __grid_constant__ ModelDev<T> M, const __grid_constant__ DerivDev D,
                                                         const DerivArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const Stash<T, NT> st{reinterpret_cast<T*>(smem_raw) + threadIdx.x};
  const int64_t ngroups = (a.C + NT - 1) / NT;
  for (int64_t g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const int64_t b = g * NT + threadIdx.x;
    const bool active = b < a.C;
    const int64_t bl = active ? b : a.C - 1;
    DerivIO<T> io;
    io.q = {a.q + bl, a.ld};
    io.v = {a.v + bl, a.ld};
    io.vd = {a.vd + bl, a.ld};
    if (EXT) io.wext = {a.wext + bl, a.ld};
    io.s = a.s + bl;
    io.sld = a.sld;
    io.active = active;
    deriv_world_sample<T, Stash<T, NT>, EXT>(M, D, io, st);
  }
}

// grid.y: the 52 components of (Ic, G, F), then with EXT the 6 of W
template <class T, int NT, bool EXT>
__global__ void __launch_bounds__(NT) deriv_accum_kernel(const __grid_constant__ ModelDev<T> M, const __grid_constant__ DerivDev D,
                                                         const DerivArgs<T> a) {
  const int64_t b = (int64_t)blockIdx.x * NT + threadIdx.x;
  if (b >= a.C) return;
  if (EXT && blockIdx.y >= kBodyRows) deriv_accumulate_wrench<T>(M, D, a.s + b, a.sld, blockIdx.y - kBodyRows);
  else deriv_accumulate<T>(M, D, a.s + b, a.sld, blockIdx.y);
}

// grid = (bodies, sample groups), bodies fastest: the CTAs that are resident together work on the SAME samples, so the per-coordinate
// rows a body shares with its relatives are served by L2 instead of being streamed from HBM once per body
// TAU: the inverse-dynamics call with tau_out
template <class T, int NT, bool EXT, bool TAU>
__global__ void __launch_bounds__(NT) deriv_pairs_kernel(const __grid_constant__ DerivDev D, const __grid_constant__ DerivAnc A,
                                                         const DerivArgs<T> a) {
  const int64_t b = (int64_t)blockIdx.y * NT + threadIdx.x;
  if (b >= a.C) return;
  deriv_pairs<T, EXT, TAU>(D, A, a.s + b, a.sld, a.dq + b, a.dv + b, a.ld, blockIdx.x, true, TAU ? a.tau + b : nullptr);
}

// inverse-dynamics Jacobians only: grid = (sample groups, nv columns)
template <class T, int NT>
__global__ void __launch_bounds__(NT) deriv_expand_kernel(const __grid_constant__ DerivDev D, const DerivArgs<T> a) {
  const int64_t b = (int64_t)blockIdx.x * NT + threadIdx.x;
  if (b >= a.C) return;
  deriv_expand_column<T>(D, a.s + (int64_t)D.h_base * a.sld + b, a.sld, a.dq + b, a.dv + b, a.Mo ? a.Mo + b : nullptr, a.ld, blockIdx.y, true);
}

// only for models whose factor does not fit into shared memory next to the right-hand sides (deriv_solve_kernel<T, false>)
template <class T, int NT>
__global__ void __launch_bounds__(NT) deriv_factor_kernel(const __grid_constant__ DerivDev D, const __grid_constant__ DerivAnc A,
                                                          const DerivArgs<T> a) {
  const int64_t b = (int64_t)blockIdx.x * NT + threadIdx.x;
  if (b >= a.C) return;
  deriv_factor<T>(D, A, a.s + (int64_t)D.h_base * a.sld + b, a.sld);
}

// blockDim = (32, W): lane = sample, warp = column subset.  HS: M of the block's 32 samples is staged in shared memory, factored
// there by all W warps together (row k's updates of its ancestors' rows are independent of each other: warp w takes the
// ancestors at depth w, w + W, ...; two barriers per row) and then re-used by all 2 nv columns.  Otherwise the factor was made
// by deriv_factor_kernel and is read from the scratch.  DTAU: also the columns 2 nv .. 3 nv - 1, those of M^-1 (into a.dtau).
template <class T, bool HS, bool DTAU>
__global__ void deriv_solve_kernel(const __grid_constant__ DerivDev D, const __grid_constant__ DerivAnc A, const DerivArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* sm = reinterpret_cast<T*>(smem_raw);
  const int lane = threadIdx.x, w = threadIdx.y, W = blockDim.y;
  const int nv = D.nv, nnz = D.nnz;
  T* Hs = sm + lane;
  T* xs = sm + (HS ? (size_t)nnz * 32 : 0) + (size_t)w * nv * 32 + lane;
  const int64_t ngroups = (a.C + 31) / 32;
  for (int64_t g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const int64_t b = g * 32 + lane;
    const bool active = b < a.C;
    const int64_t bl = active ? b : a.C - 1;
    const T* Hg = a.s + (int64_t)D.h_base * a.sld + bl;
    if (HS) {
      __syncthreads();      // the previous group's columns are done with Hs
      for (int r = w; r < nnz; r += W) Hs[r * 32] = Hg[(int64_t)r * a.sld];
      for (int k = nv - 1; k >= 0; --k) {
        const int rk = D.rowstart[k], dk = D.depth[k];
        __syncthreads();    // row k has received the updates of all its descendants
        const T inv = T(1) / Hs[(rk + dk) * 32];
        for (int di = w; di < dk; di += W) {
          const int ri = D.rowstart[A.anc[rk + di]];
          const T f = Hs[(rk + di) * 32] * inv;
          for (int d = di; d >= 0; --d) Hs[(ri + d) * 32] -= f * Hs[(rk + d) * 32];
        }
        __syncthreads();    // everybody has read row k
        for (int di = w; di < dk; di += W) Hs[(rk + di) * 32] *= inv;
        if (w == 0) Hs[(rk + dk) * 32] = inv;
      }
      __syncthreads();
    }
    const int ncols = DTAU ? 3 * nv : 2 * nv;
    for (int c = w; c < ncols; c += W) {
      const int blk = c < nv ? 0 : (DTAU && c >= 2 * nv ? 2 : 1);
      const int vj = c - blk * nv;
      T* col = (blk == 0 ? a.dq : blk == 1 ? a.dv : a.dtau) + (int64_t)vj * nv * a.ld + bl;
      if (HS) {
        const T* Hl = Hs;
        deriv_solve_column<T>(D, A, [Hl](int row) { return Hl[row * 32]; }, xs, 32, col, a.ld, vj, active, blk == 2);
      } else {
        const int64_t sld = a.sld;
        deriv_solve_column<T>(D, A, [Hg, sld](int row) { return Hg[(int64_t)row * sld]; }, xs, 32, col, a.ld, vj, active, blk == 2);
      }
    }
  }
}

// ---- model-specialised solve kernel (rbd_deriv_jit.cpp): compiled with NVRTC on the first large call (or ahead of time by
// rbd_model_precompile_derivatives), cubin cached on disk, module cached per (tables, dtype, device) ----
struct JitSolve {
  int state = 0;                 // 1 = ready, -1 = unavailable (the generic kernel serves the call)
  cudaLibrary_t lib = nullptr;
  cudaKernel_t kernel = nullptr;
  DerivJitPlan plan;
  size_t smem = 0;
  int bps = 0;
};
std::mutex g_jit_mu;
std::map<std::string, JitSolve> g_jit;

bool jit_enabled() {
  const char* e = std::getenv("RBD_JIT");
  if (e && e[0] == '0') return false;
  e = std::getenv("RBD_DERIV_JIT");
  return !(e && e[0] == '0');
}
int64_t jit_min_batch() {
  if (const char* e = std::getenv("RBD_JIT_MIN_BATCH")) return std::max<int64_t>(1, std::atoll(e));
  return 4096;
}
// cubin for the model's solve kernel (from the cache, or compiled when `compile`); no GPU needed.  dtau: the variant with the third
// block of columns (d v̇ / d tau), a text and a cubin of its own
bool jit_solve_cubin(const DerivDev& D, const DerivAnc& A, bool f64, bool dtau, bool compile, DerivJitPlan& plan, std::vector<char>& cubin,
                     std::string& err) {
  if (D.nnz * 32 * (f64 ? 8 : 4) > 200 * 1024) { err = "factor does not fit into shared memory"; return false; }
  if (!deriv_jit_plan(D, f64, plan, dtau ? 3 : 2)) { err = "too many velocity coordinates for a register-resident solve"; return false; }
  std::string src;
  deriv_jit_source(D, A, f64, plan, src);
  const std::string sfx = std::string(dtau ? "_tau" : "") + (f64 ? "_f64" : "_f32");
  if (const char* dump = std::getenv("RBD_DERIV_DUMP")) {           // inspection: nvcc -cubin -Xptxas -v on the dumped text
    if (FILE* f = fopen((std::string(dump) + sfx + ".cu").c_str(), "w")) { fwrite(src.data(), 1, src.size(), f); fclose(f); }
  }
  bool from_cache = false;
  return jit_compile_text("deriv" + sfx, src, true, cubin, compile, &from_cache, err);
}
JitSolve* jit_solve_get(const DerivDev& D, const DerivAnc& A, bool f64, bool dtau, int64_t B, const DeviceProps& p) {
  if (!jit_enabled()) return nullptr;
  std::string key((const char*)&D, sizeof(D));
  key.append((const char*)A.anc, sizeof(int16_t) * D.nnz);
  key.push_back(f64 ? 'd' : 'f');
  key.push_back((char)p.dev);
  if (dtau) key.push_back('t');
  std::lock_guard<std::mutex> lk(g_jit_mu);
  JitSolve& e = g_jit[key];
  if (e.state == 1) return &e;
  if (e.state == -1) return nullptr;
  std::vector<char> cubin;
  std::string err;
  if (!jit_solve_cubin(D, A, f64, dtau, B >= jit_min_batch(), e.plan, cubin, err)) {
    if (err != "no cached cubin") {
      e.state = -1;
      if (std::getenv("RBD_JIT_VERBOSE")) fprintf(stderr, "rbd_b200: derivative solve kernel not specialised: %s\n", err.c_str());
    }
    return nullptr;
  }
  e.smem = (size_t)D.nnz * 32 * (f64 ? 8 : 4);
  cudaError_t ce = cudaLibraryLoadData(&e.lib, cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0);
  if (ce == cudaSuccess) ce = cudaLibraryGetKernel(&e.kernel, e.lib, "rbd_deriv_solve");
  if (ce == cudaSuccess) ce = cudaFuncSetAttribute((const void*)e.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)e.smem);
  if (ce == cudaSuccess) ce = cudaFuncSetAttribute((const void*)e.kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  if (ce == cudaSuccess) ce = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&e.bps, (const void*)e.kernel, 32 * e.plan.warps, e.smem);
  if (ce != cudaSuccess || e.bps < 1) {
    cudaGetLastError();
    if (std::getenv("RBD_JIT_VERBOSE")) fprintf(stderr, "rbd_b200: derivative solve kernel failed to load: %s\n", cudaGetErrorString(ce));
    if (e.lib) { cudaLibraryUnload(e.lib); e.lib = nullptr; }
    e.state = -1;
    return nullptr;
  }
  e.state = 1;
  return &e;
}

// One call of either entry point.  Forward (rbd_dynamics_derivatives_ext): tau in, vd out, dq / dv = d v̇ / d(q, v), dtau = M^-1 or
// NULL.  Inverse (rbd_inverse_dynamics_derivatives): vd in, dq / dv = d tau / d(q, v), tau and M out or NULL.  wext may be NULL.
template <class T> struct DerivCall {
  bool inverse;
  const T* q; const T* v; const T* tau_in; const T* wext;
  T* vd;                 // forward: written; inverse: the caller's v̇ (read only)
  T* dq; T* dv; T* dtau; T* tau_out; T* M;
  bool vd_given = false;  // forward: vd already holds v̇ at (q, v, tau) and the forward dynamics is not run again
};

template <class T>
int derivatives_t(const char* fn, const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const DerivCall<T>& r, cudaStream_t stream) {
  const HostModel& hm = model->hm;
  const ModelDev<T>& M = dev_model<T>(hm);
  DerivDev D;
  DerivAnc A;
  if (!build_deriv_dev(M, D, A))
    return api_fail(RBD_EUNSUPPORTED, std::string(fn) + ": more than 128 velocity coordinates or 4096 mass-matrix entries");
  if (D.nv == 0) return RBD_OK;        // nothing to differentiate (only fixed joints): no outputs have any rows
  DeviceProps p;
  RBD_CUDA_TRY(device_props(p));
  // solve kernel geometry: warps per block so that factor + right-hand sides fit, maximising resident warps
  const int ncols = r.dtau ? 3 * D.nv : 2 * D.nv;
  const size_t hbytes = (size_t)D.nnz * 32 * sizeof(T), xbytes = (size_t)D.nv * 32 * sizeof(T);
  int bestW = 0, bestNb = 0;
  bool hs = true;
  for (int nb = 1; nb <= 4; ++nb) {
    const int64_t avail = std::min<int64_t>(p.max_smem_optin, p.smem_per_sm / nb - 1024) - (int64_t)hbytes;
    if (avail < (int64_t)xbytes) continue;
    const int W = (int)std::min<int64_t>(std::min(16, ncols), avail / (int64_t)xbytes);
    if (W * nb > bestW * bestNb) { bestW = W; bestNb = nb; }
  }
  if (const char* e = std::getenv("RBD_DERIV_GLOBAL_FACTOR")) { if (e[0] == '1') bestW = 0; }   // tests: exercise the fallback
  if (bestW == 0) {       // factor too large for shared memory: read it from the scratch
    hs = false;
    bestW = (int)std::min<int64_t>(std::min(8, ncols), p.max_smem_optin / (int64_t)xbytes);
    bestNb = 1;
  }
  JitSolve* js = hs && !r.inverse ? jit_solve_get(D, A, sizeof(T) == 8, r.dtau != nullptr, B, p) : nullptr;
  if (r.wext) deriv_dev_add_wrenches(D);       // after the lookup: the solve kernel does not depend on the wrench rows
  // chunk size from the scratch budget
  int64_t budget_mb = 2048;
  if (const char* e = std::getenv("RBD_DERIV_SCRATCH_MB")) budget_mb = std::max<int64_t>(1, std::atoll(e));
  const int64_t per_sample = (int64_t)D.rows * (int64_t)sizeof(T);
  int64_t C = std::min<int64_t>(B, std::max<int64_t>(kNT, (budget_mb << 20) / per_sample / kNT * kNT));
  // deriv_pairs_kernel puts the sample groups of a chunk in grid.y (bodies fastest, see there), which holds at most 65535 blocks
  C = std::min<int64_t>(C, (int64_t)65535 * kNT);
  const int64_t sld = (C + 31) / 32 * 32;
  StreamAlloc scratch_;
  if (cudaError_t e = scratch_.alloc((size_t)per_sample * sld, stream))
    return api_fail_cuda(e, std::string(fn) + ": scratch allocation (lower RBD_DERIV_SCRATCH_MB)");
  T* scratch = (T*)scratch_.p;
  const size_t solve_smem = (hs ? hbytes : 0) + (size_t)bestW * xbytes;
  const size_t world_smem = (size_t)std::max(1, kin_rows(hm)) * kNT * sizeof(T);
  const bool ext = r.wext != nullptr, dtau = r.dtau != nullptr, tau = r.tau_out != nullptr;
  auto kworld = ext ? deriv_world_kernel<T, kNT, true> : deriv_world_kernel<T, kNT, false>;
  auto kaccum = ext ? deriv_accum_kernel<T, kNT, true> : deriv_accum_kernel<T, kNT, false>;
  auto kpairs = ext ? (tau ? deriv_pairs_kernel<T, kNT, true, true> : deriv_pairs_kernel<T, kNT, true, false>)
                    : (tau ? deriv_pairs_kernel<T, kNT, false, true> : deriv_pairs_kernel<T, kNT, false, false>);
  auto ksolve_s = dtau ? deriv_solve_kernel<T, true, true> : deriv_solve_kernel<T, true, false>;
  auto ksolve_g = dtau ? deriv_solve_kernel<T, false, true> : deriv_solve_kernel<T, false, false>;
  int bps_world = 0, bps_solve = 0;
  if (int rc = kernel_config((const void*)kworld, kNT, world_smem, p, bps_world)) return rc;
  if (!r.inverse)
    if (int rc = kernel_config(hs ? (const void*)ksolve_s : (const void*)ksolve_g, 32 * bestW, solve_smem, p, bps_solve)) return rc;
  const int ncomp = kBodyRows + (ext ? 6 : 0);
  auto at = [](auto* ptr, int64_t b0) { return ptr ? ptr + b0 : nullptr; };
  for (int64_t b0 = 0; b0 < B; b0 += C) {
    const int64_t c = std::min<int64_t>(C, B - b0);
    T* vd = r.vd + b0;
    // v̇ itself: the library's own forward dynamics (model-specialised kernels when available)
    if (!r.inverse && !r.vd_given)
      if (int rc = rbd_dynamics(model, dtype, c, ld, r.q + b0, r.v + b0, at(r.tau_in, b0), at(r.wext, b0), vd, nullptr, stream)) return rc;
    DerivArgs<T> a{r.q + b0, r.v + b0, vd, r.dq + b0, r.dv + b0, scratch, ld, sld, c,
                   at(r.wext, b0), at(r.dtau, b0), at(r.tau_out, b0), at(r.M, b0)};
    const int gx = (int)((c + kNT - 1) / kNT);
    const LaunchShape world{std::min(gx, 8 * p.sms), kNT, (int)world_smem}, accum{gx * ncomp, kNT}, pairs{gx * D.nb, kNT},
        factor{gx, kNT}, expand{gx * D.nv, kNT};
    kworld<<<world.grid, kNT, world_smem, stream>>>(M, D, a);
    if (int rc = api_launched(&world)) return rc;
    kaccum<<<dim3(gx, ncomp), kNT, 0, stream>>>(M, D, a);
    if (int rc = api_launched(&accum)) return rc;
    kpairs<<<dim3(D.nb, gx), kNT, 0, stream>>>(D, A, a);
    if (int rc = api_launched(&pairs)) return rc;
    if (r.inverse) {
      deriv_expand_kernel<T, kNT><<<dim3(gx, D.nv), kNT, 0, stream>>>(D, a);
      if (int rc = api_launched(&expand)) return rc;
      continue;
    }
    if (!hs) {
      deriv_factor_kernel<T, kNT><<<gx, kNT, 0, stream>>>(D, A, a);
      if (int rc = api_launched(&factor)) return rc;
    }
    if (js) {
      const T* Hg = scratch + (int64_t)D.h_base * sld;
      long long sld_ = sld, ld_ = ld, c_ = c;
      T* dq_ = r.dq + b0; T* dv_ = r.dv + b0; T* dt_ = a.dtau;
      void* params[] = {(void*)&Hg, (void*)&sld_, (void*)&dq_, (void*)&dv_, (void*)&ld_, (void*)&c_, (void*)&dt_};   // 2 blocks: the first 6
      const LaunchShape solve{(int)std::min<int64_t>((c + 31) / 32, (int64_t)js->bps * p.sms), 32 * js->plan.warps, (int)js->smem, js->bps};
      RBD_CUDA_TRY(cudaLaunchKernel((const void*)js->kernel, dim3(solve.grid), dim3(solve.block), params, js->smem, stream));
      api_note_launch(&solve);
      continue;
    }
    const LaunchShape solve{(int)std::min<int64_t>((c + 31) / 32, (int64_t)bestNb * p.sms), 32 * bestW, (int)solve_smem, bestNb};
    if (hs) ksolve_s<<<solve.grid, dim3(32, bestW), solve_smem, stream>>>(D, A, a);
    else ksolve_g<<<solve.grid, dim3(32, bestW), solve_smem, stream>>>(D, A, a);
    if (int rc = api_launched(&solve)) return rc;
  }
  return RBD_OK;
}

// rbd_dynamics_derivatives and its _ext form: one set of checks, one implementation
int32_t derivatives_entry(const char* fn, const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                          const void* tau, const void* wext, void* vd_out, void* dvd_dq_out, void* dvd_dv_out, void* dvd_dtau_out,
                          void* stream) {
  if (int rc = api_check(model, dtype, B, ld)) return rc;
  const ApiCall call;
  if (B == 0) return RBD_OK;
  if (!q || !v || !vd_out || !dvd_dq_out || !dvd_dv_out)
    return api_fail(RBD_EINVAL, std::string(fn) + ": q, v, vd_out, dvd_dq_out and dvd_dv_out must not be NULL");
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype == RBD_F32) {
    const DerivCall<float> r{false, (const float*)q, (const float*)v, (const float*)tau, (const float*)wext, (float*)vd_out,
                             (float*)dvd_dq_out, (float*)dvd_dv_out, (float*)dvd_dtau_out, nullptr, nullptr};
    return derivatives_t<float>(fn, model, dtype, B, ld, r, s);
  }
  const DerivCall<double> r{false, (const double*)q, (const double*)v, (const double*)tau, (const double*)wext, (double*)vd_out,
                            (double*)dvd_dq_out, (double*)dvd_dv_out, (double*)dvd_dtau_out, nullptr, nullptr};
  return derivatives_t<double>(fn, model, dtype, B, ld, r, s);
}

}  // namespace

namespace rbd {
int dynamics_derivatives_dense(const rbd_model* model, int32_t dtype, int64_t B, const void* q, const void* v, const void* tau,
                               const void* vd, void* dq, void* dv, void* dtau, cudaStream_t stream) {
  const char* fn = "rbd_integrate_derivatives";
  if (dtype == RBD_F32) {
    DerivCall<float> r{false, (const float*)q, (const float*)v, (const float*)tau, nullptr, (float*)const_cast<void*>(vd),
                       (float*)dq, (float*)dv, (float*)dtau, nullptr, nullptr};
    r.vd_given = true;
    return derivatives_t<float>(fn, model, dtype, B, B, r, stream);
  }
  DerivCall<double> r{false, (const double*)q, (const double*)v, (const double*)tau, nullptr, (double*)const_cast<void*>(vd),
                      (double*)dq, (double*)dv, (double*)dtau, nullptr, nullptr};
  r.vd_given = true;
  return derivatives_t<double>(fn, model, dtype, B, B, r, stream);
}
}  // namespace rbd

extern "C" int32_t rbd_dynamics_derivatives_ext(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                                                const void* tau, const void* wext, void* vd_out, void* dvd_dq_out, void* dvd_dv_out,
                                                void* dvd_dtau_out, void* stream) {
  return derivatives_entry("rbd_dynamics_derivatives_ext", model, dtype, B, ld, q, v, tau, wext, vd_out, dvd_dq_out, dvd_dv_out, dvd_dtau_out,
                           stream);
}

extern "C" int32_t rbd_dynamics_derivatives(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                                            const void* tau, void* vd_out, void* dvd_dq_out, void* dvd_dv_out, void* stream) {
  return derivatives_entry("rbd_dynamics_derivatives", model, dtype, B, ld, q, v, tau, nullptr, vd_out, dvd_dq_out, dvd_dv_out, nullptr,
                           stream);
}

extern "C" int32_t rbd_inverse_dynamics_derivatives(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q,
                                                    const void* v, const void* vd, const void* wext, void* tau_out, void* dtau_dq_out,
                                                    void* dtau_dv_out, void* M_out, void* stream) {
  if (int rc = api_check(model, dtype, B, ld)) return rc;
  const ApiCall call;
  if (B == 0) return RBD_OK;
  if (!q || !v || !vd || !dtau_dq_out || !dtau_dv_out)
    return api_fail(RBD_EINVAL, "rbd_inverse_dynamics_derivatives: q, v, vd, dtau_dq_out and dtau_dv_out must not be NULL");
  cudaStream_t s = (cudaStream_t)stream;
  const char* fn = "rbd_inverse_dynamics_derivatives";
  if (dtype == RBD_F32) {
    const DerivCall<float> r{true, (const float*)q, (const float*)v, nullptr, (const float*)wext, (float*)const_cast<void*>(vd),
                             (float*)dtau_dq_out, (float*)dtau_dv_out, nullptr, (float*)tau_out, (float*)M_out};
    return derivatives_t<float>(fn, model, dtype, B, ld, r, s);
  }
  const DerivCall<double> r{true, (const double*)q, (const double*)v, nullptr, (const double*)wext, (double*)const_cast<void*>(vd),
                            (double*)dtau_dq_out, (double*)dtau_dv_out, nullptr, (double*)tau_out, (double*)M_out};
  return derivatives_t<double>(fn, model, dtype, B, ld, r, s);
}

// Ahead-of-time compilation of the model's solve kernel into the cubin cache (no GPU needed): the analogue of rbd_model_precompile
// for this entry point.  RBD_EUNSUPPORTED if NVRTC is missing or the model does not qualify (the generic kernel then serves it).
static int32_t precompile_derivatives(rbd_model* model, int32_t dtype, bool dtau, const char* fn) {
  if (!model) return api_fail(RBD_EINVAL, "model handle is NULL");
  if (dtype != RBD_F32 && dtype != RBD_F64) return api_fail(RBD_EINVAL, std::string(fn) + ": fp32 / fp64 only");
  DerivDev D;
  DerivAnc A;
  if (!build_deriv_dev(model->hm.dev64, D, A)) return api_fail(RBD_EUNSUPPORTED, "model too large for rbd_dynamics_derivatives");
  DerivJitPlan plan;
  std::vector<char> cubin;
  std::string err;
  if (!jit_solve_cubin(D, A, dtype == RBD_F64, dtau, true, plan, cubin, err)) return api_fail(RBD_EUNSUPPORTED, err);
  return RBD_OK;
}
extern "C" int32_t rbd_model_precompile_derivatives(rbd_model* model, int32_t dtype) {
  return precompile_derivatives(model, dtype, false, "rbd_model_precompile_derivatives");
}
extern "C" int32_t rbd_model_precompile_derivatives_ext(rbd_model* model, int32_t dtype, int32_t with_dtau) {
  return precompile_derivatives(model, dtype, with_dtau != 0, "rbd_model_precompile_derivatives_ext");
}
