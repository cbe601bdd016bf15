// Model-specialised kernels: compile (rbd_jit.cpp), load (cudaLibraryLoadData) and launch.  Host-only C++ on the CUDA runtime.
//
// The kernels are persistent and claim groups of 32 samples from one counter: single-warp blocks with their stash in shared
// memory, or one mixed CTA per SM whose extra warps keep their stash in L2 (rbd_jit_kernels.cuh).  Device properties, error
// mapping and the launch record are the shared plumbing of rbd_handle.h; the cubin kernels get exact shared-memory sizes here.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "rbd_handle.h"
#include "rbd_jit.h"

namespace rbd {
namespace {

constexpr int kMixWarps = 16;       // warps of the mixed CTA: 16 x 32 threads x 128 registers = the whole register file

struct Env {
  bool jit = true;
  int64_t min_batch = 1 << 15;      // below this a missing cubin is not compiled on the fly (generic kernels serve the call)
  Env() {
    if (const char* e = getenv("RBD_JIT")) jit = e[0] != '0';
    if (const char* e = getenv("RBD_JIT_MIN_BATCH")) min_batch = atoll(e);
  }
};
const Env& env() { static const Env e; return e; }

}  // namespace

int jit_variant() {
  const char* e = getenv("RBD_JIT_VARIANT");
  return e ? atoi(e) : 0;
}

cudaError_t queue_begin(rbd_model* m, cudaStream_t stream, QueueCtx& ctx) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  unsigned slot;
  {
    std::lock_guard<std::mutex> lk(m->queue_mu);
    if (m->queue_device != dev) {       // first use (or the caller moved to another device): (re)allocate the counters
      if (m->counters) { cudaFree(m->counters); m->counters = nullptr; }
      if ((e = cudaMalloc((void**)&m->counters, kCounterRing * 2 * sizeof(unsigned long long))) != cudaSuccess) return e;
      m->queue_device = dev;
    }
    slot = m->next_call++;
  }
  ctx.counter = m->counters + 2 * (slot % kCounterRing);
  ctx.flag = reinterpret_cast<int*>(ctx.counter + 1);
  return cudaMemsetAsync(ctx.counter, 0, 2 * sizeof(unsigned long long), stream);
}

void spec_release(rbd_model* m) {
  std::lock_guard<std::mutex> lk(m->spec_mu);
  for (auto& kv : m->spec) if (kv.second.lib) cudaLibraryUnload(kv.second.lib);
  m->spec.clear();
}

// Straight-line programs far beyond the instruction caches run at the SM's instruction-fetch rate instead of its issue rate,
// and an fp64 stash halves the resident warps: against the generic (looping, cache-resident) kernels the fp32 programs win,
// a large fp64 program (Atlas ABA) loses.  fp32 programs are therefore always specialised, fp64 programs only below an
// estimated size.
bool spec_worthwhile(const HostModel& hm, const SpecKey& key) {
  if (!key.f64) return true;
  // small stashes (CRBA: 2 rows per body, kinematics: the pending branch nodes only): fp64 keeps its resident warps
  if (key.algo == SPEC_CRBA || key.algo == SPEC_KIN) return true;
  const int est = hm.nb * (key.algo == SPEC_ABA ? 410 : 190);
  return est <= 6500;
}

int spec_prepare(rbd_model* m, const SpecKey& key, bool load_on_device, std::string& err) {
  std::lock_guard<std::mutex> lk(m->spec_mu);
  SpecEntry& se = m->spec[spec_key_bits(key)];
  if (se.state == 1) return RBD_OK;
  if (se.state == -1 && load_on_device) { err = se.why; return RBD_EUNSUPPORTED; }
  std::vector<char> cubin;
  bool cached = false;
  if (!jit_get_cubin(m->hm, key, cubin, true, &cached, nullptr, err)) {
    se.state = -1; se.why = err;
    return RBD_EUNSUPPORTED;
  }
  if (!load_on_device) return RBD_OK;      // precompile only (CPU build step): the cubin is in the cache now
  cudaError_t e = cudaLibraryLoadData(&se.lib, cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0);
  if (e == cudaSuccess) e = cudaLibraryGetKernel(&se.k_smem, se.lib, "rbd_jit_smem");
  if (e == cudaSuccess) e = cudaLibraryGetKernel(&se.k_mix, se.lib, "rbd_jit_mix");
  cudaFuncAttributes fa{};
  if (e == cudaSuccess) { e = cudaFuncGetAttributes(&fa, (const void*)se.k_smem); se.regs_smem = fa.numRegs; }
  if (e == cudaSuccess) { e = cudaFuncGetAttributes(&fa, (const void*)se.k_mix); se.regs_mix = fa.numRegs; }
  se.rows = spec_shared_rows(m->hm, key);       // one warp's shared rows: stash (the others are registers) and trig cache
  const size_t smem = (size_t)std::max(1, se.rows) * 32 * (key.f64 ? 8 : 4);
  DeviceProps p;
  if (e == cudaSuccess) e = device_props(p);
  se.mix_sw = std::min<int>(kMixWarps, (int)(p.max_smem_optin / smem));
  if (e == cudaSuccess) e = cudaFuncSetAttribute((const void*)se.k_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e == cudaSuccess) e = cudaFuncSetAttribute((const void*)se.k_smem, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  if (e == cudaSuccess && se.mix_sw > 0)
    e = cudaFuncSetAttribute((const void*)se.k_mix, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(smem * se.mix_sw));
  if (e == cudaSuccess) e = cudaFuncSetAttribute((const void*)se.k_mix, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  if (e != cudaSuccess) {
    cudaGetLastError();
    se.state = -1;
    se.why = err = std::string("loading the specialised cubin: ") + cudaGetErrorString(e);
    if (se.lib) { cudaLibraryUnload(se.lib); se.lib = nullptr; }
    return RBD_EUNSUPPORTED;
  }
  se.from_cache = cached;
  se.state = 1;
  return RBD_OK;
}

int spec_try_launch(rbd_model* m, const SpecKey& key, const SpecLaunchArgs& a, cudaStream_t stream, bool& used, const int** gate) {
  used = false;
  if (gate) *gate = nullptr;
  const Env& ev = env();
  if (!ev.jit || !spec_worthwhile(m->hm, key)) return RBD_OK;
  if (a.ld * (key.f64 ? 8 : 4) >= (1ll << 32)) return RBD_OK;   // the generated code forms row offsets as 32 x 32 -> 64-bit products of the byte stride
  const int rows = spec_stash_rows(m->hm, key);
  if (rows > 256) return RBD_OK;                     // larger stashes leave too few warps per SM: the generic kernels serve
  DeviceProps p;
  RBD_CUDA_TRY(device_props(p));
  const size_t es = key.f64 ? 8 : 4;
  if ((size_t)std::max(1, rows) * 32 * es > (size_t)p.max_smem_optin) return RBD_OK;
  SpecEntry* se = nullptr;
  {
    std::lock_guard<std::mutex> lk(m->spec_mu);
    se = &m->spec[spec_key_bits(key)];
  }
  if (key.algo == SPEC_KIN) {        // the 64-bit map key carries only a hash of the jacobian path: use the entry only for ITS path
    std::lock_guard<std::mutex> lk(m->spec_mu);
    if (!se->kin_set) { std::memcpy(se->kin_sign, key.kin_sign, sizeof se->kin_sign); se->kin_set = true; }
    else if (std::memcmp(se->kin_sign, key.kin_sign, sizeof se->kin_sign) != 0) return RBD_OK;
  }
  if (se->state == -1) return RBD_OK;
  if (se->state == 0) {
    if (a.B < ev.min_batch) {          // small call and nothing loaded yet: use a cached cubin if there is one, never compile
      std::vector<char> probe;
      std::string e2;
      bool cached = false;
      if (!jit_get_cubin(m->hm, key, probe, false, &cached, nullptr, e2)) return RBD_OK;
    }
    std::string e2;
    if (spec_prepare(m, key, true, e2) != RBD_OK) {      // generic kernels take over; the reason is kept in the entry
      if (getenv("RBD_JIT_VERBOSE")) fprintf(stderr, "[rbd_b200] specialised kernels unavailable: %s\n", e2.c_str());
      return RBD_OK;
    }
  }
  const int64_t ngroups = (a.B + 31) / 32;
  const size_t smem = (size_t)std::max(1, se->rows) * 32 * es;      // shared-memory stash of one warp
  // Experiments only (tools/time_stash.py): RBD_JIT_SMEM_PAD_BLOCKS=k pads the single-warp blocks' shared memory so that at most
  // k of them fit on an SM, to measure throughput against resident warps with the program unchanged.
  size_t smem_blk = smem;
  if (const char* e = getenv("RBD_JIT_SMEM_PAD_BLOCKS")) {
    const int k = atoi(e);
    if (k > 0) smem_blk = std::max(smem, std::min((size_t)p.max_smem_optin, (size_t)(p.smem_per_sm / k) - 1024));
    RBD_CUDA_TRY(cudaFuncSetAttribute((const void*)se->k_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_blk));
  }
  int bps = 0;
  RBD_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, (const void*)se->k_smem, 32, smem_blk));
  if (bps < 1) return RBD_OK;
  // The mixed CTA (rbd_jit_kernels.cuh) is worth trying when it puts at least 15 % more warps on the SM than shared-memory blocks
  // alone and there is a group of samples for each of its warps; which of the two is faster depends on the program, so the first
  // call large enough to tell times both once and keeps the winner (not while capturing a graph).  RBD_JIT_VARIANT=1 / 2 forces one.
  const int mix_warps = std::min(kMixWarps, 65536 / (((se->regs_mix + 7) / 8) * 8 * 32));
  const int mix_sw = std::min(se->mix_sw, mix_warps);
  const bool mix_ok = mix_sw >= 1 && mix_warps * 100 >= bps * 115 && ngroups >= (int64_t)mix_warps * p.sms;
  struct KArgs {
    const void* q; const void* v; const void* in2; void* o0; void* o1; long long ld, B; unsigned long long* counter; int* flag;
    void* peers[8]; long long peer_ld, peer_col0; void* mc; int npeers;
    void* ko[8];
    void* l2_stash; int smem_warps;
  };
  int* last_flag = nullptr;
  LaunchShape shape;
  auto run = [&](int variant) -> cudaError_t {        // 1 = shared-memory blocks, 2 = mixed CTA
    QueueCtx ctx;
    cudaError_t e = queue_begin(m, stream, ctx);
    if (e != cudaSuccess) return e;
    KArgs ka = {a.q, a.v, a.in2, a.o0, a.o1, (long long)a.ld, (long long)a.B, ctx.counter, ctx.flag, {}, (long long)a.peer_ld,
                (long long)a.peer_col0, a.mc, a.npeers, {}, nullptr, mix_sw};
    for (int i = 0; i < a.npeers && i < 8; ++i) ka.peers[i] = a.peers[i];
    for (int i = 0; i < 8; ++i) ka.ko[i] = a.ko[i];
    void* params[] = {&ka};
    if (variant == 2) {
      e = cudaMallocAsync(&ka.l2_stash, (size_t)(mix_warps - mix_sw) * p.sms * smem, stream);
      if (e == cudaSuccess) e = cudaLaunchKernel((const void*)se->k_mix, dim3(p.sms), dim3(32 * mix_warps), params, smem * mix_sw, stream);
      if (ka.l2_stash) cudaFreeAsync(ka.l2_stash, stream);
      shape = {p.sms, 32 * mix_warps, (int)(smem * mix_sw), 1};
    } else {
      const int grid = (int)std::min<int64_t>(ngroups, (int64_t)bps * p.sms);
      e = cudaLaunchKernel((const void*)se->k_smem, dim3(grid), dim3(32), params, smem_blk, stream);
      shape = {grid, 32, (int)smem_blk, bps};
    }
    last_flag = ctx.flag;
    return e;
  };
  cudaError_t e = cudaSuccess;
  int variant = 1;
  const int force = jit_variant();
  if (force && mix_ok) variant = force == 2 ? 2 : 1;
  else if (mix_ok) {
    variant = se->choice;
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(stream, &cap);
    if (variant == 0 && cap == cudaStreamCaptureStatusNone && a.B >= (int64_t)p.sms * 32 * 64) {
      // each variant once to warm up, then timed; the outputs are simply overwritten with the same values
      float best = 0.f;
      cudaEvent_t t0, t1;
      cudaEventCreate(&t0); cudaEventCreate(&t1);
      for (int v = 1; v <= 2 && e == cudaSuccess; ++v) {
        e = run(v);
        if (e == cudaSuccess) e = cudaEventRecord(t0, stream);
        if (e == cudaSuccess) e = run(v);
        if (e == cudaSuccess) e = cudaEventRecord(t1, stream);
        if (e == cudaSuccess) e = cudaEventSynchronize(t1);
        float ms = 0.f;
        if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, t0, t1);
        if (e == cudaSuccess && (variant == 0 || ms < best)) { best = ms; variant = v; }
      }
      cudaEventDestroy(t0); cudaEventDestroy(t1);
      if (e == cudaSuccess) se->choice = variant;
    }
    if (variant == 0) variant = 1;
  }
  if (e == cudaSuccess) e = run(variant);
  if (e != cudaSuccess) return api_fail_cuda(e, "specialised kernel launch");
  api_note_launch(&shape, true);
  if (gate && !key.f64) *gate = last_flag;
  used = true;
  return RBD_OK;
}

}  // namespace rbd
