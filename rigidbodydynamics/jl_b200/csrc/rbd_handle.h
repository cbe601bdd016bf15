// The opaque model handle of the C ABI (include/rbd_b200.h), shared by rbd_b200.cu (generic kernels, entry points) and
// rbd_spec.cpp (model-specialised kernels).
#pragma once
#include <cuda_runtime.h>

#include <map>
#include <mutex>
#include <string>

#include "../../../include/rbd_b200.h"
#include "rbd_codegen.h"
#include "rbd_model.h"

namespace rbd {

// One model-specialised program, loaded from a cubin: shared-memory blocks and the mixed shared-memory / L2 CTA.
struct SpecEntry {
  int state = 0;                 // 0 = not tried, 1 = ready, -1 = unavailable (generic kernels are used)
  cudaLibrary_t lib = nullptr;
  cudaKernel_t k_smem = nullptr, k_mix = nullptr;
  int regs_smem = 0, regs_mix = 0;
  int mix_sw = 0;                // warps of the mixed CTA whose stash fits its shared memory
  int choice = 0;                // 0 = not timed yet, 1 = shared-memory blocks, 2 = mixed CTA (for batches that fill the SMs)
  int rows = 0;
  bool from_cache = false;
  std::string why;               // reason for state -1
  int8_t kin_sign[kMaxBodies] = {0};   // SPEC_KIN: the path this entry was generated for
  bool kin_set = false;
};

constexpr int kCounterRing = 256;   // work-queue counters, one per call in flight

}  // namespace rbd

struct rbd_model {
  rbd::HostModel hm;
  // staging for the *_host entry points (allocated on first use, owned by the handle)
  std::mutex host_mu;
  void* d_stage[3] = {nullptr, nullptr, nullptr};
  size_t stage_bytes = 0;
  cudaStream_t streams[3] = {nullptr, nullptr, nullptr};
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  // work queues of the model-specialised kernels (per device)
  std::mutex queue_mu;
  int queue_device = -1;
  unsigned long long* counters = nullptr;     // [kCounterRing][2] device memory: work-queue counter, "needs generic kernel" flag
  unsigned next_call = 0;
  // model-specialised kernels, keyed by SpecKey bits
  std::mutex spec_mu;
  std::map<uint64_t, rbd::SpecEntry> spec;
};

namespace rbd {

// Resources of one work-queue launch: a zeroed work-queue counter and flag (the zeroing is enqueued on `stream`).
struct QueueCtx {
  unsigned long long* counter = nullptr;
  int* flag = nullptr;       // zeroed with the counter; raised by a specialised kernel that met an angle beyond its fast sin / cos
};
// Returns a cudaError_t (cudaSuccess = 0).
cudaError_t queue_begin(rbd_model* m, cudaStream_t stream, QueueCtx& ctx);

inline uint64_t spec_key_bits(const SpecKey& k) {
  uint64_t b = (uint64_t)k.algo | (k.f64 ? 8u : 0u) | (k.has_in2 ? 16u : 0u) | (k.has_out1 ? 32u : 0u) | (k.lower ? 64u : 0u) | (k.peers ? 128u : 0u);
  if (k.algo == SPEC_KIN) {      // output subset and jacobian path: 8 mask bits + a 40-bit hash of the path signs (the entry keeps the
    uint64_t h = 1469598103934665603ull;   // signs themselves and is only used when they match, see spec_try_launch)
    for (int i = 0; i < kMaxBodies; ++i) { h ^= (uint8_t)k.kin_sign[i]; h *= 1099511628211ull; }
    b |= ((uint64_t)(k.kin_mask & 0xff) << 8) | ((h >> 24) << 24);
  }
  return b;
}

struct SpecLaunchArgs {
  const void* q; const void* v; const void* in2;
  void* o0; void* o1;
  int64_t ld, B;
  // key.peers: o0 is unused; row k of sample b goes to peers[p][k * peer_ld + peer_col0 + b] for every p < npeers
  void* const* peers = nullptr;
  void* mc = nullptr;            // NVLS multicast mapping of the peers' arrays, or NULL
  int npeers = 0;
  int64_t peer_ld = 0, peer_col0 = 0;
  void* ko[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // SPEC_KIN: the rbd_kinematics_out pointers
};
// Tries the model-specialised kernels for (model, key).  `used` = false (and RBD_OK) when they are unavailable, not yet
// compiled and the batch is below the compile threshold, or the batch is too small: the caller then runs the generic kernels.
// `gate` (fp32 only, else NULL): device flag the specialised kernels raise when a sample needs the library sin / cos; the caller
// must enqueue the generic kernel gated on it right behind.
int spec_try_launch(rbd_model* m, const SpecKey& key, const SpecLaunchArgs& a, cudaStream_t stream, bool& used,
                    rbd_launch_info& li, const int** gate, std::string& err);
// Compile (or load from the cubin cache) without launching; RBD_OK / RBD_EUNSUPPORTED.
int spec_prepare(rbd_model* m, const SpecKey& key, bool load_on_device, std::string& err);
void spec_release(rbd_model* m);

// rbd_b200.cu's per-thread error text / argument checks / launch statistics, for the library's other translation units
int api_fail(int status, const std::string& msg);
int api_check(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld);
void api_note_launch(int grid, int block, int smem_bytes, int blocks_per_sm);
// rbd_b200.cu's RK4 driver for rbd_integrate_trajectory (q_traj / v_traj) and rbd_integrate_vjp's recompute (stages: one step,
// its four stages kept in stage_rows(nq, nv) x B rows, no finishing step).  fp32 / fp64, arguments checked by the caller.
inline int64_t stage_rows(int64_t nq, int64_t nv) { return 4 * nq + 12 * nv; }
int integrate_record(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, void* q, void* v, const void* tau, int64_t step_stride,
                     int64_t stage_stride, double dt, int nsteps, void* q_traj, void* v_traj, void* stages, cudaStream_t stream);
// rbd_adjoint.cu's forward-dynamics VJP on dense [rows x B] arrays (no external wrenches); outputs may be NULL
int dynamics_vjp_dense(const rbd_model* model, int32_t dtype, int64_t B, const void* q, const void* v, const void* vd, const void* vd_bar,
                       void* q_bar_cfg, void* v_bar, void* tau_bar, cudaStream_t stream);

}  // namespace rbd
