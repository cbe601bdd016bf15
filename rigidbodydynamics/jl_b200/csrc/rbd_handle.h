// The opaque model handle of the C ABI (include/rbd_b200.h) and the host plumbing that every translation unit of the library
// launches through (rbd_b200.cu: generic kernels, entry points; rbd_spec.cpp: model-specialised kernels; rbd_deriv.cu, rbd_loops.cu,
// rbd_adjoint.cu, rbd_integrate_vjp.cu).
#pragma once
#include <cuda_runtime.h>

#include <map>
#include <memory>
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
// Tries the model-specialised kernels for (model, key) and notes the launch as specialised.  `used` = false (and RBD_OK) when
// they are unavailable, not yet compiled and the batch is below the compile threshold, or the batch is too small: the caller
// then runs the generic kernels.  `gate` (fp32 only, else NULL): device flag the specialised kernels raise when a sample needs
// the library sin / cos; the caller must enqueue the generic kernel gated on it right behind (under a KeepLaunchRecord).
int spec_try_launch(rbd_model* m, const SpecKey& key, const SpecLaunchArgs& a, cudaStream_t stream, bool& used, const int** gate);
// Compile (or load from the cubin cache) without launching; RBD_OK / RBD_EUNSUPPORTED.
int spec_prepare(rbd_model* m, const SpecKey& key, bool load_on_device, std::string& err);
void spec_release(rbd_model* m);
// RBD_JIT_VARIANT (read at every call): 1 = shared-memory kernels only, 2 = the specialised kernels use the mixed CTA, 0 = unset
int jit_variant();

// ---- host plumbing shared by the library's translation units (rbd_b200.cu implements it) ----------------------------------
// Per-thread error text and argument checks.  A failed CUDA call returns RBD_ENOMEM if it was an allocation, else RBD_ECUDA.
int api_fail(int status, const std::string& msg);
int api_fail_cuda(cudaError_t e, const std::string& what);
#define RBD_CUDA_TRY(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) return ::rbd::api_fail_cuda(e_, #expr); } while (0)
int api_check(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld);

// The current device, cached per device.  The first query on a device keeps freed blocks of its stream-ordered pool cached
// (cudaMemPoolAttrReleaseThreshold): every entry point takes its workspaces from that pool per call.
struct DeviceProps { int dev = 0, sms = 0, max_smem_optin = 0, smem_per_sm = 0, l2_bytes = 0; };
cudaError_t device_props(DeviceProps& p);
// Checks that `smem` bytes of dynamic shared memory fit a block, opts the kernel into large dynamic shared memory with the
// maximum shared-memory carveout ONCE per (kernel, device) -- the attribute is process-global per kernel, so setting it to each
// call's exact size would race between host threads using different model handles -- and returns the resident blocks per SM.
// Kernels without dynamic shared memory keep the default carveout (their workspace traffic goes through L1).
int kernel_config(const void* kernel, int block, size_t smem, const DeviceProps& p, int& blocks_per_sm);

// A stream-ordered allocation, freed on its stream when it goes out of scope (after the launches using it were enqueued).
struct StreamAlloc {
  void* p = nullptr;
  cudaStream_t stream = nullptr;
  StreamAlloc() = default;
  StreamAlloc(const StreamAlloc&) = delete;
  StreamAlloc& operator=(const StreamAlloc&) = delete;
  ~StreamAlloc() { if (p) cudaFreeAsync(p, stream); }
  cudaError_t alloc(size_t bytes, cudaStream_t s) { stream = s; return cudaMallocAsync(&p, bytes, s); }
};

// Launch record (rbd_get_launch_info): the outermost C-ABI call on a thread resets it (one ApiCall at its entry); calls nested
// in it (rbd_dynamics_result -> rbd_dynamics, rbd_dynamics_derivatives -> rbd_dynamics) add to it.
struct ApiCall {
  ApiCall();
  ~ApiCall();
  ApiCall(const ApiCall&) = delete;
  ApiCall& operator=(const ApiCall&) = delete;
};
struct LaunchShape { int grid = 0, block = 0, smem = 0, blocks_per_sm = 0; };
// Counts one enqueued kernel.  With a shape the record describes that kernel; the elementwise kernels around the dynamics
// kernels (RK4 stages, integrate-VJP phases, the gather scatter) are counted only.
void api_note_launch(const LaunchShape* shape = nullptr, bool specialised = false);
// The status of the kernel launch just enqueued (cudaGetLastError); noted as above when it succeeded.
int api_launched(const LaunchShape* shape = nullptr);
// Restores the record, except its count, at scope exit: a gated generic fallback (and rbd_dynamics_result's by-products) add
// their launches while the record keeps describing the kernel that serves the call.
struct KeepLaunchRecord {
  rbd_launch_info saved;
  KeepLaunchRecord();
  ~KeepLaunchRecord();
  KeepLaunchRecord(const KeepLaunchRecord&) = delete;
  KeepLaunchRecord& operator=(const KeepLaunchRecord&) = delete;
};

// A persistent launch: min(groups, blocks_per_SM x SMs) blocks of `block` threads looping over the groups, plus -- when
// `work_per_thread` > 0 -- a stream-ordered workspace of that many bytes per resident thread (and `work_extra` bytes behind it),
// freed when the plan goes out of scope.  `work_cap` > 0 trims the grid so that the workspace stays within that many bytes.
// The caller launches `kernel<<<grid, block, smem, stream>>>` with its own arguments, then returns api_launched(&plan).
struct LaunchPlan : LaunchShape { StreamAlloc work; };
int plan_persistent(const void* kernel, int block, size_t smem, int64_t ngroups, cudaStream_t stream, LaunchPlan& plan,
                    size_t work_per_thread = 0, size_t work_extra = 0, size_t work_cap = 0);
// One request to rbd_b200.cu's RK4 driver, in the form the C entry points receive it (include/rbd_b200.h).  q, v and the contact
// state s are [rows x B] with leading dimension ld; the torques of (step s, stage i) start at tau + s * tau_step_stride +
// i * tau_stage_stride (NULL: zero).
struct Rollout {
  void* q; void* v; void* s;
  const void* tau;
  int64_t tau_step_stride, tau_stage_stride;
  double dt;
  int nsteps;
  void* q_traj = nullptr; void* v_traj = nullptr; void* s_traj = nullptr;   // [(nsteps + 1) x rows x B] each, or all NULL
  void* stages = nullptr;                      // rbd_integrate_vjp's recompute, see stage_rows
  const rbd_contact_desc* contact = nullptr;   // the contact rollout, or the loop rollout's contact pass
  const rbd_loop_desc* loops = nullptr;        // every stage's dynamics is the KKT solve (loop_stage_launch)
  const rbd_pd_desc* pd = nullptr;             // feedback evaluated at every stage
  const void* pd_bounds = nullptr;             // pd's effort bounds already on the device ([2 nv]: lo, then hi), or NULL: integrate
                                               // copies them from the host arrays of pd (rbd_integrate_pd_vjp's recompute passes its copy)
  const rbd_task_pd_desc* task = nullptr;      // task-space feedback at every stage (pd NULL; its joint term takes pd's place);
                                               // never set together with `stages`
};
// The recompute of one step (nsteps = 1, ld = B) keeps its four stages in stage_rows(nq, nv) x B rows of `stages` (4 ns more with
// contact, for the ṡ_i) and skips the finishing step.  With a controller (pd) pd_stage_rows(nv, computed_torque) x B more follow:
// the four stages' applied torques τ_i (nv rows each), then in computed-torque mode the four v̇_des,i (nv rows each), the
// inverse dynamics' input; rbd_integrate_pd_vjp's adjoint reads both.
inline int64_t stage_rows(int64_t nq, int64_t nv) { return 4 * nq + 12 * nv; }
inline int64_t pd_stage_rows(int64_t nv, bool computed_torque) { return (computed_torque ? 8 : 4) * nv; }
// Runs the rollout (fp32 / fp64, arguments checked by the caller).  RBD_OK at once when B == 0, or when nsteps == 0 and nothing is
// recorded.  The loop rollout takes its contact pass only when there are contact pairs.
int integrate(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const Rollout& r, cudaStream_t stream);
// rbd_loops.cu's forward dynamics of one stage of the loop rollout: v̇ = the KKT solve of rbd_dynamics_loops at the stage state
// (q, v) with torques tau (NULL: zero), every array [rows x B] dense.  With `contact` (ns > 0) the contact pass runs first in the
// same kernel at the stage state s0 + wa ṡ_prev (ṡ_prev NULL at stage 0), writes ṡ and feeds its wrenches to the solve.  `plan`
// starts empty; the first stage fills it (device descriptors, grid, workspace) and the caller keeps it for every stage of the call.
struct LoopStagePlan;
struct LoopStageArgs {
  const void* q; const void* v; const void* tau;
  const void* s0; const void* sdp; void* sd;     // contact state (contact only)
  void* vd;
  double wa;                                     // dt a_i
  int64_t B;
};
int loop_stage_launch(const rbd_model* model, int32_t dtype, const rbd_loop_desc& loops, const rbd_contact_desc* contact,
                      const LoopStageArgs& a, std::shared_ptr<LoopStagePlan>& plan, cudaStream_t stream);
// rbd_b200.cu's descriptor checks of rbd_contact_dynamics (fn: the entry point named in the message)
int api_check_contact(const rbd_model* model, const rbd_contact_desc* contact, const char* fn);
// rbd_loops.cu's descriptor checks of rbd_dynamics_loops
int api_check_loops(const rbd_model* model, const rbd_loop_desc* loops);
// rbd_adjoint.cu's forward-dynamics VJP on dense [rows x B] arrays (no external wrenches); outputs may be NULL
int dynamics_vjp_dense(const rbd_model* model, int32_t dtype, int64_t B, const void* q, const void* v, const void* vd, const void* vd_bar,
                       void* q_bar_cfg, void* v_bar, void* tau_bar, cudaStream_t stream);
// ... and the inverse-dynamics VJP on dense arrays (no external wrenches): q̄_cfg, v̄, v̇̄ of τ = ID(q, v, v̇) from τ̄; outputs may be NULL
int inverse_dynamics_vjp_dense(const rbd_model* model, int32_t dtype, int64_t B, const void* q, const void* v, const void* vd,
                               const void* tau_bar, void* q_bar_cfg, void* v_bar, void* vd_bar, cudaStream_t stream);
// The model limits of rbd_dynamics_vjp / rbd_inverse_dynamics_vjp (those of rbd_dynamics_derivatives): RBD_OK or RBD_EUNSUPPORTED
int check_vjp_limits(const HostModel& hm, const char* who);
// rbd_b200.cu's controller checks of rbd_integrate_task_pd (the joint term's JointPD checks, then check_task_pd), leading dimension ld
int api_check_task_ctrl(const char* fn, const rbd_model* model, int64_t ld, const rbd_task_pd_desc* ctrl);
// rbd_task_pd_torques on dense [rows x B] arrays (arguments checked by the caller): tau_out the applied torques; in computed-torque
// mode also v̇_des, the inverse dynamics' input, into vdes_out [nv x B] when it is not NULL
int task_pd_law(const rbd_model* model, int32_t dtype, int64_t B, const void* q, const void* v, const void* tau_ff, const rbd_task_pd_desc& c,
                int step, void* tau_out, void* vdes_out, cudaStream_t stream);

}  // namespace rbd
