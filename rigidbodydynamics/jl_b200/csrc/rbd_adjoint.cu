// rbd_dynamics_vjp / rbd_inverse_dynamics_vjp: reverse-mode products of dynamics! and inverse_dynamics! (csrc/rbd_adjoint.cuh has
// the mathematics); rbd_task_kinematics_vjp: the reverse mode of rbd_task_kinematics (csrc/rbd_task_adjoint.cuh).
//
// One generic persistent kernel per entry point, one thread per sample, one launch per call: blocks of one warp looping over groups
// of 32 samples, launched through plan_persistent (rbd_handle.h).  The per-sample working set -- 54 rows per body plus μ -- lives
// in its stream-ordered workspace of adjoint_rows() rows x RESIDENT threads, laid out [row][thread] so a warp's access to a row is
// one coalesced line; it is capped at kWorkspaceCap bytes by trimming the grid.  The forward VJP's solve
// (aba_sample) keeps its stash in shared memory like the generic ABA kernel.  The task VJP has the same structure, with
// task_adjoint_rows() rows per resident thread.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <memory>
#include <string>
#include <utility>

#include "../../../include/rbd_b200.h"
// rbd_sincos.cuh defines one out-of-line __device__ function with external linkage; this translation unit gets its own copy
#define sincos_slow sincos_slow_adjoint_tu
#include "rbd_adjoint.cuh"
#include "rbd_handle.h"
#include "rbd_task_adjoint.cuh"

using namespace rbd;

namespace {

constexpr int kNT = 32;                               // one warp per block; warps never synchronise
constexpr size_t kWorkspaceCap = size_t(512) << 20;   // bytes of workspace per call at most (fewer resident warps beyond it)

template <class T> struct VjpArgs {
  const T *q, *v, *vd, *wext, *wbar;            // wbar: ν̄ (forward) / τ̄ (inverse)
  T *qt, *qc, *vb, *vdb, *taub, *wb;            // outputs, NULL = not wanted
  T* work;                                      // [rows][grid * NT]
  const T* zero;                                // one 0 (the solve's velocity column)
  T g[3];                                       // gravity (the model passed to the forward kernel has g = 0)
  int64_t ld, B;
};

template <class T> __device__ __forceinline__ AdjIO<T> make_io(const VjpArgs<T>& a, int64_t bl, bool active, int64_t tid) {
  AdjIO<T> io;
  io.q = {a.q + bl, a.ld};
  io.v = {a.v + bl, a.ld};
  io.vd = {a.vd + bl, a.ld};
  io.wext = {a.wext ? a.wext + bl : nullptr, a.ld};
  io.qt = {a.qt ? a.qt + bl : nullptr, a.ld, active};
  io.qc = {a.qc ? a.qc + bl : nullptr, a.ld, active};
  io.vb = {a.vb ? a.vb + bl : nullptr, a.ld, active};
  io.vdb = {a.vdb ? a.vdb + bl : nullptr, a.ld, active};
  io.wb = {a.wb ? a.wb + bl : nullptr, a.ld, active};
  io.s = {a.work + tid, (int64_t)gridDim.x * kNT};       // workspace column of this resident thread
  return io;
}

// forward-dynamics VJP: M is the model with ZERO gravity (the solve); a.g carries the real one for the sweep
template <class T>
__global__ void __launch_bounds__(kNT, 1) dynamics_vjp_kernel(const __grid_constant__ ModelDev<T> M, const VjpArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const Stash<T, kNT> st{reinterpret_cast<T*>(smem_raw) + threadIdx.x};
  const int64_t tid = (int64_t)blockIdx.x * kNT + threadIdx.x;
  const int64_t ngroups = (a.B + kNT - 1) / kNT;
  for (int64_t g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const int64_t b = g * kNT + threadIdx.x;
    const bool active = b < a.B;
    const int64_t bl = active ? b : a.B - 1;      // inactive lanes recompute the last sample, stores are masked
    const AdjIO<T> io = make_io(a, bl, active, tid);
    const Col<T> wbar{a.wbar + bl, a.ld};
    const ColOut<T> taub{a.taub ? a.taub + bl : nullptr, a.ld, active};
    dynamics_vjp_sample<T>(M, a.g, io, wbar, taub, a.zero, st);
  }
}

template <class T>
__global__ void __launch_bounds__(kNT, 1) inverse_dynamics_vjp_kernel(const __grid_constant__ ModelDev<T> M, const VjpArgs<T> a) {
  const int64_t tid = (int64_t)blockIdx.x * kNT + threadIdx.x;
  const int64_t ngroups = (a.B + kNT - 1) / kNT;
  for (int64_t g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const int64_t b = g * kNT + threadIdx.x;
    const bool active = b < a.B;
    const int64_t bl = active ? b : a.B - 1;
    const AdjIO<T> io = make_io(a, bl, active, tid);
    adjoint_sample<T>(M, a.g, io, Col<T>{a.wbar + bl, a.ld}, T(1));
  }
}

template <class T>
int vjp_t(const rbd_model* model, bool fd, int64_t B, int64_t ld, VjpArgs<T> a, cudaStream_t stream) {
  const HostModel& hm = model->hm;
  ModelDev<T> M = dev_model<T>(hm);
  for (int k = 0; k < 3; ++k) a.g[k] = M.g[k];
  if (fd)
    for (int k = 0; k < 3; ++k) M.g[k] = T(0);
  const void* kernel = fd ? (const void*)dynamics_vjp_kernel<T> : (const void*)inverse_dynamics_vjp_kernel<T>;
  const size_t smem = fd ? (size_t)std::max(1, (int)M.nrows) * kNT * sizeof(T) : 0;
  const size_t row_bytes = (size_t)adjoint_rows(hm.nb, hm.nv) * sizeof(T);
  LaunchPlan pl;        // the workspace, then the zero
  if (int rc = plan_persistent(kernel, kNT, smem, (B + kNT - 1) / kNT, stream, pl, row_bytes, sizeof(T), kWorkspaceCap)) return rc;
  a.work = (T*)pl.work.p;
  a.zero = a.work + row_bytes / sizeof(T) * pl.grid * kNT;
  RBD_CUDA_TRY(cudaMemsetAsync(const_cast<T*>(a.zero), 0, sizeof(T), stream));
  if (fd) dynamics_vjp_kernel<T><<<pl.grid, pl.block, pl.smem, stream>>>(M, a);
  else inverse_dynamics_vjp_kernel<T><<<pl.grid, pl.block, pl.smem, stream>>>(M, a);
  return api_launched(&pl);
}

template <class T>
VjpArgs<T> args(int64_t B, int64_t ld, const void* q, const void* v, const void* vd, const void* wext, const void* wbar,
                void* qt, void* qc, void* vb, void* vdb, void* taub, void* wb) {
  VjpArgs<T> a{};
  a.q = (const T*)q; a.v = (const T*)v; a.vd = (const T*)vd; a.wext = (const T*)wext; a.wbar = (const T*)wbar;
  a.qt = (T*)qt; a.qc = (T*)qc; a.vb = (T*)vb; a.vdb = (T*)vdb; a.taub = (T*)taub; a.wb = (T*)wb;
  a.ld = ld; a.B = B;
  return a;
}

// ---- task-space kinematics VJP ----
template <class T> struct TaskVjpArgs {
  const T *q, *v, *vd;
  const T *tr, *pt, *tw, *pv, *J, *Jp, *acc, *pacc;   // cotangents, NULL = zero
  T *qt, *qc, *vb, *vdb;                              // outputs, NULL = not wanted
  T* work;                                            // [rows][grid * NT]
  int64_t ld, B;
};
static_assert(sizeof(ModelDev<double>) + sizeof(TaskDev<double>) + sizeof(TaskVjpArgs<double>) <= 32764,
              "task_vjp_kernel's parameters exceed the kernel-parameter limit");

template <class T>
__global__ void __launch_bounds__(kNT, 1)
task_vjp_kernel(const __grid_constant__ ModelDev<T> M, const __grid_constant__ TaskDev<T> D, const TaskVjpArgs<T> a) {
  const int64_t tid = (int64_t)blockIdx.x * kNT + threadIdx.x;
  const int64_t ngroups = (a.B + kNT - 1) / kNT;
  for (int64_t g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const int64_t b = g * kNT + threadIdx.x;
    const bool active = b < a.B;
    const int64_t bl = active ? b : a.B - 1;      // inactive lanes recompute the last sample, stores are masked
    TaskBarIO<T> io;
    auto in = [&](const T* p) { return Col<T>{p ? p + bl : nullptr, a.ld}; };
    auto out = [&](T* p) { return ColOut<T>{p ? p + bl : nullptr, a.ld, active}; };
    io.q = in(a.q); io.v = in(a.v); io.vd = in(a.vd);
    io.tr = in(a.tr); io.pt = in(a.pt); io.tw = in(a.tw); io.pv = in(a.pv);
    io.J = in(a.J); io.Jp = in(a.Jp); io.acc = in(a.acc); io.pacc = in(a.pacc);
    io.qt = out(a.qt); io.qc = out(a.qc); io.vb = out(a.vb); io.vdb = out(a.vdb);
    io.s = {a.work + tid, (int64_t)gridDim.x * kNT};
    task_vjp_sample<T>(M, D, io);
  }
}

// rows x B block of a [rows x ld] array set to zero
template <class T> int zero_rows(T* p, int rows, int64_t B, int64_t ld, cudaStream_t stream) {
  if (p && rows > 0) RBD_CUDA_TRY(cudaMemset2DAsync(p, ld * sizeof(T), 0, B * sizeof(T), rows, stream));
  return RBD_OK;
}

template <class T>
int task_vjp_t(const rbd_model* model, int64_t B, int64_t ld, const void* q, const void* v, const void* vd, const rbd_task_desc& d,
               const rbd_task_out& o, void* qt, void* qc, void* vb, void* vdb, cudaStream_t stream) {
  const HostModel& hm = model->hm;
  if (d.ntasks == 0) {                  // nothing depends on anything: the requested gradients are zero
    for (auto [p, rows] : {std::pair<void*, int>{qt, hm.nv}, {qc, hm.nq}, {vb, hm.nv}, {vdb, hm.nv}})
      if (int rc = zero_rows<T>((T*)p, rows, B, ld, stream)) return rc;
    return RBD_OK;
  }
  const ModelDev<T>& M = dev_model<T>(hm);
  std::unique_ptr<TaskDev<T>> D(new TaskDev<T>());
  const int nnamed = build_task_vjp_dev<T>(hm, d, *D);
  TaskVjpArgs<T> a{(const T*)q, (const T*)v, (const T*)vd, (const T*)o.transform, (const T*)o.point, (const T*)o.twist,
                   (const T*)o.point_velocity, (const T*)o.geometric_jacobian, (const T*)o.point_jacobian, (const T*)o.acceleration,
                   (const T*)o.point_acceleration, (T*)qt, (T*)qc, (T*)vb, (T*)vdb, nullptr, ld, B};
  const size_t row_bytes = (size_t)task_adjoint_rows(hm.nb, nnamed) * sizeof(T);
  LaunchPlan pl;
  if (int rc = plan_persistent((const void*)task_vjp_kernel<T>, kNT, 0, (B + kNT - 1) / kNT, stream, pl, row_bytes, 0, kWorkspaceCap))
    return rc;
  a.work = (T*)pl.work.p;
  task_vjp_kernel<T><<<pl.grid, pl.block, pl.smem, stream>>>(M, *D, a);
  return api_launched(&pl);
}

}  // namespace

// Same model limits as rbd_dynamics_derivatives
int rbd::check_vjp_limits(const HostModel& hm, const char* who) {
  DerivDev D;
  DerivAnc A;
  if (!build_deriv_dev(hm.dev64, D, A))
    return api_fail(RBD_EUNSUPPORTED, std::string(who) + ": more than 128 velocity coordinates or 4096 mass-matrix entries");
  return RBD_OK;
}

int rbd::inverse_dynamics_vjp_dense(const rbd_model* model, int32_t dtype, int64_t B, const void* q, const void* v, const void* vd,
                                    const void* tau_bar, void* q_bar_cfg, void* v_bar, void* vd_bar, cudaStream_t s) {
  return dtype == RBD_F32
             ? vjp_t<float>(model, false, B, B, args<float>(B, B, q, v, vd, nullptr, tau_bar, nullptr, q_bar_cfg, v_bar, vd_bar, nullptr, nullptr), s)
             : vjp_t<double>(model, false, B, B, args<double>(B, B, q, v, vd, nullptr, tau_bar, nullptr, q_bar_cfg, v_bar, vd_bar, nullptr, nullptr), s);
}

int rbd::dynamics_vjp_dense(const rbd_model* model, int32_t dtype, int64_t B, const void* q, const void* v, const void* vd,
                            const void* vd_bar, void* q_bar_cfg, void* v_bar, void* tau_bar, cudaStream_t s) {
  return dtype == RBD_F32
             ? vjp_t<float>(model, true, B, B, args<float>(B, B, q, v, vd, nullptr, vd_bar, nullptr, q_bar_cfg, v_bar, nullptr, tau_bar, nullptr), s)
             : vjp_t<double>(model, true, B, B, args<double>(B, B, q, v, vd, nullptr, vd_bar, nullptr, q_bar_cfg, v_bar, nullptr, tau_bar, nullptr), s);
}

extern "C" int32_t rbd_dynamics_vjp(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                                    const void* tau, const void* wext, const void* vd, const void* vd_bar, void* q_bar_tan,
                                    void* q_bar_cfg, void* v_bar, void* tau_bar, void* wext_bar, void* stream) {
  if (int rc = api_check(model, dtype, B, ld)) return rc;
  const ApiCall call;
  if (B == 0 || model->hm.nv == 0) return RBD_OK;
  if (!q || !v || !vd || !vd_bar) return api_fail(RBD_EINVAL, "rbd_dynamics_vjp: q, v, vd and vd_bar must not be NULL");
  if (int rc = check_vjp_limits(model->hm, "rbd_dynamics_vjp")) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  (void)tau;     // tau enters only through v̇, which is given: accepted so that the call mirrors rbd_dynamics
  return dtype == RBD_F32
             ? vjp_t<float>(model, true, B, ld, args<float>(B, ld, q, v, vd, wext, vd_bar, q_bar_tan, q_bar_cfg, v_bar, nullptr, tau_bar, wext_bar), s)
             : vjp_t<double>(model, true, B, ld, args<double>(B, ld, q, v, vd, wext, vd_bar, q_bar_tan, q_bar_cfg, v_bar, nullptr, tau_bar, wext_bar), s);
}

extern "C" int32_t rbd_inverse_dynamics_vjp(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                                            const void* vd, const void* wext, const void* tau_bar, void* q_bar_tan, void* q_bar_cfg,
                                            void* v_bar, void* vd_bar, void* wext_bar, void* stream) {
  if (int rc = api_check(model, dtype, B, ld)) return rc;
  const ApiCall call;
  if (B == 0 || model->hm.nv == 0) return RBD_OK;
  if (!q || !v || !vd || !tau_bar) return api_fail(RBD_EINVAL, "rbd_inverse_dynamics_vjp: q, v, vd and tau_bar must not be NULL");
  if (int rc = check_vjp_limits(model->hm, "rbd_inverse_dynamics_vjp")) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  return dtype == RBD_F32
             ? vjp_t<float>(model, false, B, ld, args<float>(B, ld, q, v, vd, wext, tau_bar, q_bar_tan, q_bar_cfg, v_bar, vd_bar, nullptr, wext_bar), s)
             : vjp_t<double>(model, false, B, ld, args<double>(B, ld, q, v, vd, wext, tau_bar, q_bar_tan, q_bar_cfg, v_bar, vd_bar, nullptr, wext_bar), s);
}

extern "C" int32_t rbd_task_kinematics_vjp(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                                           const void* vd, const rbd_task_desc* tasks, const rbd_task_out* out_bar, void* q_bar_tan,
                                           void* q_bar_cfg, void* v_bar, void* vd_bar, void* stream) {
  const ApiCall call;
  if (!model) return api_fail(RBD_EINVAL, "rbd_task_kinematics_vjp: model handle is NULL");
  if (dtype != RBD_F32 && dtype != RBD_F64) return api_fail(RBD_EUNSUPPORTED, "rbd_task_kinematics_vjp: fp32 and fp64 only");
  if (B < 0 || ld < B)
    return api_fail(RBD_EDIM, "rbd_task_kinematics_vjp: batch size / leading dimension mismatch (need ld >= B >= 0)");
  if (!q || !out_bar) return api_fail(RBD_EINVAL, "rbd_task_kinematics_vjp: q and out_bar must not be NULL");
  std::string err;
  if (int rc = check_task_desc(model->hm.nb, tasks, err)) return api_fail(rc, "rbd_task_kinematics_vjp: " + err);
  if (!v && (out_bar->twist || out_bar->point_velocity || out_bar->acceleration || out_bar->point_acceleration))
    return api_fail(RBD_EINVAL, "rbd_task_kinematics_vjp: twist / point_velocity / acceleration / point_acceleration cotangents need v");
  if (B == 0) return RBD_OK;
  cudaStream_t s = (cudaStream_t)stream;
  return dtype == RBD_F32 ? task_vjp_t<float>(model, B, ld, q, v, vd, *tasks, *out_bar, q_bar_tan, q_bar_cfg, v_bar, vd_bar, s)
                          : task_vjp_t<double>(model, B, ld, q, v, vd, *tasks, *out_bar, q_bar_tan, q_bar_cfg, v_bar, vd_bar, s);
}
