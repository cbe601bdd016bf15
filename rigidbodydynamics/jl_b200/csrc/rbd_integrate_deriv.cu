// rbd_integrate_derivatives: the Jacobians of every recorded RK4 step, forward mode (csrc/rbd_integrate_deriv.cuh has the
// mathematics).
//
// The (step, sample) pairs of the call are one batch, flattened step-major and processed in chunks.  Per chunk:
//   gather         the chunk's start states (and torques) from the trajectory blocks into dense [rows x C] arrays
//   recompute      rbd_b200.cu's one-step rollout with its stages kept (Rollout.stages), as rbd_integrate_vjp's backward step does
//   stage 0        lin_stage_kernel, then the stage Jacobians (dynamics_derivatives_dense), which are δv̇_0
//   stages 1..3    lin_stage_kernel, the stage Jacobians, lin_product_kernel (δv̇_i = Dq X + Dv Y + Dτ Z)
//   finish         lin_finish_kernel writes the rows of A and B
// lin_stage_kernel / lin_finish_kernel: one thread per (sample, joint, seed column), grid = (sample groups, bodies, 3 nv columns).
// lin_product_kernel: lane = sample, each thread an R x CG tile of δv̇; grid = (tiles, sample groups), tiles fastest, so the CTAs
// resident together read the same samples' D, X and Y rows and the re-reads of a row by the other tiles are served by L2.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cstdlib>
#include <string>
#include <type_traits>

#include "../../../include/rbd_b200.h"
#define sincos_slow sincos_slow_integrate_deriv_tu
#include "rbd_handle.h"
#include "rbd_integrate_deriv.cuh"

using namespace rbd;

namespace {

constexpr int kNT = 128;
constexpr int kTileR = 4, kTileC = 8;      // lin_product_kernel's tile: 32 accumulators, 24 loads per 64 FMAs

template <class T> struct GatherArgs {
  const T* q_traj; const T* v_traj; const T* tau;
  int64_t step_stride;
  T* q; T* v; T* t;                       // [nq / nv / nv x C]
  int64_t n0, C, B;
  int nq, nv;
};

// rows of the (step, sample) pairs n0 .. n0 + C - 1 from their [rows x B] blocks into dense [rows x C] arrays
template <class T>
__global__ void __launch_bounds__(256) lin_gather_kernel(const GatherArgs<T> a) {
  const int64_t rows = a.nq + a.nv + (a.tau ? a.nv : 0), total = rows * a.C;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = e / a.C, c = e - r * a.C, n = a.n0 + c, s = n / a.B, b = n - s * a.B;
    if (r < a.nq) a.q[e] = a.q_traj[(s * a.nq + r) * a.B + b];
    else if (r < a.nq + a.nv) a.v[e - a.nq * a.C] = a.v_traj[(s * a.nv + r - a.nq) * a.B + b];
    else a.t[e - (a.nq + a.nv) * a.C] = a.tau[s * a.step_stride + (r - a.nq - a.nv) * a.B + b];
  }
}

template <class T>
__global__ void __launch_bounds__(kNT) lin_stage_kernel(const __grid_constant__ ModelDev<T> M, const LinArgs<T> a) {
  const BodyDev<T>& bd = M.body[blockIdx.y];
  if (bd.kind == K_FIXED) return;
  for (int64_t b = (int64_t)blockIdx.x * kNT + threadIdx.x; b < a.ld; b += (int64_t)gridDim.x * kNT) lin_stage_joint(bd, a, b, blockIdx.z);
}

template <class T>
__global__ void __launch_bounds__(kNT) lin_finish_kernel(const __grid_constant__ ModelDev<T> M, const LinArgs<T> a) {
  const BodyDev<T>& bd = M.body[blockIdx.y];
  if (bd.kind == K_FIXED) return;
  for (int64_t b = (int64_t)blockIdx.x * kNT + threadIdx.x; b < a.ld; b += (int64_t)gridDim.x * kNT) lin_finish_joint(bd, a, b, blockIdx.z);
}

// grid.x = row tiles x column groups (row tiles fastest), grid.y = sample groups
template <class T>
__global__ void __launch_bounds__(kNT) lin_product_kernel(const LinArgs<T> a, const int nrt) {
  const int r0 = (blockIdx.x % nrt) * kTileR, c0 = (blockIdx.x / nrt) * kTileC;
  for (int64_t b = (int64_t)blockIdx.y * kNT + threadIdx.x; b < a.ld; b += (int64_t)gridDim.y * kNT)
    lin_product_tile<T, kTileR, kTileC>(a, b, r0, c0);
}

// rows per (step, sample) pair of the workspace: gathered q, v (and τ), the recompute's stages, and the seven [3 nv^2] arrays
int64_t lin_rows(int64_t nq, int64_t nv, bool tau) { return nq + nv + (tau ? nv : 0) + stage_rows(nq, nv) + 21 * nv * nv; }

struct LinCall {
  const void *q_traj, *v_traj, *tau;
  int64_t tau_step_stride;
  double dt;
  int nsteps;
  void *A, *B;
};

template <class T>
int integrate_derivatives_t(const rbd_model* model, int32_t dtype, int64_t B, const LinCall& r, cudaStream_t stream) {
  const HostModel& hm = model->hm;
  const ModelDev<T>& M = dev_model<T>(hm);
  const int64_t nq = hm.nq, nv = hm.nv, N = (int64_t)r.nsteps * B, nv2 = nv * nv;
  const T* tau = (const T*)r.tau;
  DeviceProps p;
  RBD_CUDA_TRY(device_props(p));
  // chunk size from the scratch budget of the dynamics Jacobians (which keep their own scratch within it as well)
  int64_t budget_mb = 2048;
  if (const char* e = std::getenv("RBD_DERIV_SCRATCH_MB")) budget_mb = std::max<int64_t>(1, std::atoll(e));
  const int64_t per_sample = lin_rows(nq, nv, tau != nullptr) * (int64_t)sizeof(T);
  int64_t C = std::min<int64_t>(N, std::max<int64_t>(kNT, (budget_mb << 20) / per_sample / kNT * kNT));
  C = std::min<int64_t>(C, (int64_t)65535 * kNT);      // lin_product_kernel's grid.y
  StreamAlloc work;
  if (cudaError_t e = work.alloc((size_t)per_sample * C, stream))
    return api_fail_cuda(e, "rbd_integrate_derivatives: workspace allocation (lower RBD_DERIV_SCRATCH_MB)");
  const double ca[4] = {0.0, 0.5, 0.5, 1.0}, cb[4] = {1.0 / 6, 1.0 / 3, 1.0 / 3, 1.0 / 6};   // runge_kutta_4, as integrate_t
  const int nrt = (int)((nv + kTileR - 1) / kTileR), nct = (int)((3 * nv + kTileC - 1) / kTileC);
  for (int64_t n0 = 0; n0 < N; n0 += C) {
    const int64_t c = std::min<int64_t>(C, N - n0);
    T* next = (T*)work.p;
    auto take = [&](int64_t rows) { T* o = next; next += rows * c; return o; };
    T *q0 = take(nq), *v0 = take(nv), *t0 = take(tau ? nv : 0), *stages = take(stage_rows(nq, nv));
    T *D = take(3 * nv2), *vd = take(3 * nv2), *X = take(3 * nv2), *Y = take(3 * nv2), *P = take(3 * nv2), *SP = take(3 * nv2),
      *SV = take(3 * nv2);
    const GatherArgs<T> ga{(const T*)r.q_traj, (const T*)r.v_traj, tau, r.tau_step_stride, q0, v0, t0, n0, c, B, (int)nq, (int)nv};
    const int64_t gtotal = (nq + nv + (tau ? nv : 0)) * c;
    lin_gather_kernel<T><<<(int)std::min<int64_t>((gtotal + 255) / 256, (int64_t)p.sms * 8), 256, 0, stream>>>(ga);
    if (int rc = api_launched()) return rc;
    Rollout rec{q0, v0, nullptr, tau ? t0 : nullptr, 0, 0, r.dt, 1};
    rec.stages = stages;
    if (int rc = integrate(model, dtype, c, c, rec, stream)) return rc;
    LinArgs<T> a{};
    a.q0 = q0;
    for (int i = 0; i < 4; ++i) {
      a.qs[i] = stages + (size_t)i * nq * c; a.vs[i] = stages + (4 * nq + (size_t)i * nv) * c;
      a.pd[i] = stages + (4 * nq + (4 + (size_t)i) * nv) * c;
      a.wa[i] = (T)(r.dt * ca[i]); a.wb[i] = (T)cb[i];
    }
    a.D = D; a.X = X; a.Y = Y; a.P = P; a.SP = SP; a.SV = SV; a.vd = vd;
    a.A = (T*)r.A; a.Bt = (T*)r.B;
    a.ld = c; a.n0 = n0; a.B = B; a.nv = (int)nv; a.dt = (T)r.dt;
    const dim3 gj((unsigned)std::min<int64_t>((c + kNT - 1) / kNT, (int64_t)p.sms * 8), (unsigned)hm.nb, (unsigned)(3 * nv));
    const dim3 gp((unsigned)(nrt * nct), (unsigned)((c + kNT - 1) / kNT));
    for (int i = 0; i < 4; ++i) {
      a.i = i;
      a.vdp = i == 1 ? D : vd;
      lin_stage_kernel<T><<<gj, kNT, 0, stream>>>(M, a);
      if (int rc = api_launched()) return rc;
      const T* vdi = stages + (4 * nq + (8 + (size_t)i) * nv) * c;
      if (int rc = dynamics_derivatives_dense(model, dtype, c, a.qs[i], a.vs[i], tau ? t0 : nullptr, vdi, D, D + nv2 * c, D + 2 * nv2 * c,
                                              stream))
        return rc;
      if (i == 0) continue;
      lin_product_kernel<T><<<gp, kNT, 0, stream>>>(a, nrt);
      if (int rc = api_launched()) return rc;
    }
    a.vdp = vd;
    lin_finish_kernel<T><<<gj, kNT, 0, stream>>>(M, a);
    if (int rc = api_launched()) return rc;
  }
  return RBD_OK;
}

}  // namespace

extern "C" int32_t rbd_integrate_derivatives(const rbd_model* model, int32_t dtype, int64_t B, const void* q_traj, const void* v_traj,
                                             const void* tau, int64_t tau_step_stride, int64_t tau_stage_stride, double dt,
                                             int32_t nsteps, void* A_out, void* B_out, void* stream) {
  const std::string fn = "rbd_integrate_derivatives";
  auto fail = [&](int status, const char* what) { return api_fail(status, fn + ": " + what); };
  if (int rc = api_check(model, dtype, B, B)) return rc;
  const ApiCall call;
  if (dtype != RBD_F32 && dtype != RBD_F64) return fail(RBD_EUNSUPPORTED, "fp32 and fp64 only");
  if (int rc = check_vjp_limits(model->hm, fn.c_str())) return rc;
  if (nsteps < 0 || !(dt > 0)) return fail(RBD_EINVAL, "need dt > 0 and nsteps >= 0");
  if (tau_step_stride < 0) return fail(RBD_EINVAL, "the torque step stride must be >= 0");
  if (tau_stage_stride != 0) return fail(RBD_EINVAL, "per-stage torque schedules are not supported (tau_stage_stride must be 0)");
  if (!A_out && !B_out) return fail(RBD_EINVAL, "A_out and B_out must not both be NULL");
  if (B == 0 || nsteps == 0 || model->hm.nv == 0) return RBD_OK;
  if (!q_traj || !v_traj) return fail(RBD_EINVAL, "q_traj and v_traj must not be NULL");
  const LinCall r{q_traj, v_traj, tau, tau_step_stride, dt, nsteps, A_out, B_out};
  cudaStream_t s = (cudaStream_t)stream;
  return dtype == RBD_F32 ? integrate_derivatives_t<float>(model, dtype, B, r, s) : integrate_derivatives_t<double>(model, dtype, B, r, s);
}
