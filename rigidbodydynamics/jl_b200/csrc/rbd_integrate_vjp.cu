// rbd_integrate_vjp: reverse mode through a Munthe-Kaas RK4 rollout (csrc/rbd_integrate_adjoint.cuh has the mathematics).
//
// Per step, last to first: the four stages are recomputed from the recorded state at the step's start (rbd_b200.cu's stage kernels
// and dynamics kernels, the model-specialised programs included); then five elementwise phases alternate with the four
// forward-dynamics VJPs of rbd_adjoint.cu:
//   finish + L3 | VJP 3 | G3 + L2 | VJP 2 | G2 + L1 | VJP 1 | G1 + L0 | VJP 0 | G0 (+ the trajectory adjoints of the step's start)
// An elementwise phase is one thread per (sample, joint) for the joints with non-linear maps (blockIdx.y = body) and, when the
// batch allows, a vectorised kernel over the revolute / prismatic rows (16-byte accesses, like integrate_stage_linear_kernel).
// Every launch, the recompute's and the VJPs' included, counts in the call's launch record (rbd_handle.h).
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <string>

#include "../../../include/rbd_b200.h"
#define sincos_slow sincos_slow_integrate_vjp_tu
#include "rbd_handle.h"
#include "rbd_integrate_adjoint.cuh"

using namespace rbd;

namespace {

template <class T>
__global__ void __launch_bounds__(128) integrate_adjoint_kernel(const __grid_constant__ ModelDev<T> M, const AdjStepArgs<T> a,
                                                                const bool skip_linear) {
  const BodyDev<T>& bd = M.body[blockIdx.y];
  if (bd.kind == K_FIXED) return;
  if (skip_linear && (bd.kind == K_REV || bd.kind == K_PRIS)) return;
  for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < a.ld; b += (int64_t)gridDim.x * blockDim.x) adj_joint(bd, a, b);
}

// revolute / prismatic rows, VEC samples per thread; each lane runs adj_lin like adj_joint does
template <class T>
__global__ void __launch_bounds__(256) integrate_adjoint_linear_kernel(const __grid_constant__ ModelDev<T> M, const AdjStepArgs<T> a) {
  using V = typename VecOf<T>::type;
  constexpr int N = VecOf<T>::N;
  const BodyDev<T>& bd = M.body[blockIdx.y];
  if (bd.kind != K_REV && bd.kind != K_PRIS) return;
  const int64_t qo = (int64_t)bd.qrow * a.ld, vo = (int64_t)bd.vrow * a.ld, nvec = a.ld / N;
  auto ld = [&](const T* p, int64_t off, int64_t i, T* x) {
    const V w = reinterpret_cast<const V*>(p + off)[i];
    memcpy(x, &w, sizeof(V));
  };
  auto st = [&](T* p, int64_t off, int64_t i, const T* x) {
    V w;
    memcpy(&w, x, sizeof(V));
    reinterpret_cast<V*>(p + off)[i] = w;
  };
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    T qb[N], vb[N], phib[N], qcb[N], vvb[N], vsb[N], taub[N], qtb[N], vtb[N], qb0[N], vb0[N];
    ld(a.qb, qo, i, qb); ld(a.vb, vo, i, vb); ld(a.phib, vo, i, phib);
    const bool mid = a.g < 4;
    if (mid) {
      ld(a.qcb, qo, i, qcb); ld(a.vvb, vo, i, vvb); ld(a.vsb, vo, i, vsb); ld(a.qb0, qo, i, qb0); ld(a.vb0, vo, i, vb0);
      if (a.tau_bar) ld(a.taub, vo, i, taub);
      if (a.qtb) ld(a.qtb, qo, i, qtb);
      if (a.vtb) ld(a.vtb, vo, i, vtb);
    }
    T o_qb[N], o_vb[N], o_qb0[N], o_vb0[N], o_phib[N], o_vdb[N], o_vsb[N], o_tau[N];
#pragma unroll
    for (int c = 0; c < N; ++c) {
      LinIn<T> x;
      LinOut<T> o;
      x.qb = qb[c]; x.vb = vb[c]; x.phib = phib[c];
      if (mid) {
        x.qcb = qcb[c]; x.vvb = vvb[c]; x.vsb = vsb[c]; x.qb0 = qb0[c]; x.vb0 = vb0[c];
        x.taub = a.tau_bar ? taub[c] : T(0); x.qtb = a.qtb ? qtb[c] : T(0); x.vtb = a.vtb ? vtb[c] : T(0);
      }
      adj_lin(a, x, o);
      o_qb[c] = o.qb; o_vb[c] = o.vb; o_qb0[c] = o.qb0; o_vb0[c] = o.vb0; o_phib[c] = o.phib; o_vdb[c] = o.vdb; o_vsb[c] = o.vsb;
      o_tau[c] = o.tau;
    }
    st(a.qb0, qo, i, o_qb0); st(a.vb0, vo, i, o_vb0);
    if (!mid) st(a.phib, vo, i, o_phib);
    if (mid && a.tau_bar) {
      T t[N];
      ld(a.tau_bar, vo, i, t);
#pragma unroll
      for (int c = 0; c < N; ++c) t[c] += o_tau[c];
      st(a.tau_bar, vo, i, t);
    }
    if (a.g == 0) { st(a.qb, qo, i, o_qb); st(a.vb, vo, i, o_vb); }
    if (a.l >= 0) { st(a.vsb, vo, i, o_vsb); st(a.vdb, vo, i, o_vdb); }
  }
}

// q̄ (configuration coordinates) -> tangent and minimal-norm configuration forms: between steps (in place) and for the outputs
template <class T> struct OutArgs { const T* q; const T* qb; T* qt; T* qc; int64_t B; };
template <class T>
__global__ void __launch_bounds__(128) integrate_adjoint_out_kernel(const __grid_constant__ ModelDev<T> M, const OutArgs<T> a) {
  const BodyDev<T>& bd = M.body[blockIdx.y];
  if (bd.kind == K_FIXED) return;
  for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < a.B; b += (int64_t)gridDim.x * blockDim.x)
    adj_out(bd, a.q, a.qb, a.qt, a.qc, a.B, b);
}

template <class T>
int integrate_vjp_t(const rbd_model* model, int32_t dtype, int64_t B, const T* q_traj, const T* v_traj, const T* tau, int64_t step_stride,
                    int64_t stage_stride, double dt, int nsteps, const T* qtb, const T* vtb, T* q0t, T* q0c, T* v0b, T* taub,
                    cudaStream_t stream) {
  const HostModel& hm = model->hm;
  const ModelDev<T>& M = dev_model<T>(hm);
  const int64_t nq = hm.nq, nv = hm.nv;
  DeviceProps p;
  RBD_CUDA_TRY(device_props(p));
  // workspace: the four stages, then q̄_cfg / q̄ / q̄0 / q̄s (nq rows each), v̄ / τ̄ / v̄ / v̄0 / v̄s / v̇̄ / Φ̄ (nv rows each)
  const int64_t srows = stage_rows(nq, nv), rows = srows + 4 * nq + 7 * nv;
  StreamAlloc work;
  RBD_CUDA_TRY(work.alloc((size_t)rows * B * sizeof(T), stream));
  T* stages = (T*)work.p;
  T* next = stages + srows * B;
  auto take = [&](int64_t r) { T* o = next; next += r * B; return o; };
  T *qcb = take(nq), *qb = take(nq), *qb0 = take(nq), *qsb = take(nq);
  T *vvb = take(nv), *tb = take(nv), *vb = take(nv), *vb0 = take(nv), *vsb = take(nv), *vdb = take(nv), *phib = take(nv);
  const size_t qbytes = (size_t)nq * B * sizeof(T), vbytes = (size_t)nv * B * sizeof(T);
  if (qtb) RBD_CUDA_TRY(cudaMemcpyAsync(qb, qtb + (size_t)nsteps * nq * B, qbytes, cudaMemcpyDeviceToDevice, stream));
  else RBD_CUDA_TRY(cudaMemsetAsync(qb, 0, qbytes, stream));
  if (vtb) RBD_CUDA_TRY(cudaMemcpyAsync(vb, vtb + (size_t)nsteps * nv * B, vbytes, cudaMemcpyDeviceToDevice, stream));
  else RBD_CUDA_TRY(cudaMemsetAsync(vb, 0, vbytes, stream));
  bool has_other = false;
  for (int i = 0; i < hm.nb; ++i) has_other |= (M.body[i].kind != K_REV && M.body[i].kind != K_PRIS && M.body[i].kind != K_FIXED);
  constexpr int N = VecOf<T>::N;
  const size_t va = sizeof(typename VecOf<T>::type);
  auto aligned = [&](const T* x, int64_t stride) { return !x || ((uintptr_t)x % va == 0 && stride % N == 0); };
  const bool vec_ok = B % N == 0 && B >= 1024 && aligned(taub, step_stride) && aligned(taub, stage_stride) && aligned(qtb, 0) &&
                      aligned(vtb, 0) && aligned(q_traj, 0);
  const int grid = (int)std::min<int64_t>((B + 127) / 128, (int64_t)p.sms * 8);
  const int grid_lin = (int)std::min<int64_t>((B / N + 255) / 256, (int64_t)p.sms * 4);
  const double ca[4] = {0.0, 0.5, 0.5, 1.0}, cb[4] = {1.0 / 6, 1.0 / 3, 1.0 / 3, 1.0 / 6};   // runge_kutta_4, as integrate_t
  AdjStepArgs<T> a{};
  for (int i = 0; i < 4; ++i) {
    a.qs[i] = stages + (size_t)i * nq * B; a.vs[i] = stages + (4 * nq + (size_t)i * nv) * B;
    a.pd[i] = stages + (4 * nq + (4 + (size_t)i) * nv) * B;
    a.wa[i] = (T)(dt * ca[i]); a.wb[i] = (T)cb[i];
  }
  const T* vd[4];
  for (int i = 0; i < 4; ++i) vd[i] = stages + (4 * nq + (8 + (size_t)i) * nv) * B;
  a.qcb = qcb; a.vvb = vvb; a.taub = tb;
  a.qb = qb; a.vb = vb; a.qb0 = qb0; a.vb0 = vb0; a.qsb = qsb; a.vsb = vsb; a.vdb = vdb; a.phib = phib;
  a.ld = B; a.dt = (T)dt;
  for (int s = nsteps - 1; s >= 0; --s) {
    const T* q0 = q_traj + (size_t)s * nq * B;
    const T* v0 = v_traj + (size_t)s * nv * B;
    if (int rc = integrate_record(model, dtype, B, B, const_cast<T*>(q0), const_cast<T*>(v0), tau ? tau + s * step_stride : nullptr,
                                  step_stride, stage_stride, dt, 1, nullptr, nullptr, stages, stream)) return rc;
    a.q0 = q0;
    a.qtb = qtb ? qtb + (size_t)s * nq * B : nullptr;
    a.vtb = vtb ? vtb + (size_t)s * nv * B : nullptr;
    for (int g = 4; g >= 0; --g) {
      a.g = g; a.l = g == 4 ? 3 : g - 1;
      a.tau_bar = (taub && g < 4) ? taub + s * step_stride + g * stage_stride : nullptr;
      if (vec_ok) {
        integrate_adjoint_linear_kernel<T><<<dim3(grid_lin, hm.nb), 256, 0, stream>>>(M, a);
        if (int rc = api_launched()) return rc;
      }
      if (!vec_ok || has_other) {
        integrate_adjoint_kernel<T><<<dim3(grid, hm.nb), 128, 0, stream>>>(M, a, vec_ok);
        if (int rc = api_launched()) return rc;
      }
      if (a.l < 0) {
        if (s > 0) {
          integrate_adjoint_out_kernel<T><<<dim3(grid, hm.nb), 128, 0, stream>>>(M, OutArgs<T>{q0, qb, nullptr, qb, B});
          if (int rc = api_launched()) return rc;
        }
        continue;
      }
      if (int rc = dynamics_vjp_dense(model, dtype, B, a.qs[a.l], a.vs[a.l], vd[a.l], vdb, qcb, vvb, taub ? tb : nullptr, stream)) return rc;
    }
  }
  if (q0t || q0c) {
    integrate_adjoint_out_kernel<T><<<dim3(grid, hm.nb), 128, 0, stream>>>(M, OutArgs<T>{q_traj, qb, q0t, q0c, B});
    if (int rc = api_launched()) return rc;
  }
  if (v0b) RBD_CUDA_TRY(cudaMemcpyAsync(v0b, vb, vbytes, cudaMemcpyDeviceToDevice, stream));
  return RBD_OK;
}

}  // namespace

extern "C" int32_t rbd_integrate_vjp(const rbd_model* model, int32_t dtype, int64_t B, const void* q_traj, const void* v_traj,
                                     const void* tau, int64_t tau_step_stride, int64_t tau_stage_stride, double dt, int32_t nsteps,
                                     const void* q_traj_bar, const void* v_traj_bar, void* q0_bar_tan, void* q0_bar_cfg, void* v0_bar,
                                     void* tau_bar, void* stream) {
  if (int rc = api_check(model, dtype, B, B)) return rc;
  const ApiCall call;
  if (dtype != RBD_F32 && dtype != RBD_F64) return api_fail(RBD_EUNSUPPORTED, "rbd_integrate_vjp: fp32 and fp64 only");
  if (nsteps < 0 || !(dt > 0)) return api_fail(RBD_EINVAL, "rbd_integrate_vjp: need dt > 0 and nsteps >= 0");
  if (tau_step_stride < 0 || tau_stage_stride < 0) return api_fail(RBD_EINVAL, "rbd_integrate_vjp: torque strides must be >= 0");
  if (!tau && tau_bar) return api_fail(RBD_EINVAL, "rbd_integrate_vjp: tau_bar needs tau");
  if (B == 0 || model->hm.nv == 0) return RBD_OK;
  if (!q_traj || !v_traj) return api_fail(RBD_EINVAL, "rbd_integrate_vjp: q_traj and v_traj must not be NULL");
  cudaStream_t s = (cudaStream_t)stream;
  return dtype == RBD_F32
             ? integrate_vjp_t<float>(model, dtype, B, (const float*)q_traj, (const float*)v_traj, (const float*)tau, tau_step_stride,
                                      tau_stage_stride, dt, nsteps, (const float*)q_traj_bar, (const float*)v_traj_bar, (float*)q0_bar_tan,
                                      (float*)q0_bar_cfg, (float*)v0_bar, (float*)tau_bar, s)
             : integrate_vjp_t<double>(model, dtype, B, (const double*)q_traj, (const double*)v_traj, (const double*)tau, tau_step_stride,
                                       tau_stage_stride, dt, nsteps, (const double*)q_traj_bar, (const double*)v_traj_bar,
                                       (double*)q0_bar_tan, (double*)q0_bar_cfg, (double*)v0_bar, (double*)tau_bar, s);
}
