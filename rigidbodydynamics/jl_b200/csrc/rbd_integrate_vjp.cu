// rbd_integrate_vjp: reverse mode through a Munthe-Kaas RK4 rollout (csrc/rbd_integrate_adjoint.cuh has the mathematics).
//
// Per step, last to first: the four stages are recomputed from the recorded state at the step's start (rbd_b200.cu's stage kernels
// and dynamics kernels, the model-specialised programs included); then five elementwise phases alternate with the four
// forward-dynamics VJPs of rbd_adjoint.cu:
//   finish + L3 | VJP 3 | G3 + L2 | VJP 2 | G2 + L1 | VJP 1 | G1 + L0 | VJP 0 | G0 (+ the trajectory adjoints of the step's start)
// An elementwise phase is one thread per (sample, joint) for the joints with non-linear maps (blockIdx.y = body) and, when the
// batch allows, a vectorised kernel over the revolute / prismatic rows (16-byte accesses, like integrate_stage_linear_kernel).
// Every launch, the recompute's and the VJPs' included, counts in the call's launch record (rbd_handle.h).
// rbd_integrate_contact_vjp (rbd_contact_adjoint.cuh) is the same driver over rbd_integrate_contact's recompute, with
// contact_vjp_kernel in place of each stage's forward-dynamics VJP; it also carries the contact state's adjoint.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <memory>
#include <optional>
#include <string>
#include <type_traits>
#include <vector>

#include "../../../include/rbd_b200.h"
#define sincos_slow sincos_slow_integrate_vjp_tu
#include "rbd_contact_adjoint.cuh"
#include "rbd_handle.h"
#include "rbd_task_pd_adjoint.cuh"

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

// rbd_integrate_pd_vjp: the two phase kernels above with the controller's adjoint of stage g in the mid phases
// (rbd_integrate_adjoint.cuh's pd_adj_joint); the open-loop instantiations above stay as they are.
template <class T>
__global__ void __launch_bounds__(128) integrate_adjoint_pd_kernel(const __grid_constant__ ModelDev<T> M, const AdjStepArgs<T> a,
                                                                   const PdAdjArgs<T> c, const bool skip_linear) {
  const BodyDev<T>& bd = M.body[blockIdx.y];
  if (bd.kind == K_FIXED) return;
  if (skip_linear && (bd.kind == K_REV || bd.kind == K_PRIS)) return;
  for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < a.ld; b += (int64_t)gridDim.x * blockDim.x)
    adj_joint<T, true>(bd, a, b, &c);
}

// revolute / prismatic rows, VEC samples per thread: per lane the arithmetic of adj_joint<T, true>'s revolute / prismatic branch
template <class T>
__global__ void __launch_bounds__(256) integrate_adjoint_pd_linear_kernel(const __grid_constant__ ModelDev<T> M, const AdjStepArgs<T> a,
                                                                          const PdAdjArgs<T> c) {
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
  auto add = [&](T* p, int64_t off, int64_t i, const T* x, T sign) {     // p += sign x (sign = ±1: exact)
    T y[N];
    ld(p, off, i, y);
#pragma unroll
    for (int k = 0; k < N; ++k) y[k] += sign * x[k];
    st(p, off, i, y);
  };
  const int64_t go = (int64_t)bd.vrow * c.g_ld;
  const T lo = c.tau ? c.lo[bd.vrow] : T(0), hi = c.tau ? c.hi[bd.vrow] : T(0);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    T qb[N], vb[N], phib[N], qcb[N], vvb[N], vsb[N], taub[N], qtb[N], vtb[N], qb0[N], vb0[N];
    ld(a.qb, qo, i, qb); ld(a.vb, vo, i, vb); ld(a.phib, vo, i, phib);
    const bool mid = a.g < 4;
    T kpw[N], kdw[N], vrw[N], eb[N];      // the law's adjoint: w e (-> K̄p), w (v_s - v_ref) (-> K̄d), Kd w (-> v̄_ref), ē
    if (mid) {
      ld(a.qcb, qo, i, qcb); ld(a.vvb, vo, i, vvb); ld(a.vsb, vo, i, vsb); ld(a.qb0, qo, i, qb0); ld(a.vb0, vo, i, vb0);
      ld(a.taub, vo, i, taub);
      if (a.qtb) ld(a.qtb, qo, i, qtb);
      if (a.vtb) ld(a.vtb, vo, i, vtb);
      T qs[N], vs[N], qr[N], vr[N], kp[N], kd[N], tau[N], w[N], idq[N], idv[N];
      ld(a.qs[a.g], qo, i, qs); ld(a.vs[a.g], vo, i, vs); ld(c.qref, qo, i, qr);
      if (c.vref) ld(c.vref, vo, i, vr);
      if (c.g_ld) { ld(c.kp, go, i, kp); ld(c.kd, go, i, kd); }
      if (c.tau) ld(c.tau, vo, i, tau);
      if (c.idvd) { ld(c.idvd, vo, i, w); ld(c.idq, qo, i, idq); ld(c.idv, vo, i, idv); }
#pragma unroll
      for (int k = 0; k < N; ++k) {
        if (c.tau) taub[k] = pd_mask(taub[k], tau[k], lo, hi);
        if (!c.idvd) w[k] = taub[k];
        const T kpk = c.g_ld ? kp[k] : c.kp[bd.vrow], kdk = c.g_ld ? kd[k] : c.kd[bd.vrow];
        const T e = qs[k] - qr[k], dv = vs[k] - (c.vref ? vr[k] : T(0));
        kpw[k] = w[k] * e; kdw[k] = w[k] * dv; vrw[k] = kdk * w[k];
        eb[k] = -kpk * w[k];
        T cq = c.idvd ? idq[k] : T(0), cv = c.idvd ? idv[k] : T(0);      // pd_adj_joint's order of operations
        cv -= vrw[k];
        cq += eb[k];
        qcb[k] += cq; vvb[k] += cv;
      }
      if (c.kpb) add(c.kpb, vo, i, kpw, T(-1));
      if (c.kdb) add(c.kdb, vo, i, kdw, T(-1));
      if (c.vrefb) add(c.vrefb, vo, i, vrw, T(1));
      if (c.vdrefb) add(c.vdrefb, vo, i, w, T(1));
      if (c.qrefb) add(c.qrefb, qo, i, eb, T(-1));
    }
    T o_qb[N], o_vb[N], o_qb0[N], o_vb0[N], o_phib[N], o_vdb[N], o_vsb[N], o_tau[N];
#pragma unroll
    for (int c_ = 0; c_ < N; ++c_) {
      LinIn<T> x;
      LinOut<T> o;
      x.qb = qb[c_]; x.vb = vb[c_]; x.phib = phib[c_];
      if (mid) {
        x.qcb = qcb[c_]; x.vvb = vvb[c_]; x.vsb = vsb[c_]; x.qb0 = qb0[c_]; x.vb0 = vb0[c_];
        x.taub = taub[c_]; x.qtb = a.qtb ? qtb[c_] : T(0); x.vtb = a.vtb ? vtb[c_] : T(0);
      }
      adj_lin(a, x, o);
      o_qb[c_] = o.qb; o_vb[c_] = o.vb; o_qb0[c_] = o.qb0; o_vb0[c_] = o.vb0; o_phib[c_] = o.phib; o_vdb[c_] = o.vdb; o_vsb[c_] = o.vsb;
      o_tau[c_] = o.tau;
    }
    st(a.qb0, qo, i, o_qb0); st(a.vb0, vo, i, o_vb0);
    if (!mid) st(a.phib, vo, i, o_phib);
    if (mid && a.tau_bar) add(a.tau_bar, vo, i, o_tau, T(1));
    if (a.g == 0) { st(a.qb, qo, i, o_qb); st(a.vb, vo, i, o_vb); }
    if (a.l >= 0) { st(a.vsb, vo, i, o_vsb); st(a.vdb, vo, i, o_vdb); }
  }
}

// computed-torque mode with effort bounds: τ̄ of a stage -> the seed m = τ̄ 1[lo < τ < hi] of its inverse-dynamics VJP, in place
template <class T> struct PdMaskArgs { T* taub; const T* tau; const T* lo; const T* hi; int64_t nv, B; };
template <class T>
__global__ void __launch_bounds__(256) pd_mask_kernel(const PdMaskArgs<T> a) {
  const int64_t total = a.nv * a.B;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = e / a.B;
    a.taub[e] = pd_mask(a.taub[e], a.tau[e], a.lo[k], a.hi[k]);
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

// The contact rollout's stage adjoint (rbd_contact_adjoint.cuh): in place of the forward-dynamics VJP of a stage, one thread per
// sample, persistent like dynamics_vjp_kernel (the solve's stash in shared memory, the workspace one column per resident thread).
template <class T> struct ContactVjpArgs {
  const T *q, *v, *vd, *vdb;          // stage l: (qs, vs, v̇), ν̄
  T *qc, *vb, *taub;                  // q̄_cfg, v̄, τ̄ (NULL: not wanted)
  const T *s0, *sdp, *stb;            // rbd_contact_adjoint.cuh's ContactVjpIO
  T *sb1, *sacc, *sdc;
  T* work;
  const T* zero;
  T g[3];
  T wa, wdb;
  int l;
  int64_t B;
};
template <class T>
__global__ void __launch_bounds__(32, 1) contact_vjp_kernel(const __grid_constant__ ModelDev<T> M, const __grid_constant__ ContactDev<T> C,
                                                            const __grid_constant__ ContactVjpArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const Stash<T, 32> st{reinterpret_cast<T*>(smem_raw) + threadIdx.x};
  const int64_t tid = (int64_t)blockIdx.x * 32 + threadIdx.x;
  const int64_t ngroups = (a.B + 31) / 32;
  for (int64_t g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const int64_t b = g * 32 + threadIdx.x;
    const bool active = b < a.B;
    const int64_t bl = active ? b : a.B - 1;      // inactive lanes recompute the last sample, stores are masked
    ContactVjpIO<T> io;
    io.q = {a.q + bl, a.B}; io.v = {a.v + bl, a.B}; io.vd = {a.vd + bl, a.B}; io.vdb = {a.vdb + bl, a.B};
    io.qc = {a.qc + bl, a.B, active};
    io.taub = {a.taub ? a.taub + bl : nullptr, a.B, active};
    io.vb = a.vb + bl;
    io.s0 = a.s0 + bl; io.sdp = a.sdp ? a.sdp + bl : nullptr; io.stb = a.stb ? a.stb + bl : nullptr;
    io.sb1 = a.sb1 + bl; io.sacc = a.sacc + bl; io.sdc = a.sdc + bl;
    io.ld = a.B; io.wa = a.wa; io.wdb = a.wdb; io.l = a.l;
    io.s = {a.work + tid, (int64_t)gridDim.x * 32};
    io.active = active;
    contact_vjp_sample<T>(M, a.g, C, io, a.zero, st);
  }
}

// The task-space law's adjoint (rbd_task_pd_adjoint.cuh) at one stage of rbd_integrate_task_pd_vjp, and rbd_task_pd_torques_vjp:
// one thread per sample, persistent, the workspace one column per resident thread.  Each thread owns its sample's rows of every
// output, so the additions need no atomics.
static_assert(sizeof(ModelDev<double>) + sizeof(TaskPdDev<double>) + sizeof(TaskPdVjpArgs<double>) <= 32764,
              "task_pd_vjp_kernel's parameters exceed the kernel-parameter limit");
template <class T>
__global__ void __launch_bounds__(32, 1)
task_pd_vjp_kernel(const __grid_constant__ ModelDev<T> M, const __grid_constant__ TaskPdDev<T> D, const TaskPdVjpArgs<T> a) {
  const int64_t tid = (int64_t)blockIdx.x * 32 + threadIdx.x;
  const int64_t ngroups = (a.B + 31) / 32;
  for (int64_t g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const int64_t b = g * 32 + threadIdx.x;
    const bool active = b < a.B;
    task_pd_vjp_column<T>(M, D, a, active ? b : a.B - 1, active, Scr<T>{a.work + tid, (int64_t)gridDim.x * 32});
  }
}

// the task kernel's descriptor and one plan (grid, workspace) for every launch of a call
template <class T> struct TaskPdVjpPlan {
  std::unique_ptr<TaskPdDev<T>> D;
  LaunchPlan plan;
  int init(const HostModel& hm, const rbd_task_pd_desc& c, int64_t B, cudaStream_t stream) {
    D.reset(new TaskPdDev<T>());
    const size_t row_bytes = (size_t)build_task_pd_vjp_dev<T>(hm, c, *D) * sizeof(T);
    return plan_persistent((const void*)task_pd_vjp_kernel<T>, 32, 0, (B + 31) / 32, stream, plan, row_bytes, 0, size_t(512) << 20);
  }
  int launch(const ModelDev<T>& M, TaskPdVjpArgs<T> a, cudaStream_t stream) {
    a.work = (T*)plan.work.p;
    task_pd_vjp_kernel<T><<<plan.grid, plan.block, plan.smem, stream>>>(M, *D, a);
    return api_launched(&plan);
  }
};

// One request to the rollout adjoint, in the form the C entry points receive it (include/rbd_b200.h): the recorded trajectories
// [(nsteps + 1) x rows x B] and their adjoints (NULL: zero), the torques as Rollout has them, the outputs (each NULL: not wanted),
// and the optional contact descriptor and controller, with the adjoints of the controller's arrays (NULL: none wanted).
struct RolloutVjp {
  const void *q_traj, *v_traj, *s_traj;
  const void* tau;
  int64_t tau_step_stride, tau_stage_stride;
  double dt;
  int nsteps;
  const void *q_traj_bar, *v_traj_bar, *s_traj_bar;
  void *q0_bar_tan, *q0_bar_cfg, *v0_bar, *s0_bar, *tau_bar;
  const rbd_contact_desc* contact = nullptr;
  const rbd_pd_desc* pd = nullptr;
  const rbd_pd_bar* pd_bar = nullptr;
  const rbd_task_pd_desc* task = nullptr;      // pd NULL: the joint term, if any, is task->joint
  const rbd_task_pd_bar* task_bar = nullptr;
};

// the effort bounds [2 nv] (lo, then hi) in T, copied from the host arrays (pageable memory, as integrate_t copies them) to dev
template <class T>
int upload_bounds(T* dev, const double* lo, const double* hi, int64_t nv, cudaStream_t stream) {
  std::vector<T> h(2 * nv);
  for (int64_t k = 0; k < nv; ++k) { h[k] = (T)lo[k]; h[nv + k] = (T)hi[k]; }
  RBD_CUDA_TRY(cudaMemcpyAsync(dev, h.data(), 2 * nv * sizeof(T), cudaMemcpyHostToDevice, stream));
  return RBD_OK;
}

template <class T>
int launch_pd_mask(const PdMaskArgs<T>& ma, int sms, cudaStream_t stream) {
  pd_mask_kernel<T><<<(int)std::min<int64_t>((ma.nv * ma.B + 255) / 256, (int64_t)sms * 8), 256, 0, stream>>>(ma);
  return api_launched();
}

// The JointPD law's adjoint at step s: the references and their adjoints of step s, as integrate_t reads the references.  The
// caller adds the mask and, in computed-torque mode, the inverse-dynamics VJP's rows.
template <class T>
PdAdjArgs<T> pd_adj_step(const rbd_pd_desc& pd, const rbd_pd_bar* bar, int64_t s) {
  const size_t qo = (size_t)s * pd.q_ref_step_stride, vo = (size_t)s * pd.v_ref_step_stride;
  const rbd_pd_bar cb = bar ? *bar : rbd_pd_bar{};
  PdAdjArgs<T> c{};
  c.qref = (const T*)pd.q_ref + qo;
  c.vref = pd.v_ref ? (const T*)pd.v_ref + vo : nullptr;
  c.kp = (const T*)pd.kp; c.kd = (const T*)pd.kd; c.g_ld = pd.gain_ld;
  c.kpb = (T*)cb.kp; c.kdb = (T*)cb.kd;
  c.qrefb = cb.q_ref ? (T*)cb.q_ref + qo : nullptr;
  c.vrefb = cb.v_ref ? (T*)cb.v_ref + vo : nullptr;
  c.vdrefb = cb.vd_ref ? (T*)cb.vd_ref + vo : nullptr;
  return c;
}

// ... and the task law's: the task references, gains and their adjoints of step s.  The caller adds the state, the seed, where
// q̄ / v̄ go, and the joint term.
template <class T>
TaskPdVjpArgs<T> task_vjp_step(const rbd_task_pd_desc& c, const rbd_task_pd_bar* bar, int64_t s) {
  const size_t xo = (size_t)s * c.x_ref_step_stride, xdo = (size_t)s * c.xd_ref_step_stride;
  const rbd_task_pd_bar cb = bar ? *bar : rbd_task_pd_bar{};
  TaskPdVjpArgs<T> ta{};
  ta.xref = (const T*)c.x_ref + xo; ta.xdref = c.xd_ref ? (const T*)c.xd_ref + xdo : nullptr;
  ta.kp = (const T*)c.kp; ta.kd = (const T*)c.kd; ta.gain_ld = c.gain_ld;
  ta.kpb = (T*)cb.kp; ta.kdb = (T*)cb.kd;
  ta.xrefb = cb.x_ref ? (T*)cb.x_ref + xo : nullptr; ta.xdrefb = cb.xd_ref ? (T*)cb.xd_ref + xdo : nullptr;
  return ta;
}

template <class T>
int integrate_vjp_t(const rbd_model* model, int64_t B, const RolloutVjp& r, cudaStream_t stream) {
  const int32_t dtype = std::is_same<T, float>::value ? RBD_F32 : RBD_F64;
  const HostModel& hm = model->hm;
  const ModelDev<T>& M = dev_model<T>(hm);
  const T *q_traj = (const T*)r.q_traj, *v_traj = (const T*)r.v_traj, *s_traj = (const T*)r.s_traj, *tau = (const T*)r.tau;
  const T *qtb = (const T*)r.q_traj_bar, *vtb = (const T*)r.v_traj_bar, *stb = (const T*)r.s_traj_bar;
  T *q0t = (T*)r.q0_bar_tan, *q0c = (T*)r.q0_bar_cfg, *v0b = (T*)r.v0_bar, *s0b = (T*)r.s0_bar, *taub = (T*)r.tau_bar;
  const int64_t step_stride = r.tau_step_stride, stage_stride = r.tau_stage_stride;
  const double dt = r.dt;
  const int nsteps = r.nsteps;
  const rbd_contact_desc* cd = r.contact;
  std::unique_ptr<ContactDev<T>> C;
  if (cd) {
    C.reset(new ContactDev<T>());
    build_contact_dev<T>(hm.nb, hm.pos.data(), hm.alignT.data(), *cd, *C);
  }
  const int64_t nq = hm.nq, nv = hm.nv, ns = cd ? (int64_t)3 * cd->npoints * cd->nhalfspaces : 0;
  // task-space control: its joint term, if any, takes the JointPD controller's place in the phase kernels
  const rbd_task_pd_desc* task = r.task;
  const rbd_pd_desc* pd = task ? task->joint : r.pd;
  const rbd_pd_bar* pd_bar = task ? (task->joint && r.task_bar ? r.task_bar->joint : nullptr) : r.pd_bar;
  const bool closed = pd || task;
  const bool ct = task ? task->mode == RBD_PD_COMPUTED_TORQUE : pd && pd->mode == RBD_PD_COMPUTED_TORQUE;
  const double* effort_lo = task ? task->effort_lo : (pd ? pd->effort_lo : nullptr);
  const double* effort_hi = task ? task->effort_hi : (pd ? pd->effort_hi : nullptr);
  const bool bounds = effort_lo != nullptr;
  TaskPdVjpPlan<T> tplan;
  if (task && nsteps > 0)
    if (int rc = tplan.init(hm, *task, B, stream)) return rc;
  DeviceProps p;
  RBD_CUDA_TRY(device_props(p));
  // workspace: the four stages (with contact: and their ṡ_i; with a controller: their applied torques and, in computed-torque mode,
  // v̇_des), then q̄_cfg / q̄ / q̄0 / q̄s (nq rows each), v̄ / τ̄ / v̄ / v̄0 / v̄s / v̇̄ / Φ̄ (nv rows each), then with contact s̄1 / s̄0 / the
  // carried dt a_i s̄_i (ns rows each), then in computed-torque mode the inverse-dynamics VJP's q̄_cfg (nq) / v̄ / v̇̄_des (nv), then
  // the effort bounds (2 nv values)
  const int64_t prow = stage_rows(nq, nv) + 4 * ns;
  const int64_t srows = prow + (closed ? pd_stage_rows(nv, ct) : 0);
  const int64_t rows = srows + 4 * nq + 7 * nv + 3 * ns + (ct ? nq + 2 * nv : 0);
  StreamAlloc work;
  RBD_CUDA_TRY(work.alloc(((size_t)rows * B + (bounds ? 2 * nv : 0)) * sizeof(T), stream));
  T* stages = (T*)work.p;
  T* next = stages + srows * B;
  auto take = [&](int64_t r) { T* o = next; next += r * B; return o; };
  T *qcb = take(nq), *qb = take(nq), *qb0 = take(nq), *qsb = take(nq);
  T *vvb = take(nv), *tb = take(nv), *vb = take(nv), *vb0 = take(nv), *vsb = take(nv), *vdb = take(nv), *phib = take(nv);
  T *sb1 = take(ns), *sacc = take(ns), *sdc = take(ns);
  T *idq = take(ct ? nq : 0), *idv = take(ct ? nv : 0), *idvd = take(ct ? nv : 0);
  // the controller: device bounds (copied from pageable memory, as integrate_t does), the recompute's per-stage rows
  const T* lo = nullptr;
  const T* hi = nullptr;
  if (bounds) {
    T* dev = (T*)work.p + (size_t)rows * B;
    if (int rc = upload_bounds(dev, effort_lo, effort_hi, nv, stream)) return rc;
    lo = dev; hi = dev + nv;
  }
  const T* tau_applied[4] = {nullptr, nullptr, nullptr, nullptr};
  const T* vd_des[4] = {nullptr, nullptr, nullptr, nullptr};
  for (int i = 0; i < 4 && closed; ++i) {
    tau_applied[i] = stages + (prow + (size_t)i * nv) * B;
    if (ct) vd_des[i] = stages + (prow + (4 + (size_t)i) * nv) * B;
  }
  const bool want_tb = taub || closed;      // the controller's adjoint reads τ̄ of every stage
  const size_t qbytes = (size_t)nq * B * sizeof(T), vbytes = (size_t)nv * B * sizeof(T);
  if (qtb) RBD_CUDA_TRY(cudaMemcpyAsync(qb, qtb + (size_t)nsteps * nq * B, qbytes, cudaMemcpyDeviceToDevice, stream));
  else RBD_CUDA_TRY(cudaMemsetAsync(qb, 0, qbytes, stream));
  if (vtb) RBD_CUDA_TRY(cudaMemcpyAsync(vb, vtb + (size_t)nsteps * nv * B, vbytes, cudaMemcpyDeviceToDevice, stream));
  else RBD_CUDA_TRY(cudaMemsetAsync(vb, 0, vbytes, stream));
  const size_t sbytes = (size_t)ns * B * sizeof(T);
  if (ns && stb) RBD_CUDA_TRY(cudaMemcpyAsync(sb1, stb + (size_t)nsteps * ns * B, sbytes, cudaMemcpyDeviceToDevice, stream));
  else if (ns) RBD_CUDA_TRY(cudaMemsetAsync(sb1, 0, sbytes, stream));
  // the contact stage adjoint: one plan (grid, workspace and the solve's zero) for the whole call
  ContactVjpArgs<T> cva{};
  std::optional<LaunchPlan> cplan;
  ModelDev<T> Mz;
  if (cd && nsteps > 0) {
    Mz = M;
    for (int k = 0; k < 3; ++k) { cva.g[k] = M.g[k]; Mz.g[k] = T(0); }
    const size_t row_bytes = (size_t)contact_vjp_rows(hm.nb, hm.nv) * sizeof(T);
    cplan.emplace();
    if (int rc = plan_persistent((const void*)contact_vjp_kernel<T>, 32, (size_t)std::max(1, (int)M.nrows) * 32 * sizeof(T), (B + 31) / 32,
                                 stream, *cplan, row_bytes, sizeof(T), size_t(512) << 20)) return rc;
    cva.work = (T*)cplan->work.p;
    cva.zero = cva.work + row_bytes / sizeof(T) * cplan->grid * 32;
    RBD_CUDA_TRY(cudaMemsetAsync(const_cast<T*>(cva.zero), 0, sizeof(T), stream));
    cva.vdb = vdb; cva.qc = qcb; cva.vb = vvb; cva.taub = (taub || closed) ? tb : nullptr;
    cva.sb1 = sb1; cva.sacc = sacc; cva.sdc = sdc; cva.B = B;
  }
  bool has_other = false;
  for (int i = 0; i < hm.nb; ++i) has_other |= (M.body[i].kind != K_REV && M.body[i].kind != K_PRIS && M.body[i].kind != K_FIXED);
  constexpr int N = VecOf<T>::N;
  const size_t va = sizeof(typename VecOf<T>::type);
  auto aligned = [&](const T* x, int64_t stride) { return !x || ((uintptr_t)x % va == 0 && stride % N == 0); };
  bool vec_ok = B % N == 0 && B >= 1024 && aligned(taub, step_stride) && aligned(taub, stage_stride) && aligned(qtb, 0) &&
                aligned(vtb, 0) && aligned(q_traj, 0);
  if (pd) {     // ... and every controller array and controller adjoint (kp_bar / kd_bar are [nv x B] whatever gain_ld is)
    const rbd_pd_bar cb = pd_bar ? *pd_bar : rbd_pd_bar{};
    vec_ok = vec_ok && aligned((const T*)pd->q_ref, pd->q_ref_step_stride) && aligned((const T*)pd->v_ref, pd->v_ref_step_stride) &&
             (pd->gain_ld == 0 || (aligned((const T*)pd->kp, 0) && aligned((const T*)pd->kd, 0))) && aligned((const T*)cb.kp, 0) &&
             aligned((const T*)cb.kd, 0) && aligned((const T*)cb.q_ref, pd->q_ref_step_stride) &&
             aligned((const T*)cb.v_ref, pd->v_ref_step_stride) && aligned((const T*)cb.vd_ref, pd->v_ref_step_stride);
  }
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
    const T* s0 = cd ? s_traj + (size_t)s * ns * B : nullptr;
    Rollout rec{const_cast<T*>(q0), const_cast<T*>(v0), const_cast<T*>(s0), tau ? tau + s * step_stride : nullptr, step_stride,
                stage_stride, dt, 1};
    rec.stages = stages;
    rec.contact = cd;
    rbd_pd_desc pds{};      // the recompute is a one-step rollout: the controller's references start at step s
    rbd_task_pd_desc tds{};
    if (pd) {
      pds = *pd;
      const size_t vo = (size_t)s * pd->v_ref_step_stride;
      pds.q_ref = (const T*)pd->q_ref + (size_t)s * pd->q_ref_step_stride;
      pds.v_ref = pd->v_ref ? (const T*)pd->v_ref + vo : nullptr;
      pds.vd_ref = pd->vd_ref ? (const T*)pd->vd_ref + vo : nullptr;
      rec.pd = &pds;
      rec.pd_bounds = lo;      // the bounds copied above: one host copy per call
    }
    if (task) {
      tds = *task;
      tds.x_ref = (const T*)task->x_ref + (size_t)s * task->x_ref_step_stride;
      tds.xd_ref = task->xd_ref ? (const T*)task->xd_ref + (size_t)s * task->xd_ref_step_stride : nullptr;
      tds.joint = pd ? &pds : nullptr;
      rec.task = &tds;
      rec.pd = nullptr;
      rec.pd_bounds = lo;
    }
    if (int rc = integrate(model, dtype, B, B, rec, stream)) return rc;
    a.q0 = q0;
    a.qtb = qtb ? qtb + (size_t)s * nq * B : nullptr;
    a.vtb = vtb ? vtb + (size_t)s * nv * B : nullptr;
    PdAdjArgs<T> c{};
    if (pd) {
      c = pd_adj_step<T>(*pd, pd_bar, s);
      c.lo = lo; c.hi = hi;
      if (ct) { c.idq = idq; c.idv = idv; c.idvd = idvd; }
    }
    for (int g = 4; g >= 0; --g) {
      a.g = g; a.l = g == 4 ? 3 : g - 1;
      a.tau_bar = (taub && g < 4) ? taub + s * step_stride + g * stage_stride : nullptr;
      // computed-torque mode and task-space control: masked before the inverse-dynamics / task VJP
      c.tau = (bounds && !ct && !task && g < 4) ? tau_applied[g] : nullptr;
      if (vec_ok) {
        if (pd) integrate_adjoint_pd_linear_kernel<T><<<dim3(grid_lin, hm.nb), 256, 0, stream>>>(M, a, c);
        else integrate_adjoint_linear_kernel<T><<<dim3(grid_lin, hm.nb), 256, 0, stream>>>(M, a);
        if (int rc = api_launched()) return rc;
      }
      if (!vec_ok || has_other) {
        if (pd) integrate_adjoint_pd_kernel<T><<<dim3(grid, hm.nb), 128, 0, stream>>>(M, a, c, vec_ok);
        else integrate_adjoint_kernel<T><<<dim3(grid, hm.nb), 128, 0, stream>>>(M, a, vec_ok);
        if (int rc = api_launched()) return rc;
      }
      if (a.l < 0) {
        if (s > 0) {
          integrate_adjoint_out_kernel<T><<<dim3(grid, hm.nb), 128, 0, stream>>>(M, OutArgs<T>{q0, qb, nullptr, qb, B});
          if (int rc = api_launched()) return rc;
        }
        continue;
      }
      const int l = a.l;
      if (cd) {
        const T* sd = stages + (size_t)stage_rows(nq, nv) * B;
        cva.q = a.qs[l]; cva.v = a.vs[l]; cva.vd = vd[l];
        cva.s0 = s0; cva.sdp = l ? sd + (size_t)(l - 1) * ns * B : nullptr;
        cva.stb = (l == 0 && stb) ? stb + (size_t)s * ns * B : nullptr;
        cva.wa = a.wa[l]; cva.wdb = (T)dt * a.wb[l]; cva.l = l;
        contact_vjp_kernel<T><<<cplan->grid, cplan->block, cplan->smem, stream>>>(Mz, *C, cva);
        if (int rc = api_launched(&*cplan)) return rc;
      } else if (int rc = dynamics_vjp_dense(model, dtype, B, a.qs[l], a.vs[l], vd[l], vdb, qcb, vvb, want_tb ? tb : nullptr, stream)) {
        return rc;
      }
      // computed-torque mode and task-space control: m = τ̄ masked by the applied torque, the seed of the VJPs below
      if (bounds && (ct || task))
        if (int rc = launch_pd_mask(PdMaskArgs<T>{tb, tau_applied[l], lo, hi, nv, B}, p.sms, stream)) return rc;
      if (ct)     // the inverse-dynamics VJP at (q_s, v_s, v̇_des) seeded with m
        if (int rc = inverse_dynamics_vjp_dense(model, dtype, B, a.qs[l], a.vs[l], vd_des[l], tb, idq, idv, idvd, stream)) return rc;
      if (task) {     // the task law's adjoint at (q_s, v_s) with the references of step s, seeded with m (torque) or v̇̄_des
        TaskPdVjpArgs<T> ta = task_vjp_step<T>(*task, r.task_bar, s);
        ta.q = a.qs[l]; ta.v = a.vs[l]; ta.w = ct ? idvd : tb;
        // where the next phase kernel reads q̄ / v̄: the PD phase kernels add the inverse-dynamics VJP's rows themselves, the
        // open-loop ones do not, so without a joint term those are folded into the dynamics VJP's rows here
        ta.qacc = ct && pd ? idq : qcb; ta.vacc = ct && pd ? idv : vvb;
        ta.qfold = ct && !pd ? idq : nullptr; ta.vfold = ct && !pd ? idv : nullptr;
        ta.B = B;
        if (int rc = tplan.launch(M, ta, stream)) return rc;
      }
    }
  }
  if (q0t || q0c) {
    integrate_adjoint_out_kernel<T><<<dim3(grid, hm.nb), 128, 0, stream>>>(M, OutArgs<T>{q_traj, qb, q0t, q0c, B});
    if (int rc = api_launched()) return rc;
  }
  if (v0b) RBD_CUDA_TRY(cudaMemcpyAsync(v0b, vb, vbytes, cudaMemcpyDeviceToDevice, stream));
  if (ns && s0b) RBD_CUDA_TRY(cudaMemcpyAsync(s0b, sb1, sbytes, cudaMemcpyDeviceToDevice, stream));
  return RBD_OK;
}

// rbd_task_pd_torques_vjp: the law at (q, v) recomputed (task_pd_law), τ̄ masked by the applied torque, in computed-torque mode the
// inverse-dynamics VJP at (q, v, v̇_des), then one task_pd_vjp_kernel with the joint term's adjoint in the same pass, and the
// configuration covector brought to its tangent and minimal-norm forms.  Every array [rows x B].
template <class T>
int task_pd_torques_vjp_t(const rbd_model* model, int32_t dtype, int64_t B, const T* q, const T* v, const T* tau_ff,
                          const rbd_task_pd_desc& c, int step, const T* taub_out, T* qt, T* qcfg, T* vbar, T* tffb,
                          const rbd_task_pd_bar* bar, cudaStream_t stream) {
  const HostModel& hm = model->hm;
  const ModelDev<T>& M = dev_model<T>(hm);
  const int64_t nq = hm.nq, nv = hm.nv;
  const bool ct = c.mode == RBD_PD_COMPUTED_TORQUE, bounds = c.effort_lo != nullptr;
  const rbd_pd_desc* j = c.joint;
  TaskPdVjpPlan<T> tplan;
  if (int rc = tplan.init(hm, c, B, stream)) return rc;
  DeviceProps p;
  RBD_CUDA_TRY(device_props(p));
  // workspace: τ applied, m, v̇_des, v̄_ID, v̇̄_des (nv rows each), q̄ and q̄_ID (nq rows each), v̄ (nv), the bounds (2 nv values)
  StreamAlloc work;
  RBD_CUDA_TRY(work.alloc(((size_t)(6 * nv + 2 * nq) * B + 2 * nv) * sizeof(T), stream));
  T* tau = (T*)work.p;
  T *m = tau + nv * B, *vdes = m + nv * B, *idv = vdes + nv * B, *idvd = idv + nv * B, *vacc = idvd + nv * B;
  T *qacc = vacc + nv * B, *idq = qacc + nq * B;
  T* lohi = idq + nq * B;
  if (bounds)
    if (int rc = upload_bounds(lohi, c.effort_lo, c.effort_hi, nv, stream)) return rc;
  const size_t vbytes = (size_t)nv * B * sizeof(T), qbytes = (size_t)nq * B * sizeof(T);
  RBD_CUDA_TRY(cudaMemcpyAsync(m, taub_out, vbytes, cudaMemcpyDeviceToDevice, stream));
  RBD_CUDA_TRY(cudaMemsetAsync(qacc, 0, qbytes, stream));
  RBD_CUDA_TRY(cudaMemsetAsync(vacc, 0, vbytes, stream));
  if (bounds || ct)
    if (int rc = task_pd_law(model, dtype, B, q, v, tau_ff, c, step, tau, ct ? vdes : nullptr, stream)) return rc;
  if (bounds)
    if (int rc = launch_pd_mask(PdMaskArgs<T>{m, tau, lohi, lohi + nv, nv, B}, p.sms, stream)) return rc;
  if (tffb) RBD_CUDA_TRY(cudaMemcpyAsync(tffb, m, vbytes, cudaMemcpyDeviceToDevice, stream));
  if (ct)
    if (int rc = inverse_dynamics_vjp_dense(model, dtype, B, q, v, vdes, m, idq, idv, idvd, stream)) return rc;
  TaskPdVjpArgs<T> ta = task_vjp_step<T>(c, bar, step);
  ta.q = q; ta.v = v; ta.w = ct ? idvd : m;
  ta.qacc = qacc; ta.vacc = vacc;
  ta.qfold = ct && !j ? idq : nullptr; ta.vfold = ct && !j ? idv : nullptr;
  if (j) {     // the joint term at the references of `step`; in computed-torque mode it also adds the inverse-dynamics VJP's q̄ / v̄
    ta.has_joint = true;
    ta.joint = pd_adj_step<T>(*j, bar ? bar->joint : nullptr, step);
    if (ct) { ta.joint.idq = idq; ta.joint.idv = idv; ta.joint.idvd = idvd; }
  }
  ta.B = B;
  if (int rc = tplan.launch(M, ta, stream)) return rc;
  if (qt || qcfg) {
    const int grid = (int)std::min<int64_t>((B + 127) / 128, (int64_t)p.sms * 8);
    integrate_adjoint_out_kernel<T><<<dim3(grid, hm.nb), 128, 0, stream>>>(M, OutArgs<T>{q, qacc, qt, qcfg, B});
    if (int rc = api_launched()) return rc;
  }
  if (vbar) RBD_CUDA_TRY(cudaMemcpyAsync(vbar, vacc, vbytes, cudaMemcpyDeviceToDevice, stream));
  return RBD_OK;
}

// the adjoint of an array of a task-space controller exists only where the array does (fn: the entry point named in the messages)
int check_task_pd_bar(const std::string& fn, const rbd_task_pd_desc& c, const rbd_task_pd_bar* bar) {
  auto fail = [&](const char* what) { return api_fail(RBD_EINVAL, fn + ": " + what); };
  if (!bar) return RBD_OK;
  if (bar->xd_ref && !c.xd_ref) return fail("ctrl_bar->xd_ref needs ctrl->xd_ref");
  if (bar->joint && !c.joint) return fail("ctrl_bar->joint needs ctrl->joint");
  if (bar->joint && ((bar->joint->v_ref && !c.joint->v_ref) || (bar->joint->vd_ref && !c.joint->vd_ref)))
    return fail("ctrl_bar->joint->v_ref / vd_ref need the joint term's v_ref / vd_ref");
  return RBD_OK;
}

// The argument checks of the rollout VJP entry points, after api_check (fn: the entry point named in the messages); each entry
// point adds the check of the argument that names it.  The controller's are rbd_integrate_pd's / rbd_integrate_task_pd's with
// leading dimension B.  RBD_OK also when there is nothing to compute.
int check_rollout_vjp(const std::string& fn, const rbd_model* model, int32_t dtype, int64_t B, const RolloutVjp& r) {
  auto fail = [&](int status, const char* what) { return api_fail(status, fn + ": " + what); };
  if (dtype != RBD_F32 && dtype != RBD_F64) return fail(RBD_EUNSUPPORTED, "fp32 and fp64 only");
  if (r.nsteps < 0 || !(r.dt > 0)) return fail(RBD_EINVAL, "need dt > 0 and nsteps >= 0");
  if (r.tau_step_stride < 0 || r.tau_stage_stride < 0) return fail(RBD_EINVAL, "torque strides must be >= 0");
  if (!r.tau && r.tau_bar) return fail(RBD_EINVAL, "tau_bar needs tau");
  if (r.contact)
    if (int rc = api_check_contact(model, r.contact, fn.c_str())) return rc;
  if (r.pd) {
    if (int rc = api_check_pd(fn.c_str(), model, B, r.pd)) return rc;
    // the adjoint of an array exists only where the array does
    if (r.pd_bar && ((r.pd_bar->v_ref && !r.pd->v_ref) || (r.pd_bar->vd_ref && !r.pd->vd_ref)))
      return fail(RBD_EINVAL, "pd_bar->v_ref / vd_ref need pd->v_ref / vd_ref");
  }
  if (r.task) {
    if (int rc = api_check_task_ctrl(fn.c_str(), model, B, r.task)) return rc;
    if (int rc = check_task_pd_bar(fn, *r.task, r.task_bar)) return rc;
  }
  if ((r.pd && r.pd->mode == RBD_PD_COMPUTED_TORQUE) || (r.task && r.task->mode == RBD_PD_COMPUTED_TORQUE))
    if (int rc = check_vjp_limits(model->hm, fn.c_str())) return rc;
  if (B == 0 || model->hm.nv == 0) return RBD_OK;
  if (!r.q_traj || !r.v_traj) return fail(RBD_EINVAL, "q_traj and v_traj must not be NULL");
  if (r.contact && r.contact->npoints * r.contact->nhalfspaces > 0 && !r.s_traj)
    return fail(RBD_EINVAL, "s_traj must not be NULL when there are contact pairs");
  return RBD_OK;
}

// runs a checked request
int integrate_vjp(const rbd_model* model, int32_t dtype, int64_t B, const RolloutVjp& r, void* stream) {
  if (B == 0 || model->hm.nv == 0) return RBD_OK;
  cudaStream_t s = (cudaStream_t)stream;
  return dtype == RBD_F32 ? integrate_vjp_t<float>(model, B, r, s) : integrate_vjp_t<double>(model, B, r, s);
}

}  // namespace

extern "C" int32_t rbd_integrate_vjp(const rbd_model* model, int32_t dtype, int64_t B, const void* q_traj, const void* v_traj,
                                     const void* tau, int64_t tau_step_stride, int64_t tau_stage_stride, double dt, int32_t nsteps,
                                     const void* q_traj_bar, const void* v_traj_bar, void* q0_bar_tan, void* q0_bar_cfg, void* v0_bar,
                                     void* tau_bar, void* stream) {
  if (int rc = api_check(model, dtype, B, B)) return rc;
  const ApiCall call;
  const RolloutVjp r{q_traj, v_traj, nullptr, tau, tau_step_stride, tau_stage_stride, dt, nsteps, q_traj_bar, v_traj_bar, nullptr,
                     q0_bar_tan, q0_bar_cfg, v0_bar, nullptr, tau_bar};
  if (int rc = check_rollout_vjp("rbd_integrate_vjp", model, dtype, B, r)) return rc;
  return integrate_vjp(model, dtype, B, r, stream);
}

extern "C" int32_t rbd_integrate_contact_vjp(const rbd_model* model, int32_t dtype, int64_t B, const void* q_traj, const void* v_traj,
                                             const void* s_traj, const void* tau, int64_t tau_step_stride, int64_t tau_stage_stride,
                                             const rbd_contact_desc* contact, double dt, int32_t nsteps, const void* q_traj_bar,
                                             const void* v_traj_bar, const void* s_traj_bar, void* q0_bar_tan, void* q0_bar_cfg,
                                             void* v0_bar, void* s0_bar, void* tau_bar, void* stream) {
  if (int rc = api_check(model, dtype, B, B)) return rc;
  const ApiCall call;
  RolloutVjp r{q_traj, v_traj, s_traj, tau, tau_step_stride, tau_stage_stride, dt, nsteps, q_traj_bar, v_traj_bar, s_traj_bar,
               q0_bar_tan, q0_bar_cfg, v0_bar, s0_bar, tau_bar};
  r.contact = contact;
  if (int rc = check_rollout_vjp("rbd_integrate_contact_vjp", model, dtype, B, r)) return rc;
  if (!contact) return api_fail(RBD_EINVAL, "rbd_integrate_contact_vjp: contact must not be NULL");
  return integrate_vjp(model, dtype, B, r, stream);
}

extern "C" int32_t rbd_integrate_pd_vjp(const rbd_model* model, int32_t dtype, int64_t B, const void* q_traj, const void* v_traj,
                                        const void* s_traj, const void* tau, int64_t tau_step_stride, int64_t tau_stage_stride,
                                        const rbd_pd_desc* pd, const rbd_contact_desc* contact, double dt, int32_t nsteps,
                                        const void* q_traj_bar, const void* v_traj_bar, const void* s_traj_bar, void* q0_bar_tan,
                                        void* q0_bar_cfg, void* v0_bar, void* s0_bar, void* tau_bar, const rbd_pd_bar* pd_bar,
                                        void* stream) {
  if (int rc = api_check(model, dtype, B, B)) return rc;
  const ApiCall call;
  RolloutVjp r{q_traj, v_traj, s_traj, tau, tau_step_stride, tau_stage_stride, dt, nsteps, q_traj_bar, v_traj_bar, s_traj_bar,
               q0_bar_tan, q0_bar_cfg, v0_bar, s0_bar, tau_bar};
  r.contact = contact; r.pd = pd; r.pd_bar = pd_bar;
  if (int rc = check_rollout_vjp("rbd_integrate_pd_vjp", model, dtype, B, r)) return rc;
  if (!pd) return api_fail(RBD_EINVAL, "rbd_integrate_pd_vjp: pd must not be NULL");
  return integrate_vjp(model, dtype, B, r, stream);
}

extern "C" int32_t rbd_integrate_task_pd_vjp(const rbd_model* model, int32_t dtype, int64_t B, const void* q_traj, const void* v_traj,
                                             const void* s_traj, const void* tau, int64_t tau_step_stride, int64_t tau_stage_stride,
                                             const rbd_task_pd_desc* ctrl, const rbd_contact_desc* contact, double dt, int32_t nsteps,
                                             const void* q_traj_bar, const void* v_traj_bar, const void* s_traj_bar, void* q0_bar_tan,
                                             void* q0_bar_cfg, void* v0_bar, void* s0_bar, void* tau_bar, const rbd_task_pd_bar* ctrl_bar,
                                             void* stream) {
  if (int rc = api_check(model, dtype, B, B)) return rc;
  const ApiCall call;
  RolloutVjp r{q_traj, v_traj, s_traj, tau, tau_step_stride, tau_stage_stride, dt, nsteps, q_traj_bar, v_traj_bar, s_traj_bar,
               q0_bar_tan, q0_bar_cfg, v0_bar, s0_bar, tau_bar};
  r.contact = contact; r.task = ctrl; r.task_bar = ctrl_bar;
  if (int rc = check_rollout_vjp("rbd_integrate_task_pd_vjp", model, dtype, B, r)) return rc;
  if (!ctrl) return api_fail(RBD_EINVAL, "rbd_integrate_task_pd_vjp: ctrl must not be NULL");
  return integrate_vjp(model, dtype, B, r, stream);
}

extern "C" int32_t rbd_task_pd_torques_vjp(const rbd_model* model, int32_t dtype, int64_t B, const void* q, const void* v,
                                           const void* tau_ff, const rbd_task_pd_desc* ctrl, int32_t step, const void* tau_out_bar,
                                           void* q_bar_tan, void* q_bar_cfg, void* v_bar, void* tau_ff_bar,
                                           const rbd_task_pd_bar* ctrl_bar, void* stream) {
  const std::string fn = "rbd_task_pd_torques_vjp";
  auto fail = [&](int status, const std::string& what) { return api_fail(status, fn + ": " + what); };
  if (int rc = api_check(model, dtype, B, B)) return rc;
  const ApiCall call;
  if (dtype != RBD_F32 && dtype != RBD_F64) return fail(RBD_EUNSUPPORTED, "fp32 and fp64 only");
  if (int rc = api_check_task_ctrl(fn.c_str(), model, B, ctrl)) return rc;
  if (step < 0) return fail(RBD_EINVAL, "step must be >= 0");
  if (!tau_ff && tau_ff_bar) return fail(RBD_EINVAL, "tau_ff_bar needs tau_ff");
  if (int rc = check_task_pd_bar(fn, *ctrl, ctrl_bar)) return rc;
  if (ctrl->mode == RBD_PD_COMPUTED_TORQUE)
    if (int rc = check_vjp_limits(model->hm, fn.c_str())) return rc;
  if (B == 0 || model->hm.nv == 0) return RBD_OK;
  if (!q || !v || !tau_out_bar) return fail(RBD_EINVAL, "q, v and tau_out_bar must not be NULL");
  cudaStream_t s = (cudaStream_t)stream;
  return dtype == RBD_F32
             ? task_pd_torques_vjp_t<float>(model, dtype, B, (const float*)q, (const float*)v, (const float*)tau_ff, *ctrl, step,
                                            (const float*)tau_out_bar, (float*)q_bar_tan, (float*)q_bar_cfg, (float*)v_bar, (float*)tau_ff_bar,
                                            ctrl_bar, s)
             : task_pd_torques_vjp_t<double>(model, dtype, B, (const double*)q, (const double*)v, (const double*)tau_ff, *ctrl, step,
                                             (const double*)tau_out_bar, (double*)q_bar_tan, (double*)q_bar_cfg, (double*)v_bar,
                                             (double*)tau_ff_bar, ctrl_bar, s);
}
