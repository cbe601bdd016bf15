// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
// Runs rbd_integrate_derivatives ON THE CPU over the same (step, sample) batch the kernels see: the gather, the stage recompute of
// rbd_integrate (joint_stage + aba_sample, with the kernels' arithmetic), the stage Jacobians of csrc/rbd_deriv.cuh (as
// hostsim_deriv_ext.cpp) and the per-joint stages, products and finishing step of csrc/rbd_integrate_deriv.cuh, on [rows][N]
// arrays laid out like the kernels' workspace.  Also exports the per-joint maps (G / L JVPs, N and N⁺) for finite differences.
#include <string>
#include <vector>

#include "../../rigidbodydynamics/jl_b200/csrc/rbd_deriv.cuh"
#include "../../rigidbodydynamics/jl_b200/csrc/rbd_integrate_deriv.cuh"
#include "../../rigidbodydynamics/jl_b200/csrc/rbd_model.h"

using namespace rbd;

namespace {
template <class T> const ModelDev<T>& dev(const HostModel& m);
template <> const ModelDev<float>& dev<float>(const HostModel& m) { return m.dev32; }
template <> const ModelDev<double>& dev<double>(const HostModel& m) { return m.dev64; }

const double kA[4] = {0.0, 0.5, 0.5, 1.0}, kB[4] = {1.0 / 6, 1.0 / 3, 1.0 / 3, 1.0 / 6};

// the four stages of one step from column b of (q0, v0) with torques tau (NULL: zero), as hostsim_integrate_vjp.cpp's stages
template <class T>
void stages(const HostModel& hm, int64_t N, int64_t b, const T* q0, const T* v0, const T* tau, double dt, T* const* qs, T* const* vs,
            T* const* pd, T* const* vd) {
  const ModelDev<T>& M = dev<T>(hm);
  std::vector<T> stash(M.nrows + 64), phi(M.nv), vv(M.nv);
  for (int i = 0; i < 4; ++i) {
    const T wa = (T)(dt * kA[i]);
    for (int k = 0; k < M.nv; ++k) {
      const int64_t e = (int64_t)k * N + b;
      phi[k] = i ? wa * pd[i - 1][e] : T(0);
      vv[k] = i ? v0[e] + wa * vd[i - 1][e] : v0[e];
      vs[i][e] = vv[k];
    }
    const Col<T> cq0{q0 + b, N}, cphi{phi.data(), 1}, cvs{vv.data(), 1};
    const ColOut<T> oqs{qs[i] + b, N, true}, opd{pd[i] + b, N, true};
    for (int j = 0; j < M.nb; ++j) joint_stage(M.body[j], cq0, cphi, cvs, oqs, opd);
    AbaIO<T, false> io;
    io.q = {qs[i] + b, N}; io.v = {vs[i] + b, N};
    io.tau = {tau ? tau + b : nullptr, N}; io.wext = {nullptr, 1};
    io.vd = {vd[i] + b, N, true}; io.qd = {nullptr, 1, true}; io.ext = {nullptr, 1};
    Stash<T, 1> st{stash.data()};
    if (hm.general) aba_sample<T, Stash<T, 1>, true>(M, io, st);
    else aba_sample<T, Stash<T, 1>, false>(M, io, st);
  }
}

// [Dq | Dv | Dτ] of column b at (q, v, v̇), as hostsim_deriv_ext.cpp's forward run with d v̇ / d tau
template <class T>
void stage_jacobians(const HostModel& hm, int64_t N, int64_t b, const T* q, const T* v, const T* vd, T* D) {
  const ModelDev<T>& M = dev<T>(hm);
  DerivDev Dd; DerivAnc A;
  build_deriv_dev(M, Dd, A);
  const int nv = Dd.nv;
  const int64_t nv2 = (int64_t)nv * nv;
  std::vector<T> stash(kin_rows(hm) + 64), scr(Dd.rows), x(nv);
  DerivIO<T> io;
  io.q = {q + b, N}; io.v = {v + b, N}; io.vd = {vd + b, N};
  io.s = scr.data(); io.sld = 1; io.active = true;
  deriv_world_sample<T>(M, Dd, io, Stash<T, 1>{stash.data()});
  for (int c = 0; c < kBodyRows; ++c) deriv_accumulate<T>(M, Dd, scr.data(), 1, c);
  for (int K = 0; K < M.nb; ++K) deriv_pairs<T>(Dd, A, scr.data(), 1, D + b, D + nv2 * N + b, N, K, true);
  const T* H = scr.data() + Dd.h_base;
  deriv_factor<T>(Dd, A, scr.data() + Dd.h_base, 1);
  auto Hf = [H](int row) { return H[row]; };
  for (int c = 0; c < 3 * nv; ++c) {
    const int blk = c / nv, vj = c % nv;
    deriv_solve_column<T>(Dd, A, Hf, x.data(), 1, D + blk * nv2 * N + (int64_t)vj * nv * N + b, N, vj, true, blk == 2);
  }
}

template <class T>
void run(const HostModel& hm, int64_t B, const T* qt, const T* vt, const T* tau, int64_t step, double dt, int nsteps, T* Aout, T* Bout) {
  const ModelDev<T>& M = dev<T>(hm);
  const int64_t nq = M.nq, nv = M.nv, N = (int64_t)nsteps * B, nv2 = nv * nv;
  std::vector<T> q0(nq * N), v0(nv * N), t0(tau ? nv * N : 0), w((4 * nq + 12 * nv) * N), big(7 * 3 * nv2 * N);
  for (int64_t n = 0; n < N; ++n) {
    const int64_t s = n / B, b = n % B;
    for (int64_t k = 0; k < nq; ++k) q0[k * N + n] = qt[(s * nq + k) * B + b];
    for (int64_t k = 0; k < nv; ++k) v0[k * N + n] = vt[(s * nv + k) * B + b];
    if (tau)
      for (int64_t k = 0; k < nv; ++k) t0[k * N + n] = tau[s * step + k * B + b];
  }
  T *qs[4], *vs[4], *pd[4], *vd[4];
  for (int i = 0; i < 4; ++i) {
    qs[i] = w.data() + i * nq * N; vs[i] = w.data() + (4 * nq + i * nv) * N;
    pd[i] = w.data() + (4 * nq + (4 + i) * nv) * N; vd[i] = w.data() + (4 * nq + (8 + i) * nv) * N;
  }
  for (int64_t b = 0; b < N; ++b) stages(hm, N, b, q0.data(), v0.data(), tau ? t0.data() : (const T*)nullptr, dt, qs, vs, pd, vd);
  T* p = big.data();
  auto take = [&]() { T* o = p; p += 3 * nv2 * N; return o; };
  T *D = take(), *Vd = take(), *X = take(), *Y = take(), *P = take(), *SP = take(), *SV = take();
  LinArgs<T> a{};
  a.q0 = q0.data();
  for (int i = 0; i < 4; ++i) { a.qs[i] = qs[i]; a.vs[i] = vs[i]; a.pd[i] = pd[i]; a.wa[i] = (T)(dt * kA[i]); a.wb[i] = (T)kB[i]; }
  a.D = D; a.X = X; a.Y = Y; a.P = P; a.SP = SP; a.SV = SV; a.vd = Vd;
  a.A = Aout; a.Bt = Bout;
  a.ld = N; a.n0 = 0; a.B = B; a.nv = (int)nv; a.dt = (T)dt;
  for (int i = 0; i < 4; ++i) {
    a.i = i;
    a.vdp = i == 1 ? D : Vd;
    for (int64_t b = 0; b < N; ++b)
      for (int j = 0; j < M.nb; ++j)
        for (int c = 0; c < 3 * nv; ++c) lin_stage_joint(M.body[j], a, b, c);
    for (int64_t b = 0; b < N; ++b) stage_jacobians(hm, N, b, qs[i], vs[i], vd[i], D);
    if (i == 0) continue;
    for (int64_t b = 0; b < N; ++b)
      for (int r0 = 0; r0 < nv; r0 += 4)
        for (int c0 = 0; c0 < 3 * nv; c0 += 8) lin_product_tile<T, 4, 8>(a, b, r0, c0);
  }
  a.vdp = Vd;
  for (int64_t b = 0; b < N; ++b)
    for (int j = 0; j < M.nb; ++j)
      for (int c = 0; c < 3 * nv; ++c) lin_finish_joint(M.body[j], a, b, c);
}
}  // namespace

extern "C" {
int hostsim_integrate_derivatives(const rbd_model_desc* d, int dtype, int64_t B, const void* qt, const void* vt, const void* tau,
                                  int64_t step, double dt, int nsteps, void* A, void* Bm) {
  HostModel hm; std::string err;
  if (int rc = build_host_model(d, hm, err)) return rc;
  if (dtype == 0)
    run<float>(hm, B, (const float*)qt, (const float*)vt, (const float*)tau, step, dt, nsteps, (float*)A, (float*)Bm);
  else
    run<double>(hm, B, (const double*)qt, (const double*)vt, (const double*)tau, step, dt, nsteps, (double*)A, (double*)Bm);
  return 0;
}
// one joint of kind `kind`, fp64, local rows
void hostsim_joint_g_jvp(int kind, const double* q0, const double* dq0, const double* phi, const double* dphi, double* qs, double* dqs) {
  g_jvp(kind, q0, dq0, phi, dphi, qs, dqs);
}
void hostsim_joint_l_jvp(int kind, const double* q0, const double* dq0, const double* qs, const double* dqs, const double* vs,
                         const double* dvs, double* dpd) {
  l_jvp(kind, q0, dq0, qs, dqs, vs, dvs, dpd);
}
void hostsim_joint_vel_to_cfg(int kind, const double* q, const double* v, double* qd) { vel_to_cfg(kind, q, v, qd); }
void hostsim_joint_cfg_to_vel(int kind, const double* q, const double* qd, double* v) { cfg_to_vel(kind, q, qd, v); }
}
