// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
// Runs the backward pass of rbd_integrate_vjp ON THE CPU, one sample at a time: the stage recompute of rbd_integrate (joint_stage
// + aba_sample, with the kernels' arithmetic), dynamics_vjp_sample (csrc/rbd_adjoint.cuh) and the per-joint adjoints of
// csrc/rbd_integrate_adjoint.cuh, on [rows][B] arrays laid out like the kernels' workspace.  Also exports the forward trajectory
// and the per-joint coordinate maps and their adjoints, so the mathematics can be checked against finite differences without a GPU.
#include <string>
#include <vector>

#include "../../rigidbodydynamics/jl_b200/csrc/rbd_adjoint.cuh"
#include "../../rigidbodydynamics/jl_b200/csrc/rbd_integrate_adjoint.cuh"
#include "../../rigidbodydynamics/jl_b200/csrc/rbd_model.h"

using namespace rbd;

namespace {
template <class T> const ModelDev<T>& dev(const HostModel& m);
template <> const ModelDev<float>& dev<float>(const HostModel& m) { return m.dev32; }
template <> const ModelDev<double>& dev<double>(const HostModel& m) { return m.dev64; }

const double kA[4] = {0.0, 0.5, 0.5, 1.0}, kB[4] = {1.0 / 6, 1.0 / 3, 1.0 / 3, 1.0 / 6};

template <class T> struct Sched {        // torques of (step s, stage i), leading dimension B, or none
  const T* tau; int64_t step, stage;
  const T* at(int s, int i) const { return tau ? tau + s * step + i * stage : nullptr; }
};

// the four stages of one step from column b of (q0, v0), into column b of qs[i] / vs[i] / pd[i] / vd[i]  (integrate_stage_kernel)
template <class T>
void stages(const HostModel& hm, int64_t B, int64_t b, const T* q0, const T* v0, const Sched<T>& tau, int s, double dt, T* const* qs,
            T* const* vs, T* const* pd, T* const* vd) {
  const ModelDev<T>& M = dev<T>(hm);
  std::vector<T> stash(M.nrows + 64), phi(M.nv), vv(M.nv);
  for (int i = 0; i < 4; ++i) {
    const T wa = (T)(dt * kA[i]);
    for (int k = 0; k < M.nv; ++k) {
      const int64_t e = (int64_t)k * B + b;
      phi[k] = i ? wa * pd[i - 1][e] : T(0);
      vv[k] = i ? v0[e] + wa * vd[i - 1][e] : v0[e];
      vs[i][e] = vv[k];
    }
    const Col<T> cq0{q0 + b, B}, cphi{phi.data(), 1}, cvs{vv.data(), 1};
    const ColOut<T> oqs{qs[i] + b, B, true}, opd{pd[i] + b, B, true};
    for (int j = 0; j < M.nb; ++j) joint_stage(M.body[j], cq0, cphi, cvs, oqs, opd);
    AbaIO<T, false> io;
    const T* t = tau.at(s, i);
    io.q = {qs[i] + b, B}; io.v = {vs[i] + b, B};
    io.tau = {t ? t + b : nullptr, B}; io.wext = {nullptr, 1};
    io.vd = {vd[i] + b, B, true}; io.qd = {nullptr, 1, true}; io.ext = {nullptr, 1};
    Stash<T, 1> st{stash.data()};
    if (hm.general) aba_sample<T, Stash<T, 1>, true>(M, io, st);
    else aba_sample<T, Stash<T, 1>, false>(M, io, st);
  }
}

template <class T>
void traj(const HostModel& hm, int64_t B, T* qt, T* vt, const Sched<T>& tau, double dt, int nsteps) {
  const ModelDev<T>& M = dev<T>(hm);
  const int64_t nq = M.nq, nv = M.nv;
  std::vector<T> w(4 * (nq + 3 * nv) * B), phi(nv), vn(nv), dump(nv);
  T *qs[4], *vs[4], *pd[4], *vd[4];
  for (int i = 0; i < 4; ++i) {
    qs[i] = w.data() + i * nq * B; vs[i] = w.data() + (4 * nq + i * nv) * B;
    pd[i] = w.data() + (4 * nq + (4 + i) * nv) * B; vd[i] = w.data() + (4 * nq + (8 + i) * nv) * B;
  }
  for (int s = 0; s < nsteps; ++s) {
    const T* q0 = qt + s * nq * B; const T* v0 = vt + s * nv * B;
    T* q1 = qt + (s + 1) * nq * B; T* v1 = vt + (s + 1) * nv * B;
    for (int64_t b = 0; b < B; ++b) {
      stages(hm, B, b, q0, v0, tau, s, dt, qs, vs, pd, vd);
      const T tdt = (T)dt, wb[4] = {(T)kB[0], (T)kB[1], (T)kB[2], (T)kB[3]};
      for (int k = 0; k < nv; ++k) {       // SumRow4
        const int64_t e = k * B + b;
        phi[k] = tdt * (wb[0] * pd[0][e] + wb[1] * pd[1][e] + wb[2] * pd[2][e] + wb[3] * pd[3][e]);
        vn[k] = v0[e] + tdt * (wb[0] * vd[0][e] + wb[1] * vd[1][e] + wb[2] * vd[2][e] + wb[3] * vd[3][e]);
        v1[e] = vn[k];
      }
      const Col<T> cq0{q0 + b, B}, cphi{phi.data(), 1}, cvn{vn.data(), 1};
      const ColOut<T> oq{q1 + b, B, true}, odump{dump.data(), 1, false};
      for (int j = 0; j < M.nb; ++j) joint_stage(M.body[j], cq0, cphi, cvn, oq, odump);
    }
  }
}

template <class T>
void vjp(const HostModel& hm, int64_t B, const T* qt, const T* vt, const Sched<T>& tau, double dt, int nsteps, const T* qtb,
         const T* vtb, T* q0t, T* q0c, T* v0b, T* taub) {
  ModelDev<T> Mz = dev<T>(hm);
  const ModelDev<T>& M = dev<T>(hm);
  const T grav[3] = {Mz.g[0], Mz.g[1], Mz.g[2]};
  Mz.g[0] = Mz.g[1] = Mz.g[2] = T(0);
  const int64_t nq = M.nq, nv = M.nv;
  std::vector<T> w((4 * (nq + 3 * nv) + 4 * nq + 8 * nv) * B, T(0));
  T *qs[4], *vs[4], *pd[4], *vd[4];
  for (int i = 0; i < 4; ++i) {
    qs[i] = w.data() + i * nq * B; vs[i] = w.data() + (4 * nq + i * nv) * B;
    pd[i] = w.data() + (4 * nq + (4 + i) * nv) * B; vd[i] = w.data() + (4 * nq + (8 + i) * nv) * B;
  }
  T* p = w.data() + 4 * (nq + 3 * nv) * B;
  auto take = [&](int64_t rows) { T* r = p; p += rows * B; return r; };
  T *qcb = take(nq), *qb = take(nq), *qb0 = take(nq), *qsb = take(nq);
  T *vvb = take(nv), *tb = take(nv), *vb = take(nv), *vb0 = take(nv), *vsb = take(nv), *vdb = take(nv), *phib = take(nv);
  for (int64_t e = 0; e < nq * B; ++e) qb[e] = qtb ? qtb[nsteps * nq * B + e] : T(0);
  for (int64_t e = 0; e < nv * B; ++e) vb[e] = vtb ? vtb[nsteps * nv * B + e] : T(0);
  std::vector<T> work(adjoint_rows(hm.nb, hm.nv)), stash(M.nrows + 64);
  const T zero = T(0);
  for (int s = nsteps - 1; s >= 0; --s) {
    const T* q0 = qt + s * nq * B; const T* v0 = vt + s * nv * B;
    for (int64_t b = 0; b < B; ++b) stages(hm, B, b, q0, v0, tau, s, dt, qs, vs, pd, vd);
    AdjStepArgs<T> a{};
    a.q0 = q0;
    for (int i = 0; i < 4; ++i) { a.qs[i] = qs[i]; a.vs[i] = vs[i]; a.pd[i] = pd[i]; a.wa[i] = (T)(dt * kA[i]); a.wb[i] = (T)kB[i]; }
    a.qcb = qcb; a.vvb = vvb; a.taub = tb;
    a.qb = qb; a.vb = vb; a.qb0 = qb0; a.vb0 = vb0; a.qsb = qsb; a.vsb = vsb; a.vdb = vdb; a.phib = phib;
    a.qtb = qtb ? qtb + s * nq * B : nullptr; a.vtb = vtb ? vtb + s * nv * B : nullptr;
    a.ld = B; a.dt = (T)dt;
    for (int g = 4; g >= 0; --g) {
      a.g = g; a.l = g == 4 ? 3 : g - 1;
      a.tau_bar = (taub && g < 4) ? taub + s * tau.step + g * tau.stage : nullptr;
      for (int64_t b = 0; b < B; ++b)
        for (int j = 0; j < M.nb; ++j) adj_joint(M.body[j], a, b);
      if (a.l < 0) {
        if (s > 0)
          for (int64_t b = 0; b < B; ++b)
            for (int j = 0; j < M.nb; ++j) adj_out(M.body[j], q0, qb, (T*)nullptr, qb, B, b);
        continue;
      }
      const int l = a.l;
      for (int64_t b = 0; b < B; ++b) {
        AdjIO<T> io;
        io.q = {qs[l] + b, B}; io.v = {vs[l] + b, B}; io.vd = {vd[l] + b, B}; io.wext = {nullptr, B};
        io.qt = {nullptr, B, true}; io.qc = {qcb + b, B, true}; io.vb = {vvb + b, B, true}; io.vdb = {nullptr, B, true};
        io.wb = {nullptr, B, true};
        io.s = {work.data(), 1};
        dynamics_vjp_sample<T>(Mz, grav, io, Col<T>{vdb + b, B}, ColOut<T>{tb + b, B, true}, &zero, Stash<T, 1>{stash.data()});
      }
    }
  }
  // tangent and configuration forms of q̄0, v̄0
  for (int64_t b = 0; b < B; ++b)
    for (int j = 0; j < M.nb; ++j) adj_out(M.body[j], qt, qb, q0t, q0c, B, b);
  if (v0b) for (int64_t e = 0; e < nv * B; ++e) v0b[e] = vb[e];
}
}  // namespace

extern "C" {
int hostsim_integrate_traj(const rbd_model_desc* d, int dtype, int64_t B, void* qt, void* vt, const void* tau, int64_t step,
                           int64_t stage, double dt, int nsteps) {
  HostModel hm; std::string err;
  if (int rc = build_host_model(d, hm, err)) return rc;
  if (dtype == 0) traj<float>(hm, B, (float*)qt, (float*)vt, Sched<float>{(const float*)tau, step, stage}, dt, nsteps);
  else traj<double>(hm, B, (double*)qt, (double*)vt, Sched<double>{(const double*)tau, step, stage}, dt, nsteps);
  return 0;
}
int hostsim_integrate_vjp(const rbd_model_desc* d, int dtype, int64_t B, const void* qt, const void* vt, const void* tau, int64_t step,
                          int64_t stage, double dt, int nsteps, const void* qtb, const void* vtb, void* q0t, void* q0c, void* v0b,
                          void* taub) {
  HostModel hm; std::string err;
  if (int rc = build_host_model(d, hm, err)) return rc;
  if (dtype == 0)
    vjp<float>(hm, B, (const float*)qt, (const float*)vt, Sched<float>{(const float*)tau, step, stage}, dt, nsteps, (const float*)qtb,
               (const float*)vtb, (float*)q0t, (float*)q0c, (float*)v0b, (float*)taub);
  else
    vjp<double>(hm, B, (const double*)qt, (const double*)vt, Sched<double>{(const double*)tau, step, stage}, dt, nsteps,
                (const double*)qtb, (const double*)vtb, (double*)q0t, (double*)q0c, (double*)v0b, (double*)taub);
  return 0;
}
// one joint of kind `kind`, fp64, local rows: G, L and their adjoints (phib may be NULL)
void hostsim_joint_global(int kind, const double* q0, const double* phi, double* qs) { joint_global_arr(kind, q0, phi, qs); }
void hostsim_joint_rate(int kind, const double* q0, const double* qs, const double* vs, double* pd) { joint_rate_arr(kind, q0, qs, vs, pd); }
void hostsim_joint_g_adjoint(int kind, const double* q0, const double* phi, const double* qsb, double* q0b, double* phib) {
  g_adjoint(kind, q0, phi, qsb, q0b, phib);
}
void hostsim_joint_l_adjoint(int kind, const double* q0, const double* qs, const double* vs, const double* pdb, double* q0b, double* qsb,
                             double* vsb) {
  l_adjoint(kind, q0, qs, vs, pdb, q0b, qsb, vsb);
}
}
