// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
// Runs the backward pass of rbd_integrate_contact_vjp ON THE CPU, one sample at a time: the stage recompute of rbd_integrate_contact
// (joint_stage, contact_stage_pass and aba_sample, as aba_contact_kernel runs them), the elementwise phases of
// csrc/rbd_integrate_adjoint.cuh and contact_vjp_sample (csrc/rbd_contact_adjoint.cuh), on [rows][B] arrays laid out like the
// kernels' workspace.  Also exports contact_force and its adjoint for one pair, so the force law's derivative can be checked against
// finite differences branch by branch.
#include <string>
#include <vector>

#include "../../rigidbodydynamics/jl_b200/csrc/rbd_contact_adjoint.cuh"
#include "../../rigidbodydynamics/jl_b200/csrc/rbd_model.h"

using namespace rbd;

namespace {
template <class T> const ModelDev<T>& dev(const HostModel& m);
template <> const ModelDev<float>& dev<float>(const HostModel& m) { return m.dev32; }
template <> const ModelDev<double>& dev<double>(const HostModel& m) { return m.dev64; }

const double kA[4] = {0.0, 0.5, 0.5, 1.0}, kB[4] = {1.0 / 6, 1.0 / 3, 1.0 / 3, 1.0 / 6};

template <class T> struct Sched {
  const T* tau; int64_t step, stage;
  const T* at(int s, int i) const { return tau ? tau + s * step + i * stage : nullptr; }
};

// the four stages of one step from column b of (q0, v0, s0), into column b of qs / vs / pd / vd / sd
template <class T>
void stages(const HostModel& hm, const ContactDev<T>& C, int64_t B, int64_t b, const T* q0, const T* v0, const T* s0, const Sched<T>& tau,
            int s, double dt, T* const* qs, T* const* vs, T* const* pd, T* const* vd, T* const* sd) {
  const ModelDev<T>& M = dev<T>(hm);
  int8_t slot[kMaxBodies];
  const int nw = contact_wrench_slots(hm.nb, C, slot);
  std::vector<T> stash(M.nrows + 64), phi(M.nv), vv(M.nv), scratch(6 * nw + 1);
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
    ContactAbaIO<T, kAllKinds> io;
    const T* t = tau.at(s, i);
    io.q = {qs[i] + b, B}; io.v = {vs[i] + b, B};
    io.tau = {t ? t + b : nullptr, B};
    io.vd = {vd[i] + b, B, true}; io.qd = {nullptr, 1, true};
    io.ext = {scratch.data(), 1, slot};
    const ContactStageIO<T> cs{s0 + b, i ? sd[i - 1] + b : nullptr, sd[i] + b, wa, B, true};
    Stash<T, 1> st{stash.data()};
    contact_stage_pass(M, C, io.q, io.v, cs, io.ext, st, M.slot_base, kSlotRowsAba);
    if (hm.general) aba_sample<T, Stash<T, 1>, true>(M, io, st);
    else aba_sample<T, Stash<T, 1>, false>(M, io, st);
  }
}

template <class T>
void vjp(const HostModel& hm, const rbd_contact_desc& cd, int64_t B, const T* qt, const T* vt, const T* stj, const Sched<T>& tau, double dt,
         int nsteps, const T* qtb, const T* vtb, const T* stb, T* q0t, T* q0c, T* v0b, T* s0b, T* taub) {
  ModelDev<T> Mz = dev<T>(hm);
  const ModelDev<T>& M = dev<T>(hm);
  const T grav[3] = {Mz.g[0], Mz.g[1], Mz.g[2]};
  Mz.g[0] = Mz.g[1] = Mz.g[2] = T(0);
  std::vector<ContactDev<T>> Cv(1);
  build_contact_dev<T>(hm.nb, hm.pos.data(), hm.alignT.data(), cd, Cv[0]);
  const ContactDev<T>& C = Cv[0];
  const int64_t nq = M.nq, nv = M.nv, ns = 3 * (int64_t)cd.npoints * cd.nhalfspaces;
  std::vector<T> w((4 * (nq + 3 * nv) + 4 * ns + 4 * nq + 8 * nv + 3 * ns) * B + 1, T(0));
  T *qs[4], *vs[4], *pd[4], *vd[4], *sd[4];
  T* p = w.data();
  auto take = [&](int64_t rows) { T* r = p; p += rows * B; return r; };
  for (int i = 0; i < 4; ++i) qs[i] = take(nq);
  for (int i = 0; i < 4; ++i) vs[i] = take(nv);
  for (int i = 0; i < 4; ++i) pd[i] = take(nv);
  for (int i = 0; i < 4; ++i) vd[i] = take(nv);
  for (int i = 0; i < 4; ++i) sd[i] = take(ns);
  T *qcb = take(nq), *qb = take(nq), *qb0 = take(nq), *qsb = take(nq);
  T *vvb = take(nv), *tb = take(nv), *vb = take(nv), *vb0 = take(nv), *vsb = take(nv), *vdb = take(nv), *phib = take(nv);
  T *sb1 = take(ns), *sacc = take(ns), *sdc = take(ns);
  for (int64_t e = 0; e < nq * B; ++e) qb[e] = qtb ? qtb[nsteps * nq * B + e] : T(0);
  for (int64_t e = 0; e < nv * B; ++e) vb[e] = vtb ? vtb[nsteps * nv * B + e] : T(0);
  for (int64_t e = 0; e < ns * B; ++e) sb1[e] = stb ? stb[nsteps * ns * B + e] : T(0);
  std::vector<T> work(contact_vjp_rows(hm.nb, hm.nv)), stash(M.nrows + 64);
  const T zero = T(0);
  for (int s = nsteps - 1; s >= 0; --s) {
    const T* q0 = qt + s * nq * B; const T* v0 = vt + s * nv * B; const T* s0 = stj + s * ns * B;
    for (int64_t b = 0; b < B; ++b) stages(hm, C, B, b, q0, v0, s0, tau, s, dt, qs, vs, pd, vd, sd);
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
        ContactVjpIO<T> io;
        io.q = {qs[l] + b, B}; io.v = {vs[l] + b, B}; io.vd = {vd[l] + b, B}; io.vdb = {vdb + b, B};
        io.qc = {qcb + b, B, true}; io.taub = {tb + b, B, true}; io.vb = vvb + b;
        io.s0 = s0 + b; io.sdp = l ? sd[l - 1] + b : nullptr; io.stb = (l == 0 && stb) ? stb + s * ns * B + b : nullptr;
        io.sb1 = sb1 + b; io.sacc = sacc + b; io.sdc = sdc + b;
        io.ld = B; io.wa = a.wa[l]; io.wdb = (T)dt * a.wb[l]; io.l = l;
        io.s = {work.data(), 1};
        io.active = true;
        contact_vjp_sample<T>(Mz, grav, C, io, &zero, Stash<T, 1>{stash.data()});
      }
    }
  }
  for (int64_t b = 0; b < B; ++b)
    for (int j = 0; j < M.nb; ++j) adj_out(M.body[j], qt, qb, q0t, q0c, B, b);
  if (v0b) for (int64_t e = 0; e < nv * B; ++e) v0b[e] = vb[e];
  if (s0b) for (int64_t e = 0; e < ns * B; ++e) s0b[e] = sb1[e];
}

// a one-point, one-half-space descriptor for the force law: hc = (k, lambda, n), fr = (mu, k, b), unit normal n
void one_pair(const double* hc, const double* fr, const double* n, ContactDev<double>& C) {
  std::memset(&C, 0, sizeof(C));
  C.npoints = 1; C.nhalf = 1;
  for (int r = 0; r < 3; ++r) { C.hc[0][r] = hc[r]; C.fr[0][r] = fr[r]; C.hn[0][r] = n[r]; }
}
}  // namespace

extern "C" {
int hostsim_integrate_contact_vjp(const rbd_model_desc* d, int dtype, int64_t B, const void* qt, const void* vt, const void* st,
                                  const void* tau, int64_t step, int64_t stage, const rbd_contact_desc* cd, double dt, int nsteps,
                                  const void* qtb, const void* vtb, const void* stb, void* q0t, void* q0c, void* v0b, void* s0b,
                                  void* taub) {
  HostModel hm; std::string err;
  if (int rc = build_host_model(d, hm, err)) return rc;
  if (dtype == 0)
    vjp<float>(hm, *cd, B, (const float*)qt, (const float*)vt, (const float*)st, Sched<float>{(const float*)tau, step, stage}, dt, nsteps,
               (const float*)qtb, (const float*)vtb, (const float*)stb, (float*)q0t, (float*)q0c, (float*)v0b, (float*)s0b, (float*)taub);
  else
    vjp<double>(hm, *cd, B, (const double*)qt, (const double*)vt, (const double*)st, Sched<double>{(const double*)tau, step, stage}, dt,
                nsteps, (const double*)qtb, (const double*)vtb, (const double*)stb, (double*)q0t, (double*)q0c, (double*)v0b,
                (double*)s0b, (double*)taub);
  return 0;
}
// contact_force of one pair in contact (fp64): f, xd
void hostsim_contact_force(const double* hc, const double* fr, const double* n, double z, const double* vel, const double* x, double* f,
                           double* xd) {
  ContactDev<double> C;
  one_pair(hc, fr, n, C);
  contact_force(C, 0, C.hn[0], z, vel, [&](int k) { return x[k]; }, f, xd);
}
// its adjoint: (fb, xdb) -> zb, velb, xb
void hostsim_contact_force_adjoint(const double* hc, const double* fr, const double* n, double z, const double* vel, const double* x,
                                   const double* fb, const double* xdb, double* zb, double* velb, double* xb) {
  ContactDev<double> C;
  one_pair(hc, fr, n, C);
  double f[3];
  contact_force_adjoint(C, 0, C.hn[0], z, vel, x, fb, xdb, f, *zb, velb, xb);
}
}
