// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
// rbd_integrate_pd_vjp ON THE CPU.  (1) pd_adj_joint (csrc/rbd_integrate_adjoint.cuh) for one joint of one sample exactly as the
// phase kernels call it, and joint_error (csrc/rbd_pd.cuh), so that the law's adjoint can be checked against central differences of
// the law.  (2) The whole backward pass, one sample at a time on [rows][B] arrays laid out like the kernels' workspace: the closed-
// loop recompute of integrate_t (joint_stage, pd_joint, rnea_sample + the pd_finish_kernel arithmetic in computed-torque mode,
// aba_sample), dynamics_vjp_sample, the mask and adjoint_sample (the inverse-dynamics VJP) in computed-torque mode, and the phases
// adj_joint<T, true> -- the structure of tests/hostsim/hostsim_integrate_vjp.cpp with the controller added.
#include <string>
#include <vector>

#include "../../rigidbodydynamics/jl_b200/csrc/rbd_adjoint.cuh"
#include "../../rigidbodydynamics/jl_b200/csrc/rbd_integrate_adjoint.cuh"
#include "../../rigidbodydynamics/jl_b200/csrc/rbd_model.h"
#include "../../rigidbodydynamics/jl_b200/csrc/rbd_rnea_crba.cuh"

using namespace rbd;

namespace {
template <class T> const ModelDev<T>& dev(const HostModel& m);
template <> const ModelDev<float>& dev<float>(const HostModel& m) { return m.dev32; }
template <> const ModelDev<double>& dev<double>(const HostModel& m) { return m.dev64; }

const double kA[4] = {0.0, 0.5, 0.5, 1.0}, kB[4] = {1.0 / 6, 1.0 / 3, 1.0 / 3, 1.0 / 6};

// rbd_pd_desc in host form at leading dimension B, with the bounds converted to T (lo NULL: none)
template <class T> struct Ctl {
  int ct;
  const T* kp; const T* kd; int64_t g_ld;
  const T* qref; const T* vref; const T* vdref; int64_t qstride, vstride;
  const T* lo; const T* hi;
  const T* tau; int64_t step, stage;      // τ_ff (NULL: 0)
  const T* ff(int s, int i) const { return tau ? tau + s * step + i * stage : nullptr; }
};

// the four closed-loop stages of one step at column b: qs / vs / pd / vd as integrate_stage_kernel + dynamics, taui the applied
// torques, vdes v̇_des (computed-torque mode)
template <class T>
void stages(const HostModel& hm, int64_t B, int64_t b, const T* q0, const T* v0, const Ctl<T>& c, int s, double dt, T* const* qs,
            T* const* vs, T* const* pd, T* const* vd, T* const* taui, T* const* vdes) {
  const ModelDev<T>& M = dev<T>(hm);
  std::vector<T> stash(std::max(M.nrows, rnea_rows(hm)) + 64), phi(M.nv), vv(M.nv);
  const int64_t nv = M.nv;
  for (int i = 0; i < 4; ++i) {
    const T wa = (T)(dt * kA[i]);
    for (int k = 0; k < nv; ++k) {
      const int64_t e = (int64_t)k * B + b;
      phi[k] = i ? wa * pd[i - 1][e] : T(0);
      vv[k] = i ? v0[e] + wa * vd[i - 1][e] : v0[e];
      vs[i][e] = vv[k];
    }
    const Col<T> cq0{q0 + b, B}, cphi{phi.data(), 1}, cvs{vv.data(), 1};
    const ColOut<T> oqs{qs[i] + b, B, true}, opd{pd[i] + b, B, true};
    for (int j = 0; j < M.nb; ++j) joint_stage(M.body[j], cq0, cphi, cvs, oqs, opd);
    const T* qref = c.qref + s * c.qstride + b;
    const T* vref = c.vref ? c.vref + s * c.vstride + b : nullptr;
    const T* ff = c.ff(s, i);
    const int64_t gc = c.g_ld ? b : 0;
    const PdSample<T> ps{qs[i] + b, vs[i] + b, B, qref, vref,
                         c.ct ? (c.vdref ? c.vdref + s * c.vstride + b : nullptr) : (ff ? ff + b : nullptr), B, c.kp + gc, c.kd + gc,
                         c.g_ld ? c.g_ld : 1, c.ct ? nullptr : c.lo, c.ct ? nullptr : c.hi};
    for (int j = 0; j < M.nb; ++j) pd_joint(M.body[j], ps, ColOut<T>{(c.ct ? vdes[i] : taui[i]) + b, B, true});
    if (c.ct) {       // inverse_dynamics_t, then pd_finish_kernel
      RneaIO<T> io;
      io.q = {qs[i] + b, B}; io.v = {vs[i] + b, B}; io.vd = {vdes[i] + b, B};
      io.wext = {nullptr, B}; io.tau = {taui[i] + b, B, true}; io.ext = {nullptr, 1};
      rnea_sample<T>(M, io, Stash<T, 1>{stash.data()});
      for (int k = 0; k < nv; ++k) {
        const int64_t e = (int64_t)k * B + b;
        T x = taui[i][e];
        if (ff) x += ff[e];
        if (c.lo) x = clamp_t(x, c.lo[k], c.hi[k]);
        taui[i][e] = x;
      }
    }
    AbaIO<T, false> io;
    io.q = {qs[i] + b, B}; io.v = {vs[i] + b, B};
    io.tau = {taui[i] + b, B}; io.wext = {nullptr, 1};
    io.vd = {vd[i] + b, B, true}; io.qd = {nullptr, 1, true}; io.ext = {nullptr, 1};
    Stash<T, 1> st{stash.data()};
    if (hm.general) aba_sample<T, Stash<T, 1>, true>(M, io, st);
    else aba_sample<T, Stash<T, 1>, false>(M, io, st);
  }
}

template <class T> struct Work {        // the four stages and the controller's per-stage rows, [rows][B]
  std::vector<T> w;
  T *qs[4], *vs[4], *pd[4], *vd[4], *taui[4], *vdes[4];
  Work(int64_t nq, int64_t nv, int64_t B) : w((4 * nq + 20 * nv) * B, T(0)) {
    for (int i = 0; i < 4; ++i) {
      qs[i] = w.data() + i * nq * B; vs[i] = w.data() + (4 * nq + i * nv) * B;
      pd[i] = w.data() + (4 * nq + (4 + i) * nv) * B; vd[i] = w.data() + (4 * nq + (8 + i) * nv) * B;
      taui[i] = w.data() + (4 * nq + (12 + i) * nv) * B; vdes[i] = w.data() + (4 * nq + (16 + i) * nv) * B;
    }
  }
};

template <class T>
void traj(const HostModel& hm, int64_t B, T* qt, T* vt, const Ctl<T>& c, double dt, int nsteps) {
  const ModelDev<T>& M = dev<T>(hm);
  const int64_t nq = M.nq, nv = M.nv;
  Work<T> w(nq, nv, B);
  std::vector<T> phi(nv), vn(nv), dump(nv);
  for (int s = 0; s < nsteps; ++s) {
    const T* q0 = qt + s * nq * B; const T* v0 = vt + s * nv * B;
    T* q1 = qt + (s + 1) * nq * B; T* v1 = vt + (s + 1) * nv * B;
    for (int64_t b = 0; b < B; ++b) {
      stages(hm, B, b, q0, v0, c, s, dt, w.qs, w.vs, w.pd, w.vd, w.taui, w.vdes);
      const T tdt = (T)dt, wb[4] = {(T)kB[0], (T)kB[1], (T)kB[2], (T)kB[3]};
      for (int k = 0; k < nv; ++k) {       // SumRow4
        const int64_t e = k * B + b;
        phi[k] = tdt * (wb[0] * w.pd[0][e] + wb[1] * w.pd[1][e] + wb[2] * w.pd[2][e] + wb[3] * w.pd[3][e]);
        vn[k] = v0[e] + tdt * (wb[0] * w.vd[0][e] + wb[1] * w.vd[1][e] + wb[2] * w.vd[2][e] + wb[3] * w.vd[3][e]);
        v1[e] = vn[k];
      }
      const Col<T> cq0{q0 + b, B}, cphi{phi.data(), 1}, cvn{vn.data(), 1};
      const ColOut<T> oq{q1 + b, B, true}, odump{dump.data(), 1, false};
      for (int j = 0; j < M.nb; ++j) joint_stage(M.body[j], cq0, cphi, cvn, oq, odump);
    }
  }
}

// bars: kp, kd [nv x B], q_ref, v_ref, vd_ref (shapes of the controller's arrays), each added to, NULL = not wanted
template <class T>
void vjp(const HostModel& hm, int64_t B, const T* qt, const T* vt, const Ctl<T>& c, double dt, int nsteps, const T* qtb, const T* vtb,
         T* q0t, T* q0c, T* v0b, T* taub, T* const* bars) {
  ModelDev<T> Mz = dev<T>(hm);
  const ModelDev<T>& M = dev<T>(hm);
  const T grav[3] = {Mz.g[0], Mz.g[1], Mz.g[2]};
  Mz.g[0] = Mz.g[1] = Mz.g[2] = T(0);
  const int64_t nq = M.nq, nv = M.nv;
  Work<T> w(nq, nv, B);
  std::vector<T> adj((5 * nq + 10 * nv) * B, T(0));
  T* p = adj.data();
  auto take = [&](int64_t rows) { T* r = p; p += rows * B; return r; };
  T *qcb = take(nq), *qb = take(nq), *qb0 = take(nq), *qsb = take(nq);
  T *vvb = take(nv), *tb = take(nv), *vb = take(nv), *vb0 = take(nv), *vsb = take(nv), *vdb = take(nv), *phib = take(nv);
  T *idq = take(nq), *idv = take(nv), *idvd = take(nv);
  for (int64_t e = 0; e < nq * B; ++e) qb[e] = qtb ? qtb[nsteps * nq * B + e] : T(0);
  for (int64_t e = 0; e < nv * B; ++e) vb[e] = vtb ? vtb[nsteps * nv * B + e] : T(0);
  std::vector<T> work(adjoint_rows(hm.nb, hm.nv)), stash(M.nrows + 64);
  const T zero = T(0);
  for (int s = nsteps - 1; s >= 0; --s) {
    const T* q0 = qt + s * nq * B; const T* v0 = vt + s * nv * B;
    for (int64_t b = 0; b < B; ++b) stages(hm, B, b, q0, v0, c, s, dt, w.qs, w.vs, w.pd, w.vd, w.taui, w.vdes);
    AdjStepArgs<T> a{};
    a.q0 = q0;
    for (int i = 0; i < 4; ++i) { a.qs[i] = w.qs[i]; a.vs[i] = w.vs[i]; a.pd[i] = w.pd[i]; a.wa[i] = (T)(dt * kA[i]); a.wb[i] = (T)kB[i]; }
    a.qcb = qcb; a.vvb = vvb; a.taub = tb;
    a.qb = qb; a.vb = vb; a.qb0 = qb0; a.vb0 = vb0; a.qsb = qsb; a.vsb = vsb; a.vdb = vdb; a.phib = phib;
    a.qtb = qtb ? qtb + s * nq * B : nullptr; a.vtb = vtb ? vtb + s * nv * B : nullptr;
    a.ld = B; a.dt = (T)dt;
    PdAdjArgs<T> pc{};
    pc.qref = c.qref + s * c.qstride; pc.vref = c.vref ? c.vref + s * c.vstride : nullptr;
    pc.kp = c.kp; pc.kd = c.kd; pc.g_ld = c.g_ld; pc.lo = c.lo; pc.hi = c.hi;
    if (c.ct) { pc.idq = idq; pc.idv = idv; pc.idvd = idvd; }
    pc.kpb = bars[0]; pc.kdb = bars[1];
    pc.qrefb = bars[2] ? bars[2] + s * c.qstride : nullptr;
    pc.vrefb = bars[3] ? bars[3] + s * c.vstride : nullptr;
    pc.vdrefb = bars[4] ? bars[4] + s * c.vstride : nullptr;
    for (int g = 4; g >= 0; --g) {
      a.g = g; a.l = g == 4 ? 3 : g - 1;
      a.tau_bar = (taub && g < 4) ? taub + s * c.step + g * c.stage : nullptr;
      pc.tau = (c.lo && !c.ct && g < 4) ? w.taui[g] : nullptr;
      for (int64_t b = 0; b < B; ++b)
        for (int j = 0; j < M.nb; ++j) adj_joint<T, true>(M.body[j], a, b, &pc);
      if (a.l < 0) {
        if (s > 0)
          for (int64_t b = 0; b < B; ++b)
            for (int j = 0; j < M.nb; ++j) adj_out(M.body[j], q0, qb, (T*)nullptr, qb, B, b);
        continue;
      }
      const int l = a.l;
      for (int64_t b = 0; b < B; ++b) {
        AdjIO<T> io;
        io.q = {w.qs[l] + b, B}; io.v = {w.vs[l] + b, B}; io.vd = {w.vd[l] + b, B}; io.wext = {nullptr, B};
        io.qt = {nullptr, B, true}; io.qc = {qcb + b, B, true}; io.vb = {vvb + b, B, true}; io.vdb = {nullptr, B, true};
        io.wb = {nullptr, B, true};
        io.s = {work.data(), 1};
        dynamics_vjp_sample<T>(Mz, grav, io, Col<T>{vdb + b, B}, ColOut<T>{tb + b, B, true}, &zero, Stash<T, 1>{stash.data()});
        if (!c.ct) continue;
        if (c.lo)            // pd_mask_kernel
          for (int k = 0; k < nv; ++k) {
            const int64_t e = (int64_t)k * B + b;
            tb[e] = pd_mask(tb[e], w.taui[l][e], c.lo[k], c.hi[k]);
          }
        AdjIO<T> id;         // inverse_dynamics_vjp_dense
        id.q = {w.qs[l] + b, B}; id.v = {w.vs[l] + b, B}; id.vd = {w.vdes[l] + b, B}; id.wext = {nullptr, B};
        id.qt = {nullptr, B, true}; id.qc = {idq + b, B, true}; id.vb = {idv + b, B, true}; id.vdb = {idvd + b, B, true};
        id.wb = {nullptr, B, true};
        id.s = {work.data(), 1};
        adjoint_sample<T>(M, grav, id, Col<T>{tb + b, B}, T(1));
      }
    }
  }
  for (int64_t b = 0; b < B; ++b)
    for (int j = 0; j < M.nb; ++j) adj_out(M.body[j], qt, qb, q0t, q0c, B, b);
  if (v0b) for (int64_t e = 0; e < nv * B; ++e) v0b[e] = vb[e];
}

// the ABI's controller arguments -> Ctl<T> (bounds converted into `lh`)
template <class T>
Ctl<T> ctl(int ct, const void* kp, const void* kd, int64_t g_ld, const void* qref, const void* vref, const void* vdref, int64_t qs, int64_t vs,
           const double* lo, const double* hi, const void* tau, int64_t step, int64_t stage, int nv, std::vector<T>& lh) {
  lh.assign(2 * nv, T(0));
  for (int k = 0; lo && k < nv; ++k) { lh[k] = (T)lo[k]; lh[nv + k] = (T)hi[k]; }
  return Ctl<T>{ct, (const T*)kp, (const T*)kd, g_ld, (const T*)qref, (const T*)vref, (const T*)vdref, qs, vs,
                lo ? lh.data() : nullptr, lo ? lh.data() + nv : nullptr, (const T*)tau, step, stage};
}
}  // namespace

extern "C" {
// The closed-loop trajectory (qt / vt [(nsteps + 1) x rows x B], block 0 given) and its backward pass; dtype 0 = fp32, 1 = fp64.
// Controller arguments as rbd_pd_desc at leading dimension B (lo / hi host fp64 or NULL); tau with its strides as τ_ff.
int hostsim_pd_traj(const rbd_model_desc* d, int dtype, int64_t B, void* qt, void* vt, int ct, const void* kp, const void* kd, int64_t g_ld,
                    const void* qref, const void* vref, const void* vdref, int64_t qstride, int64_t vstride, const double* lo,
                    const double* hi, const void* tau, int64_t step, int64_t stage, double dt, int nsteps) {
  HostModel hm; std::string err;
  if (int rc = build_host_model(d, hm, err)) return rc;
  if (dtype == 0) {
    std::vector<float> lh;
    traj<float>(hm, B, (float*)qt, (float*)vt, ctl<float>(ct, kp, kd, g_ld, qref, vref, vdref, qstride, vstride, lo, hi, tau, step, stage,
                                                          hm.nv, lh), dt, nsteps);
  } else {
    std::vector<double> lh;
    traj<double>(hm, B, (double*)qt, (double*)vt, ctl<double>(ct, kp, kd, g_ld, qref, vref, vdref, qstride, vstride, lo, hi, tau, step,
                                                              stage, hm.nv, lh), dt, nsteps);
  }
  return 0;
}
int hostsim_pd_vjp(const rbd_model_desc* d, int dtype, int64_t B, const void* qt, const void* vt, int ct, const void* kp, const void* kd,
                   int64_t g_ld, const void* qref, const void* vref, const void* vdref, int64_t qstride, int64_t vstride, const double* lo,
                   const double* hi, const void* tau, int64_t step, int64_t stage, double dt, int nsteps, const void* qtb, const void* vtb,
                   void* q0t, void* q0c, void* v0b, void* taub, void* const* bars) {
  HostModel hm; std::string err;
  if (int rc = build_host_model(d, hm, err)) return rc;
  if (dtype == 0) {
    std::vector<float> lh;
    vjp<float>(hm, B, (const float*)qt, (const float*)vt, ctl<float>(ct, kp, kd, g_ld, qref, vref, vdref, qstride, vstride, lo, hi, tau,
                                                                     step, stage, hm.nv, lh),
               dt, nsteps, (const float*)qtb, (const float*)vtb, (float*)q0t, (float*)q0c, (float*)v0b, (float*)taub, (float* const*)bars);
  } else {
    std::vector<double> lh;
    vjp<double>(hm, B, (const double*)qt, (const double*)vt, ctl<double>(ct, kp, kd, g_ld, qref, vref, vdref, qstride, vstride, lo, hi,
                                                                         tau, step, stage, hm.nv, lh),
                dt, nsteps, (const double*)qtb, (const double*)vtb, (double*)q0t, (double*)q0c, (double*)v0b, (double*)taub,
                (double* const*)bars);
  }
  return 0;
}
// e [nv] = joint_error(kind, qref, q), fp64
void hostsim_joint_error(int kind, const double* qref, const double* q, double* e) { joint_error(kind, qref, q, e); }

// One joint of kind `kind` at one sample, fp64.  Inputs: q / qref [nq], v / vref [nv] (vref may be NULL), kp / kd [nv], taub [nv]
// (τ̄ of the stage), tau [nv] with lo / hi [nv] (the applied torque and bounds, or all NULL: no mask), and in computed-torque mode
// w [nv] (v̇̄_des; NULL: PD mode, with idq / idv zero).  Outputs: cq [nq], cv [nv], m [nv]; kpb / kdb / qrefb / vrefb / vdrefb are
// added to (each may be NULL).
void hostsim_pd_adj_joint(int kind, const double* q, const double* v, const double* qref, const double* vref, const double* kp,
                          const double* kd, const double* taub, const double* tau, const double* lo, const double* hi, const double* w,
                          double* cq, double* cv, double* m, double* kpb, double* kdb, double* qrefb, double* vrefb, double* vdrefb) {
  BodyDev<double> bd{};
  bd.kind = kind; bd.qrow = 0; bd.vrow = 0;
  AdjStepArgs<double> a{};
  a.qs[0] = q; a.vs[0] = v; a.taub = taub; a.ld = 1; a.g = 0;
  const double zeros[7] = {0, 0, 0, 0, 0, 0, 0};
  PdAdjArgs<double> c{};
  c.qref = qref; c.vref = vref; c.kp = kp; c.kd = kd; c.g_ld = 0;
  c.tau = tau; c.lo = lo; c.hi = hi;
  if (w) { c.idq = zeros; c.idv = zeros; c.idvd = w; }
  c.kpb = kpb; c.kdb = kdb; c.qrefb = qrefb; c.vrefb = vrefb; c.vdrefb = vdrefb;
  pd_adj_joint(bd, a, c, 0, cq, cv, m);
}
}
