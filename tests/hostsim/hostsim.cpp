// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
// Runs the per-sample device algorithms of csrc/rbd_device.cuh ON THE CPU (they are __host__ __device__ templates)
// so that the math of the kernels can be checked against the oracle in the CPU-only test tier, before any GPU time
// is spent.  The shipped librbd_b200.so does not contain this file and has no CPU path.
#include <cstring>
#include <string>
#include <vector>

#include "../../rigidbodydynamics/jl_b200/csrc/rbd_rnea_crba.cuh"
#include "../../rigidbodydynamics/jl_b200/csrc/rbd_kin.cuh"
#include "../../rigidbodydynamics/jl_b200/csrc/rbd_deriv.cuh"
#include "../../rigidbodydynamics/jl_b200/csrc/rbd_dual.cuh"
#include "../../rigidbodydynamics/jl_b200/csrc/rbd_integrate.cuh"
#include "../../rigidbodydynamics/jl_b200/csrc/rbd_model.h"
#include "../../rigidbodydynamics/jl_b200/csrc/rbd_codegen.h"

using namespace rbd;

namespace {
template <class T> const ModelDev<T>& dev(const HostModel& m);
template <> const ModelDev<float>& dev<float>(const HostModel& m) { return m.dev32; }
template <> const ModelDev<double>& dev<double>(const HostModel& m) { return m.dev64; }

template <class T, bool EXT>
void run_dynamics_e(const HostModel& hm, int64_t B, const T* q, const T* v, const T* tau, const T* wext, T* vd, T* qd) {
  const ModelDev<T>& M = dev<T>(hm);
  std::vector<T> stash(M.nrows + 64), scratch(6 * M.nb);
  for (int64_t b = 0; b < B; ++b) {
    AbaIO<T, EXT> io;
    io.q = {q + b, B}; io.v = {v + b, B};
    io.tau = {tau ? tau + b : nullptr, B}; io.wext = {EXT ? wext + b : nullptr, B};
    io.vd = {vd + b, B, true}; io.qd = {qd ? qd + b : nullptr, B, true};
    io.ext = {EXT ? scratch.data() : nullptr, 1};
    Stash<T, 1> st{stash.data()};
    if (EXT) ext_wrench_pass(M, io.q, io.wext, io.ext, st, M.slot_base, kSlotRowsAba);
    if (hm.general) aba_sample<T, Stash<T, 1>, true>(M, io, st);
    else aba_sample<T, Stash<T, 1>, false>(M, io, st);
  }
}
template <class T>
void run_dynamics(const HostModel& hm, int64_t B, const T* q, const T* v, const T* tau, const T* wext, T* vd, T* qd) {
  if (wext) run_dynamics_e<T, true>(hm, B, q, v, tau, wext, vd, qd);
  else run_dynamics_e<T, false>(hm, B, q, v, tau, wext, vd, qd);
}

template <class T>
void run_rnea(const HostModel& hm, int64_t B, const T* q, const T* v, const T* vd, const T* wext, T* tau) {
  const ModelDev<T>& M = dev<T>(hm);
  std::vector<T> stash(rnea_rows(hm) + 64), scratch(6 * M.nb);
  for (int64_t b = 0; b < B; ++b) {
    RneaIO<T> io;
    io.q = {q + b, B}; io.v = {v + b, B}; io.vd = {vd ? vd + b : nullptr, B};
    io.wext = {wext ? wext + b : nullptr, B};
    io.tau = {tau + b, B, true};
    io.ext = {wext ? scratch.data() : nullptr, 1};
    rnea_sample<T>(M, io, Stash<T, 1>{stash.data()});
  }
}

template <class T>
void run_kin(const HostModel& hm, int64_t B, const T* q, const T* v, const int8_t* sign, T* const* o /* 8 outputs */) {
  const ModelDev<T>& M = dev<T>(hm);
  KinDev<T> K;
  std::memset(&K, 0, sizeof(K));
  for (int p = 0; p < hm.nb; ++p) {
    for (int k = 0; k < 9; ++k) K.At[p][k] = (T)hm.alignT[9 * p + k];
    K.sign[p] = sign ? sign[hm.order[p]] : 0;
  }
  K.inv_mass = (T)(1.0 / hm.total_mass);
  std::vector<T> stash(kin_rows(hm) + 64), scratch(12 * M.nb);
  for (int64_t b = 0; b < B; ++b) {
    KinIO<T> io;
    io.q = {q + b, B}; io.v = {v ? v + b : nullptr, B};
    auto out = [&](T* p) { return ColOut<T>{p ? p + b : nullptr, B, true}; };
    io.tr = out(o[0]); io.com = out(o[1]); io.ke = out(o[2]); io.pe = out(o[3]);
    io.mom = out(o[4]); io.mrb = out(o[5]); io.A = out(o[6]); io.J = out(o[7]);
    io.poses = {o[6] ? scratch.data() : nullptr, 1};
    kin_sample<T>(M, K, io, Stash<T, 1>{stash.data()});
  }
}

template <class T>
void run_contact(const HostModel& hm, int64_t B, const T* q, const T* v, const rbd_contact_desc& cd, T* s, T* sd, T* wr) {
  const ModelDev<T>& M = dev<T>(hm);
  ContactDev<T> C;
  build_contact_dev<T>(hm.nb, hm.pos.data(), hm.alignT.data(), cd, C);
  std::vector<T> stash(kin_rows(hm) + 64);
  for (int64_t b = 0; b < B; ++b) {
    ContactIO<T> io;
    io.q = {q + b, B}; io.v = {v + b, B};
    io.s = s ? s + b : nullptr; io.sd = sd ? sd + b : nullptr; io.wr = wr + b;
    io.ld = B; io.active = true;
    contact_sample<T>(M, C, io, Stash<T, 1>{stash.data()});
  }
}

template <class T> void run_crba(const HostModel& hm, int64_t B, const T* q, T* Mout) {
  const ModelDev<T>& M = dev<T>(hm);
  std::vector<T> stash(crba_rows(hm) + 64);
  bool multi = false;
  for (int i = 0; i < M.nb; ++i) multi |= kind_nv(M.body[i].kind) > 1;
  for (int64_t b = 0; b < B; ++b) {
    CrbaIO<T> io;
    io.q = {q + b, B};
    io.M = {Mout + b, B, true};
    io.lower = false;
    if (multi) crba_sample<T, Stash<T, 1>, 6>(M, io, Stash<T, 1>{stash.data()});
    else crba_sample<T, Stash<T, 1>, 1>(M, io, Stash<T, 1>{stash.data()});
  }
}
// dv̇/dq, dv̇/dv (csrc/rbd_deriv.cuh): the five phases run one sample at a time with a scratch of one column
template <class T>
int run_derivatives(const HostModel& hm, int64_t B, const T* q, const T* v, const T* tau, T* vd, T* dq, T* dv) {
  const ModelDev<T>& M = dev<T>(hm);
  DerivDev D; DerivAnc A;
  if (!build_deriv_dev(M, D, A)) return RBD_EUNSUPPORTED;
  run_dynamics<T>(hm, B, q, v, tau, nullptr, vd, nullptr);
  std::vector<T> stash(kin_rows(hm) + 64), scr(D.rows), x(D.nv);
  for (int64_t b = 0; b < B; ++b) {
    DerivIO<T> io;
    io.q = {q + b, B}; io.v = {v + b, B}; io.vd = {vd + b, B};
    io.s = scr.data(); io.sld = 1; io.active = true;
    deriv_world_sample<T>(M, D, io, Stash<T, 1>{stash.data()});
    for (int c = 0; c < kBodyRows; ++c) deriv_accumulate<T>(M, D, scr.data(), 1, c);
    for (int K = 0; K < M.nb; ++K) deriv_pairs<T>(D, A, scr.data(), 1, dq + b, dv + b, B, K, true);
    deriv_factor<T>(D, A, scr.data() + D.h_base, 1);
    const T* H = scr.data() + D.h_base;
    auto Hf = [H](int row) { return H[row]; };
    for (int c = 0; c < 2 * D.nv; ++c) {
      T* out = (c < D.nv ? dq : dv) + (int64_t)(c % D.nv) * D.nv * B + b;
      deriv_solve_column<T>(D, A, Hf, x.data(), 1, out, B, c % D.nv, true);
    }
  }
  return 0;
}
}  // namespace

// Munthe-Kaas RK4 steps with the device coordinate maps (joint_stage) and the device ABA, one sample at a time
template <class T>
void run_integrate(const HostModel& hm, int64_t B, T* q, T* v, const T* tau, double dt, int nsteps) {
  const ModelDev<T>& M = dev<T>(hm);
  const int nq = M.nq, nv = M.nv;
  std::vector<T> stash(M.nrows + 64), q0(nq), v0(nv), qs(nq), vs(nv), phi(nv), phid(nv), vd(nv), accphi(nv), accv(nv), dump(nv);
  const double a[4] = {0.0, 0.5, 0.5, 1.0}, bw[4] = {1.0 / 6, 1.0 / 3, 1.0 / 3, 1.0 / 6};
  for (int64_t b = 0; b < B; ++b) {
    for (int s = 0; s < nsteps; ++s) {
      for (int k = 0; k < nq; ++k) q0[k] = q[(int64_t)k * B + b];
      for (int k = 0; k < nv; ++k) v0[k] = v[(int64_t)k * B + b];
      for (int i = 0; i < 4; ++i) {
        const T wa = (T)(dt * a[i]);
        for (int k = 0; k < nv; ++k) {
          const T vdp = i ? vd[k] : T(0), pdp = i ? phid[k] : T(0);
          phi[k] = wa * pdp; vs[k] = v0[k] + wa * vdp;
          accv[k] = i ? accv[k] + (T)bw[i - 1] * vdp : T(0);
        }
        const Col<T> cq0{q0.data(), 1}, cphi{phi.data(), 1}, cvs{vs.data(), 1};
        const ColOut<T> oqs{qs.data(), 1, true}, ophid{phid.data(), 1, true};
        for (int j = 0; j < M.nb; ++j) joint_stage(M.body[j], cq0, cphi, cvs, oqs, ophid);
        for (int k = 0; k < nv; ++k) accphi[k] = (i ? accphi[k] : T(0)) + (T)bw[i] * phid[k];
        AbaIO<T, false> io;
        io.q = {qs.data(), 1}; io.v = {vs.data(), 1};
        io.tau = {tau ? tau + b : nullptr, B}; io.wext = {nullptr, 1};
        io.vd = {vd.data(), 1, true}; io.qd = {nullptr, 1, true}; io.ext = {nullptr, 1};
        Stash<T, 1> st{stash.data()};
        if (hm.general) aba_sample<T, Stash<T, 1>, true>(M, io, st);
        else aba_sample<T, Stash<T, 1>, false>(M, io, st);
      }
      for (int k = 0; k < nv; ++k) {
        vs[k] = v0[k] + (T)dt * (accv[k] + (T)bw[3] * vd[k]);
        phi[k] = (T)dt * accphi[k];
        v[(int64_t)k * B + b] = vs[k];
      }
      const Col<T> cq0{q0.data(), 1}, cphi{phi.data(), 1}, cvs{vs.data(), 1};
      const ColOut<T> oq{q + b, B, true}, odump{dump.data(), 1, false};
      for (int j = 0; j < M.nb; ++j) joint_stage(M.body[j], cq0, cphi, cvs, oq, odump);
    }
  }
}

extern "C" {
// Model-specialised program (csrc/rbd_codegen.cpp) for the mechanism: flavor 0 = self-contained C++ (one sample per call),
// 1 = the per-sample CUDA function body, 3 = the whole NVRTC translation unit; fold = 0 keeps mirror-image chains straight-line
// (flavours 0-2).  Returns a malloc'ed string (free with hostsim_free) or NULL; stats = {nodes_traced, nodes_live, add, mul, div,
// neg, sincos, load, store, sld, sst, stash_rows, fold_loops, fold_bodies, pairs}.
// kin_mask / kin_sign (reference joint order, may be NULL): the rbd_kinematics variant (algo 3)
static int g_kin_mask = 0;
static int8_t g_kin_sign[rbd::kMaxBodies] = {0};
void hostsim_spec_kin(int mask, const int8_t* sign, int nb) {
  g_kin_mask = mask;
  for (int i = 0; i < rbd::kMaxBodies; ++i) g_kin_sign[i] = (sign && i < nb) ? sign[i] : 0;
}
char* hostsim_spec_source(const rbd_model_desc* d, int algo, int dtype, int has_in2, int has_out1, int flavor, int fold,
                          int* stats) {
  HostModel hm; std::string err;
  if (build_host_model(d, hm, err) != RBD_OK) return nullptr;
  SpecKey key; key.algo = algo; key.f64 = dtype == 1; key.has_in2 = (has_in2 & 1) != 0; key.has_out1 = has_out1 != 0;
  key.lower = (has_in2 & 2) != 0;      // CRBA: bit 1 of has_in2 selects the lower triangle
  if (algo == SPEC_KIN) {
    key.kin_mask = g_kin_mask;
    for (int p = 0; p < hm.nb; ++p) key.kin_sign[p] = g_kin_sign[hm.order[p]];
  }
  SpecStats st; std::string out;
  bool ok;
  if (flavor == 0) ok = spec_emit_cpu_tu(hm, key, "rbd_spec_cpu", out, &st, err, fold != 0);
  else if (flavor == 3) ok = spec_emit_cuda_tu(hm, key, out, &st, err);
  else ok = spec_emit_function(hm, key, flavor, "rbd_spec_fn", out, &st, err, fold != 0);
  if (!ok) return nullptr;
  if (stats) {
    const int v[15] = {st.nodes_traced, st.nodes_live, st.n_add, st.n_mul, st.n_div, st.n_neg, st.n_sincos, st.n_load, st.n_store,
                       st.n_sld, st.n_sst, st.stash_rows, st.n_fold_loops, st.n_fold_bodies, (int)hm.pairs.size()};
    for (int k = 0; k < 15; ++k) stats[k] = v[k];
  }
  char* r = (char*)malloc(out.size() + 1);
  std::memcpy(r, out.c_str(), out.size() + 1);
  return r;
}
void hostsim_free(char* p) { free(p); }

int hostsim_integrate(const rbd_model_desc* d, int dtype, int64_t B, void* q, void* v, const void* tau, double dt, int nsteps) {
  HostModel hm; std::string err;
  int rc = build_host_model(d, hm, err);
  if (rc) return rc;
  if (dtype == 0) run_integrate<float>(hm, B, (float*)q, (float*)v, (const float*)tau, dt, nsteps);
  else run_integrate<double>(hm, B, (double*)q, (double*)v, (const double*)tau, dt, nsteps);
  return 0;
}
int hostsim_info(const rbd_model_desc* d, int* nrows, int* general, int* nslots, int* order) {
  HostModel hm; std::string err;
  int rc = build_host_model(d, hm, err);
  if (rc) return rc;
  *nrows = hm.dev64.nrows; *general = hm.general; *nslots = hm.nslots;
  for (int i = 0; i < hm.nb; ++i) order[i] = hm.order[i];
  return 0;
}
int hostsim_dynamics(const rbd_model_desc* d, int dtype, int64_t B, const void* q, const void* v, const void* tau,
                     const void* wext, void* vd, void* qd) {
  HostModel hm; std::string err;
  int rc = build_host_model(d, hm, err);
  if (rc) return rc;
  if (dtype == 0) run_dynamics<float>(hm, B, (const float*)q, (const float*)v, (const float*)tau, (const float*)wext, (float*)vd, (float*)qd);
  else run_dynamics<double>(hm, B, (const double*)q, (const double*)v, (const double*)tau, (const double*)wext, (double*)vd, (double*)qd);
  return 0;
}
// dynamics! on Dual{Float64,6} arrays [rows][B][7]: one pass of the device code per (sample, partial direction)
int hostsim_dynamics_dual(const rbd_model_desc* d, int64_t B, const double* q, const double* v, const double* tau, double* vd) {
  HostModel hm; std::string err;
  int rc = build_host_model(d, hm, err);
  if (rc) return rc;
  const ModelDev<double>& S = hm.dev64;
  std::vector<ModelDev<Dual64>> Mv(1);
  ModelDev<Dual64>& M = Mv[0];
  M.nb = S.nb; M.nq = S.nq; M.nv = S.nv; M.nrows = S.nrows; M.slot_base = S.slot_base; M.nslots = S.nslots;
  for (int k = 0; k < 3; ++k) M.g[k] = Dual64(S.g[k]);
  for (int i = 0; i < S.nb; ++i) {
    const BodyDev<double>& s = S.body[i];
    BodyDev<Dual64>& b = M.body[i];
    for (int k = 0; k < 9; ++k) b.Rt[k] = Dual64(s.Rt[k]);
    for (int k = 0; k < 3; ++k) { b.pt[k] = Dual64(s.pt[k]); b.h[k] = Dual64(s.h[k]); }
    for (int k = 0; k < 6; ++k) b.J[k] = Dual64(s.J[k]);
    b.m = Dual64(s.m);
    b.qoff = Dual64(s.qoff);
    b.kind = s.kind; b.parent = s.parent; b.qrow = s.qrow; b.vrow = s.vrow; b.row0 = s.row0;
    b.oslot = s.oslot; b.pslot = s.pslot; b.flags = s.flags; b.refidx = s.refidx;
  }
  std::vector<Dual64> stash(M.nrows + 64);
  for (int64_t b = 0; b < B; ++b)
    for (int dir = 0; dir < 6; ++dir) {
      AbaIO<Dual64, false> io;
      io.q = {q + b * kDualWidth, B, dir};
      io.v = {v + b * kDualWidth, B, dir};
      io.tau = {tau ? tau + b * kDualWidth : nullptr, B, dir};
      io.wext = {nullptr, B, dir};
      io.vd = {vd + b * kDualWidth, B, dir, true};
      io.qd = {nullptr, B, dir, true};
      io.ext = {nullptr, 0};
      Stash<Dual64, 1> st{stash.data()};
      if (hm.general) aba_sample<Dual64, Stash<Dual64, 1>, true>(M, io, st);
      else aba_sample<Dual64, Stash<Dual64, 1>, false>(M, io, st);
    }
  return 0;
}
int hostsim_inverse_dynamics(const rbd_model_desc* d, int dtype, int64_t B, const void* q, const void* v, const void* vd,
                             const void* wext, void* tau) {
  HostModel hm; std::string err;
  int rc = build_host_model(d, hm, err);
  if (rc) return rc;
  if (dtype == 0) run_rnea<float>(hm, B, (const float*)q, (const float*)v, (const float*)vd, (const float*)wext, (float*)tau);
  else run_rnea<double>(hm, B, (const double*)q, (const double*)v, (const double*)vd, (const double*)wext, (double*)tau);
  return 0;
}
int hostsim_mass_matrix(const rbd_model_desc* d, int dtype, int64_t B, const void* q, void* M) {
  HostModel hm; std::string err;
  int rc = build_host_model(d, hm, err);
  if (rc) return rc;
  if (dtype == 0) run_crba<float>(hm, B, (const float*)q, (float*)M);
  else run_crba<double>(hm, B, (const double*)q, (double*)M);
  return 0;
}
int hostsim_kinematics(const rbd_model_desc* d, int dtype, int64_t B, const void* q, const void* v, const int8_t* sign,
                       void* const* outs) {
  HostModel hm; std::string err;
  int rc = build_host_model(d, hm, err);
  if (rc) return rc;
  if (dtype == 0) run_kin<float>(hm, B, (const float*)q, (const float*)v, sign, (float* const*)outs);
  else run_kin<double>(hm, B, (const double*)q, (const double*)v, sign, (double* const*)outs);
  return 0;
}
int hostsim_contact(const rbd_model_desc* d, int dtype, int64_t B, const void* q, const void* v, const rbd_contact_desc* cd, void* s,
                    void* sd, void* wr) {
  HostModel hm; std::string err;
  int rc = build_host_model(d, hm, err);
  if (rc) return rc;
  if (dtype == 0) run_contact<float>(hm, B, (const float*)q, (const float*)v, *cd, (float*)s, (float*)sd, (float*)wr);
  else run_contact<double>(hm, B, (const double*)q, (const double*)v, *cd, (double*)s, (double*)sd, (double*)wr);
  return 0;
}
int hostsim_derivatives(const rbd_model_desc* d, int dtype, int64_t B, const void* q, const void* v, const void* tau, void* vd, void* dq,
                        void* dv) {
  HostModel hm; std::string err;
  int rc = build_host_model(d, hm, err);
  if (rc) return rc;
  if (dtype == 0) return run_derivatives<float>(hm, B, (const float*)q, (const float*)v, (const float*)tau, (float*)vd, (float*)dq, (float*)dv);
  return run_derivatives<double>(hm, B, (const double*)q, (const double*)v, (const double*)tau, (double*)vd, (double*)dq, (double*)dv);
}
int hostsim_flags(const rbd_model_desc* d, int* flags /* [nb], preorder */) {
  HostModel hm; std::string err;
  int rc = build_host_model(d, hm, err);
  if (rc) return rc;
  for (int p = 0; p < hm.nb; ++p) flags[p] = hm.dev64.body[p].flags;
  return 0;
}
}
