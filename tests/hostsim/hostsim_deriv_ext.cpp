// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
// Runs the per-sample functions of rbd_dynamics_derivatives_ext / rbd_inverse_dynamics_derivatives (csrc/rbd_deriv.cuh) ON THE CPU:
// the world pass with the external-wrench rows, the subtree sums, the pair entries, then either the factor and the three-block solve
// (forward) or the dense expansion of M and the zeros of unrelated pairs (inverse).  One sample at a time with a scratch column of
// one row per scalar, as hostsim.cpp's run_derivatives.
#include <string>
#include <vector>

#include "../../rigidbodydynamics/jl_b200/csrc/rbd_deriv.cuh"
#include "../../rigidbodydynamics/jl_b200/csrc/rbd_model.h"

using namespace rbd;

namespace {
template <class T> const ModelDev<T>& dev(const HostModel& m);
template <> const ModelDev<float>& dev<float>(const HostModel& m) { return m.dev32; }
template <> const ModelDev<double>& dev<double>(const HostModel& m) { return m.dev64; }

// vd: the linearisation point (forward: v̇ = dynamics(q, v, tau, wext), computed by the caller; inverse: the caller's v̇).
// Forward: dq, dv = d v̇ / d(q, v), dtau = M^-1 or NULL.  Inverse: dq, dv = d tau / d(q, v), tau and Mo or NULL.
template <class T>
int run(const HostModel& hm, int inverse, int64_t B, const T* q, const T* v, const T* vd, const T* wext, T* dq, T* dv, T* dtau, T* tau,
        T* Mo) {
  const ModelDev<T>& M = dev<T>(hm);
  DerivDev D; DerivAnc A;
  if (!build_deriv_dev(M, D, A)) return RBD_EUNSUPPORTED;
  if (wext) deriv_dev_add_wrenches(D);
  const int nv = D.nv;
  std::vector<T> stash(kin_rows(hm) + 64), scr(D.rows), x(nv);
  for (int64_t b = 0; b < B; ++b) {
    DerivIO<T> io;
    io.q = {q + b, B}; io.v = {v + b, B}; io.vd = {vd + b, B};
    if (wext) io.wext = {wext + b, B};
    io.s = scr.data(); io.sld = 1; io.active = true;
    const Stash<T, 1> st{stash.data()};
    if (wext) deriv_world_sample<T, Stash<T, 1>, true>(M, D, io, st);
    else deriv_world_sample<T>(M, D, io, st);
    for (int c = 0; c < kBodyRows; ++c) deriv_accumulate<T>(M, D, scr.data(), 1, c);
    if (wext)
      for (int c = 0; c < 6; ++c) deriv_accumulate_wrench<T>(M, D, scr.data(), 1, c);
    for (int K = 0; K < M.nb; ++K) {
      T* tb = tau ? tau + b : nullptr;
      if (wext && tau) deriv_pairs<T, true, true>(D, A, scr.data(), 1, dq + b, dv + b, B, K, true, tb);
      else if (wext) deriv_pairs<T, true>(D, A, scr.data(), 1, dq + b, dv + b, B, K, true);
      else if (tau) deriv_pairs<T, false, true>(D, A, scr.data(), 1, dq + b, dv + b, B, K, true, tb);
      else deriv_pairs<T>(D, A, scr.data(), 1, dq + b, dv + b, B, K, true);
    }
    const T* H = scr.data() + D.h_base;
    if (inverse) {
      for (int vj = 0; vj < nv; ++vj) deriv_expand_column<T>(D, H, 1, dq + b, dv + b, Mo ? Mo + b : nullptr, B, vj, true);
      continue;
    }
    deriv_factor<T>(D, A, scr.data() + D.h_base, 1);
    auto Hf = [H](int row) { return H[row]; };
    const int ncols = dtau ? 3 * nv : 2 * nv;
    for (int c = 0; c < ncols; ++c) {
      const int blk = c / nv, vj = c % nv;
      T* out = (blk == 0 ? dq : blk == 1 ? dv : dtau) + (int64_t)vj * nv * B + b;
      deriv_solve_column<T>(D, A, Hf, x.data(), 1, out, B, vj, true, blk == 2);
    }
  }
  return 0;
}
}  // namespace

extern "C" {
int hostsim_deriv_ext(const rbd_model_desc* d, int inverse, int dtype, int64_t B, const void* q, const void* v, const void* vd,
                      const void* wext, void* dq, void* dv, void* dtau, void* tau, void* Mo) {
  HostModel hm; std::string err;
  int rc = build_host_model(d, hm, err);
  if (rc) return rc;
  if (dtype == 0)
    return run<float>(hm, inverse, B, (const float*)q, (const float*)v, (const float*)vd, (const float*)wext, (float*)dq, (float*)dv,
                      (float*)dtau, (float*)tau, (float*)Mo);
  return run<double>(hm, inverse, B, (const double*)q, (const double*)v, (const double*)vd, (const double*)wext, (double*)dq,
                     (double*)dv, (double*)dtau, (double*)tau, (double*)Mo);
}
}
