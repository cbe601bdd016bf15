// Generator of the model-specialised solve kernel behind rbd_dynamics_derivatives.
//
// The generic deriv_solve_kernel (rbd_deriv.cu) walks index tables and keeps each right-hand side in shared memory: ~4 shared
// memory accesses per multiply-add, and it measured at half the shared-memory bandwidth of the SM.  For a concrete mechanism every
// index of the two triangular solves is a constant, so this generator writes them out: the right-hand sides of `cg` columns
// live in REGISTERS (x<u>_<p> are scalars), each entry of the factor is read from shared memory once per `cg` columns, and the
// two sweeps are straight-line fused multiply-adds.  The factorisation itself stays the table-driven cooperative loop (its
// tables become __constant__ arrays of the module).  Same arithmetic, same operation order per column as deriv_solve_column.
// With a third block (plan.blocks == 3) the columns 2 nv .. 3 nv - 1 solve the constant right-hand sides -e_j (d v̇ / d tau =
// M^-1, into dtau); nothing is loaded for them.  With two blocks the text is exactly that of the two-block kernel alone.
#include "rbd_deriv_jit.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>

namespace rbd {

bool deriv_jit_plan(const DerivDev& D, bool f64, DerivJitPlan& plan, int blocks) {
  const int words = f64 ? 2 : 1;                     // 32-bit registers per scalar
  const int budget = f64 ? 150 : 110;                // registers for right-hand sides (measured: Atlas fp64 2 columns, fp32 3)
  int cg = budget / (D.nv * words);
  if (cg < 1) return false;
  if (cg > 4) cg = 4;
  if (const char* e = std::getenv("RBD_DERIV_CG")) cg = std::max(1, std::min(cg, std::atoi(e)));     // experiments
  const int ncols = blocks * D.nv;
  plan.blocks = blocks;
  plan.cg = cg;
  plan.ngroups = (ncols + cg - 1) / cg;
  const int wmax = 12;
  const int rounds = (plan.ngroups + wmax - 1) / wmax;
  plan.warps = (plan.ngroups + rounds - 1) / rounds;
  return true;
}

void deriv_jit_source(const DerivDev& D, const DerivAnc& A, bool f64, const DerivJitPlan& plan, std::string& out) {
  const int nv = D.nv, nnz = D.nnz, cg = plan.cg, W = plan.warps;
  char b[512];
  std::string s;
  s.reserve(1 << 18);
  auto add = [&](const char* t) { s += t; };
  snprintf(b, sizeof b, "typedef %s T;\n#define NV %d\n#define NNZ %d\n#define NW %d\n#define CG %d\n#define NGRP %d\n", f64 ? "double" : "float", nv,
           nnz, W, cg, plan.ngroups);
  add(b);
  auto table = [&](const char* name, const int16_t* v, int n) {
    s += "__constant__ short "; s += name; s += "[] = {";
    for (int i = 0; i < n; ++i) { snprintf(b, sizeof b, "%d,", (int)v[i]); s += b; }
    s += "};\n";
  };
  table("kRowstart", D.rowstart, nv);
  table("kDepth", D.depth, nv);
  table("kAnc", A.anc, nnz);
  table("kPdof", D.pdof, nv);
  // rows related to column pj (its subtree and its ancestors): bit p of (lo, hi)
  s += "__constant__ unsigned long long kRel[][2] = {";
  for (int pj = 0; pj < nv; ++pj) {
    unsigned long long m[2] = {0, 0};
    for (int p = 0; p < nv; ++p) {
      const bool rel = (p >= pj && p < pj + D.dsub[pj]) || (pj >= p && pj < p + D.dsub[p]);
      if (rel) m[p >> 6] |= 1ull << (p & 63);
    }
    snprintf(b, sizeof b, "{0x%llxull,0x%llxull},", m[0], m[1]);
    s += b;
  }
  s += "};\n";
  const bool tau = plan.blocks == 3;
  add("extern \"C\" __global__ void __launch_bounds__(32 * NW, 1) rbd_deriv_solve(const T* __restrict__ Hg0, long long sld, T* dq, T* dv,\n");
  add(tau ? "                                                                     long long ld, long long C, T* dtau) {\n"
          : "                                                                     long long ld, long long C) {\n");
  add(
      "  extern __shared__ __align__(16) unsigned char smem_raw[];\n"
      "  T* Hs = reinterpret_cast<T*>(smem_raw) + (threadIdx.x & 31);\n"
      "  const int w = threadIdx.x >> 5;\n"
      "  const long long ngroups = (C + 31) / 32;\n"
      "  for (long long g = blockIdx.x; g < ngroups; g += gridDim.x) {\n"
      "    const long long b = g * 32 + (threadIdx.x & 31);\n"
      "    const bool active = b < C;\n"
      "    const long long bl = active ? b : C - 1;\n"
      "    const T* Hg = Hg0 + bl;\n"
      "    __syncthreads();\n"
      "    for (int r = w; r < NNZ; r += NW) Hs[r * 32] = Hg[r * sld];\n"
      "    for (int k = NV - 1; k >= 0; --k) {\n"
      "      const int rk = kRowstart[k], dk = kDepth[k];\n"
      "      __syncthreads();\n"
      "      const T inv = T(1) / Hs[(rk + dk) * 32];\n"
      "      for (int di = w; di < dk; di += NW) {\n"
      "        const int ri = kRowstart[kAnc[rk + di]];\n"
      "        const T f = Hs[(rk + di) * 32] * inv;\n"
      "        for (int d = di; d >= 0; --d) Hs[(ri + d) * 32] -= f * Hs[(rk + d) * 32];\n"
      "      }\n"
      "      __syncthreads();\n"
      "      for (int di = w; di < dk; di += NW) Hs[(rk + di) * 32] *= inv;\n"
      "      if (w == 0) Hs[(rk + dk) * 32] = inv;\n"
      "    }\n"
      "    __syncthreads();\n"
      "    // volatile: otherwise the compiler keeps every factor entry of the first sweep in a register for the second one (and spills)\n"
      "    const volatile T* Hv = Hs;\n"
      "    for (int cgi = w; cgi < NGRP; cgi += NW) {\n");
  for (int u = 0; u < cg; ++u) {
    if (tau) {
      // the unit columns: mask = {pj}, the right-hand side -1 there (bits of p and pj in the same word compare as the loads below)
      snprintf(b, sizeof b,
               "      const int c%d = cgi * CG + %d;\n"
               "      const bool ok%d = active && c%d < 3 * NV;\n"
               "      const int cc%d = c%d < 3 * NV ? c%d : 3 * NV - 1;\n"
               "      const bool e%d = cc%d >= 2 * NV;\n"
               "      const int vj%d = cc%d < NV ? cc%d : (e%d ? cc%d - 2 * NV : cc%d - NV);\n"
               "      T* col%d = (cc%d < NV ? dq : e%d ? dtau : dv) + (long long)vj%d * NV * ld + bl;\n",
               u, u, u, u, u, u, u, u, u, u, u, u, u, u, u, u, u, u, u);
      add(b);
      snprintf(b, sizeof b,
               "      const int pj%d = kPdof[vj%d];\n"
               "      const unsigned long long ml%d = e%d ? (pj%d < 64 ? 1ull << pj%d : 0ull) : kRel[pj%d][0],\n"
               "                               mh%d = e%d ? (pj%d >= 64 ? 1ull << (pj%d - 64) : 0ull) : kRel[pj%d][1];\n",
               u, u, u, u, u, u, u, u, u, u, u, u);
      add(b);
      for (int p = 0; p < nv; ++p) {
        snprintf(b, sizeof b, "      T x%d_%d = ((%s%d >> %d) & 1ull) ? (e%d ? T(-1) : col%d[%dll * ld]) : T(0);\n", u, p, p < 64 ? "ml" : "mh", u,
                 p & 63, u, u, (int)D.vrow[p]);
        add(b);
      }
      continue;
    }
    snprintf(b, sizeof b,
             "      const int c%d = cgi * CG + %d;\n"
             "      const bool ok%d = active && c%d < 2 * NV;\n"
             "      const int cc%d = c%d < 2 * NV ? c%d : 2 * NV - 1;\n"
             "      const int vj%d = cc%d < NV ? cc%d : cc%d - NV;\n"
             "      T* col%d = (cc%d < NV ? dq : dv) + (long long)vj%d * NV * ld + bl;\n"
             "      const unsigned long long ml%d = kRel[kPdof[vj%d]][0], mh%d = kRel[kPdof[vj%d]][1];\n",
             u, u, u, u, u, u, u, u, u, u, u, u, u, u, u, u, u, u);
    add(b);
    for (int p = 0; p < nv; ++p) {
      snprintf(b, sizeof b, "      T x%d_%d = ((%s%d >> %d) & 1ull) ? col%d[%dll * ld] : T(0);\n", u, p, p < 64 ? "ml" : "mh", u, p & 63, u, (int)D.vrow[p]);
      add(b);
    }
  }
  // One basic block of ~10^3 loads and ~10^3 x cg multiply-adds makes ptxas hoist the loads until nothing fits (it then gives up
  // on registers altogether): a never-taken branch every `split` factor entries bounds its scheduling regions.
  int split = 24, since = 0;
  if (const char* e = std::getenv("RBD_DERIV_SPLIT")) split = std::atoi(e);
  auto maybe_split = [&]() { if (split > 0 && ++since >= split) { since = 0; add("      if (ld < 0) asm volatile(\"trap;\");\n"); } };
  // L^-T
  for (int i = nv - 1; i >= 0; --i) {
    const int ri = D.rowstart[i];
    for (int d = D.depth[i] - 1; d >= 0; --d) {
      const int j = A.anc[ri + d];
      snprintf(b, sizeof b, "      { const T h = Hv[%d];", (ri + d) * 32);
      add(b);
      for (int u = 0; u < cg; ++u) { snprintf(b, sizeof b, " x%d_%d -= h * x%d_%d;", u, j, u, i); add(b); }
      add(" }\n");
      maybe_split();
    }
  }
  for (int p = 0; p < nv; ++p) {
    snprintf(b, sizeof b, "      { const T h = Hv[%d];", (D.rowstart[p] + D.depth[p]) * 32);
    add(b);
    for (int u = 0; u < cg; ++u) { snprintf(b, sizeof b, " x%d_%d *= h;", u, p); add(b); }
    add(" }\n");
  }
  // L^-1 and the stores.  The store addresses are the load addresses; left to itself the compiler keeps all 2 * cg * nv of them
  // alive across the sweeps (and spills): an opaque copy of ld makes it recompute each one where it is used.
  add("      long long ld2;\n      asm volatile(\"mov.b64 %0, %1;\" : \"=l\"(ld2) : \"l\"(ld));\n");
  for (int i = 0; i < nv; ++i) {
    const int ri = D.rowstart[i];
    for (int d = D.depth[i] - 1; d >= 0; --d) {
      const int j = A.anc[ri + d];
      snprintf(b, sizeof b, "      { const T h = Hv[%d];", (ri + d) * 32);
      add(b);
      for (int u = 0; u < cg; ++u) { snprintf(b, sizeof b, " x%d_%d -= h * x%d_%d;", u, i, u, j); add(b); }
      add(" }\n");
      maybe_split();
    }
    for (int u = 0; u < cg; ++u) {
      snprintf(b, sizeof b, "      if (ok%d) col%d[%dll * ld2] = -x%d_%d;\n", u, u, (int)D.vrow[i], u, i);
      add(b);
    }
  }
  add("    }\n  }\n}\n");
  out.swap(s);
}

}  // namespace rbd
