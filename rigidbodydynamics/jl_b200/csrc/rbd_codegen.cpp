// Model-specialised code generation (see rbd_codegen.h, rbd_sym.h).  Host-only C++.
#include "rbd_codegen.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <unordered_map>

#include "rbd_rnea_crba.cuh"
#include "rbd_sym.h"
#include "rbd_kin.cuh"

namespace rbd {
namespace {

constexpr int kGeneratorVersion = 26;   // bump when the emitted code changes (part of the cubin cache key)

template <class F> const ModelDev<F>& devm(const HostModel& m);
template <> const ModelDev<float>& devm<float>(const HostModel& m) { return m.dev32; }
template <> const ModelDev<double>& devm<double>(const HostModel& m) { return m.dev64; }

struct TraceScope {
  SymTrace* prev;
  explicit TraceScope(SymTrace* t) : prev(sym_trace()) { sym_trace() = t; }
  ~TraceScope() { sym_trace() = prev; }
};

// Drops upper-triangle stores of the mass matrix when only the lower one is wanted (mass_matrix! fills M.data's lower
// triangle only, mechanism_algorithms.jl:248-272): a store to row i + j*nv with i < j is not recorded.
struct LowerFilter { int nv; };

bool run_trace(const HostModel& hm, const SpecKey& key, SymTrace& tr, int& stash_rows, std::string& err) {
  tr.single = !key.f64;
  TraceScope scope(&tr);
  std::unique_ptr<ModelDev<Sym>> M(new ModelDev<Sym>());
  if (key.f64) sym_model(hm.dev64, *M); else sym_model(hm.dev32, *M);
  const SymStash st;
  if (key.algo == SPEC_ABA) {
    AbaIO<Sym, false, kAllKinds> io;
    io.q = {A_Q, true}; io.v = {A_V, true}; io.tau = {A_TAU, key.has_in2}; io.wext = {A_WEXT, false};
    io.vd = {A_OUT0, true}; io.qd = {A_OUT1, key.has_out1};
    io.ext = {false};
    if (hm.general) aba_sample<Sym, SymStash, true>(*M, io, st);
    else aba_sample<Sym, SymStash, false>(*M, io, st);
    stash_rows = hm.dev64.nrows;
    return true;
  }
  if (key.algo == SPEC_RNEA) {
    RneaIO<Sym> io;
    io.q = {A_Q, true}; io.v = {A_V, true}; io.vd = {A_VD_IN, key.has_in2}; io.wext = {A_WEXT, false};
    io.tau = {A_OUT0, true};
    io.ext = {false};
    rnea_sample<Sym>(*M, io, st);
    stash_rows = rnea_rows(hm);
    return true;
  }
  if (key.algo == SPEC_CRBA) {
    CrbaIO<Sym> io;
    io.q = {A_Q, true};
    io.M = {A_OUT0, true};
    io.lower = key.lower;
    crba_sample<Sym, SymStash, 6>(*M, io, st);      // KMAX 6 covers every joint kind; unused columns are never touched
    stash_rows = crba_rows(hm);
    return true;
  }
  if (key.algo == SPEC_KIN) {
    std::unique_ptr<KinDev<Sym>> K(new KinDev<Sym>());
    for (int p = 0; p < hm.nb; ++p) {
      for (int k = 0; k < 9; ++k) K->At[p][k] = Sym(hm.alignT[9 * p + k]);
      K->sign[p] = key.kin_sign[p];
    }
    K->inv_mass = Sym(1.0 / hm.total_mass);
    KinIO<Sym> io;
    io.q = {A_Q, true}; io.v = {A_V, key.has_in2};
    auto out = [&](int k) { return ColOut<Sym>{A_K0 + k, (key.kin_mask >> k & 1) != 0}; };
    io.tr = out(0); io.com = out(1); io.ke = out(2); io.pe = out(3); io.mom = out(4); io.mrb = out(5); io.A = out(6); io.J = out(7);
    if (key.kin_mask == (1 << 6) && 6 * hm.nv + kSlotRowsMomMat * hm.nslots <= 256) {
      // the momentum matrix on its own: the two body-frame sweeps (nothing but the result columns crosses them)
      momentum_matrix_sample<Sym, SymStash>(*M, io.q, io.A, st);
      stash_rows = spec_stash_rows(hm, key);
      return true;
    }
    std::vector<int32_t> poses;            // the momentum matrix' return sweep re-uses the traced poses themselves (Scr<Sym>::fwd)
    io.poses = {io.A.valid(), &poses};
    kin_sample<Sym, SymStash>(*M, *K, io, st);
    stash_rows = std::max(1, kin_rows(hm));
    return true;
  }
  err = "spec: algorithm not specialisable";
  return false;
}

struct Emitter {
  const SymTrace& tr;
  const SpecKey& key;
  int flavor;
  std::vector<uint8_t> live;
  std::string out;
  SpecStats stats;

  int split_every = 0;           // CUDA flavours: RBD_SPLIT() (a never-taken branch = basic-block boundary) every N statements
  std::vector<int32_t> uses;     // live uses of every node
  std::vector<uint8_t> fused;    // product folded into the FMA of its single consumer

  // Explicit fused multiply-adds (the translation units are compiled with --fmad=false): a product with exactly one use, by an
  // addition or subtraction, is folded into it.  Doing the contraction HERE rather than leaving it to the compiler makes the
  // kernel and the CPU flavour bit-identical.
  void plan_fma() {
    const auto& N = tr.nodes;
    uses.assign(N.size(), 0);
    fused.assign(N.size(), 0);
    for (size_t i = 0; i < N.size(); ++i) {
      if (!live[i]) continue;
      const SymNode& n = N[i];
      if (n.op == S_COS) continue;
      if (n.a >= 0) ++uses[n.a];
      if (n.b >= 0) ++uses[n.b];
    }
    for (size_t i = 0; i < N.size(); ++i) {
      if (!live[i]) continue;
      const SymNode& n = N[i];
      if (n.op != S_ADD && n.op != S_SUB) continue;
      // prefer the later-computed product (it is the one on the critical path)
      const int cand[2] = {std::max(n.a, n.b), std::min(n.a, n.b)};
      for (int c : cand)
        if (N[c].op == S_MUL && uses[c] == 1 && !fused[c]) { fused[c] = 1; fma_of[i] = c; break; }
    }
  }
  std::unordered_map<size_t, int32_t> fma_of;   // add / sub node -> the product folded into it

  Emitter(const SymTrace& t, const SpecKey& k, int f) : tr(t), key(k), flavor(f), live(t.nodes.size(), 0) {}

  void mark() {      // nodes are in topological order: one backward sweep
    const auto& N = tr.nodes;
    for (int i = (int)N.size() - 1; i >= 0; --i) {
      const SymNode& n = N[i];
      if (n.op == S_STORE || n.op == S_SST || n.op == S_SFENCE || n.op == S_XST) live[i] = 1;
      if (!live[i]) continue;
      if (n.op == S_COS) { live[n.b] = 1; continue; }      // the pair is emitted at its sin node, which carries the argument
      if (n.a >= 0) live[n.a] = 1;
      if (n.b >= 0) live[n.b] = 1;
    }
  }

  std::string lit(double v) const {
    char buf[64];
    if (key.f64) snprintf(buf, sizeof buf, "%.17g", v);
    else snprintf(buf, sizeof buf, "%.9g", v);
    std::string s(buf);
    if (s.find_first_of(".eEn") == std::string::npos) s += ".0";      // "n": inf / nan never occur for model constants
    if (!key.f64) s += "f";
    return s;
  }
  std::string ref(int id) const {
    const SymNode& n = tr.nodes[id];
    if (n.op == S_CONST) return "RBD_K(" + lit(n.c) + ")";
    return "t" + std::to_string(id);
  }
  static const char* arr_name(int arr) {
    switch (arr) {
      case A_Q: return "q";
      case A_V: return "v";
      case A_TAU: return "in2";
      case A_VD_IN: return "in2";
      case A_WEXT: return "wext";
      case A_OUT0: return "o0";
      case A_OUT1: return "o1";
      case A_K0: return "ko0"; case A_K1: return "ko1"; case A_K2: return "ko2"; case A_K3: return "ko3";
      case A_K4: return "ko4"; case A_K5: return "ko5"; case A_K6: return "ko6"; case A_K7: return "ko7";
    }
    return "?";
  }

  void emit() {
    mark();
    plan_fma();
    const auto& N = tr.nodes;
    char line[256];
    stats.nodes_traced = (int)N.size();
    int since = 0;
    for (size_t i = 0; i < N.size(); ++i) {
      if (!live[i]) continue;
      const SymNode& n = N[i];
      if (n.op != S_CONST) ++stats.nodes_live;
      if (fused[i]) continue;
      if (split_every > 0 && n.op != S_CONST && n.op != S_COS && ++since >= split_every && !(n.op == S_SLD && n.grp != (int)i)) {
        out += "RBD_SPLIT();\n";
        since = 0;
      }
      switch (n.op) {
        case S_CONST: break;
        case S_ADD:
        case S_SUB: {
          ++stats.n_add;
          auto it = fma_of.find(i);
          if (it == fma_of.end()) {
            snprintf(line, sizeof line, "const rbd_v t%zu = %s(%s, %s);\n", i, n.op == S_ADD ? "RBD_ADD" : "RBD_SUB", ref(n.a).c_str(), ref(n.b).c_str());
          } else {
            const SymNode& p = N[it->second];
            const int other = it->second == n.a ? n.b : n.a;
            const char* f = n.op == S_ADD ? "RBD_FMA" : (it->second == n.a ? "RBD_FMS" /* x*y - c */ : "RBD_FNMA" /* c - x*y */);
            snprintf(line, sizeof line, "const rbd_v t%zu = %s(%s, %s, %s);\n", i, f, ref(p.a).c_str(), ref(p.b).c_str(), ref(other).c_str());
          }
          out += line;
          break;
        }
        case S_MUL: ++stats.n_mul; snprintf(line, sizeof line, "const rbd_v t%zu = RBD_MUL(%s, %s);\n", i, ref(n.a).c_str(), ref(n.b).c_str()); out += line; break;
        case S_DIV:
          ++stats.n_div;
          if (tr.is_const(n.a, 1.0)) snprintf(line, sizeof line, "const rbd_v t%zu = RBD_RCP(%s);\n", i, ref(n.b).c_str());
          else snprintf(line, sizeof line, "const rbd_v t%zu = RBD_DIV(%s, %s);\n", i, ref(n.a).c_str(), ref(n.b).c_str());
          out += line;
          break;
        case S_NEG: ++stats.n_neg; snprintf(line, sizeof line, "const rbd_v t%zu = RBD_NEG(%s);\n", i, ref(n.a).c_str()); out += line; break;
        case S_SIN:
          ++stats.n_sincos;
          snprintf(line, sizeof line, "rbd_v t%zu, t%zu; RBD_SINCOS(%s, t%zu, t%zu);\n", i, i + 1, ref(n.a).c_str(), i, i + 1);
          out += line;
          break;
        case S_COS: break;
        case S_LOAD:
          ++stats.n_load;
          if (n.arr == A_V) ++stats.n_load_v;
          snprintf(line, sizeof line, "const rbd_v t%zu = RBD_LDG(%s, %d);\n", i, arr_name(n.arr), n.row);
          out += line;
          break;
        case S_STORE:
          ++stats.n_store;
          if (key.peers && n.arr == A_OUT0 && flavor != FLAVOR_CPU) snprintf(line, sizeof line, "RBD_STG_PEERS(%d, %s);\n", n.row, ref(n.a).c_str());
          else snprintf(line, sizeof line, "RBD_STG(%s, %d, %s);\n", arr_name(n.arr), n.row, ref(n.a).c_str());
          out += line;
          break;
        case S_SLD: {
          ++stats.n_sld;
          snprintf(line, sizeof line, "const rbd_v t%zu = RBD_SLD(%d);\n", i, n.row);
          out += line;
          break;
        }
        case S_SST:
          ++stats.n_sst;
          snprintf(line, sizeof line, "RBD_SST(%d, %s);\n", n.row, ref(n.a).c_str());
          out += line;
          break;
        case S_SFENCE: out += "RBD_SFENCE();\n"; break;
        case S_XLD: snprintf(line, sizeof line, "const rbd_v t%zu = RBD_XLD(%d);\n", i, n.row); out += line; break;
        case S_XST: snprintf(line, sizeof line, "RBD_XST(%d, %s);\n", n.row, ref(n.a).c_str()); out += line; break;
      }
    }
  }
};

}  // namespace

bool spec_emit_function(const HostModel& hm, const SpecKey& key, int flavor, const std::string& name, std::string& out,
                        SpecStats* stats, std::string& err) {
  SymTrace tr;
  int rows = 0;
  if (!run_trace(hm, key, tr, rows, err)) return false;
  Emitter em(tr, key, flavor);
  if (flavor != FLAVOR_CPU) {
    // One basic block of 10^4 instructions lets ptxas stretch live ranges until it spills (Atlas: 128 registers + 350 B of
    // local memory, -10 % throughput); a never-taken branch every few hundred statements bounds its scheduling regions.
    em.split_every = 192;
    if (const char* e = getenv("RBD_JIT_SPLIT")) em.split_every = atoi(e);
  }
  em.emit();
  em.stats.stash_rows = rows;
  if (stats) *stats = em.stats;
  const char* F = key.f64 ? "double" : "float";
  std::string sig;
  if (flavor == FLAVOR_CPU) {
    sig = std::string("extern \"C\" void ") + name + "(const " + F + "* q, const " + F + "* v, const " + F + "* in2, " + F + "* o0, " +
          F + "* o1, long long ld, " + F + "* sh" + (key.algo == SPEC_KIN ? std::string(", ") + F + "* const* ko)" : std::string(")"));
  } else {
    sig = std::string("__device__ __forceinline__ void ") + name + "(const rbd_f* __restrict__ q, const rbd_f* __restrict__ v, "
          "const rbd_f* __restrict__ in2, rbd_f* __restrict__ o0, rbd_f* __restrict__ o1, const long long ld, const bool active, "
          "int* flag, const RbdJitArgs& pa, const long long pb, RBD_STASH_ARG)";
  }
  out += sig + " {\n";
  if (flavor != FLAVOR_CPU) out += "RBD_FN_BEGIN\n";
  if (key.algo == SPEC_KIN) out += flavor == FLAVOR_CPU ? "RBD_KIN_BEGIN_CPU\n" : "RBD_KIN_BEGIN\n";
  out += em.out;
  if (flavor != FLAVOR_CPU) out += "RBD_FN_END\n";
  out += "}\n";
  return true;
}

int spec_stash_rows(const HostModel& hm, const SpecKey& key) {
  if (key.algo == SPEC_KIN) {
    const int two_sweep = 6 * hm.nv + kSlotRowsMomMat * hm.nslots;
    return (key.kin_mask == (1 << 6) && two_sweep <= 256) ? two_sweep : std::max(1, kin_rows(hm));
  }
  return key.algo == SPEC_ABA ? hm.dev64.nrows : (key.algo == SPEC_RNEA ? rnea_rows(hm) : std::max(1, crba_rows(hm)));
}

uint64_t spec_hash(const HostModel& hm, const SpecKey& key) {
  uint64_t h = 0xcbf29ce484222325ull;
  auto mix = [&](const void* p, size_t n) {
    const unsigned char* b = (const unsigned char*)p;
    for (size_t i = 0; i < n; ++i) { h ^= b[i]; h *= 0x100000001b3ull; }
  };
  const int hdr[9] = {kGeneratorVersion, key.algo, key.f64, key.has_in2, key.has_out1, key.lower, hm.nb, hm.general, key.peers};
  mix(hdr, sizeof hdr);
  if (key.algo == SPEC_KIN) { mix(&key.kin_mask, sizeof key.kin_mask); mix(key.kin_sign, sizeof key.kin_sign); }
  if (key.f64) {
    const ModelDev<double>& M = hm.dev64;
    mix(&M, offsetof(ModelDev<double>, body) + sizeof(BodyDev<double>) * (size_t)M.nb);
  } else {
    const ModelDev<float>& M = hm.dev32;
    mix(&M, offsetof(ModelDev<float>, body) + sizeof(BodyDev<float>) * (size_t)M.nb);
  }
  return h;
}

bool spec_emit_cuda_tu(const HostModel& hm, const SpecKey& key, std::string& out, SpecStats* stats, std::string& err) {
  // the per-sample function first (its statistics go into the header)
  std::string fn_smem;
  SpecStats st;
  if (!spec_emit_function(hm, key, FLAVOR_SMEM, "rbd_spec_smem", fn_smem, &st, err)) return false;
  if (stats) *stats = st;
  char buf[768];
  const int rows = spec_stash_rows(hm, key);
  snprintf(buf, sizeof buf,
           "// generated by librbd_b200.so (rbd_codegen.cpp) for one mechanism: %d live nodes (%d add/sub, %d mul, %d div, %d sincos, "
           "%d global loads, %d stash loads, %d stash stores)\n"
           "#define RBD_SPEC_F64 %d\n#define RBD_SPEC_NQ %d\n#define RBD_SPEC_NV %d\n#define RBD_SPEC_ROWS %d\n"
           "#define RBD_SPEC_HAS_IN2 %d\n#define RBD_SPEC_HAS_OUT1 %d\n#define RBD_SPEC_OUT0_ROWS %d\n#define RBD_SPEC_OUT1_ROWS %d\n"
           "#define RBD_SPEC_ROW32 %d\n#define RBD_SPEC_KIN %d\n#define RBD_SPEC_USES_V %d\n#include \"rbd_jit_prelude.cuh\"\n",
           st.nodes_live, st.n_add, st.n_mul, st.n_div, st.n_sincos, st.n_load, st.n_sld, st.n_sst,
           key.f64 ? 1 : 0, hm.nq, hm.nv, rows, key.has_in2 ? 1 : 0, key.has_out1 ? 1 : 0, key.algo == SPEC_CRBA ? hm.nv * hm.nv : hm.nv, hm.nq,
           key.algo == SPEC_CRBA ? 1 : 0, key.algo == SPEC_KIN ? 1 : 0, st.n_load_v > 0 ? 1 : 0);
  out += buf;
  out += "#define RBD_FLAVOR_SMEM 1\n#include \"rbd_jit_flavor.cuh\"\n" + fn_smem;
  out += "#include \"rbd_jit_kernels.cuh\"\n";
  return true;
}

bool spec_emit_cpu_tu(const HostModel& hm, const SpecKey& key, const std::string& name, std::string& out, SpecStats* stats,
                      std::string& err) {
  out += "// generated by librbd_b200.so (rbd_codegen.cpp): model-specialised program, CPU flavour (test tier)\n"
         "#include \"rbd_device.cuh\"\n"
         "#define RBD_LDG(p, r) p[(long long)(r) * ld]\n#define RBD_STG(p, r, x) p[(long long)(r) * ld] = (x)\n"
         "#define RBD_SLD(r) sh[r]\n#define RBD_SST(r, x) sh[r] = (x)\n#define RBD_SFENCE()\n"
         "#define RBD_RCP(x) (1 / (x))\n#define RBD_DIV(a, b) ((a) / (b))\n#define RBD_SINCOS(x, s, c) rbd::sincos_t(x, s, c)\n"
         "#define RBD_K(x) (x)\n#define RBD_ADD(a, b) ((a) + (b))\n#define RBD_SUB(a, b) ((a) - (b))\n#define RBD_MUL(a, b) ((a) * (b))\n"
         "#define RBD_KIN_BEGIN_CPU rbd_v *ko0 = ko[0], *ko1 = ko[1], *ko2 = ko[2], *ko3 = ko[3], *ko4 = ko[4], *ko5 = ko[5], *ko6 = ko[6], *ko7 = ko[7]; (void)ko0; (void)ko1; (void)ko2; (void)ko3; (void)ko4; (void)ko5; (void)ko6; (void)ko7;\n"
         "#define RBD_NEG(a) (-(a))\n#define RBD_FMA(a, b, c) std::fma(a, b, c)\n#define RBD_FMS(a, b, c) std::fma(a, b, -(c))\n"
         "#define RBD_FNMA(a, b, c) std::fma(-(a), b, c)\n";
  out += std::string("typedef ") + (key.f64 ? "double" : "float") + " rbd_v;\n";
  return spec_emit_function(hm, key, FLAVOR_CPU, name, out, stats, err);
}

}  // namespace rbd
