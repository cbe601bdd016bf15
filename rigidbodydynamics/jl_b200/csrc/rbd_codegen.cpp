// Model-specialised code generation (see rbd_codegen.h, rbd_sym.h).  Host-only C++.
#include "rbd_codegen.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <array>
#include <functional>
#include <map>
#include <memory>
#include <set>
#include <unordered_map>
#include <unordered_set>

#include "rbd_rnea_crba.cuh"
#include "rbd_sym.h"
#include "rbd_kin.cuh"

namespace rbd {
namespace {

constexpr int kGeneratorVersion = 31;   // bump when the emitted code changes (part of the cubin cache key)
constexpr int kRegRowsAba = -1;         // register-resident stash rows of the fp32 forward-dynamics programs (-1: all eligible)
constexpr int kSmemPerSm = 233472;      // H100: 228 KB of shared memory per SM ...
constexpr int kSmemReservedPerBlock = 1024;   // ... of which each resident block takes 1 KB for the system

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

bool run_trace(const HostModel& hm, const SpecKey& key, bool trig, SymTrace& tr, int& stash_rows, std::string& err) {
  tr.single = !key.f64;
  TraceScope scope(&tr);
  std::unique_ptr<ModelDev<Sym>> M(new ModelDev<Sym>());
  const std::vector<FoldPair>* pairs = key.algo == SPEC_ABA ? &hm.pairs : nullptr;
  if (key.f64) sym_model(hm.dev64, *M, pairs); else sym_model(hm.dev32, *M, pairs);
  if (pairs)
    for (const FoldPair& fp : *pairs)
      for (int pass = 1; pass <= 3; ++pass) {
        const int a = pass == 2 ? fp.l0 + 2 * fp.len - 1 : fp.l0, b = pass == 2 ? fp.l0 + fp.len - 1 : fp.l0 + fp.len;
        tr.fresh_steps.insert({pass, a});
        tr.fresh_steps.insert({pass, b});
        // the step before the pair already requests the first body's joint scalars (prefetch_body)
        if (pass == 2) tr.fresh_steps.insert(a + 1 < hm.nb ? std::make_pair(2, a + 1) : std::make_pair(1, -1));
        else if (a > 1) tr.fresh_steps.insert({pass, a - 1});
        else if (pass == 3) tr.fresh_steps.insert({2, -1});
      }
  SymStash st;
  st.trig = trig && key.algo == SPEC_ABA;
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
  int split_folded = 0;          // the same for a program with folded chains
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
    if (n.op == S_CONST || n.op == S_PARAM) return "RBD_K(" + lit(n.c) + ")";   // straight-line code: a parameter is its value
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
  bool stmt_node(int i) const {
    const int op = tr.nodes[i].op;
    return live[i] && op != S_CONST && op != S_LOAD && op != S_PARAM;
  }

  // Text of statement i: name(j) = variable of node j, opnd(j, k) = operand k (0: a, 1: b) of node j, row(j) = its row expression.
  using NameFn = std::function<std::string(int)>;
  using OpFn = std::function<std::string(int, int)>;
  std::string stmt(int i, const NameFn& name, const OpFn& opnd, const NameFn& row) {
    const SymNode& n = tr.nodes[i];
    const std::string v = "const rbd_v " + name(i) + " = ";
    switch (n.op) {
      case S_ADD:
      case S_SUB: {
        ++stats.n_add;
        auto it = fma_of.find(i);
        if (it == fma_of.end()) return v + (n.op == S_ADD ? "RBD_ADD(" : "RBD_SUB(") + opnd(i, 0) + ", " + opnd(i, 1) + ");\n";
        const int p = it->second;
        const char* f = n.op == S_ADD ? "RBD_FMA" : (p == n.a ? "RBD_FMS" /* x*y - c */ : "RBD_FNMA" /* c - x*y */);
        return v + f + "(" + opnd(p, 0) + ", " + opnd(p, 1) + ", " + opnd(i, p == n.a ? 1 : 0) + ");\n";
      }
      case S_MUL: ++stats.n_mul; return v + "RBD_MUL(" + opnd(i, 0) + ", " + opnd(i, 1) + ");\n";
      case S_DIV:
        ++stats.n_div;
        if (tr.is_const(n.a, 1.0)) return v + "RBD_RCP(" + opnd(i, 1) + ");\n";
        return v + "RBD_DIV(" + opnd(i, 0) + ", " + opnd(i, 1) + ");\n";
      case S_NEG: ++stats.n_neg; return v + "RBD_NEG(" + opnd(i, 0) + ");\n";
      case S_SIN:
        ++stats.n_sincos;
        return "rbd_v " + name(i) + ", " + name(i + 1) + "; RBD_SINCOS(" + opnd(i, 0) + ", " + name(i) + ", " + name(i + 1) + ");\n";
      case S_LOAD:
        ++stats.n_load;
        if (n.arr == A_V) ++stats.n_load_v;
        return v + "RBD_LDG(" + arr_name(n.arr) + ", " + row(i) + ");\n";
      case S_STORE:
        ++stats.n_store;
        if (key.peers && n.arr == A_OUT0 && flavor != FLAVOR_CPU) return "RBD_STG_PEERS(" + row(i) + ", " + opnd(i, 0) + ");\n";
        return std::string("RBD_STG(") + arr_name(n.arr) + ", " + row(i) + ", " + opnd(i, 0) + ");\n";
      case S_SLD:
        ++stats.n_sld;
        if (reg_row(n.arr, n.row)) return v + rname(n.arr, n.row) + ";\n";
        return v + (n.arr == R_TRIG ? "RBD_TLD(" : "RBD_SLD(") + row(i) + ");\n";
      case S_SST:
        ++stats.n_sst;
        if (reg_row(n.arr, n.row)) return rname(n.arr, n.row) + " = " + opnd(i, 0) + ";\n";
        return (n.arr == R_TRIG ? "RBD_TST(" : "RBD_SST(") + row(i) + ", " + opnd(i, 0) + ");\n";
      case S_SFENCE: return "RBD_SFENCE();\n";
      case S_XLD: return v + "RBD_XLD(" + row(i) + ");\n";
      case S_XST: return "RBD_XST(" + row(i) + ", " + opnd(i, 0) + ");\n";
    }
    return "";
  }
  std::string split_point(int i, int& since) {
    const SymNode& n = tr.nodes[i];
    if (split_every > 0 && n.op != S_COS && ++since >= split_every && !(n.op == S_SLD && n.grp != i)) {
      since = 0;
      return "RBD_SPLIT();\n";
    }
    return "";
  }

  // ---- folding mirror-image chains ------------------------------------------------------------------------------------
  // In each ABA pass the two chains of a HostModel pair are walked back to back: segment A (the first walked: the left chain
  // outward, the right chain inward), then segment B.  B is folded onto A when it is the same program statement by statement:
  // same operations and FMA contractions, operands that correspond (B's own statements <-> A's, parameters by slot, global
  // loads and stash rows by a per-statement row offset), except for the nodes inside each body's trace_conn brackets (the
  // link to the parent, which differs between a first child and a sibling).  A is then emitted once as the body of a
  // two-iteration loop: iteration 0 is A, iteration 1 is B; rows become row_A + it * offset, parameters come from a
  // per-instance table, the connection nodes run in a branch on the iteration, and every value the loop hands on is
  // assigned to a variable declared before it.  Both iterations execute exactly the statements of the straight-line program.
  struct Fold {
    int a0 = 0, mid = 0, b1 = 0, instA = 0, first = 0, len = 0, pass = 0;
    std::vector<int32_t> la, lb;                                     // matched statements of A and B, in order
    std::vector<std::vector<int32_t>> ca, cb;                        // connection statements of step k
    std::vector<int> cat;                                            // matched statements before connection k (-1: none)
    std::unordered_map<int32_t, int> connk;                          // connection statement -> k
    std::unordered_map<int32_t, int32_t> b2a;
    std::unordered_set<int32_t> amatched;
    std::unordered_map<int32_t, std::array<std::string, 2>> opa;    // operand texts of A's statements
    std::unordered_map<int32_t, int> drow;                           // A statement -> row offset of its B twin
    std::map<int32_t, int> dload;                                    // A-side load -> row offset of B's
    std::vector<std::array<int32_t, 3>> pv;                          // per-instance values: A node, B node, connection k (-1: none)
    std::set<std::pair<int32_t, int32_t>> pvs;
    std::vector<int32_t> outs;                                       // nodes of A or B used after the loop
  };
  bool fold = true;
  int total_rows = 0;            // stash rows of the algorithm's layout
  const HostModel* hm = nullptr;
  std::vector<Fold> folds;
  std::vector<int32_t> fold_at, in_fold;
  std::vector<uint8_t> remat;

  static std::string pvname(int32_t x, int32_t y) { return "x" + std::to_string(x) + "_" + std::to_string(y); }

  // operand x of an A statement against operand y of its B twin
  struct Bind { int kind = 0, x = -1, y = -1, d = 0, k = -1; std::string txt; };
  bool bind(const Fold& f, int x, int y, Bind& o) const {
    const SymNode& nx = tr.nodes[x];
    const SymNode& ny = tr.nodes[y];
    o = Bind();
    if (nx.op == S_CONST || ny.op == S_CONST) { o.txt = ref(x); return x == y; }
    if (nx.op == S_PARAM || ny.op == S_PARAM) {
      o.txt = "RBD_PAR(" + std::to_string(nx.row) + ")";
      return nx.op == ny.op && nx.row == ny.row && nx.arr == f.instA && ny.arr == 1 - f.instA;
    }
    const bool xl = nx.op == S_LOAD, yl = ny.op == S_LOAD;
    if (xl && yl && nx.arr == ny.arr) {
      o.kind = 1; o.x = x; o.d = ny.row - nx.row;
      auto it = f.dload.find(x);
      o.txt = "l" + std::to_string(x);
      return it == f.dload.end() || it->second == o.d;
    }
    const bool xa = x >= f.a0 && x < f.mid, yb = y >= f.mid && y < f.b1;
    if (!xl && xa && f.amatched.count(x)) {
      auto it = f.b2a.find(y);
      o.txt = "u" + std::to_string(x);
      return yb && it != f.b2a.end() && it->second == x;
    }
    // otherwise a per-instance value: a load, a node before the pair, or a connection node, on either side
    const bool xcon = !xl && xa && f.connk.count(x), ycon = !yl && yb && f.connk.count(y);
    if (!(xl || xcon || (x < f.a0 && !fused[x]))) return false;
    if (!(yl || ycon || (y < f.a0 && !fused[y]))) return false;
    if (x == y) { o.txt = ref(x); return true; }                     // the same value outside the pair
    const int kx = xcon ? f.connk.at(x) : -1, ky = ycon ? f.connk.at(y) : -1;
    if (kx >= 0 && ky >= 0 && kx != ky) return false;
    o.kind = 2; o.x = x; o.y = y; o.k = std::max(kx, ky);
    o.txt = pvname(x, y);
    return true;
  }
  void commit(Fold& f, const Bind& b) {
    if (b.kind == 1) f.dload[b.x] = b.d;
    if (b.kind == 2 && f.pvs.insert({b.x, b.y}).second) f.pv.push_back({b.x, b.y, b.k});
  }
  // operand text inside a connection branch (side 0: A, 1: B); "" = not expressible
  std::string conn_ref(const Fold& f, int side, int x) const {
    const SymNode& n = tr.nodes[x];
    if (n.op == S_CONST) return ref(x);
    if (n.op == S_PARAM) return n.arr == (side ? 1 - f.instA : f.instA) ? "RBD_PAR(" + std::to_string(n.row) + ")" : "";
    if (n.op == S_LOAD) return std::string("RBD_LDG(") + arr_name(n.arr) + ", " + std::to_string(n.row) + ")";
    if (f.connk.count(x) && (side ? x >= f.mid : x < f.mid)) return "c" + std::to_string(x);
    if (side == 0 && f.amatched.count(x)) return "u" + std::to_string(x);
    if (side == 1) { auto it = f.b2a.find(x); if (it != f.b2a.end()) return "u" + std::to_string(it->second); }
    if (x < f.a0 && !fused[x]) return ref(x);
    return "";
  }

  bool try_fold(Fold& f, const std::vector<int>& sa, const std::vector<int>& sb, const std::map<int, std::vector<int>>& conn_of_step) {
    const auto& N = tr.nodes;
    const int L = (int)sa.size();
    f.ca.assign(L, {}); f.cb.assign(L, {}); f.cat.assign(L, -1);
    std::vector<std::array<int, 2>> ra(L, {-1, -1}), rb(L, {-1, -1});
    auto conn_range = [&](int step, std::array<int, 2>& r) {
      auto it = conn_of_step.find(step);
      if (it == conn_of_step.end()) return true;
      if (it->second.size() != 2 || !tr.conns[it->second[0]].begin || tr.conns[it->second[1]].begin) return false;
      r = {tr.conns[it->second[0]].node, tr.conns[it->second[1]].node};
      return true;
    };
    for (int k = 0; k < L; ++k) {
      if (!conn_range(sa[k], ra[k]) || !conn_range(sb[k], rb[k]) || (ra[k][0] < 0) != (rb[k][0] < 0)) return false;
      for (int i = ra[k][0]; i >= 0 && i < ra[k][1]; ++i) if (stmt_node(i)) { f.ca[k].push_back(i); f.connk[i] = k; }
      for (int i = rb[k][0]; i >= 0 && i < rb[k][1]; ++i) if (stmt_node(i)) { f.cb[k].push_back(i); f.connk[i] = k; }
    }
    for (int i = f.a0; i < f.mid; ++i) if (stmt_node(i) && !f.connk.count(i)) f.la.push_back(i);
    for (int i = f.mid; i < f.b1; ++i) if (stmt_node(i) && !f.connk.count(i)) f.lb.push_back(i);
    if (f.la.size() != f.lb.size() || f.la.empty()) return false;
    for (int k = 0; k < L; ++k) {
      if (ra[k][0] < 0) continue;
      const int na = (int)(std::lower_bound(f.la.begin(), f.la.end(), ra[k][0]) - f.la.begin());
      const int nb = (int)(std::lower_bound(f.lb.begin(), f.lb.end(), rb[k][0]) - f.lb.begin());
      if (na != nb) return false;
      f.cat[k] = na;
    }
    f.amatched.insert(f.la.begin(), f.la.end());
    // a contraction never crosses the boundary of A, B or the pair
    for (const auto& e : fma_of) {
      const int i = (int)e.first, p = e.second;
      auto seg = [&](int x) { return x < f.a0 || x >= f.b1 ? 0 : (x < f.mid ? 1 : 2); };
      if (seg(i) != seg(p) && seg(i) != 0) return false;         // (out of the pair: see the values handed on below)
    }
    for (size_t k = 0; k < f.la.size(); ++k) {
      const int a = f.la[k], b = f.lb[k];
      const SymNode& na = N[a];
      const SymNode& nb = N[b];
      f.b2a[b] = a;
      if (na.op != nb.op || fused[a] != fused[b]) return false;
      auto fa = fma_of.find(a), fb = fma_of.find(b);
      if ((fa == fma_of.end()) != (fb == fma_of.end())) return false;
      if (fa != fma_of.end()) {
        auto m = f.b2a.find(fb->second);
        if (m == f.b2a.end() || m->second != fa->second) return false;
      }
      std::array<std::string, 2>& txt = f.opa[a];
      Bind b0, b1;
      switch (na.op) {
        case S_ADD: case S_MUL: case S_SUB: case S_DIV: {
          bool ok = bind(f, na.a, nb.a, b0) && bind(f, na.b, nb.b, b1);
          if (!ok && (na.op == S_ADD || na.op == S_MUL)) ok = bind(f, na.a, nb.b, b0) && bind(f, na.b, nb.a, b1);
          if (!ok) return false;
          if (b0.kind == 1 && b1.kind == 1 && b0.x == b1.x && b0.d != b1.d) return false;
          commit(f, b0); commit(f, b1);
          txt = {b0.txt, b1.txt};
          break;
        }
        case S_NEG: case S_SIN: case S_SST: case S_STORE: case S_COS:
          if (!bind(f, na.a, nb.a, b0)) return false;
          commit(f, b0);
          txt[0] = b0.txt;
          if (na.op == S_COS) { auto m = f.b2a.find(nb.b); if (m == f.b2a.end() || m->second != na.b) return false; }
          if (na.op == S_STORE && na.arr != nb.arr) return false;
          if (na.op == S_SST && na.arr != nb.arr) return false;
          if (na.op == S_SST || na.op == S_STORE) f.drow[a] = nb.row - na.row;
          break;
        case S_SLD:
          if (na.arr != nb.arr) return false;
          f.drow[a] = nb.row - na.row;
          break;
        case S_SFENCE: break;
        default: return false;
      }
    }
    for (int k = 0; k < L; ++k) {
      for (int x : f.ca[k]) for (int o : {N[x].a, N[x].b}) if (o >= 0 && N[x].op != S_COS && conn_ref(f, 0, o).empty()) return false;
      for (int x : f.cb[k]) for (int o : {N[x].a, N[x].b}) if (o >= 0 && N[x].op != S_COS && conn_ref(f, 1, o).empty()) return false;
    }
    // values the loop hands on
    std::set<int32_t> outs;
    for (size_t i = f.b1; i < N.size(); ++i) {
      if (!live[i]) continue;
      for (int o : {N[i].a, N[i].b})
        if (o >= f.a0 && o < f.b1 && stmt_node(o)) {
          if (fused[o]) {          // a product contracted into a statement after the loop: its operands are handed on
            for (int po : {N[o].a, N[o].b}) if (po >= f.a0 && po < f.b1 && stmt_node(po)) outs.insert(po);
          } else {
            outs.insert(o);
          }
        }
    }
    f.outs.assign(outs.begin(), outs.end());
    return true;
  }

  void analyse_folds() {
    const auto& N = tr.nodes;
    fold_at.assign(N.size(), -1);
    in_fold.assign(N.size(), -1);
    remat.assign(N.size(), 0);
    if (!hm || hm->pairs.empty() || tr.steps.empty()) return;
    std::map<std::pair<int, int>, int> sidx;
    for (size_t s = 0; s < tr.steps.size(); ++s) sidx[{tr.steps[s].pass, tr.steps[s].body}] = (int)s;
    std::map<int, std::vector<int>> conn_of_step;
    for (size_t c = 0; c < tr.conns.size(); ++c) conn_of_step[tr.conns[c].step].push_back((int)c);
    for (int pass = 1; pass <= 3; ++pass)
      for (const FoldPair& fp : hm->pairs) {
        if (fp.l0 < 1) continue;
        std::vector<int> sa, sb;
        bool ok = true;
        for (int k = 0; k < fp.len && ok; ++k) {
          const int a = pass == 2 ? fp.l0 + 2 * fp.len - 1 - k : fp.l0 + k;
          const int b = pass == 2 ? fp.l0 + fp.len - 1 - k : fp.l0 + fp.len + k;
          auto ia = sidx.find({pass, a}), ib = sidx.find({pass, b});
          ok = ia != sidx.end() && ib != sidx.end();
          if (ok) { sa.push_back(ia->second); sb.push_back(ib->second); }
        }
        if (!ok || sb.back() + 1 >= (int)tr.steps.size()) continue;
        Fold f;
        f.pass = pass; f.len = fp.len; f.instA = pass == 2 ? 1 : 0;
        f.first = pass == 2 ? fp.l0 + 2 * fp.len - 1 : fp.l0;
        f.a0 = tr.steps[sa[0]].node; f.mid = tr.steps[sb[0]].node; f.b1 = tr.steps[sb.back() + 1].node;
        if (!try_fold(f, sa, sb, conn_of_step)) continue;
        fold_at[f.a0] = (int)folds.size();
        for (int i = f.a0; i < f.b1; ++i) in_fold[i] = (int)folds.size();
        folds.push_back(std::move(f));
      }
  }

  std::string outer_operand(int x) {
    const SymNode& n = tr.nodes[x];
    if (n.op == S_LOAD && in_fold[x] >= 0 && !remat[x]) {     // a load inside a loop is simply issued again
      remat[x] = 1;
      ++stats.n_load;
      out += "const rbd_v t" + std::to_string(x) + " = RBD_LDG(" + arr_name(n.arr) + ", " + std::to_string(n.row) + ");\n";
    }
    return ref(x);
  }

  // ---- register-resident stash rows ------------------------------------------------------------------------------------
  // A stash row that no statement addresses as row + rbd_it * Δ (Δ != 0) has one name in every statement that touches it, so it
  // can be an ordinary variable instead of shared memory: the trunk bodies' rows and the pending slot of a folded program, any
  // row of a straight-line one.  Up to `reg_budget` such rows (-1: all) become registers, chosen by accesses per statement of
  // live range (a value is live from its store to the last load before the next store); the other rows are renumbered
  // 0 .. shared_rows - 1 in their order.  The statements are the same either way, so the results are bit-identical.
  // The trig cache (region R_TRIG) is planned the same way on its own rows, every eligible one a register unless the budget is
  // 0; its shared rows follow the stash's in each warp's shared memory (RBD_TLD / RBD_TST).
  int reg_budget = 0;
  std::vector<int> rowmap[R_COUNT];   // row of a region -> shared-memory row of that region, -1: register
  std::vector<int> regs[R_COUNT];     // register rows, ascending
  int shared_rows = 0;                // shared rows of the stash
  int trig_rows = 0;                  // shared rows of the trig cache

  bool reg_row(int g, int r) const { return r >= 0 && r < (int)rowmap[g].size() && rowmap[g][r] == -1; }
  static std::string rname(int g, int r) { return (g == R_TRIG ? "rbd_sc" : "rbd_r") + std::to_string(r); }
  int srow(int g, int r) const { return r < (int)rowmap[g].size() ? rowmap[g][r] : r; }
  bool stash_op(int j) const { return tr.nodes[j].op == S_SLD || tr.nodes[j].op == S_SST; }
  std::string row_text(int j) const { return std::to_string(stash_op(j) ? srow(tr.nodes[j].arr, tr.nodes[j].row) : tr.nodes[j].row); }

  // returns the number of shared rows of region g
  int plan_region(int g, int total_rows, int budget) {
    const auto& N = tr.nodes;
    auto in = [&](size_t i) { return live[i] && stash_op((int)i) && N[i].arr == g; };
    std::vector<int>& map = rowmap[g];
    int nrows = total_rows;
    for (size_t i = 0; i < N.size(); ++i)
      if (in(i)) nrows = std::max(nrows, N[i].row + 1);
    map.resize(nrows);
    for (int r = 0; r < nrows; ++r) map[r] = r;
    if (g == R_STASH && budget == 0) return total_rows;
    std::vector<uint8_t> indexed(nrows, 0), touched(nrows, 0);
    for (const Fold& f : folds)
      for (const auto& e : f.drow) {
        const SymNode& n = N[e.first];
        if (e.second == 0 || !stash_op(e.first) || n.arr != g || fused[e.first]) continue;
        indexed[n.row] = indexed[n.row + e.second] = 1;
      }
    std::vector<int64_t> acc(nrows, 0), span(nrows, 0), open(nrows, -1), last(nrows, -1);
    for (size_t i = 0; i < N.size(); ++i) {
      if (!in(i)) continue;
      const int r = N[i].row;
      touched[r] = 1;
      ++acc[r];
      if (N[i].op == S_SST) {
        if (open[r] >= 0 && last[r] > open[r]) span[r] += last[r] - open[r];
        open[r] = (int64_t)i;
      } else {
        if (open[r] < 0) open[r] = (int64_t)i;
        last[r] = (int64_t)i;
      }
    }
    std::vector<int> cand;
    for (int r = 0; r < nrows; ++r) {
      if (open[r] >= 0 && last[r] > open[r]) span[r] += last[r] - open[r];
      if (touched[r] && !indexed[r]) cand.push_back(r);
    }
    std::stable_sort(cand.begin(), cand.end(), [&](int x, int y) { return acc[x] * (span[y] + 1) > acc[y] * (span[x] + 1); });
    if (budget >= 0 && (int)cand.size() > budget) cand.resize(budget);
    regs[g] = cand;
    std::sort(regs[g].begin(), regs[g].end());
    for (int r : regs[g]) map[r] = -1;
    int shared = 0;
    for (int r = 0; r < nrows; ++r)
      if (map[r] >= 0) map[r] = touched[r] ? shared++ : -2;    // -2: never accessed (no slot, never emitted)
    return shared;
  }
  void plan_rows(int total_rows) {
    shared_rows = plan_region(R_STASH, total_rows, reg_budget);
    if (reg_budget != 0) stats.reg_rows = (int)regs[R_STASH].size();
    trig_rows = plan_region(R_TRIG, 0, reg_budget == 0 ? 0 : -1);
    stats.trig_rows = trig_rows;
    stats.trig_reg_rows = (int)regs[R_TRIG].size();
  }
  std::string reg_decls() const {
    std::string s;
    for (int g = 0; g < R_COUNT; ++g)
      for (int r : regs[g]) s += "rbd_v " + rname(g, r) + " = RBD_K(" + lit(0.0) + ");\n";
    return s;
  }

  void emit_fold(const Fold& f, int& since) {
    const auto& N = tr.nodes;
    auto rowx = [](int row, int d) { return d ? "(" + std::to_string(row) + " + rbd_it * " + std::to_string(d) + ")" : std::to_string(row); };
    auto srowx = [&](int g, int row, int d) { return rowx(srow(g, row), d ? srow(g, row + d) - srow(g, row) : 0); };
    char hdr[160];
    snprintf(hdr, sizeof hdr, "// ABA pass %d: bodies %d..%d and their mirror images run one copy of the code\n", f.pass,
             std::min(f.first, f.first + (f.pass == 2 ? 1 - f.len : f.len - 1)), std::max(f.first, f.first + (f.pass == 2 ? 1 - f.len : f.len - 1)));
    out += hdr;
    for (int x : f.outs) out += "rbd_v t" + std::to_string(x) + ";\n";
    out += "#pragma unroll 1\nfor (int rbd_it = 0; rbd_it < 2; ++rbd_it) {\n";
    out += "const int rbd_s = rbd_it ^ " + std::to_string(f.instA) + "; (void)rbd_s;\n";
    for (const auto& e : f.dload) {
      const int x = e.first;
      if (x >= f.a0 && x < f.mid && !f.connk.count(x)) continue;
      ++stats.n_load;
      out += "const rbd_v l" + std::to_string(x) + " = RBD_LDG(" + arr_name(N[x].arr) + ", " + rowx(N[x].row, e.second) + ");\n";
    }
    for (const auto& p : f.pv) {
      if (p[2] >= 0) out += "rbd_v " + pvname(p[0], p[1]) + ";\n";
      else out += "const rbd_v " + pvname(p[0], p[1]) + " = rbd_it ? " + conn_ref(f, 1, p[1]) + " : " + conn_ref(f, 0, p[0]) + ";\n";
    }
    const NameFn uname = [](int j) { return "u" + std::to_string(j); };
    const NameFn cname = [](int j) { return "c" + std::to_string(j); };
    const OpFn aop = [&](int j, int k) { return f.opa.at(j)[k]; };
    const NameFn arow = [&](int j) {
      auto it = f.drow.find(j);
      const int d = it == f.drow.end() ? 0 : it->second;
      return stash_op(j) ? srowx(N[j].arr, N[j].row, d) : rowx(N[j].row, d);
    };
    const NameFn absrow = [&](int j) { return row_text(j); };
    std::set<int32_t> outset(f.outs.begin(), f.outs.end());
    auto branches = [&](size_t at) {
      for (size_t k = 0; k < f.ca.size(); ++k) {
        if (f.cat[k] != (int)at) continue;
        bool any = !f.ca[k].empty() || !f.cb[k].empty();
        for (const auto& p : f.pv) any = any || p[2] == (int)k;
        if (!any) continue;
        for (int side = 0; side < 2; ++side) {
          out += side ? "} else {\n" : "if (rbd_it == 0) {\n";
          const OpFn cop = [&, side](int j, int q) { return conn_ref(f, side, q ? N[j].b : N[j].a); };
          for (int x : side ? f.cb[k] : f.ca[k]) {
            if (!fused[x] && N[x].op != S_COS) out += stmt(x, cname, cop, absrow);
            if (outset.count(x)) out += "t" + std::to_string(x) + " = c" + std::to_string(x) + ";\n";
          }
          for (const auto& p : f.pv)
            if (p[2] == (int)k) out += pvname(p[0], p[1]) + " = " + conn_ref(f, side, p[side]) + ";\n";
        }
        out += "}\n";
      }
    };
    size_t j = 0;
    for (int i = f.a0; i < f.mid; ++i) {
      if (N[i].op == S_LOAD && f.dload.count(i) && !f.connk.count(i)) {
        ++stats.n_load;
        out += "const rbd_v l" + std::to_string(i) + " = RBD_LDG(" + arr_name(N[i].arr) + ", " + rowx(N[i].row, f.dload.at(i)) + ");\n";
        continue;
      }
      if (j < f.la.size() && f.la[j] == i) {
        branches(j);
        ++j;
        if (fused[i] || N[i].op == S_COS) continue;
        out += split_point(i, since);
        out += stmt(i, uname, aop, arow);
      }
    }
    branches(f.la.size());
    std::string oa, ob;
    for (int x : f.outs) {
      if (f.connk.count(x)) continue;
      if (x < f.mid) oa += "t" + std::to_string(x) + " = u" + std::to_string(x) + ";\n";
      else ob += "t" + std::to_string(x) + " = u" + std::to_string(f.b2a.at(x)) + ";\n";
    }
    if (!oa.empty() || !ob.empty()) out += "if (rbd_it == 0) {\n" + oa + "} else {\n" + ob + "}\n";
    out += "}\n";
    ++stats.n_fold_loops;
    stats.n_fold_bodies += f.len;
  }

  void plan() {
    mark();
    plan_fma();
    if (fold) analyse_folds();
    if (!folds.empty()) split_every = split_folded;
    if (!fold) { fold_at.assign(tr.nodes.size(), -1); in_fold.assign(tr.nodes.size(), -1); remat.assign(tr.nodes.size(), 0); }
    plan_rows(total_rows);
  }

  void emit() {      // after plan()
    const auto& N = tr.nodes;
    stats.nodes_traced = (int)N.size();
    for (size_t i = 0; i < N.size(); ++i) if (live[i] && N[i].op != S_CONST && N[i].op != S_PARAM) ++stats.nodes_live;
    const NameFn tname = [](int j) { return "t" + std::to_string(j); };
    const OpFn top = [&](int j, int k) { return outer_operand(k ? N[j].b : N[j].a); };
    const NameFn trow = [&](int j) { return row_text(j); };
    int since = 0;
    for (size_t i = 0; i < N.size(); ++i) {
      if (fold_at[i] >= 0) {
        const Fold& f = folds[fold_at[i]];
        emit_fold(f, since);
        i = f.b1 - 1;
        continue;
      }
      if (!live[i]) continue;
      const SymNode& n = N[i];
      if (fused[i] || n.op == S_CONST || n.op == S_PARAM || n.op == S_COS) continue;
      if (n.op == S_LOAD && in_fold[i] >= 0) continue;
      out += split_point((int)i, since);
      if (n.op == S_LOAD) remat[i] = 1;
      out += stmt((int)i, tname, top, trow);
    }
  }

  // per-instance parameter table of the folded loops
  std::string param_table() const {
    if (folds.empty() || tr.npar == 0) return "";
    std::vector<double> tab[2];
    tab[0].assign(tr.npar, 0.0); tab[1].assign(tr.npar, 0.0);
    for (const SymNode& n : tr.nodes) if (n.op == S_PARAM) tab[n.arr][n.row] = n.c;
    std::string s = flavor == FLAVOR_CPU ? "static const rbd_v" : "__constant__ rbd_f";
    s += " rbd_par_tab[2][" + std::to_string(tr.npar) + "] = {";
    for (int k = 0; k < 2; ++k) {
      s += k ? "}, {" : "{";
      for (int j = 0; j < tr.npar; ++j) s += (j ? ", " : "") + lit(tab[k][j]);
    }
    s += "}};\n#undef RBD_PAR\n#define RBD_PAR(k_) rbd_par_tab[rbd_s][k_]\n";
    return s;
  }
};

}  // namespace

namespace {

// Shared-memory rows of a planned program's stash (RBD_SPEC_ROWS): the compacted rows when some are registers, else the
// algorithm's layout.
int smem_stash_rows(const HostModel& hm, const SpecKey& key, const Emitter& em) {
  return em.stats.reg_rows ? em.shared_rows : spec_stash_rows(hm, key);
}

// Traces `key` and plans its program (`em`, over `tr`).  The trig cache (spec_trig) is kept only if its shared rows cost no
// resident single-warp blocks; otherwise the program is traced again without it (the cache only saves recomputation).
bool plan_program(const HostModel& hm, const SpecKey& key, int flavor, bool fold, SymTrace& tr, std::unique_ptr<Emitter>& em,
                  std::string& err) {
  for (bool trig = spec_trig(key);; trig = false) {
    em.reset();
    tr = SymTrace();
    int rows = 0;
    if (!run_trace(hm, key, trig, tr, rows, err)) return false;
    em.reset(new Emitter(tr, key, flavor));
    em->hm = &hm;
    em->fold = fold;
    em->total_rows = rows;
    em->reg_budget = spec_reg_rows(key);
    if (flavor != FLAVOR_CPU) {
      // One basic block of 10^4 instructions lets ptxas stretch live ranges until it spills (Atlas: 128 registers + 350 B of
      // local memory, -10 % throughput); a never-taken branch every few hundred statements bounds its scheduling regions.
      // A folded program's loops already end basic blocks every few hundred statements, and there the extra branches only cost
      // (Atlas fp32 forward dynamics on H100 at 400 W: 800 M evals/s with a branch every 192 statements, 856 M without).
      em->split_every = 192;
      em->split_folded = 0;
      if (const char* e = getenv("RBD_JIT_SPLIT")) em->split_every = em->split_folded = atoi(e);
    }
    em->plan();
    const int stash = smem_stash_rows(hm, key, *em);
    if (!trig || spec_smem_blocks(key, stash + em->trig_rows) >= spec_smem_blocks(key, stash)) return true;
  }
}

}  // namespace

bool spec_emit_function(const HostModel& hm, const SpecKey& key, int flavor, const std::string& name, std::string& out,
                        SpecStats* stats, std::string& err, bool fold) {
  SymTrace tr;
  std::unique_ptr<Emitter> pem;
  if (!plan_program(hm, key, flavor, fold, tr, pem, err)) return false;
  Emitter& em = *pem;
  em.emit();
  em.stats.stash_rows = em.total_rows;
  em.stats.shared_rows = em.shared_rows;
  if (stats) *stats = em.stats;
  out += em.param_table();
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
  if (flavor == FLAVOR_CPU && em.trig_rows) out += "rbd_v rbd_trig[" + std::to_string(em.trig_rows) + "];\n";
  out += em.reg_decls();
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

int spec_reg_rows(const SpecKey& key) {
  if (key.algo != SPEC_ABA || key.f64) return 0;
  if (const char* e = getenv("RBD_JIT_REG_ROWS")) return atoi(e);
  return kRegRowsAba;
}

int spec_smem_blocks(const SpecKey& key, int shared_rows) {
  if (const char* e = getenv("RBD_JIT_SMEM_BLOCKS")) return std::max(1, std::min(32, atoi(e)));
  const int bytes = std::max(1, shared_rows) * 32 * (key.f64 ? 8 : 4);
  // A program with register rows is compiled for at most 8 blocks, two warps per SM sub-partition and up to 255 registers each:
  // Atlas fp32 forward dynamics runs 6 % faster that way than at the 11 blocks its 156 shared rows allow (168 registers, 128 B
  // of spills; DESIGN.md section 7).
  return std::max(1, std::min(spec_reg_rows(key) != 0 ? 8 : 16, kSmemPerSm / (bytes + kSmemReservedPerBlock)));
}

bool spec_trig(const SpecKey& key) {
  if (key.algo != SPEC_ABA || key.f64) return false;
  const char* e = getenv("RBD_JIT_TRIG");
  return !e || e[0] != '0';
}

int spec_shared_rows(const HostModel& hm, const SpecKey& key) {
  if (spec_reg_rows(key) == 0 && !spec_trig(key)) return spec_stash_rows(hm, key);
  SymTrace tr;
  std::unique_ptr<Emitter> em;
  std::string err;
  if (!plan_program(hm, key, FLAVOR_SMEM, true, tr, em, err)) return spec_stash_rows(hm, key);
  return smem_stash_rows(hm, key, *em) + em->trig_rows;
}

uint64_t spec_hash(const HostModel& hm, const SpecKey& key) {
  uint64_t h = 0xcbf29ce484222325ull;
  auto mix = [&](const void* p, size_t n) {
    const unsigned char* b = (const unsigned char*)p;
    for (size_t i = 0; i < n; ++i) { h ^= b[i]; h *= 0x100000001b3ull; }
  };
  const char* blocks = getenv("RBD_JIT_SMEM_BLOCKS");
  const int hdr[12] = {kGeneratorVersion, key.algo, key.f64, key.has_in2, key.has_out1, key.lower, hm.nb, hm.general, key.peers,
                       spec_reg_rows(key), blocks ? atoi(blocks) : 0, spec_trig(key)};
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
  char buf[1024];
  const int rows = st.reg_rows ? st.shared_rows : spec_stash_rows(hm, key);     // shared-memory rows of the stash (smem_stash_rows)
  snprintf(buf, sizeof buf,
           "// generated by librbd_b200.so (rbd_codegen.cpp) for one mechanism: %d live nodes (%d add/sub, %d mul, %d div, %d sincos, "
           "%d global loads, %d stash loads, %d stash stores; %d stash rows in registers; trig cache: %d rows in shared memory, "
           "%d in registers)\n"
           "#define RBD_SPEC_SMEM_BLOCKS %d\n"
           "#define RBD_SPEC_F64 %d\n#define RBD_SPEC_NQ %d\n#define RBD_SPEC_NV %d\n#define RBD_SPEC_ROWS %d\n#define RBD_SPEC_TRIG_ROWS %d\n"
           "#define RBD_SPEC_HAS_IN2 %d\n#define RBD_SPEC_HAS_OUT1 %d\n#define RBD_SPEC_OUT0_ROWS %d\n#define RBD_SPEC_OUT1_ROWS %d\n"
           "#define RBD_SPEC_ROW32 %d\n#define RBD_SPEC_KIN %d\n#define RBD_SPEC_USES_V %d\n#include \"rbd_jit_prelude.cuh\"\n",
           st.nodes_live, st.n_add, st.n_mul, st.n_div, st.n_sincos, st.n_load, st.n_sld, st.n_sst, st.reg_rows, st.trig_rows,
           st.trig_reg_rows, spec_smem_blocks(key, rows + st.trig_rows), key.f64 ? 1 : 0, hm.nq, hm.nv, rows, st.trig_rows, key.has_in2 ? 1 : 0, key.has_out1 ? 1 : 0, key.algo == SPEC_CRBA ? hm.nv * hm.nv : hm.nv, hm.nq,
           key.algo == SPEC_CRBA ? 1 : 0, key.algo == SPEC_KIN ? 1 : 0, st.n_load_v > 0 ? 1 : 0);
  out += buf;
  out += "#define RBD_FLAVOR_SMEM 1\n#include \"rbd_jit_flavor.cuh\"\n" + fn_smem;
  out += "#include \"rbd_jit_kernels.cuh\"\n";
  return true;
}

bool spec_emit_cpu_tu(const HostModel& hm, const SpecKey& key, const std::string& name, std::string& out, SpecStats* stats,
                      std::string& err, bool fold) {
  out += "// generated by librbd_b200.so (rbd_codegen.cpp): model-specialised program, CPU flavour (test tier)\n"
         "#include \"rbd_device.cuh\"\n"
         "#define RBD_LDG(p, r) p[(long long)(r) * ld]\n#define RBD_STG(p, r, x) p[(long long)(r) * ld] = (x)\n"
         "#define RBD_SLD(r) sh[r]\n#define RBD_SST(r, x) sh[r] = (x)\n#define RBD_SFENCE()\n"
         "#define RBD_TLD(r) rbd_trig[r]\n#define RBD_TST(r, x) rbd_trig[r] = (x)\n"
         "#define RBD_RCP(x) (1 / (x))\n#define RBD_DIV(a, b) ((a) / (b))\n#define RBD_SINCOS(x, s, c) rbd::sincos_t(x, s, c)\n"
         "#define RBD_K(x) (x)\n#define RBD_ADD(a, b) ((a) + (b))\n#define RBD_SUB(a, b) ((a) - (b))\n#define RBD_MUL(a, b) ((a) * (b))\n"
         "#define RBD_KIN_BEGIN_CPU rbd_v *ko0 = ko[0], *ko1 = ko[1], *ko2 = ko[2], *ko3 = ko[3], *ko4 = ko[4], *ko5 = ko[5], *ko6 = ko[6], *ko7 = ko[7]; (void)ko0; (void)ko1; (void)ko2; (void)ko3; (void)ko4; (void)ko5; (void)ko6; (void)ko7;\n"
         "#define RBD_NEG(a) (-(a))\n#define RBD_FMA(a, b, c) std::fma(a, b, c)\n#define RBD_FMS(a, b, c) std::fma(a, b, -(c))\n"
         "#define RBD_FNMA(a, b, c) std::fma(-(a), b, c)\n";
  out += std::string("typedef ") + (key.f64 ? "double" : "float") + " rbd_v;\n";
  return spec_emit_function(hm, key, FLAVOR_CPU, name, out, stats, err, fold);
}

}  // namespace rbd
