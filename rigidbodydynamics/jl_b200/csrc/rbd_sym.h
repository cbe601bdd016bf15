// Expression tracer for model-specialised kernels (host-only C++).
//
// The per-sample algorithms of rbd_device.cuh / rbd_rnea_crba.cuh are templates on the scalar type T.  Instantiated on
// the HOST with T = Sym they do not compute numbers: every arithmetic operator appends a node to a straight-line program
// (the "trace") and returns its index.  Because the flattened mechanism is concrete while tracing, every branch on joint
// kinds / flags / tree structure is resolved, every model constant (tree transforms, inertias, class angles) is a literal,
// and the usual algebraic identities (x*0, x*1, x+0, constant folding, common sub-expressions) are applied as nodes are
// created -- structural zeros of the spatial inertias and tree offsets vanish from the program.  rbd_codegen.cpp turns the
// trace into CUDA source that rbd_jit.cpp compiles with NVRTC at rbd_model_create time: the model-specialised kernel the
// generic (runtime tree walk) kernels fall back from.  The same trace emitted as plain C++ is what the CPU test tier checks
// against the oracle.
//
// What is traced is THE SAME code the generic kernels run, so parity of the specialised kernel follows from parity of the
// templates; nothing about the algorithms is restated here.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#include <map>
#include <set>
#include <string>
#include <tuple>
#include <unordered_map>
#include <vector>

#include "rbd_device.cuh"
#include "rbd_model.h"

namespace rbd {

enum SymOp : int32_t {
  S_CONST = 0,
  S_ADD, S_SUB, S_MUL, S_DIV, S_NEG,
  S_SIN, S_COS,          // the two results of one sincos_t(a): always created as a pair (cos node id = sin node id + 1)
  S_LOAD,                // global input:  arr = which array, row
  S_STORE,               // global output: arr, row, a = value
  S_SLD,                 // stash load:  row; grp = id of the first load of its ldv<N> batch
  S_SST,                 // stash store: row, a = value
  S_SFENCE,              // stash store fence: where a thread re-reads its own stash writes (a no-op in shared memory)
  S_XLD, S_XST,          // per-thread global scratch (body-frame external wrenches): row[, a]
  S_PARAM,               // model constant of one instance of a folded chain pair: row = slot, arr = instance (0 left, 1 right), c = value
};

// arrays a traced algorithm may touch (the code generator maps them to kernel arguments)
enum SymArr : int32_t { A_Q = 0, A_V, A_TAU, A_VD_IN, A_WEXT, A_OUT0, A_OUT1,
                        A_K0, A_K1, A_K2, A_K3, A_K4, A_K5, A_K6, A_K7,      // the eight outputs of rbd_kinematics, in rbd_kinematics_out order
                        A_COUNT };

struct SymNode {
  int32_t op;
  int32_t a, b;
  int32_t arr, row, grp;
  double c;
};

struct SymTrace {
  std::vector<SymNode> nodes;
  std::unordered_map<uint64_t, std::vector<int32_t>> cse;   // hash of (op, a, b / constant bits) -> candidates
  std::unordered_map<uint64_t, int32_t> last_load;          // (arr, row) -> most recent load node
  bool single = true;                                        // fold constants in fp32 (kernels for float) or fp64
  int load_window = 400;                                     // a repeated load this close to the previous one re-uses it
  // trace_step / trace_conn marks (rbd_device.cuh): node index where each ABA body step begins, and the connection brackets
  struct Step { int32_t pass, body, node; };
  struct Conn { int32_t node, step; bool begin; };
  std::vector<Step> steps;
  std::vector<Conn> conns;
  // steps (pass, body) that begin the walk of a folded chain: loads issued before one are not re-used after it, so that both
  // chains of a pair start from their own loads (and re-use nothing computed before them)
  std::set<std::pair<int32_t, int32_t>> fresh_steps;
  int32_t load_floor = 0;
  // Parameter leaves (S_PARAM).  A model constant that differs between the two instances of a folded pair is not a literal but
  // an opaque leaf: never folded into or sign-normalised like a constant, one node per instance (so the two instances' code
  // stays apart), one slot shared by both.  An expression of parameters and constants only is folded like a constant
  // expression, per instance, into a derived parameter; its slot is keyed by the operation and the operand slots / constants,
  // so mirror-image instances get the same slot.
  int npar = 0;
  std::map<std::tuple<int32_t, int64_t, uint64_t, int64_t, uint64_t>, int32_t> dslot;
  std::map<std::pair<int32_t, int32_t>, int32_t> dnode;      // (slot, instance) -> derived parameter node

  int32_t push(const SymNode& n) { nodes.push_back(n); return (int32_t)nodes.size() - 1; }
  double rnd(double x) const { return single ? (double)(float)x : x; }
  bool is_const(int32_t id) const { return nodes[id].op == S_CONST; }
  bool is_const(int32_t id, double v) const { return nodes[id].op == S_CONST && nodes[id].c == v; }
  double cval(int32_t id) const { return nodes[id].c; }

  int32_t constant(double v) {
    v = rnd(v);
    if (v == 0.0) v = 0.0;     // -0 -> +0
    uint64_t bits;
    std::memcpy(&bits, &v, 8);
    const uint64_t h = bits * 0x9E3779B97F4A7C15ull + 1;
    for (int32_t id : cse[h]) if (nodes[id].op == S_CONST && nodes[id].c == v) return id;
    const int32_t id = push({S_CONST, -1, -1, 0, 0, 0, v});
    cse[h].push_back(id);
    return id;
  }
  int32_t param(int32_t slot, int32_t inst, double v) { return push({S_PARAM, -1, -1, inst, slot, 0, rnd(v)}); }
  bool is_par(int32_t id) const { return nodes[id].op == S_PARAM; }
  bool is_lit(int32_t id) const { return is_const(id) || is_par(id); }
  // both operands constants or parameters, at least one a parameter, not of different instances
  bool par_fold(int32_t a, int32_t b) const {
    if (!is_lit(a) || (b >= 0 && !is_lit(b))) return false;
    if (!is_par(a) && !(b >= 0 && is_par(b))) return false;
    return !(b >= 0 && is_par(a) && is_par(b) && nodes[a].arr != nodes[b].arr);
  }
  int32_t derive(int32_t op, int32_t a, int32_t b, double v) {
    v = rnd(v);
    if (v == 0.0) v = 0.0;
    auto key = [&](int32_t x, int64_t& kind, uint64_t& bits) {
      kind = x < 0 ? -1 : (is_par(x) ? nodes[x].row : -2);
      bits = 0;
      if (x >= 0 && !is_par(x)) std::memcpy(&bits, &nodes[x].c, 8);
    };
    int64_t ka, kb; uint64_t va, vb;
    key(a, ka, va); key(b, kb, vb);
    if ((op == S_ADD || op == S_MUL) && std::make_pair(ka, va) > std::make_pair(kb, vb)) { std::swap(ka, kb); std::swap(va, vb); }
    auto it = dslot.emplace(std::make_tuple(op, ka, va, kb, vb), npar);
    if (it.second) ++npar;
    const int32_t slot = it.first->second;
    const int32_t inst = is_par(a) ? nodes[a].arr : nodes[b].arr;
    auto nd = dnode.find({slot, inst});
    if (nd != dnode.end()) return nd->second;
    const int32_t id = push({S_PARAM, -1, -1, inst, slot, 0, v});
    dnode[{slot, inst}] = id;
    return id;
  }
  int32_t pure(int32_t op, int32_t a, int32_t b) {
    const uint64_t h = ((uint64_t)(uint32_t)op << 58) ^ ((uint64_t)(uint32_t)a * 0xD6E8FEB86659FD93ull) ^ ((uint64_t)(uint32_t)(b + 7) * 0xA24BAED4963EE407ull);
    for (int32_t id : cse[h]) if (nodes[id].op == op && nodes[id].a == a && nodes[id].b == b) return id;
    const int32_t id = push({op, a, b, 0, 0, 0, 0.0});
    cse[h].push_back(id);
    return id;
  }
  int32_t neg(int32_t a) {
    if (is_const(a)) return constant(-cval(a));
    if (is_par(a)) return derive(S_NEG, a, -1, -cval(a));
    if (nodes[a].op == S_NEG) return nodes[a].a;
    if (nodes[a].op == S_SUB) return sub(nodes[a].b, nodes[a].a);
    return pure(S_NEG, a, -1);
  }
  int32_t add(int32_t a, int32_t b) {
    if (is_const(a) && is_const(b)) return constant(cval(a) + cval(b));
    if (is_const(a, 0.0)) return b;
    if (is_const(b, 0.0)) return a;
    if (par_fold(a, b)) return derive(S_ADD, a, b, cval(a) + cval(b));
    if (nodes[b].op == S_NEG) return sub(a, nodes[b].a);
    if (nodes[a].op == S_NEG) return sub(b, nodes[a].a);
    if (a > b) std::swap(a, b);
    return pure(S_ADD, a, b);
  }
  int32_t sub(int32_t a, int32_t b) {
    if (is_const(a) && is_const(b)) return constant(cval(a) - cval(b));
    if (a == b) return constant(0.0);
    if (is_const(b, 0.0)) return a;
    if (is_const(a, 0.0)) return neg(b);
    if (par_fold(a, b)) return derive(S_SUB, a, b, cval(a) - cval(b));
    if (nodes[b].op == S_NEG) return add(a, nodes[b].a);
    return pure(S_SUB, a, b);
  }
  int32_t mul(int32_t a, int32_t b) {
    if (is_const(a) && is_const(b)) return constant(cval(a) * cval(b));
    if (is_const(a, 0.0) || is_const(b, 0.0)) return constant(0.0);
    if (is_const(a, 1.0)) return b;
    if (is_const(b, 1.0)) return a;
    if (is_const(a, -1.0)) return neg(b);
    if (is_const(b, -1.0)) return neg(a);
    if (par_fold(a, b)) return derive(S_MUL, a, b, cval(a) * cval(b));
    // keep signs out of products so that x*y and (-x)*y share one node (negation is a free operand modifier on the GPU)
    bool negate = false;
    if (nodes[a].op == S_NEG) { a = nodes[a].a; negate = !negate; }
    if (nodes[b].op == S_NEG) { b = nodes[b].a; negate = !negate; }
    if (is_const(a) && cval(a) < 0) { a = constant(-cval(a)); negate = !negate; }
    if (is_const(b) && cval(b) < 0) { b = constant(-cval(b)); negate = !negate; }
    if (is_const(a, 1.0)) return negate ? neg(b) : b;
    if (is_const(b, 1.0)) return negate ? neg(a) : a;
    if (a > b) std::swap(a, b);
    const int32_t p = pure(S_MUL, a, b);
    return negate ? neg(p) : p;
  }
  int32_t div(int32_t a, int32_t b) {
    if (is_const(a) && is_const(b)) return constant(cval(a) / cval(b));
    if (is_const(a, 0.0)) return constant(0.0);
    if (is_const(b, 1.0)) return a;
    if (par_fold(a, b)) return derive(S_DIV, a, b, cval(a) / cval(b));
    if (is_const(b)) return mul(a, constant(1.0 / cval(b)));   // only exact for powers of two; used for T(0.5)-style scalings
    if (is_par(b)) return mul(a, derive(S_DIV, constant(1.0), b, 1.0 / cval(b)));   // the same, with the reciprocal a parameter
    return pure(S_DIV, a, b);
  }
  void sincos(int32_t a, int32_t& s, int32_t& c) {
    if (is_const(a)) { s = constant(std::sin(cval(a))); c = constant(std::cos(cval(a))); return; }
    if (is_par(a)) { s = derive(S_SIN, a, -1, std::sin(cval(a))); c = derive(S_COS, a, -1, std::cos(cval(a))); return; }
    const uint64_t h = ((uint64_t)S_SIN << 58) ^ ((uint64_t)(uint32_t)a * 0xD6E8FEB86659FD93ull);
    for (int32_t id : cse[h]) if (nodes[id].op == S_SIN && nodes[id].a == a) { s = id; c = id + 1; return; }
    s = push({S_SIN, a, -1, 0, 0, 0, 0.0});
    c = push({S_COS, a, s, 0, 0, 0, 0.0});
    cse[h].push_back(s);
  }
  int32_t load(int32_t arr, int32_t row) {
    const uint64_t key = ((uint64_t)(uint32_t)arr << 32) | (uint32_t)row;
    auto it = last_load.find(key);
    if (it != last_load.end() && (int32_t)nodes.size() - it->second <= load_window && it->second >= load_floor) return it->second;
    const int32_t id = push({S_LOAD, -1, -1, arr, row, 0, 0.0});
    last_load[key] = id;
    return id;
  }
  void store(int32_t arr, int32_t row, int32_t v) { push({S_STORE, v, -1, arr, row, 0, 0.0}); }
  int32_t sld(int32_t row, int32_t grp) { const int32_t id = push({S_SLD, -1, -1, 0, row, grp, 0.0}); return id; }
  void sst(int32_t row, int32_t v) { push({S_SST, v, -1, 0, row, 0, 0.0}); }
  void sfence() { if (!nodes.empty() && nodes.back().op == S_SFENCE) return; push({S_SFENCE, -1, -1, 0, 0, 0, 0.0}); }
  int32_t xld(int32_t row) { return push({S_XLD, -1, -1, 0, row, 0, 0.0}); }
  void xst(int32_t row, int32_t v) { push({S_XST, v, -1, 0, row, 0, 0.0}); }
};

inline SymTrace*& sym_trace() { static thread_local SymTrace* t = nullptr; return t; }

// The traced scalar.  Default-constructed = "uninitialised" (id -1), like an uninitialised float.
struct Sym {
  int32_t id;
  Sym() : id(-1) {}
  Sym(double v) : id(sym_trace()->constant(v)) {}
  Sym(float v) : id(sym_trace()->constant((double)v)) {}
  Sym(int v) : id(sym_trace()->constant((double)v)) {}
  struct Raw {};
  Sym(Raw, int32_t i) : id(i) {}
};
inline Sym mk(int32_t id) { return Sym(Sym::Raw{}, id); }

template <> inline void trace_step<Sym>(int pass, int i) {
  SymTrace* t = sym_trace();
  t->steps.push_back({pass, i, (int32_t)t->nodes.size()});
  if (t->fresh_steps.count({pass, i})) t->load_floor = (int32_t)t->nodes.size();
}
template <> inline void trace_conn<Sym>(bool begin) {
  SymTrace* t = sym_trace();
  t->conns.push_back({(int32_t)t->nodes.size(), (int32_t)t->steps.size() - 1, begin});
}
inline Sym operator+(const Sym& a, const Sym& b) { return mk(sym_trace()->add(a.id, b.id)); }
inline Sym operator-(const Sym& a, const Sym& b) { return mk(sym_trace()->sub(a.id, b.id)); }
inline Sym operator*(const Sym& a, const Sym& b) { return mk(sym_trace()->mul(a.id, b.id)); }
inline Sym operator/(const Sym& a, const Sym& b) { return mk(sym_trace()->div(a.id, b.id)); }
inline Sym operator-(const Sym& a) { return mk(sym_trace()->neg(a.id)); }
inline Sym& operator+=(Sym& a, const Sym& b) { a = a + b; return a; }
inline Sym& operator-=(Sym& a, const Sym& b) { a = a - b; return a; }
inline Sym& operator*=(Sym& a, const Sym& b) { a = a * b; return a; }
inline void sincos_t(const Sym& x, Sym& s, Sym& c) {
  int32_t si, ci;
  sym_trace()->sincos(x.id, si, ci);
  s = mk(si); c = mk(ci);
}

// ---- views: the same interfaces the device code uses, recording instead of touching memory --------------------------
template <> struct Col<Sym> {
  int32_t arr;
  bool present;
  Sym operator()(int row) const { return mk(sym_trace()->load(arr, row)); }
  bool valid() const { return present; }
};
template <> struct ColRW<Sym> {
  int32_t arr;
  bool present;
  Sym operator()(int row) const { return mk(sym_trace()->load(arr, row)); }
  bool valid() const { return present; }
};
template <> struct ColOut<Sym> {
  int32_t arr;
  bool present;
  void st(int row, const Sym& v) const { if (present) sym_trace()->store(arr, row, v.id); }
  bool valid() const { return present; }
};
// Per-thread scratch.  With `fwd` the rows are not memory at all: a value written in one sweep is simply the SAME traced value when
// it is read back in the next (the compiler keeps it in a register or spills it to local memory, which is per-thread and
// coalesced like the generic kernels' scratch column).
template <> struct Scr<Sym> {
  bool present;
  std::vector<int32_t>* fwd = nullptr;
  Sym get(int row) const { return fwd ? mk((*fwd)[row]) : mk(sym_trace()->xld(row)); }
  void st(int row, const Sym& v) const {
    if (fwd) { if ((int)fwd->size() <= row) fwd->resize(row + 1, -1); (*fwd)[row] = v.id; }
    else sym_trace()->xst(row, v.id);
  }
  bool valid() const { return present; }
};
struct SymStash {
  Sym ld(int row) const {
    SymTrace* t = sym_trace();
    const int32_t id = (int32_t)t->nodes.size();
    return mk(t->sld(row, id));
  }
  void st(int row, const Sym& v) const { sym_trace()->sst(row, v.id); }
  void add(int row, const Sym& v) const { fence_st(); st(row, ld(row) + v); }
  template <int N> void ldv(int row, Sym* out) const {
    SymTrace* t = sym_trace();
    const int32_t first = (int32_t)t->nodes.size();
    for (int k = 0; k < N; ++k) out[k] = mk(t->sld(row + k, first));
  }
  void fence_st() const { sym_trace()->sfence(); }
  const SymStash& slots() const { return *this; }
};

// Model constants as literals of the trace; with `pairs`, the constants that differ between the two chains of a pair are
// parameter leaves instead (see SymTrace::param).
template <class F> inline void sym_model(const ModelDev<F>& S, ModelDev<Sym>& D, const std::vector<FoldPair>* pairs = nullptr) {
  D.nb = S.nb; D.nq = S.nq; D.nv = S.nv; D.nrows = S.nrows; D.slot_base = S.slot_base; D.nslots = S.nslots;
  for (int k = 0; k < 3; ++k) D.g[k] = Sym((double)S.g[k]);
  D.pad_ = Sym(0.0);
  for (int i = 0; i < S.nb; ++i) {
    const BodyDev<F>& s = S.body[i];
    BodyDev<Sym>& d = D.body[i];
    for (int k = 0; k < 9; ++k) d.Rt[k] = Sym((double)s.Rt[k]);
    for (int k = 0; k < 3; ++k) { d.pt[k] = Sym((double)s.pt[k]); d.h[k] = Sym((double)s.h[k]); }
    for (int k = 0; k < 6; ++k) d.J[k] = Sym((double)s.J[k]);
    d.m = Sym((double)s.m);
    d.qoff = Sym((double)s.qoff);
    d.kind = s.kind; d.parent = s.parent; d.qrow = s.qrow; d.vrow = s.vrow; d.row0 = s.row0;
    d.oslot = s.oslot; d.pslot = s.pslot; d.flags = s.flags; d.refidx = s.refidx;
  }
  if (!pairs) return;
  SymTrace* t = sym_trace();
  for (const FoldPair& fp : *pairs)
    for (int k = 0; k < fp.len; ++k) {
      const BodyDev<F>& sl = S.body[fp.l0 + k];
      const BodyDev<F>& sr = S.body[fp.l0 + fp.len + k];
      BodyDev<Sym>& dl = D.body[fp.l0 + k];
      BodyDev<Sym>& dr = D.body[fp.l0 + fp.len + k];
      auto split = [&](F a, F b, Sym& da, Sym& db) {
        if (a == b) return;
        const int32_t slot = t->npar++;
        da = mk(t->param(slot, 0, (double)a));
        db = mk(t->param(slot, 1, (double)b));
      };
      for (int j = 0; j < 9; ++j) split(sl.Rt[j], sr.Rt[j], dl.Rt[j], dr.Rt[j]);
      for (int j = 0; j < 3; ++j) { split(sl.pt[j], sr.pt[j], dl.pt[j], dr.pt[j]); split(sl.h[j], sr.h[j], dl.h[j], dr.h[j]); }
      for (int j = 0; j < 6; ++j) split(sl.J[j], sr.J[j], dl.J[j], dr.J[j]);
      split(sl.m, sr.m, dl.m, dr.m);
      split(sl.qoff, sr.qoff, dl.qoff, dr.qoff);
    }
}

}  // namespace rbd
