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
#include <string>
#include <unordered_map>
#include <vector>

#include "rbd_device.cuh"

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
  int32_t pure(int32_t op, int32_t a, int32_t b) {
    const uint64_t h = ((uint64_t)(uint32_t)op << 58) ^ ((uint64_t)(uint32_t)a * 0xD6E8FEB86659FD93ull) ^ ((uint64_t)(uint32_t)(b + 7) * 0xA24BAED4963EE407ull);
    for (int32_t id : cse[h]) if (nodes[id].op == op && nodes[id].a == a && nodes[id].b == b) return id;
    const int32_t id = push({op, a, b, 0, 0, 0, 0.0});
    cse[h].push_back(id);
    return id;
  }
  int32_t neg(int32_t a) {
    if (is_const(a)) return constant(-cval(a));
    if (nodes[a].op == S_NEG) return nodes[a].a;
    if (nodes[a].op == S_SUB) return sub(nodes[a].b, nodes[a].a);
    return pure(S_NEG, a, -1);
  }
  int32_t add(int32_t a, int32_t b) {
    if (is_const(a) && is_const(b)) return constant(cval(a) + cval(b));
    if (is_const(a, 0.0)) return b;
    if (is_const(b, 0.0)) return a;
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
    if (is_const(b)) return mul(a, constant(1.0 / cval(b)));   // only exact for powers of two; used for T(0.5)-style scalings
    return pure(S_DIV, a, b);
  }
  void sincos(int32_t a, int32_t& s, int32_t& c) {
    if (is_const(a)) { s = constant(std::sin(cval(a))); c = constant(std::cos(cval(a))); return; }
    const uint64_t h = ((uint64_t)S_SIN << 58) ^ ((uint64_t)(uint32_t)a * 0xD6E8FEB86659FD93ull);
    for (int32_t id : cse[h]) if (nodes[id].op == S_SIN && nodes[id].a == a) { s = id; c = id + 1; return; }
    s = push({S_SIN, a, -1, 0, 0, 0, 0.0});
    c = push({S_COS, a, s, 0, 0, 0, 0.0});
    cse[h].push_back(s);
  }
  int32_t load(int32_t arr, int32_t row) {
    const uint64_t key = ((uint64_t)(uint32_t)arr << 32) | (uint32_t)row;
    auto it = last_load.find(key);
    if (it != last_load.end() && (int32_t)nodes.size() - it->second <= load_window) return it->second;
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

// Model constants as literals of the trace.
template <class F> inline void sym_model(const ModelDev<F>& S, ModelDev<Sym>& D) {
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
}

}  // namespace rbd
