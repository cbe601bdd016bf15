// Forward-mode dual numbers for config 4 of BASELINE.json: `dynamics!` on `ForwardDiff.Dual{Tag,Float64,6}` inputs
// (the reference reaches its generic-scalar path through StateCache, examples/5; src/caches.jl:46-64).
//
// Memory layout at the boundary = Julia's: a `Dual{Tag,Float64,6}` is an isbits struct of 7 contiguous Float64
// (value, 6 partials), so a Matrix{Dual}(B, n) is [n][B][7] doubles: element (row k, sample b) starts at ((k*ld + b) * 7).
//
// Mapping: one THREAD per (sample, partial direction).  Partial directions are independent of each other given the value,
// so thread (b, d) carries Dual1 = (value, d-th partial) through the very same templated ABA code; the 6 threads of a sample
// sit in adjacent lanes, their value loads coalesce into one request and their partial loads are contiguous.
#pragma once
#include <type_traits>

#include "rbd_device.cuh"

namespace rbd {

template <class F> struct Dual1 {
  F v, d;
  RBD_HD Dual1() : v(0), d(0) {}
  RBD_HD Dual1(F a) : v(a), d(0) {}
  RBD_HD Dual1(F a, F b) : v(a), d(b) {}
  template <class U> RBD_HD explicit Dual1(const Dual1<U>& o) : v((F)o.v), d((F)o.d) {}
  RBD_HD explicit Dual1(int a) : v((F)a), d(0) {}
  // a constant of another floating type, e.g. T(0.5) with T = Dual1<float>: rounded like F(0.5)
  template <class U, class = typename std::enable_if<std::is_floating_point<U>::value && !std::is_same<U, F>::value>::type>
  RBD_HD Dual1(U a) : v((F)a), d(0) {}
};
template <class F> RBD_HD Dual1<F> operator+(const Dual1<F>& a, const Dual1<F>& b) { return {a.v + b.v, a.d + b.d}; }
template <class F> RBD_HD Dual1<F> operator-(const Dual1<F>& a, const Dual1<F>& b) { return {a.v - b.v, a.d - b.d}; }
template <class F> RBD_HD Dual1<F> operator-(const Dual1<F>& a) { return {-a.v, -a.d}; }
template <class F> RBD_HD Dual1<F> operator*(const Dual1<F>& a, const Dual1<F>& b) { return {a.v * b.v, a.v * b.d + a.d * b.v}; }
template <class F> RBD_HD Dual1<F> operator/(const Dual1<F>& a, const Dual1<F>& b) {
  const F inv = F(1) / b.v;
  const F q = a.v * inv;
  return {q, (a.d - q * b.d) * inv};
}
template <class F> RBD_HD Dual1<F>& operator+=(Dual1<F>& a, const Dual1<F>& b) { a.v += b.v; a.d += b.d; return a; }
template <class F> RBD_HD Dual1<F>& operator-=(Dual1<F>& a, const Dual1<F>& b) { a.v -= b.v; a.d -= b.d; return a; }
template <class F> RBD_HD Dual1<F>& operator*=(Dual1<F>& a, const Dual1<F>& b) { a = a * b; return a; }

RBD_HD void sincos_t(const Dual1<double>& x, Dual1<double>& s, Dual1<double>& c) {
  double sv, cv;
  sincos_t(x.v, sv, cv);
  s = {sv, cv * x.d};
  c = {cv, -sv * x.d};
}

using Dual64 = Dual1<double>;
#define RBD_DUAL_TYPES 1
constexpr int kDualWidth = 7;   // doubles per Dual{Float64,6}

// rows x batch views over arrays of 7-double duals; `p` is pre-offset to this thread's sample, `dir` selects the partial
template <> struct Col<Dual64> {
  const double* p;
  int64_t ld;
  int dir;
  RBD_HD Dual64 operator()(int row) const {
    const double* e = p + (int64_t)row * ld * kDualWidth;
    return {e[0], e[1 + dir]};
  }
  RBD_HD bool valid() const { return p != nullptr; }
};
template <> struct ColOut<Dual64> {
  double* p;
  int64_t ld;
  int dir;
  bool active;
  RBD_HD void st(int row, const Dual64& x) const {
    if (!active) return;
    double* e = p + (int64_t)row * ld * kDualWidth;
    if (dir == 0) e[0] = x.v;
    e[1 + dir] = x.d;
  }
  RBD_HD bool valid() const { return p != nullptr; }
};

}  // namespace rbd
