// Model-specialised solve kernel of rbd_dynamics_derivatives: source generator (host C++), see rbd_deriv_jit.cpp.
#pragma once
#include <string>

#include "rbd_deriv.cuh"

namespace rbd {

struct DerivJitPlan {
  int cg = 0;        // columns solved together by one thread (their right-hand sides live in registers)
  int warps = 0;     // warps per CTA
  int ngroups = 0;   // column groups = ceil(blocks nv / cg)
  int blocks = 2;    // blocks of nv columns: d v̇ / dq, d v̇ / dv and, with 3, d v̇ / d tau = M^-1
};
// Chooses cg / warps for the model; false if the right-hand sides of even one column do not fit into registers.
bool deriv_jit_plan(const DerivDev& D, bool f64, DerivJitPlan& plan, int blocks = 2);
// CUDA source of `extern "C" __global__ rbd_deriv_solve(const T* H, long long sld, T* dq, T* dv, long long ld, long long C)`, with
// a last parameter `T* dtau` when plan.blocks == 3.
void deriv_jit_source(const DerivDev& D, const DerivAnc& A, bool f64, const DerivJitPlan& plan, std::string& out);

}  // namespace rbd
