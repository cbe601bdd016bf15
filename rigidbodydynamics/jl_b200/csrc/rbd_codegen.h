// Model-specialised code generation: trace the templated per-sample algorithms on a concrete mechanism (rbd_sym.h) and emit
// the resulting straight-line program as CUDA (compiled by NVRTC in rbd_jit.cpp) or as plain C++ (CPU test tier).
#pragma once
#include <string>

#include "rbd_model.h"

namespace rbd {

enum SpecAlgo : int { SPEC_ABA = 0, SPEC_RNEA = 1, SPEC_CRBA = 2, SPEC_KIN = 3 };

struct SpecKey {
  int algo = SPEC_ABA;
  bool f64 = false;      // scalar type of the kernel
  bool has_in2 = true;   // ABA: tau given (else zero torques); RNEA: vd given (else dynamics_bias)
  bool has_out1 = false; // ABA: q̇ output requested
  bool lower = false;    // CRBA: lower triangle only
  bool peers = false;    // ABA: v̇ is stored into every peer GPU's gathered array (rbd_dynamics_gather) instead of o0
  // KIN (rbd_kinematics): bit k of kin_mask = output k of rbd_kinematics_out requested; has_in2 = v given; kin_sign = the geometric jacobian's path, PREORDER positions
  int kin_mask = 0;
  int8_t kin_sign[kMaxBodies] = {0};
};

struct SpecStats {
  int nodes_traced = 0, nodes_live = 0;
  int n_add = 0, n_mul = 0, n_div = 0, n_neg = 0, n_sincos = 0, n_load = 0, n_store = 0, n_sld = 0, n_sst = 0;
  int stash_rows = 0;
  int n_load_v = 0;      // global loads of the v array (0: the kernel shell does not prefetch it)
  int n_fold_loops = 0;  // (pass, chain pair) steps emitted once as a two-iteration loop for both mirror-image chains
  int n_fold_bodies = 0; // body steps whose code those loops share (summed over passes)
  int reg_rows = 0;      // stash rows kept in registers (RBD_JIT_REG_ROWS)
  int shared_rows = 0;   // stash rows left in shared memory (RBD_SPEC_ROWS of the CUDA flavour)
  int trig_rows = 0;     // trig cache rows in shared memory, after the stash's (RBD_SPEC_TRIG_ROWS; spec_trig)
  int trig_reg_rows = 0; // trig cache rows in registers
};

enum SpecFlavor : int { FLAVOR_CPU = 0, FLAVOR_SMEM = 1 };

// Body of one per-sample function `name(...)` for the given flavour (see rbd_jit_prelude.cuh for the calling convention).
// Returns false (with `err`) if the model / key cannot be specialised.  `fold` = false keeps mirror-image chains straight-line
// (the reference form the folded program is tested against; not a user option).
bool spec_emit_function(const HostModel& hm, const SpecKey& key, int flavor, const std::string& name, std::string& out,
                        SpecStats* stats, std::string& err, bool fold = true);

// Whole NVRTC translation unit for `key`: defines + the per-sample function + the kernel shell of the prelude.
bool spec_emit_cuda_tu(const HostModel& hm, const SpecKey& key, std::string& out, SpecStats* stats, std::string& err);
// Rows of the algorithm's stash layout, and the rows of one warp's shared memory in the generated program: the stash rows it
// keeps there (the others are registers, see spec_reg_rows) plus those of its trig cache (spec_trig).  The latter runs the
// tracer, it is meant for once per loaded program.
int spec_stash_rows(const HostModel& hm, const SpecKey& key);
int spec_shared_rows(const HostModel& hm, const SpecKey& key);
// Whether the program keeps a trig cache: (sin, cos) of every revolute joint computed once in the first ABA pass and read back in
// the other two (trig_keep, rbd_device.cuh).  fp32 forward dynamics only, and only where its shared rows cost no resident
// blocks; RBD_JIT_TRIG=0 turns it off.
bool spec_trig(const SpecKey& key);
// Whether sums are planned as FMA chains (Emitter::plan_chains): by default in forward-dynamics and kinematics programs;
// RBD_JIT_FMA_CHAIN=0 / 1 turns them off / on for every program (off: one product per add, the planning before them).  And the
// number of terms above which a sum is split into two chains joined by one add (RBD_JIT_FMA_CAP; 0: never).
bool spec_fma_chain(const SpecKey& key);
int spec_fma_cap();
// Whether an fp32 program's reciprocals are the branch-free fast path under the range gate (rbd_jit_prelude.cuh, RBD_RCP);
// RBD_JIT_RCP=0 keeps the library's __frcp_rn.
bool spec_rcp_gate(const SpecKey& key);
// Budget of register-resident stash rows for `key` (-1: every eligible row); RBD_JIT_REG_ROWS overrides it for forward dynamics.
int spec_reg_rows(const SpecKey& key);
// Minimum resident single-warp blocks per SM rbd_jit_smem is compiled for (its register cap): as many as the shared stash
// allows on a 228 KB SM, at most 16 (128 registers), at most 8 (255 registers) with register rows; RBD_JIT_SMEM_BLOCKS overrides it.
int spec_smem_blocks(const SpecKey& key, int shared_rows);

// Self-contained C++ translation unit (needs csrc/ on the include path) defining `extern "C" void name(q, v, in2, o0, o1, ld, sh)`
// for ONE sample: column pointers with leading dimension ld, `sh` = stash_rows scalars of scratch.  Test tier only.
bool spec_emit_cpu_tu(const HostModel& hm, const SpecKey& key, const std::string& name, std::string& out, SpecStats* stats,
                      std::string& err, bool fold = true);

// 64-bit content hash of a model + key + generator version (cubin cache key).
uint64_t spec_hash(const HostModel& hm, const SpecKey& key);

}  // namespace rbd
