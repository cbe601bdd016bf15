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
};

enum SpecFlavor : int { FLAVOR_CPU = 0, FLAVOR_SMEM = 1 };

// Body of one per-sample function `name(...)` for the given flavour (see rbd_jit_prelude.cuh for the calling convention).
// Returns false (with `err`) if the model / key cannot be specialised.  `fold` = false keeps mirror-image chains straight-line
// (the reference form the folded program is tested against; not a user option).
bool spec_emit_function(const HostModel& hm, const SpecKey& key, int flavor, const std::string& name, std::string& out,
                        SpecStats* stats, std::string& err, bool fold = true);

// Whole NVRTC translation unit for `key`: defines + the per-sample function + the kernel shell of the prelude.
bool spec_emit_cuda_tu(const HostModel& hm, const SpecKey& key, std::string& out, SpecStats* stats, std::string& err);
int spec_stash_rows(const HostModel& hm, const SpecKey& key);

// Self-contained C++ translation unit (needs csrc/ on the include path) defining `extern "C" void name(q, v, in2, o0, o1, ld, sh)`
// for ONE sample: column pointers with leading dimension ld, `sh` = stash_rows scalars of scratch.  Test tier only.
bool spec_emit_cpu_tu(const HostModel& hm, const SpecKey& key, const std::string& name, std::string& out, SpecStats* stats,
                      std::string& err, bool fold = true);

// 64-bit content hash of a model + key + generator version (cubin cache key).
uint64_t spec_hash(const HostModel& hm, const SpecKey& key);

}  // namespace rbd
