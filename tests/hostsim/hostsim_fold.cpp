// Test shim for the folding of mirror-image chains (rbd_codegen.cpp): the ABA program of a mechanism with and without the fold,
// and the chain pairs the flattener exports.  Built by tests/test_fold.py.
#include <cstdlib>
#include <cstring>
#include <string>

#include "rbd_codegen.h"
#include "rbd_model.h"

using namespace rbd;

extern "C" {
// stats = {nodes_live, fold_loops, fold_bodies, pairs}; returns a malloc'ed string or NULL
char* fold_spec_source(const rbd_model_desc* d, int dtype, int has_in2, int has_out1, int fold, int* stats) {
  HostModel hm; std::string err;
  if (build_host_model(d, hm, err) != RBD_OK) return nullptr;
  SpecKey key; key.algo = SPEC_ABA; key.f64 = dtype == 1; key.has_in2 = has_in2 != 0; key.has_out1 = has_out1 != 0;
  SpecStats st; std::string out;
  if (!spec_emit_cpu_tu(hm, key, "rbd_spec_cpu", out, &st, err, fold != 0)) return nullptr;
  stats[0] = st.nodes_live; stats[1] = st.n_fold_loops; stats[2] = st.n_fold_bodies; stats[3] = (int)hm.pairs.size();
  char* r = (char*)malloc(out.size() + 1);
  std::memcpy(r, out.c_str(), out.size() + 1);
  return r;
}
void fold_free(char* p) { free(p); }
}
