// Stash access macros of the generated per-sample function (no include guard: the header undefines and redefines them).
#undef RBD_STASH_ARG
#undef RBD_SLD
#undef RBD_SST
#undef RBD_SFENCE
#undef RBD_TLD
#undef RBD_TST
#if defined(RBD_FLAVOR_SMEM)
// shared memory, [row][lane] of a single warp: conflict-free, constant offsets.  volatile: with every row a compile-time constant the
// compiler would otherwise forward each pass-1 store to its pass-2 load THROUGH REGISTERS (and spill them) -- the stash exists to
// get those values out of the register file.  (That holds for the stash as a whole; the generator keeps a bounded set of rows
// that are never indexed by a folded loop's iteration -- the trunk's and the pending slot -- in plain variables, rbd_codegen.cpp.)
#define RBD_STASH_ARG volatile rbd_f* sh
#define RBD_SLD(r) sh[(r) * 32]
#define RBD_SST(r, val_) sh[(r) * 32] = (val_)
#define RBD_SFENCE()
// the trig cache (rbd_codegen.cpp, spec_trig): its own rows, after the stash's in the warp's shared memory
#define RBD_TLD(r) sh[(RBD_SPEC_ROWS + (r)) * 32]
#define RBD_TST(r, val_) sh[(RBD_SPEC_ROWS + (r)) * 32] = (val_)
#endif
