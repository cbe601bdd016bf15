// Persistent kernel around the generated per-sample function (see rbd_jit_prelude.cuh): warps claim groups of 32 consecutive
// samples from an atomic counter; the next group's input lines are prefetched into L2 while the current one is computed; warps
// never synchronise with each other.  Two ways to fill an SM with warps (rbd_spec.cpp picks one per model and entry point):
//   rbd_jit_smem   single-warp blocks with their stash in shared memory ([row][lane]), as many per SM as the stash allows;
//   rbd_jit_mix    one CTA per SM of up to 16 warps: those shared memory can hold keep their stash there, the others in a global
//                  scratch small enough to stay in the 50 MB L2 -- the register file holds 16 warps where shared memory holds 8
//                  Atlas stashes.  (Tried and dropped: multi-warp CTAs walking the program as a convoy behind CTA
// barriers every 64 ... 1024 statements, to share instruction fetches -- no measurable change, DESIGN.md section 4.8.)
#pragma once

#define RBD_QUEUE_LOOP(CALL)                                                                        \
  const int lane = threadIdx.x & 31;                                                                \
  const long long ngroups = (a.B + 31) / 32;                                                        \
  long long g = rbd_claim_group(a.counter);                                                         \
  while (g < ngroups) {                                                                             \
    const long long gn = rbd_claim_group(a.counter);                                                \
    if (gn < ngroups) {                                                                             \
      const long long bn = gn * 32;                                                                 \
      rbd_prefetch_rows(a.q, RBD_SPEC_NQ, a.ld, bn);                                                \
      if (RBD_SPEC_USES_V) rbd_prefetch_rows(a.v, RBD_SPEC_NV, a.ld, bn);   /* not when the program never reads v */ \
      if (RBD_SPEC_HAS_IN2) rbd_prefetch_rows(a.in2, RBD_SPEC_NV, a.ld, bn);                        \
    }                                                                                               \
    const long long b = g * 32 + lane;                                                              \
    const bool active = b < a.B;                                                                    \
    const long long bl = active ? b : a.B - 1;   /* inactive lanes recompute the last sample, stores are masked */ \
    CALL(a.q + bl, a.v + bl, RBD_SPEC_HAS_IN2 ? a.in2 + bl : (const rbd_f*)0, a.o0 + bl,             \
         RBD_SPEC_HAS_OUT1 ? a.o1 + bl : (rbd_f*)0, a.ld, active, a.flag, a, bl);                    \
    g = gn;                                                                                         \
  }

// Register cap of the single-warp blocks: as many blocks as the shared stash lets reside (RBD_SPEC_SMEM_BLOCKS, at most 16) share
// the register file, so 8 resident Atlas warps get up to 255 registers each instead of 128.
extern "C" __global__ void __launch_bounds__(32, RBD_SPEC_F64 ? 1 : RBD_SPEC_SMEM_BLOCKS) rbd_jit_smem(const RbdJitArgs a) {
  extern __shared__ __align__(16) unsigned char rbd_smem_raw[];
  volatile rbd_f* sh = reinterpret_cast<volatile rbd_f*>(rbd_smem_raw) + threadIdx.x;
#define RBD_CALL_SMEM(q_, v_, i_, o0_, o1_, ld_, act_, fl_, pa_, pb_) rbd_spec_smem(q_, v_, i_, o0_, o1_, ld_, act_, fl_, pa_, pb_, sh)
  RBD_QUEUE_LOOP(RBD_CALL_SMEM)
}

// All warps run the same program through a generic stash pointer, so the SM fetches ONE instruction stream (two kernels side by
// side starve each other's instruction supply, DESIGN.md 4.8).
#define RBD_STASH_ROWS (RBD_SPEC_ROWS + RBD_SPEC_TRIG_ROWS > 0 ? RBD_SPEC_ROWS + RBD_SPEC_TRIG_ROWS : 1)   /* + the trig cache */
extern "C" __global__ void __launch_bounds__(512, 1) rbd_jit_mix(const RbdJitArgs a) {
  extern __shared__ __align__(16) unsigned char rbd_smem_raw[];
  const unsigned w = threadIdx.x >> 5;
  const unsigned sw = (unsigned)a.smem_warps, gw = blockDim.x / 32u - sw;
  volatile rbd_f* sh = w < sw ? reinterpret_cast<volatile rbd_f*>(rbd_smem_raw) + w * (RBD_STASH_ROWS * 32u) + (threadIdx.x & 31u)
                              : a.l2_stash + ((unsigned long long)blockIdx.x * gw + (w - sw)) * (RBD_STASH_ROWS * 32u) + (threadIdx.x & 31u);
  RBD_QUEUE_LOOP(RBD_CALL_SMEM)
}
