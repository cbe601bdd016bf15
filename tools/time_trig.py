#!/usr/bin/env python
"""Trig cache of the fp32 forward-dynamics program (RBD_JIT_TRIG), measured on Atlas fp32 `dynamics!` at 2^20 samples.

Both variants run in one process, alternating, over `rounds` windows each (CUDA events, 20 launches per window after a warm-up),
with the shared-memory blocks forced (RBD_JIT_VARIANT=1).  Each variant is its own model handle, generated under its own
RBD_JIT_TRIG (part of the cubin cache key):
  off   RBD_JIT_TRIG=0: every ABA pass evaluates sin / cos of the joint angles (the program before the cache)
  on    the default: pass 1 keeps (sin, cos), passes 2 and 3 read them back
The outputs must be equal bit for bit.  Prints one JSON line with the card name, power limit and SM clock read in the same process.
    python tools/time_trig.py [rounds]      (default 5)"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import rigidbodydynamics.jl_b200 as rbd  # noqa: E402
from tools.time_stash import gpu_facts, window  # noqa: E402

B = 1 << 20
VARIANTS = {"off": "0", "on": "1"}


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    os.environ["RBD_JIT_VARIANT"] = "1"
    os.environ.pop("RBD_JIT_REG_ROWS", None)
    g = torch.Generator(device="cuda").manual_seed(3)
    base = rbd.load_model("atlas", floating=True)
    st0 = rbd.MechanismState(base, B, torch.float32)
    rbd.rand_(st0, np.random.default_rng(1))
    tau = torch.rand((st0.nv, B), dtype=torch.float32, device="cuda", generator=g)
    runs = {}
    for n, trig in VARIANTS.items():      # one model handle per variant, generated and loaded under its setting
        os.environ["RBD_JIT_TRIG"] = trig
        mech = rbd.load_model("atlas", floating=True)
        st = rbd.MechanismState(mech, B, torch.float32)
        st.q.copy_(st0.q)
        st.v.copy_(st0.v)
        res = rbd.DynamicsResult(mech, B, torch.float32)
        fn = (lambda res=res, st=st: rbd.dynamics_(res, st, tau, want_qd=False))
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        li = rbd.launch_info()
        runs[n] = {"fn": fn, "res": res, "ms": [], "launch": {"specialised": li.specialised, "grid": li.grid, "block": li.block,
                                                              "smem_bytes": li.smem_bytes, "blocks_per_sm": li.blocks_per_sm}}
    facts = gpu_facts()
    for _ in range(rounds):
        for n, trig in VARIANTS.items():
            os.environ["RBD_JIT_TRIG"] = trig
            runs[n]["fn"]()
            torch.cuda.synchronize()
            runs[n]["ms"].append(window(runs[n]["fn"]))
    facts_after = gpu_facts()
    results = []
    for n, r in runs.items():
        best = min(r["ms"])
        results.append({"variant": n, "ms": [round(m, 4) for m in r["ms"]], "best_ms": round(best, 4),
                        "Mevals_s": round(B / best / 1e3, 1), "launch": r["launch"]})
    on, off = min(runs["on"]["ms"]), min(runs["off"]["ms"])
    print(json.dumps({"tool": "time_trig", **facts, "sm_clock_after": facts_after.get("sm_clock"), "B": B, "results": results,
                      "speedup": round(off / on, 4), "identical": bool(torch.equal(runs["on"]["res"].vd, runs["off"]["res"].vd))}),
          flush=True)


if __name__ == "__main__":
    main()
