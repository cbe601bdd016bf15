#!/usr/bin/env python
"""Register-resident stash rows and the register cap of rbd_jit_smem, measured on Atlas fp32 `dynamics!` at 2^20 samples.

All variants run in one process, alternating, best of three windows (CUDA events, 20 launches per window after a warm-up),
with the shared-memory blocks forced (RBD_JIT_VARIANT=1).  Each variant is its own model handle, generated under its own
environment (RBD_JIT_REG_ROWS, RBD_JIT_SMEM_BLOCKS: both part of the cubin cache key; RBD_JIT_SMEM_PAD_BLOCKS, read at every
call, pads the blocks' shared memory to put at most k of them on an SM):
  parent      no register rows, 16 blocks in the launch bounds (128 registers): the program before register rows
  cap         no register rows, launch bounds from the shared stash (8 blocks: up to 255 registers)
  reg<N>      N register rows (all = every eligible row), launch bounds by the default rule (at most 8 blocks with register rows)
  regall_b<k> every eligible row in registers, launch bounds for k blocks
  default     the defaults (every eligible row, 8 blocks)
  pad<k>      the parent program with at most k blocks per SM
The outputs of every variant must equal the parent's bit for bit.  Prints one JSON line with the card name, power limit and
SM clock read in the same process.
    python tools/time_stash.py [variant ...]      (default: all)"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import rigidbodydynamics.jl_b200 as rbd  # noqa: E402

B = 1 << 20
VARIANTS = {
    "parent": {"RBD_JIT_REG_ROWS": "0", "RBD_JIT_SMEM_BLOCKS": "16"},
    "cap": {"RBD_JIT_REG_ROWS": "0"},
    "reg8": {"RBD_JIT_REG_ROWS": "8"},
    "reg16": {"RBD_JIT_REG_ROWS": "16"},
    "reg27": {"RBD_JIT_REG_ROWS": "27"},
    "reg40": {"RBD_JIT_REG_ROWS": "40"},
    "regall": {"RBD_JIT_REG_ROWS": "-1"},
    "regall_b8": {"RBD_JIT_REG_ROWS": "-1", "RBD_JIT_SMEM_BLOCKS": "8"},
    "regall_b11": {"RBD_JIT_REG_ROWS": "-1", "RBD_JIT_SMEM_BLOCKS": "11"},
    "default": {},
    **{f"pad{k}": {"RBD_JIT_REG_ROWS": "0", "RBD_JIT_SMEM_BLOCKS": "16", "RBD_JIT_SMEM_PAD_BLOCKS": str(k)} for k in (4, 5, 6, 7, 8)},
}
KNOBS = ("RBD_JIT_REG_ROWS", "RBD_JIT_SMEM_BLOCKS", "RBD_JIT_SMEM_PAD_BLOCKS")


def set_env(env):
    for k in KNOBS:
        os.environ.pop(k, None)
    os.environ.update(env)


def gpu_facts():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm, smmax = (s.strip() for s in out.split(","))
        return {"gpu": name, "power_limit": pl, "sm_clock": sm, "max_sm_clock": smmax}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(), "nvidia_smi": repr(e)}


def window(fn, reps=20):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    names = sys.argv[1:] or list(VARIANTS)
    os.environ["RBD_JIT_VARIANT"] = "1"
    g = torch.Generator(device="cuda").manual_seed(3)
    base = rbd.load_model("atlas", floating=True)
    st0 = rbd.MechanismState(base, B, torch.float32)
    rbd.rand_(st0, np.random.default_rng(1))
    tau = torch.rand((st0.nv, B), dtype=torch.float32, device="cuda", generator=g)
    runs = {}
    for n in names:                       # one model handle per variant, generated and loaded under its environment
        set_env(VARIANTS[n])
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
    for _ in range(3):
        for n in names:
            set_env(VARIANTS[n])
            runs[n]["fn"]()
            torch.cuda.synchronize()
            runs[n]["ms"].append(window(runs[n]["fn"]))
    facts_after = gpu_facts()
    ref = runs[names[0]]["res"].vd
    results = []
    for n in names:
        r = runs[n]
        best = min(r["ms"])
        results.append({"variant": n, "env": VARIANTS[n], "ms": [round(m, 4) for m in r["ms"]], "best_ms": round(best, 4),
                        "Mevals_s": round(B / best / 1e3, 1), "launch": r["launch"],
                        f"equal_to_{names[0]}": bool(torch.equal(r["res"].vd, ref))})
    print(json.dumps({"tool": "time_stash", **facts, "sm_clock_after": facts_after.get("sm_clock"), "B": B, "results": results}),
          flush=True)


if __name__ == "__main__":
    main()
