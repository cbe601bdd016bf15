#!/usr/bin/env python
"""Sum planning (RBD_JIT_FMA_CHAIN, RBD_JIT_FMA_CAP) and the gated reciprocal (RBD_JIT_RCP) of the model-specialised programs,
measured on Atlas fp32 `dynamics!` at 2^20 samples.

Every variant runs in one process, alternating, over `rounds` windows each (CUDA events, 20 launches per window after a warm-up),
with the shared-memory blocks forced (RBD_JIT_VARIANT=1).  Each variant is its own model handle, generated and compiled under its
own settings (all part of the cubin cache key) into a fresh cache directory:
  old        RBD_JIT_FMA_CHAIN=0: one product contracted into each add / sub (the planning before the chains)
  chain      sums as FMA chains, no length cap (RBD_JIT_FMA_CAP=0)
  chain4     sums as FMA chains, a sum of more than 4 terms split into two chains
each as `-lib` with the library's __frcp_rn (RBD_JIT_RCP=0) and as `-rcp` with the branch-free reciprocal under the range gate.
For each variant the loaded cubin's rbd_jit_smem is read back: SASS instructions, registers, stack and spill bytes (cuobjdump).
v̇ must be within 1e-4 (relative to the column's largest) of the old planning's: reassociation changes the last bits.
Prints one JSON line with the card name, power limit and SM clock read in the same process.
    python tools/time_emit.py [rounds]      (default 5)"""
import glob
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import rigidbodydynamics.jl_b200 as rbd  # noqa: E402
from tools.time_stash import gpu_facts, window  # noqa: E402

B = 1 << 20
PLANS = {"old": {"RBD_JIT_FMA_CHAIN": "0"}, "chain": {"RBD_JIT_FMA_CAP": "0"}, "chain4": {"RBD_JIT_FMA_CAP": "4"}}
VARIANTS = {f"{p}-{r}": {**env, "RBD_JIT_RCP": "1" if r == "rcp" else "0"} for p, env in PLANS.items() for r in ("lib", "rcp")}
KNOBS = ("RBD_JIT_FMA_CHAIN", "RBD_JIT_FMA_CAP", "RBD_JIT_RCP")


def set_env(env):
    for k in KNOBS:
        os.environ.pop(k, None)
    os.environ.update(env)


def cubin_facts(path):
    """rbd_jit_smem of one cubin: SASS instructions (NOPs excluded), registers, stack and spill bytes."""
    cuobjdump = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    try:
        sass = subprocess.run([cuobjdump, "-sass", "-fun", "rbd_jit_smem", path], capture_output=True, text=True, timeout=120).stdout
        res = subprocess.run([cuobjdump, "-res-usage", path], capture_output=True, text=True, timeout=120).stdout
    except Exception as e:  # noqa: BLE001
        return {"cuobjdump": repr(e)}
    ops = re.findall(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", sass)
    ops = [o for o in ops if o != "NOP"]
    out = {"sass": len(ops), "CALL": sum(o.startswith("CALL") for o in ops), "BSSY": sum(o.startswith("BSSY") for o in ops)}
    m = re.search(r"Function rbd_jit_smem:\s*\n\s*(.*)", res)
    if m:
        for k, v in re.findall(r"(REG|STACK|LOCAL):(\d+)", m.group(1)):
            out[k.lower()] = int(v)
    return out


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
    with tempfile.TemporaryDirectory(prefix="rbd_time_emit_") as tmp:
        for n, env in VARIANTS.items():      # one model handle per variant, generated and loaded under its settings
            set_env(env)
            os.environ["RBD_JIT_CACHE"] = os.path.join(tmp, n)
            os.makedirs(os.environ["RBD_JIT_CACHE"])
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
            cubins = glob.glob(os.path.join(tmp, n, "*aba_f32*.cubin"))
            runs[n] = {"fn": fn, "res": res, "ms": [], "env": env,
                       "launch": {"specialised": li.specialised, "grid": li.grid, "block": li.block, "smem_bytes": li.smem_bytes,
                                  "blocks_per_sm": li.blocks_per_sm},
                       "cubin": cubin_facts(cubins[0]) if len(cubins) == 1 else {"cubins": len(cubins)}}
        facts = gpu_facts()
        for _ in range(rounds):
            for n, r in runs.items():
                set_env(r["env"])
                r["fn"]()
                torch.cuda.synchronize()
                r["ms"].append(window(r["fn"]))
        facts_after = gpu_facts()
    ref = runs["old-lib"]["res"].vd
    scale = ref.abs().amax(0).clamp_min(1.0)
    results = []
    for n, r in runs.items():
        best = min(r["ms"])
        diff = float(((r["res"].vd - ref).abs().amax(0) / scale).max())
        results.append({"variant": n, "ms": [round(m, 4) for m in r["ms"]], "best_ms": round(best, 4),
                        "Mevals_s": round(B / best / 1e3, 1), "vs_old_lib": round(min(runs["old-lib"]["ms"]) / best, 4),
                        "max_rel_diff_vs_old_lib": diff, "ok": diff < 1e-4, "launch": r["launch"], **r["cubin"]})
    print(json.dumps({"tool": "time_emit", **facts, "sm_clock_after": facts_after.get("sm_clock"), "B": B, "results": results}),
          flush=True)


if __name__ == "__main__":
    main()
