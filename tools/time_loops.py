"""Times rbd_dynamics_loops (dynamics! with kinematic loops) and prints one JSON line.

Cases: the four-bar linkage (fp64 and fp32, 2^20 samples) and Atlas in double support (both feet welded to the world by Fixed loop
joints, nl = 12; fp32 at 2^20, fp64 at 2^16), each next to rbd_dynamics on the same spanning tree, the two timed alternately in the
same process.  Kernel time by CUDA events over repeated launches after a warm-up.  The error is the max relative error against the
fp64 host restatement (tests/loops_oracle.py) on a seeded strided subsample.  The card's name and power limit are read in the same
run.  Usage: python tools/time_loops.py [--reps N]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import rigidbodydynamics.jl_b200 as rbd  # noqa: E402
from tests.loops_oracle import FOUR_BAR_Q0, LoopOracle, atlas_double_support, four_bar  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
    except Exception:                       # nvidia-smi unavailable: the name from the runtime, power unknown
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def event_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def case(name, mech, B, dtype, reps, rng, q=None):
    st = rbd.MechanismState(mech, B, dtype)
    if q is None:
        rbd.rand_(st, rng)
    else:
        st.q.copy_(torch.from_numpy(q(B, rng)).to(dtype))
        st.v.copy_(torch.from_numpy(rng.standard_normal((st.nv, B))).to(dtype))
    tau = torch.from_numpy(rng.random((st.nv, B))).to(dtype).cuda()
    res, tree = rbd.DynamicsResult(mech, B, dtype), rbd.DynamicsResult(mech, B, dtype)
    ld = rbd.loop_desc(mech)
    loops = lambda: rbd.dynamics_loops_(res, st, tau, loops=ld, want_qd=False)
    handle = st.handle.ptr
    lib = rbd.load_library()
    code = 1 if dtype == torch.float64 else 0
    stream = torch.cuda.current_stream().cuda_stream
    plain = lambda: lib.rbd_dynamics(handle, code, B, B, st.q.data_ptr(), st.v.data_ptr(), tau.data_ptr(), None, tree.vd.data_ptr(),
                                     None, stream)
    for _ in range(3):
        loops()
        plain()
    torch.cuda.synchronize()
    t_loop, t_tree = [], []
    for _ in range(3):                      # alternate the two, keep the best window of each
        t_loop.append(event_ms(loops, reps))
        t_tree.append(event_ms(plain, reps))
    idx = torch.arange(3, B, max(1, B // 512), device="cuda")
    ref = LoopOracle(mech).dynamics(*(x[:, idx].double().cpu().numpy() for x in (st.q, st.v, tau)))
    err = {}
    for key, got in (("vd", res.vd), ("lam", res.lam)):
        g = got[:, idx].double().cpu().numpy()
        err[key] = float((np.abs(g - ref[key]).max(0) / np.maximum(1.0, np.abs(ref[key]).max(0))).max())
    ms = min(t_loop)
    return {"case": name, "dtype": str(dtype).replace("torch.", ""), "B": B, "nv": st.nv, "nl": ld.nc,
            "loops_ms": round(ms, 4), "loops_Msamples_per_s": round(B / ms / 1e3, 2), "rbd_dynamics_tree_ms": round(min(t_tree), 4),
            "max_rel_err_vs_oracle": err, "subsample": int(idx.numel())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_loops.py needs a CUDA device")
    rng = np.random.default_rng(2024)
    name, power = card()
    fb, atlas = four_bar(), atlas_double_support()
    near = lambda B, r: FOUR_BAR_Q0[:, None] + 0.2 * r.standard_normal((3, B))
    rows = [case("four_bar", fb, 1 << 20, torch.float64, args.reps, rng, near),
            case("four_bar", fb, 1 << 20, torch.float32, args.reps, rng, near),
            case("atlas_double_support", atlas, 1 << 20, torch.float32, args.reps, rng),
            case("atlas_double_support", atlas, 1 << 16, torch.float64, args.reps, rng)]
    print(json.dumps({"tool": "time_loops", "gpu": name, "power_limit": power, "results": rows}), flush=True)


if __name__ == "__main__":
    main()
