#!/usr/bin/env python
"""Shared-memory kernels alone vs the mixed CTA with its L2 stash (RBD_JIT_VARIANT=1 / 2, read at every call), alternating,
kernel time by CUDA events, Atlas floating base.  One JSON line per configuration; outputs of the two variants must be equal.
    python tools/time_mix.py [config ...]      (default: all)"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import rigidbodydynamics.jl_b200 as rbd  # noqa: E402


def timed(fn, reps=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def state(mech, B, dtype, seed):
    st = rbd.MechanismState(mech, B, dtype)
    rbd.rand_(st, np.random.default_rng(seed))
    return st


def configs(mech):
    g = torch.Generator(device="cuda").manual_seed(3)
    nb = len(mech.joints)

    def dyn(B, dtype, wext=False):
        st = state(mech, B, dtype, 1)
        tau = torch.rand((st.nv, B), dtype=dtype, device="cuda", generator=g)
        w = torch.rand((6 * nb, B), dtype=dtype, device="cuda", generator=g) if wext else None
        res = rbd.DynamicsResult(mech, B, dtype)
        return (lambda: rbd.dynamics_(res, st, tau, w, want_qd=False)), (lambda: res.vd), B

    def inv(B, dtype, wext=False):
        st = state(mech, B, dtype, 2)
        vd = torch.rand((st.nv, B), dtype=dtype, device="cuda", generator=g)
        w = torch.rand((6 * nb, B), dtype=dtype, device="cuda", generator=g) if wext else None
        out = torch.empty_like(vd)
        return (lambda: rbd.inverse_dynamics_(out, st, vd, w)), (lambda: out), B

    def dual(B):          # as bench.py's config 4: value + 6 partials of the non-quaternion coordinates
        st = state(mech, B, torch.float64, 4)
        qd = torch.zeros((st.nq, B, 7), dtype=torch.float64, device="cuda")
        qd[..., 0] = st.q
        qd[4:, :, 1:] = torch.rand((st.nq - 4, B, 6), dtype=torch.float64, device="cuda", generator=g)
        vd_, td = (torch.rand((st.nv, B, 7), dtype=torch.float64, device="cuda", generator=g) for _ in range(2))
        out = torch.empty_like(vd_)
        return (lambda: rbd.dynamics_dual_(out, st, qd, vd_, td)), (lambda: out), B

    return {
        "f32_dynamics_b1048576": lambda: dyn(1 << 20, torch.float32),
        "f64_dynamics_b65536": lambda: dyn(1 << 16, torch.float64),
        "f64_dynamics_b1048576": lambda: dyn(1 << 20, torch.float64),
        "f32_dynamics_extwrench_b1048576": lambda: dyn(1 << 20, torch.float32, True),
        "f32_inverse_dynamics_b1048576": lambda: inv(1 << 20, torch.float32),
        "f32_inverse_dynamics_extwrench_b1048576": lambda: inv(1 << 20, torch.float32, True),
        "f64_inverse_dynamics_b1048576": lambda: inv(1 << 20, torch.float64),
        "dual64x6_dynamics_b8192": lambda: dual(8192),
    }


def main():
    mech = rbd.load_model("atlas", floating=True)
    cfgs = configs(mech)
    for name in sys.argv[1:] or list(cfgs):
        fn, out, B = cfgs[name]()
        ms = {"1": [], "2": []}
        res, info = {}, {}
        for _ in range(2):
            for v in ("1", "2"):
                os.environ["RBD_JIT_VARIANT"] = v
                ms[v].append(timed(fn))
                li = rbd.launch_info()
                info[v] = {"block": li.block, "grid": li.grid, "smem": li.smem_bytes, "specialised": li.specialised}
                res[v] = out().clone()
        del os.environ["RBD_JIT_VARIANT"]
        print(json.dumps({"config": name, "smem_only_Mevals_s": [round(B / m / 1e3, 1) for m in ms["1"]],
                          "mixed_Mevals_s": [round(B / m / 1e3, 1) for m in ms["2"]], "launch": info,
                          "equal": bool(torch.equal(res["1"], res["2"]))}), flush=True)


if __name__ == "__main__":
    main()
