"""Times the backward pass of a rollout (rbd_integrate_vjp) against the forward RK4 step (rbd_integrate) and prints one JSON line.

Cases: floating Atlas (fp32 at 2^20, fp64 at 2^16) and the 7-DoF iiwa14 arm (fp32 at 2^20), constant torques, `--steps` steps.
Forward and backward are timed alternately in the same process by CUDA events over repeated calls after a warm-up, best of three
windows; rates are sample-steps per second.  A separate torch.profiler run splits one backward call into the stage recompute
(rbd_integrate's stage and dynamics kernels), the forward-dynamics VJPs (dynamics_vjp_kernel) and the new elementwise adjoint
kernels (integrate_adjoint*).  The workspace is computed from its row counts (it is allocated by the library's stream-ordered
allocator, not torch's).  The card's name and power limit are read in the same run.
Usage: python tools/time_integrate_vjp.py [--steps N] [--reps N]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import rigidbodydynamics.jl_b200 as rbd  # noqa: E402
from tools.time_loops import card, event_ms  # noqa: E402

DT = 1e-3


def case(name, mech, B, dtype, steps, reps, rng):
    st = rbd.MechanismState(mech, B, dtype)
    rbd.rand_(st, rng)
    nq, nv = st.nq, st.nv
    tau = torch.from_numpy(rng.random((nv, B))).to(dtype).cuda()
    q0, v0 = st.q.clone(), st.v.clone()
    qt, vt = rbd.simulate_trajectory_(st, steps, tau, dt=DT)
    qtb, vtb = torch.randn_like(qt), torch.randn_like(vt)
    e = lambda rows: torch.empty((rows, B), dtype=dtype, device="cuda")
    qc, vb, tb = e(nq), e(nv), torch.zeros_like(tau)
    lib = rbd.load_library()
    from rigidbodydynamics.jl_b200.state import _DT

    def fwd():
        st.q.copy_(q0); st.v.copy_(v0)
        rbd._cabi.check(lib.rbd_integrate(st.handle.ptr, _DT[dtype], B, B, st.q.data_ptr(), st.v.data_ptr(), tau.data_ptr(), DT, steps,
                                          torch.cuda.current_stream().cuda_stream))

    def bwd():
        rbd.integrate_vjp_(mech, qt, vt, tau, dt=DT, q_traj_bar=qtb, v_traj_bar=vtb, q0_bar_cfg=qc, v0_bar=vb, tau_bar=tb)
    for _ in range(2):
        fwd(); bwd()
    torch.cuda.synchronize()
    t = {"forward": [], "backward": []}
    for _ in range(3):
        t["forward"].append(event_ms(fwd, reps))
        t["backward"].append(event_ms(bwd, reps))
    fms, bms = min(t["forward"]) / steps, min(t["backward"]) / steps
    # per-kernel split of one backward call
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        bwd()
        torch.cuda.synchronize()
    split = {"recompute": 0.0, "dynamics_vjp": 0.0, "elementwise_adjoint": 0.0, "other": 0.0}
    for ev in prof.key_averages():
        us = getattr(ev, "device_time_total", None)
        if us is None:
            us = ev.cuda_time_total
        if us <= 0:
            continue
        k = ev.key
        if "integrate_adjoint" in k:
            split["elementwise_adjoint"] += us
        elif "dynamics_vjp_kernel" in k:
            split["dynamics_vjp"] += us
        elif "integrate_stage" in k or "aba" in k or "rbd_jit" in k or "rbd_spec" in k:
            split["recompute"] += us
        elif "Memcpy" in k or "Memset" in k or "elementwise" in k.lower():
            split["other"] += us
        else:
            split["recompute"] += us     # the model-specialised dynamics kernels carry generated names
    tot = sum(split.values())
    size = 4 if dtype == torch.float32 else 8
    ws_rows = (4 * nq + 12 * nv) + 4 * nq + 7 * nv          # rbd_integrate_vjp's own workspace
    rec_rows = 2 * nq + 10 * nv                               # integrate_t's workspace during the recompute
    return {"case": name, "dtype": str(dtype).replace("torch.", ""), "B": B, "nq": nq, "nv": nv, "steps": steps,
            "forward_step_ms": round(fms, 4), "backward_step_ms": round(bms, 4),
            "forward_M_sample_steps_per_s": round(B / fms / 1e3, 2), "backward_M_sample_steps_per_s": round(B / bms / 1e3, 2),
            "backward_over_forward": round(bms / fms, 2),
            "split_share": {k: round(v / tot, 4) for k, v in split.items()} if tot else None,
            "workspace_MB": round(ws_rows * B * size / 2**20, 1), "recompute_workspace_MB": round(rec_rows * B * size / 2**20, 1),
            "finite": bool(torch.isfinite(qc).all() and torch.isfinite(vb).all() and torch.isfinite(tb).all())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_integrate_vjp.py needs a CUDA device")
    rng = np.random.default_rng(2026)
    name, power = card()
    atlas, arm = rbd.load_model("atlas", floating=True), rbd.load_model("iiwa14", floating=False)
    rows = [case("atlas", atlas, 1 << 20, torch.float32, args.steps, args.reps, rng),
            case("atlas", atlas, 1 << 16, torch.float64, args.steps, args.reps, rng),
            case("iiwa14", arm, 1 << 20, torch.float32, args.steps, args.reps, rng)]
    print(json.dumps({"tool": "time_integrate_vjp", "gpu": name, "power_limit": power, "results": rows}), flush=True)


if __name__ == "__main__":
    main()
