"""Times closed-loop rollouts (rbd_integrate_pd) against the open-loop rollout and prints one JSON line.

Atlas (floating base) at 2^20 samples in fp32 and 2^16 in fp64.  Three paths alternate in one process, timed by CUDA events over
repeated calls after a warm-up, best of three windows:
  (a) open loop    simulate_ with a per-step torque schedule [steps, nv, B]            (rbd_integrate_schedule)
  (b) PD           simulate_ with JointPD, per-sample gains, a held target and v_ref    (rbd_integrate_pd, PD mode)
      and the same with gains shared by the batch and no v_ref (less controller traffic)
  (c) CT           the same in computed-torque mode                                     (rbd_integrate_pd, two more kernels per stage)
Reported: ms per RK4 step, sample-steps/s and the ratio to (a).  The card's name and power limit are read in the same run.
With --profile DIR, one extra run of each path under torch.profiler writes a kernel table there (not part of the timing).
Usage: python tools/time_pd.py [--steps N] [--reps N] [--profile DIR]
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


def case(B, dtype, steps, reps, rng, profile_dir=None):
    mech = rbd.load_model("atlas", floating=True)
    st = rbd.MechanismState(mech, B, dtype)
    rbd.rand_(st, rng)
    st.v.mul_(0.2)
    q0, v0 = st.q.clone(), st.v.clone()
    nv = st.nv
    sched = torch.from_numpy(rng.random((steps, nv, B)) - 0.5).to(dtype).cuda()
    # gains a user would pick: per DoF and sample, w^2 and 2 w (critical damping, w = 20 rad/s) times the joint's effective inertia
    # 1 / (M^-1)_kk at the initial configuration -- gains not scaled to Atlas' light links make PD mode unstable at this dt, and
    # samples that diverge would send the fp32 specialised program to its generic fallback at every stage
    M = rbd.mass_matrix(st).view(nv, nv, B).permute(2, 0, 1).double()
    eff = (1.0 / torch.linalg.inv(M).diagonal(dim1=1, dim2=2)).t().contiguous()
    del M
    w = 20.0
    kp = (w * w * eff).to(dtype).contiguous()
    kd = (2 * w * eff).to(dtype).contiguous()
    del eff
    vref = torch.zeros_like(v0)
    pd = rbd.JointPD(kp, kd, q0.clone(), vref)
    # computed-torque gains act on accelerations: w^2 and 2 w themselves, varied per sample
    f = torch.from_numpy(rng.uniform(0.5, 1.5, (nv, B))).to(dtype).cuda()
    ct = rbd.JointPD((w * w * f).contiguous(), (2 * w * f).contiguous(), q0.clone(), vref, computed_torque=True)
    T = steps * DT - 1e-9

    def run(ctrl):
        def f():
            st.q.copy_(q0); st.v.copy_(v0)
            rbd.simulate_(st, T, sched, dt=DT, controller=ctrl)
        return f
    pd_lean = rbd.JointPD(kp.min(1).values.contiguous(), kd.min(1).values.contiguous(), q0.clone())
    paths = {"open_loop": run(None), "pd": run(pd), "pd_shared_gains_no_vref": run(pd_lean), "computed_torque": run(ct)}
    for f in paths.values():                  # warm-up: module loads, specialised kernels, allocator
        f(); f()
    torch.cuda.synchronize()
    for k, f in paths.items():
        f()
        if not (bool(torch.isfinite(st.q).all()) and bool(torch.isfinite(st.v).all())):
            raise SystemExit(f"time_pd: the {k} rollout diverged")
    best = {k: float("inf") for k in paths}
    for _ in range(3):
        for k, f in paths.items():
            best[k] = min(best[k], event_ms(f, reps))
    out = {}
    for k, ms in best.items():
        step_ms = ms / steps
        out[k] = {"ms_per_step": round(step_ms, 4), "sample_steps_per_s": float(f"{B / (step_ms * 1e-3):.4g}"),
                  "vs_open_loop": round(ms / best["open_loop"], 3)}
    if profile_dir:
        from torch.profiler import ProfilerActivity, profile
        for k, f in paths.items():
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                f()
                torch.cuda.synchronize()
            with open(os.path.join(profile_dir, f"pd_{str(dtype)[6:]}_{k}.txt"), "w") as fh:
                fh.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=25))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--profile", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_pd: no CUDA device")
    if a.profile:
        os.makedirs(a.profile, exist_ok=True)
    name, power = card()
    rng = np.random.default_rng(0)
    res = {"card": name, "power_limit": power, "steps": a.steps, "dt": DT}
    res["atlas_fp32_2^20"] = case(1 << 20, torch.float32, a.steps, a.reps, rng, a.profile)
    res["atlas_fp64_2^16"] = case(1 << 16, torch.float64, a.steps, a.reps, rng, a.profile)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
