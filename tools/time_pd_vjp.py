"""Times the backward step of closed-loop rollouts (rbd_integrate_pd_vjp) against the open-loop backward step (rbd_integrate_vjp)
and prints one JSON line.

Atlas (floating base) at 2^20 samples in fp32 and 2^16 in fp64, with the gains and step size of tools/time_pd.py.  A trajectory of
`steps` steps is recorded once per path; then the four backward passes alternate in one process, timed by CUDA events over repeated
calls after a warm-up, best of three windows:
  open_loop         integrate_vjp_ over the open-loop trajectory
  pd                integrate_pd_vjp_, per-sample gains, held q_ref and v_ref, every controller gradient requested
  pd_shared_gains   the same with gains shared by the batch and no v_ref
  computed_torque   computed-torque mode, per-sample gains (one more inverse-dynamics VJP per stage)
Reported: ms per backward step and the ratio to open_loop.  The card's name and power limit are read in the same run.  With
--profile DIR, one extra call of each path under torch.profiler writes a kernel table there (not part of the timing).
Usage: python tools/time_pd_vjp.py [--steps N] [--reps N] [--profile DIR]
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
from rigidbodydynamics.jl_b200.autodiff import _model_handle, _pd_trajectory, _trajectory  # noqa: E402
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
    M = rbd.mass_matrix(st).view(nv, nv, B).permute(2, 0, 1).double()       # gains as tools/time_pd.py picks them
    eff = (1.0 / torch.linalg.inv(M).diagonal(dim1=1, dim2=2)).t().contiguous()
    del M
    w = 20.0
    kp = (w * w * eff).to(dtype).contiguous()
    kd = (2 * w * eff).to(dtype).contiguous()
    del eff
    vref = torch.zeros_like(v0)
    f = torch.from_numpy(rng.uniform(0.5, 1.5, (nv, B))).to(dtype).cuda()
    ctrls = {"pd": rbd.JointPD(kp, kd, q0.clone(), vref),
             "pd_shared_gains": rbd.JointPD(kp.min(1).values.contiguous(), kd.min(1).values.contiguous(), q0.clone()),
             "computed_torque": rbd.JointPD((w * w * f).contiguous(), (2 * w * f).contiguous(), q0.clone(), vref, computed_torque=True)}
    h = _model_handle(mech)
    step = nv * B
    qtb = torch.zeros((steps + 1, st.nq, B), dtype=dtype, device="cuda")
    vtb = torch.zeros((steps + 1, nv, B), dtype=dtype, device="cuda")
    qtb[-1].normal_(); vtb[-1].normal_()
    qc, vb, tb = torch.empty_like(q0), torch.empty_like(v0), torch.zeros_like(sched)
    kpb, kdb = torch.zeros_like(v0), torch.zeros_like(v0)

    def open_loop():
        qt, vt = _trajectory(h, q0, v0, sched, 0, steps, step, 0, DT)
        return lambda: rbd.integrate_vjp_(mech, qt, vt, sched, dt=DT, q_traj_bar=qtb, v_traj_bar=vtb, q0_bar_cfg=qc, v0_bar=vb,
                                          tau_bar=tb)

    def closed(ctl):
        qt, vt, _ = _pd_trajectory(h, q0, v0, None, sched, 0, steps, step, 0, ctl, None, DT, "time_pd_vjp")
        qrb = torch.zeros_like(ctl.q_ref)
        vrb = None if ctl.v_ref is None else torch.zeros_like(ctl.v_ref)
        return lambda: rbd.integrate_pd_vjp_(mech, qt, vt, sched, controller=ctl, dt=DT, q_traj_bar=qtb, v_traj_bar=vtb, q0_bar_cfg=qc,
                                             v0_bar=vb, tau_bar=tb, kp_bar=kpb, kd_bar=kdb, q_ref_bar=qrb, v_ref_bar=vrb)
    paths = {"open_loop": open_loop()}
    paths.update({k: closed(c) for k, c in ctrls.items()})
    for k, fn in paths.items():               # warm-up: module loads, specialised kernels, allocator
        fn(); fn()
        torch.cuda.synchronize()
        if not (bool(torch.isfinite(qc).all()) and bool(torch.isfinite(vb).all())):
            raise SystemExit(f"time_pd_vjp: the {k} gradients are not finite")
    best = {k: float("inf") for k in paths}
    for _ in range(3):
        for k, fn in paths.items():
            best[k] = min(best[k], event_ms(fn, reps))
    out = {}
    for k, ms in best.items():
        out[k] = {"ms_per_backward_step": round(ms / steps, 3), "vs_open_loop": round(ms / best["open_loop"], 3)}
    if profile_dir:
        from torch.profiler import ProfilerActivity, profile
        for k, fn in paths.items():
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            with open(os.path.join(profile_dir, f"pd_vjp_{str(dtype)[6:]}_{k}.txt"), "w") as fh:
                fh.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=25))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--profile", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_pd_vjp: no CUDA device")
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
