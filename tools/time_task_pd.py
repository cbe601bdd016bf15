"""Times task-space feedback (rbd_integrate_task_pd, rbd_task_pd_torques) and prints one JSON line.

Atlas (floating base) with four tasks -- the hands as points (w.r.t. the world), the feet as poses -- at 2^20 samples in fp32 and
2^16 in fp64, 20 RK4 steps at dt = 1e-3.  Paths alternate in one process, timed by CUDA events over repeated calls after a warm-up,
best of three windows:
  open_loop         simulate_ with a per-step torque schedule                         (rbd_integrate_schedule)
  joint_pd          simulate_ with JointPD (per-sample gains, held target)             (rbd_integrate_pd)
  task_pd           TaskPD in torque mode on top of the same JointPD                    (rbd_integrate_task_pd: + 1 kernel / stage)
  task_ct           TaskPD in computed-torque mode with a JointPD damping term           (+ inverse dynamics, finishing kernel)
Reported: ms per RK4 step and the ratio to open_loop.  The law at one state: rbd_task_pd_torques (torque mode, no joint term)
against the composition a user writes without it -- rbd_task_kinematics, the law in torch, rbd_task_kinematics_vjp's v_bar
(tests/test_task_pd.py: composed_task_torques) -- at the same states, ms per call.  Card name and power limit from the same run.
With --profile DIR, one extra run of the one-shot paths under torch.profiler writes a kernel table there.
Usage: python tools/time_task_pd.py [--steps N] [--reps N] [--profile DIR]
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
from rigidbodydynamics.jl_b200.kinematics import TaskFrame  # noqa: E402
from tests.test_task_pd import composed_task_torques  # noqa: E402
from tools.time_loops import card, event_ms  # noqa: E402

DT = 1e-3


def case(B, dtype, steps, reps, rng, profile_dir=None):
    mech = rbd.load_model("atlas", floating=True)
    st = rbd.MechanismState(mech, B, dtype)
    rbd.rand_(st, rng)
    st.v.mul_(0.2)
    st.q[4:7].zero_()
    st.q[6] = 0.9
    q0, v0 = st.q.clone(), st.v.clone()
    nv = st.nv
    sched = torch.from_numpy(rng.random((steps, nv, B)) - 0.5).to(dtype).cuda()
    # joint gains as tools/time_pd.py: critical damping at 20 rad/s times each joint's effective inertia at the start
    M = rbd.mass_matrix(st).view(nv, nv, B).permute(2, 0, 1).double()
    eff = (1.0 / torch.linalg.inv(M).diagonal(dim1=1, dim2=2)).t().contiguous()
    del M
    w = 20.0
    joint = rbd.JointPD((w * w * eff).to(dtype).contiguous(), (2 * w * eff).to(dtype).contiguous(), q0.clone())
    del eff
    dev = lambda a: torch.as_tensor(np.asarray(a, np.float64)).to(dtype).cuda()      # noqa: E731
    tasks = [TaskFrame(mech.findbody("l_hand"), None, [0.0, 0.1, 0.0]), TaskFrame(mech.findbody("r_hand"), None, [0.0, -0.1, 0.0]),
             TaskFrame(mech.findbody("l_foot")), TaskFrame(mech.findbody("r_foot"))]
    kinds = ["point", "point", "pose", "pose"]
    pts = torch.empty((6, B), dtype=dtype, device="cuda")
    rbd.task_kinematics_(st, tasks[:2], point=pts)
    x_ref = torch.cat([pts + 0.05, rbd.relative_transform(st, tasks[2].body), rbd.relative_transform(st, tasks[3].body)]).contiguous()
    kp, kd = dev([50.0] * 6 + [20.0] * 12), dev([5.0] * 6 + [2.0] * 12)
    task_pd = rbd.TaskPD(tasks, kinds, kp, kd, x_ref, joint=joint)
    damp = rbd.JointPD(dev([0.0] * nv), dev([20.0] * nv), q0.clone(), computed_torque=True)
    task_ct = rbd.TaskPD(tasks, kinds, kp * 4, kd * 4, x_ref, joint=damp, computed_torque=True)
    T = steps * DT - 1e-9

    def run(ctrl):
        def f():
            st.q.copy_(q0); st.v.copy_(v0)
            rbd.simulate_(st, T, sched, dt=DT, controller=ctrl)
        return f
    paths = {"open_loop": run(None), "joint_pd": run(joint), "task_pd": run(task_pd), "task_ct": run(task_ct)}
    law = rbd.TaskPD(tasks, kinds, kp, kd, x_ref)
    one = {"task_pd_torques": lambda: rbd.task_pd_torques(st, law), "composition": lambda: composed_task_torques(st, law)}
    st.q.copy_(q0); st.v.copy_(v0)
    a, b = one["task_pd_torques"](), one["composition"]()
    agree = float(((a - b).abs().amax(0) / b.abs().amax(0).clamp(min=1)).max())
    for f in list(paths.values()) + list(one.values()):      # warm-up: module loads, specialised kernels, allocator
        f(); f()
    torch.cuda.synchronize()
    for k, f in paths.items():
        f()
        if not (bool(torch.isfinite(st.q).all()) and bool(torch.isfinite(st.v).all())):
            raise SystemExit(f"time_task_pd: the {k} rollout diverged")
    st.q.copy_(q0); st.v.copy_(v0)
    best = {k: float("inf") for k in list(paths) + list(one)}
    for _ in range(3):
        for k, f in paths.items():
            best[k] = min(best[k], event_ms(f, reps))
        st.q.copy_(q0); st.v.copy_(v0)
        for k, f in one.items():
            best[k] = min(best[k], event_ms(f, 10 * reps))
    out = {}
    for k in paths:
        out[k] = {"ms_per_step": round(best[k] / steps, 4), "vs_open_loop": round(best[k] / best["open_loop"], 3)}
    for k in one:
        out[k] = {"ms_per_call": round(best[k], 4)}
    out["composition_over_task_pd_torques"] = round(best["composition"] / best["task_pd_torques"], 2)
    out["one_shot_relative_difference"] = float(f"{agree:.3g}")
    if profile_dir:
        from torch.profiler import ProfilerActivity, profile
        for k, f in one.items():
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                f()
                torch.cuda.synchronize()
            with open(os.path.join(profile_dir, f"task_pd_{str(dtype)[6:]}_{k}.txt"), "w") as fh:
                fh.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=25))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--profile", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_task_pd: no CUDA device")
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
