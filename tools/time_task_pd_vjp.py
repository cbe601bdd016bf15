"""Times the backward step of task-space closed-loop rollouts (rbd_integrate_task_pd_vjp) and prints one JSON line.

Atlas (floating base) at 2^20 samples in fp32 and 2^16 in fp64: both hands as point tasks and both feet as pose tasks (the tasks of
tools/time_task_pd.py), with a JointPD damping term.  Trajectories of `steps` steps are recorded once per path; then the paths
alternate in one process, timed by CUDA events over repeated calls after a warm-up, best of three windows:
  task_pd_backward           integrate_task_pd_vjp_ in torque mode, every controller gradient requested
  task_ct_backward           the same in computed-torque mode (one more inverse-dynamics VJP per stage)
  task_pd_forward            the recorded TaskPD rollout itself (rbd_integrate_task_pd), for scale
  joint_pd_backward          integrate_pd_vjp_ with the damping term alone, for scale
Reported: ms per step.  The card's name and power limit are read in the same run.
Usage: python tools/time_task_pd_vjp.py [--steps N] [--reps N]
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
from rigidbodydynamics.jl_b200.autodiff import _model_handle, _pd_trajectory, _task_trajectory  # noqa: E402
from rigidbodydynamics.jl_b200.kinematics import TaskFrame  # noqa: E402
from tools.time_loops import card, event_ms  # noqa: E402

DT = 1e-3


def case(B, dtype, steps, reps, rng):
    mech = rbd.load_model("atlas", floating=True)
    st = rbd.MechanismState(mech, B, dtype)
    rbd.rand_(st, rng)
    st.v.mul_(0.2)
    q0, v0 = st.q.clone(), st.v.clone()
    nv = st.nv
    f = mech.findbody
    tasks = [TaskFrame(f("l_hand"), None, np.array([0.0, 0.1, 0.0])), TaskFrame(f("r_hand"), None, np.array([0.0, -0.1, 0.0])),
             TaskFrame(f("l_foot"), None, None), TaskFrame(f("r_foot"), None, None)]
    kinds = ["point", "point", "pose", "pose"]
    with torch.no_grad():
        out = rbd.autodiff.task_kinematics(mech, q0, tasks=tasks, outputs=("transform", "point"))
    x_ref = []
    for k, t in enumerate(tasks):                 # targets: the current values, the points moved by 5 cm
        if kinds[k] == "point":
            x_ref.append(out["point"][3 * k:3 * k + 3] + 0.05)
        else:
            x_ref.append(out["transform"][12 * k:12 * k + 12])
    x_ref = torch.cat(x_ref).contiguous()
    R = 18
    kp = torch.full((R,), 100.0, dtype=dtype, device="cuda")
    kd = torch.full((R,), 10.0, dtype=dtype, device="cuda")
    zero, damp = torch.zeros(nv, dtype=dtype, device="cuda"), torch.full((nv,), 2.0, dtype=dtype, device="cuda")
    h = _model_handle(mech)
    qtb = torch.zeros((steps + 1, st.nq, B), dtype=dtype, device="cuda")
    vtb = torch.zeros((steps + 1, nv, B), dtype=dtype, device="cuda")
    qtb[-1].normal_(); vtb[-1].normal_()
    qc, vb = torch.empty_like(q0), torch.empty_like(v0)
    kpb, kdb = torch.zeros((R, B), dtype=dtype, device="cuda"), torch.zeros((R, B), dtype=dtype, device="cuda")
    xrb = torch.zeros_like(x_ref)

    def task_path(ct):
        j = rbd.JointPD(zero, damp, q0.clone(), computed_torque=ct)
        ctl = rbd.TaskPD(tasks, kinds, kp, kd, x_ref, joint=j, computed_torque=ct)
        qt, vt, _ = _task_trajectory(h, mech, q0, v0, None, None, 0, steps, 0, 0, ctl, None, DT, "time_task_pd_vjp")
        jb = [torch.zeros_like(v0), torch.zeros_like(v0), torch.zeros_like(q0), None, None]
        bwd = lambda: rbd.integrate_task_pd_vjp_(mech, qt, vt, controller=ctl, dt=DT, q_traj_bar=qtb, v_traj_bar=vtb,  # noqa: E731
                                                 q0_bar_cfg=qc, v0_bar=vb, kp_bar=kpb, kd_bar=kdb, x_ref_bar=xrb, joint_bars=jb)
        fwd = lambda: _task_trajectory(h, mech, q0, v0, None, None, 0, steps, 0, 0, ctl, None, DT, "time_task_pd_vjp")  # noqa: E731
        return bwd, fwd

    def joint_path():
        j = rbd.JointPD(zero, damp, q0.clone())
        qt, vt, _ = _pd_trajectory(h, q0, v0, None, None, 0, steps, 0, 0, j, None, DT, "time_task_pd_vjp")
        return lambda: rbd.integrate_pd_vjp_(mech, qt, vt, controller=j, dt=DT, q_traj_bar=qtb, v_traj_bar=vtb, q0_bar_cfg=qc,
                                             v0_bar=vb)
    pd_b, pd_f = task_path(False)
    ct_b, _ = task_path(True)
    paths = {"task_pd_backward": pd_b, "task_ct_backward": ct_b, "task_pd_forward": pd_f, "joint_pd_backward": joint_path()}
    for k, fn in paths.items():               # warm-up: module loads, specialised kernels, allocator
        fn(); fn()
        torch.cuda.synchronize()
        if not (bool(torch.isfinite(qc).all()) and bool(torch.isfinite(vb).all())):
            raise SystemExit(f"time_task_pd_vjp: the {k} gradients are not finite")
    best = {k: float("inf") for k in paths}
    for _ in range(3):
        for k, fn in paths.items():
            best[k] = min(best[k], event_ms(fn, reps))
    return {k: {"ms_per_step": round(ms / steps, 3)} for k, ms in best.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_task_pd_vjp: no CUDA device")
    name, power = card()
    rng = np.random.default_rng(0)
    res = {"card": name, "power_limit": power, "steps": a.steps, "dt": DT}
    res["atlas_fp32_2^20"] = case(1 << 20, torch.float32, a.steps, a.reps, rng)
    res["atlas_fp64_2^16"] = case(1 << 16, torch.float64, a.steps, a.reps, rng)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
