"""Times rbd_task_kinematics_vjp next to the forward rbd_task_kinematics of the same outputs, in the same run, on Atlas (floating
base): fp32 at 2^20 and fp64 at 2^16, kernel time by CUDA events after warm-up, and prints the card name and power limit of the same
run.  The four end-effector tasks of tools/time_task.py (l_hand, r_hand, l_foot, r_foot relative to the world, root frame), v and
v̇ given, all four gradients requested:
  (a) cotangents on point + point_jacobian
  (b) cotangents on all eight outputs
Forward and backward are timed alternately."""
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import rigidbodydynamics.jl_b200 as rbd  # noqa: E402
from rigidbodydynamics.jl_b200.kinematics import _TASK_ROWS, TaskFrame  # noqa: E402

NAMES = ("l_hand", "r_hand", "l_foot", "r_foot")
POINTS = ([0.0, 0.1, 0.0], [0.0, -0.1, 0.0], [0.05, 0.0, -0.05], [0.05, 0.0, -0.05])
ALL = ("transform", "point", "twist", "point_velocity", "geometric_jacobian", "point_jacobian", "acceleration", "point_acceleration")


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"device: {torch.cuda.get_device_name(0)}; nvidia-smi name, power limit: {smi.stdout.strip()}", flush=True)
    m = rbd.load_model("atlas", floating=True)
    nv = m.num_velocities()
    tasks = [TaskFrame(m.findbody(n), None, p, None) for n, p in zip(NAMES, POINTS)]
    K = len(tasks)
    for dtype, B in ((torch.float32, 1 << 20), (torch.float64, 1 << 16)):
        st = rbd.MechanismState(m, B, dtype)
        rbd.rand_(st, np.random.default_rng(3))
        gen = torch.Generator(device="cuda").manual_seed(0)
        vd = torch.rand((nv, B), dtype=dtype, device="cuda", generator=gen)
        grads = {"q_bar_tan": torch.empty((nv, B), dtype=dtype, device="cuda"),
                 "q_bar_cfg": torch.empty((st.nq, B), dtype=dtype, device="cuda"),
                 "v_bar": torch.empty((nv, B), dtype=dtype, device="cuda"), "vd_bar": torch.empty((nv, B), dtype=dtype, device="cuda")}
        for label, names in (("(a) point + point_jacobian", ("point", "point_jacobian")), ("(b) all eight outputs", ALL)):
            outs = {k: torch.empty((_TASK_ROWS[k](st) * K, B), dtype=dtype, device="cuda") for k in names}
            bars = {k: torch.randn((_TASK_ROWS[k](st) * K, B), dtype=dtype, device="cuda", generator=gen) for k in names}
            fwd = lambda: rbd.task_kinematics_(st, tasks, vd, **outs)                              # noqa: E731
            bwd = lambda: rbd.autodiff.task_kinematics_vjp_(st, tasks, vd, bars=bars, **grads)      # noqa: E731
            for fn in (fwd, bwd):
                for _ in range(3):
                    fn()
            torch.cuda.synchronize()
            bwd()
            torch.cuda.synchronize()
            info = rbd.launch_info()
            tf, tb = [], []
            for _ in range(5):
                tf.append(timed(fwd, 10))
                tb.append(timed(bwd, 10))
            for g in grads.values():
                assert torch.isfinite(g).all()
            mf, mb = float(np.median(tf)), float(np.median(tb))
            print(f"{dtype} B={B} {label}: forward {mf:.3f} ms (runs {', '.join(f'{t:.3f}' for t in tf)}), backward {mb:.3f} ms "
                  f"(runs {', '.join(f'{t:.3f}' for t in tb)}), backward / forward {mb / mf:.2f}x; backward grid {info.grid} x "
                  f"{info.block}, {info.blocks_per_sm} blocks/SM, {info.kernels_launched} kernel(s)", flush=True)
            del outs, bars
        del st, grads
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
