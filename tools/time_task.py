"""Times rbd_task_kinematics on Atlas (floating base), batch 2^20, fp32 and fp64, kernel time by CUDA events after warm-up, and prints
the card name and power limit of the same run.  Four tasks: l_hand, r_hand, l_foot, r_foot relative to the world, root frame.
  (a) point + point_jacobian                       fp32 I/O 148 B in + 1776 B out = 1924 B/eval
  (b) all eight outputs with v and v̇                fp32 I/O 436 B in + 5712 B out = 6148 B/eval   (fp64: twice both)
and, alternating with (a) in the same run, today's composition of (a): four rbd_kinematics geometric-Jacobian calls, one
transforms_to_root call and the torch code that forms the point positions and the 3-row point Jacobians; both must give the
same numbers.  The HBM bound is bytes / 3.35 TB/s (H100 SXM data sheet)."""
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import rigidbodydynamics.jl_b200 as rbd  # noqa: E402
from rigidbodydynamics.jl_b200.kinematics import TaskFrame  # noqa: E402

HBM = 3.35e12
NAMES = ("l_hand", "r_hand", "l_foot", "r_foot")
POINTS = ([0.0, 0.1, 0.0], [0.0, -0.1, 0.0], [0.05, 0.0, -0.05], [0.05, 0.0, -0.05])


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
    nb, nv = len(m.joints), m.num_velocities()
    B = 1 << 20
    index = {id(j.successor): i for i, j in enumerate(m.joints)}
    bodies = [m.findbody(n) for n in NAMES]
    tasks = [TaskFrame(b, None, p, None) for b, p in zip(bodies, POINTS)]
    K = len(tasks)
    for dtype in (torch.float32, torch.float64):
        es = 4 if dtype == torch.float32 else 8
        st = rbd.MechanismState(m, B, dtype)
        rbd.rand_(st, np.random.default_rng(3))
        vd = torch.rand((nv, B), dtype=dtype, device="cuda")
        new = lambda r: torch.empty((r, B), dtype=dtype, device="cuda")     # noqa: E731
        pa = {"point": new(3 * K), "point_jacobian": new(3 * nv * K)}
        pb = {"transform": new(12 * K), "point": new(3 * K), "twist": new(6 * K), "point_velocity": new(3 * K),
              "geometric_jacobian": new(6 * nv * K), "point_jacobian": new(3 * nv * K), "acceleration": new(6 * K),
              "point_acceleration": new(3 * K)}
        # today's composition of (a)
        paths = [rbd.path(m, m.root_body, b) for b in bodies]
        Js = [new(6 * nv) for _ in bodies]
        tr = new(12 * nb)
        pts = torch.tensor(POINTS, dtype=dtype, device="cuda")                  # [K, 3]
        rows = torch.tensor([index[id(b)] for b in bodies], device="cuda")
        comp_pt, comp_jp = new(3 * K), new(3 * nv * K)

        def composition():
            for J, pth in zip(Js, paths):
                rbd.kinematics_(st, pth, geometric_jacobian=J)
            rbd.transforms_to_root_(tr, st)
            T = tr.view(nb, 12, B)[rows]                                        # [K, 12, B]
            R, p = T[:, :9].view(K, 3, 3, B), T[:, 9:]
            proot = p + torch.einsum("kijb,kj->kib", R, pts)                    # [K, 3, B]
            comp_pt.view(K, 3, B).copy_(proot)
            for k, J in enumerate(Js):
                Jc = J.view(nv, 6, B)
                w, l = Jc[:, :3], Jc[:, 3:]
                pr = proot[k].unsqueeze(0).expand_as(w)
                comp_jp.view(K, nv, 3, B)[k].copy_(l + torch.linalg.cross(w, pr, dim=1))

        fa = lambda: rbd.task_kinematics_(st, tasks, None, **pa)               # noqa: E731
        fb = lambda: rbd.task_kinematics_(st, tasks, vd, **pb)                 # noqa: E731
        for fn in (fa, fb, composition):
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        scale = max(1.0, float(comp_jp.abs().max()))
        err = max(float((pa["point"] - comp_pt).abs().max()), float((pa["point_jacobian"] - comp_jp).abs().max())) / scale
        tol = 1e-5 if dtype == torch.float32 else 1e-12
        print(f"{dtype}: task call vs composition, max |difference| / max(1, |J|) = {err:.2e} (tol {tol:g})", flush=True)
        assert err < tol
        ta, tc = [], []
        for _ in range(5):                    # alternate the two ways of computing (a)
            ta.append(timed(fa, 10))
            tc.append(timed(composition, 10))
        tb = [timed(fb, 10) for _ in range(3)]
        fa()
        torch.cuda.synchronize()
        info = rbd.launch_info()
        bytes_a = es * ((m.num_positions()) + K * (3 + 3 * nv))
        bytes_b = es * (m.num_positions() + 2 * nv + K * (12 + 3 + 6 + 3 + 6 * nv + 3 * nv + 6 + 3))
        for name, ts, byts in (("(a) point + point_jacobian", ta, bytes_a), ("(b) all eight outputs", tb, bytes_b)):
            ms = float(np.median(ts))
            rate = B / ms * 1e3
            bound = HBM / byts
            print(f"{dtype} {name}: {ms:.3f} ms (runs {', '.join(f'{t:.3f}' for t in ts)}), {rate / 1e6:.1f} M evals/s, "
                  f"{byts} B/eval, HBM bound {bound / 1e6:.0f} M evals/s, {100 * rate / bound:.1f} % of it", flush=True)
        mc = float(np.median(tc))
        print(f"{dtype} composition of (a): {mc:.3f} ms (runs {', '.join(f'{t:.3f}' for t in tc)}), {B / mc / 1e3:.1f} M evals/s; "
              f"task call speedup {mc / float(np.median(ta)):.2f}x; task kernel grid {info.grid} x {info.block}, smem {info.smem_bytes} B, "
              f"{info.blocks_per_sm} blocks/SM", flush=True)
        del st, pa, pb, Js, tr, comp_pt, comp_jp
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
