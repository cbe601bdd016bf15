"""Times rbd_kinematics_vjp next to the forward rbd_kinematics of the same outputs, in the same run, on Atlas (floating base): fp32
at 2^20 and fp64 at 2^16, kernel time by CUDA events after warm-up, and prints the card name and power limit of the same run.  v is
given and all three gradients are requested; the geometric Jacobian's path runs from l_hand to r_foot.  Cotangent sets:
  (a) center_of_mass + momentum
  (b) momentum_matrix
  (c) all eight outputs
Forward and backward are timed alternately, five windows of ten calls each, and the medians are printed.  At these batch sizes the
forward runs the model-specialised (NVRTC) program, the backward the generic kernel."""
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import rigidbodydynamics.jl_b200 as rbd  # noqa: E402
from rigidbodydynamics.jl_b200.kinematics import _ROWS  # noqa: E402

ALL = ("transforms_to_root", "center_of_mass", "kinetic_energy", "gravitational_potential_energy", "momentum", "momentum_rate_bias",
       "momentum_matrix", "geometric_jacobian")


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
    path = rbd.path(m, m.findbody("l_hand"), m.findbody("r_foot"))
    for dtype, B in ((torch.float32, 1 << 20), (torch.float64, 1 << 16)):
        st = rbd.MechanismState(m, B, dtype)
        rbd.rand_(st, np.random.default_rng(3))
        gen = torch.Generator(device="cuda").manual_seed(0)
        grads = {"q_bar_tan": torch.empty((st.nv, B), dtype=dtype, device="cuda"),
                 "q_bar_cfg": torch.empty((st.nq, B), dtype=dtype, device="cuda"),
                 "v_bar": torch.empty((st.nv, B), dtype=dtype, device="cuda")}
        for label, names in (("(a) center_of_mass + momentum", ("center_of_mass", "momentum")), ("(b) momentum_matrix", ("momentum_matrix",)),
                             ("(c) all eight outputs", ALL)):
            outs = {k: torch.empty((_ROWS[k](st), B), dtype=dtype, device="cuda") for k in names}
            bars = {k: torch.randn((_ROWS[k](st), B), dtype=dtype, device="cuda", generator=gen) for k in names}
            pth = path if "geometric_jacobian" in names else None
            fwd = lambda: rbd.kinematics_(st, pth, **outs)                                       # noqa: E731
            bwd = lambda: rbd.autodiff.kinematics_vjp_(st, pth, bars=bars, **grads)              # noqa: E731
            for fn in (fwd, bwd):
                for _ in range(3):
                    fn()
            torch.cuda.synchronize()
            fwd()
            torch.cuda.synchronize()
            finfo = rbd.launch_info()
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
            print(f"{dtype} B={B} {label}: forward {mf:.3f} ms (runs {', '.join(f'{t:.3f}' for t in tf)}; "
                  f"{'specialised' if finfo.specialised else 'generic'}), backward {mb:.3f} ms (runs {', '.join(f'{t:.3f}' for t in tb)}), "
                  f"backward / forward {mb / mf:.2f}x; backward grid {info.grid} x {info.block}, {info.blocks_per_sm} blocks/SM, "
                  f"{info.kernels_launched} kernel(s)", flush=True)
            del outs, bars
        del st, grads
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
