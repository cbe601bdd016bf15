"""Times the complete linearisation entry points against the plain analytic Jacobians (rbd_dynamics_derivatives), kernel time by CUDA
events, launch counts from launch_info(), card name and power limit printed in the same run:
  fd           dynamics_derivatives_                        d v̇ / dq, d v̇ / dv
  fd+wext      ... with external wrenches
  fd+dtau      ... with d v̇ / d tau = M^-1 (the solve's third block)
  fd+wext+dtau both
  id           inverse_dynamics_derivatives_ with wrenches  d tau / dq, d tau / dv
  id+tau+M     ... with tau and M
The variants alternate within each round; each line is the best of the rounds.  usage: time_deriv_ext.py [model] [log2 batch ...]"""
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import rigidbodydynamics.jl_b200 as rbd  # noqa: E402

name = sys.argv[1] if len(sys.argv) > 1 else "atlas"
logs = [int(a) for a in sys.argv[2:]] or [13, 14, 15, 16]
m = rbd.load_model(name, floating=(name != "iiwa14"))
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                          timeout=30).stdout.strip().splitlines()[0]
except Exception as e:          # the card name alone still comes from torch
    card = f"{torch.cuda.get_device_name(0)} (power limit not available: {e})"
print(f"card: {card}", flush=True)
ROUNDS, N = 5, 10
for dtype in (torch.float64, torch.float32):
    for lb in logs:
        B = 1 << lb
        st = rbd.MechanismState(m, B, dtype)
        rbd.rand_(st, np.random.default_rng(1))
        nv, nb = st.nv, len(m.joints)
        tau = torch.rand((nv, B), dtype=dtype, device="cuda")
        w = torch.rand((6 * nb, B), dtype=dtype, device="cuda")
        res = rbd.DynamicsResult(m, B, dtype)
        new = lambda rows: torch.empty((rows, B), dtype=dtype, device="cuda")      # noqa: E731
        dq, dv, dt, tq = new(nv * nv), new(nv * nv), new(nv * nv), new(nv)
        M = new(nv * nv)
        vd = torch.rand((nv, B), dtype=dtype, device="cuda")
        variants = {
            "fd": lambda: rbd.dynamics_derivatives_(dq, dv, res, st, tau),
            "fd+wext": lambda: rbd.dynamics_derivatives_(dq, dv, res, st, tau, w),
            "fd+dtau": lambda: rbd.dynamics_derivatives_(dq, dv, res, st, tau, None, dt),
            "fd+wext+dtau": lambda: rbd.dynamics_derivatives_(dq, dv, res, st, tau, w, dt),
            "id": lambda: rbd.inverse_dynamics_derivatives_(dq, dv, st, vd, w),
            "id+tau+M": lambda: rbd.inverse_dynamics_derivatives_(dq, dv, st, vd, w, torques=tq, massmatrix=M),
        }
        best, launches = {k: float("inf") for k in variants}, {}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for f in variants.values():
            f(); f()
        torch.cuda.synchronize()
        for _ in range(ROUNDS):
            for k, f in variants.items():
                e0.record()
                for _ in range(N):
                    f()
                e1.record()
                torch.cuda.synchronize()
                best[k] = min(best[k], e0.elapsed_time(e1) / N)
                launches[k] = rbd.launch_info().kernels_launched
        base = best["fd"]
        for k in variants:
            print(f"{name} {str(dtype)[6:]} B=2^{lb} {k:13s} {best[k]:8.3f} ms  {B / best[k] / 1e3:7.2f} M samples/s  "
                  f"{best[k] / base:5.2f}x fd  {launches[k]} launches", flush=True)
        del dq, dv, dt, tq, M, res, st, tau, w, vd
        torch.cuda.empty_cache()
