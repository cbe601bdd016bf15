"""Times the backward pass of the contact rollout (rbd_integrate_contact_vjp) and prints one JSON line.

Case: floating Atlas with four contact points per foot on a floor, standing (tools/time_contact_rollout.py), constant torques,
fp32 at 2^20 and fp64 at 2^16.  Three paths alternate in one process, timed by CUDA events over repeated calls after a warm-up,
best of three windows, in ms per RK4 step and sample-steps per second:
  (a) rbd_integrate_contact_vjp                  backward through the contact rollout (recompute + adjoint)
  (b) rbd_integrate_contact                      the forward contact rollout
  (c) rbd_integrate_vjp on the same tree         backward through the rollout without contact (DESIGN 4.13)
The card's name and power limit are read in the same run.
Usage: python tools/time_contact_vjp.py [--steps N] [--reps N]
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import rigidbodydynamics.jl_b200 as rbd  # noqa: E402
from rigidbodydynamics.jl_b200 import _cabi  # noqa: E402
from rigidbodydynamics.jl_b200.state import _DT  # noqa: E402
from tools.time_contact_rollout import DT, atlas_on_floor, standing  # noqa: E402
from tools.time_loops import card, event_ms  # noqa: E402


def case(mech, cd, B, dtype, steps, reps, rng):
    q, v, tau = standing(mech, B, rng)
    st = rbd.MechanismState(mech, B, dtype)
    nq, nv, ns = st.nq, st.nv, cd.nstates
    q0, v0 = torch.from_numpy(q).to(dtype).cuda(), torch.from_numpy(v).to(dtype).cuda()
    tq = torch.from_numpy(tau).to(dtype).cuda()
    s = torch.zeros((ns, B), dtype=dtype, device="cuda")
    st.q.copy_(q0); st.v.copy_(v0)
    qt, vt, stj = rbd.simulate_contact_trajectory_(st, steps, s, tq, dt=DT, contact=cd)
    qtb, vtb, stb = torch.zeros_like(qt), torch.randn_like(vt), torch.zeros_like(stj)
    qtb[-1].normal_(); stb[-1].normal_()
    e = lambda rows: torch.empty((rows, B), dtype=dtype, device="cuda")     # noqa: E731
    qc, vb, sb, tb = e(nq), e(nv), e(ns), torch.zeros_like(tq)
    lib = rbd.load_library()
    c, keep = cd.c_struct()
    h, dt_ = st.handle.ptr, _DT[dtype]
    stream = lambda: torch.cuda.current_stream().cuda_stream    # noqa: E731
    p = lambda x: x.data_ptr()      # noqa: E731

    def backward_contact():
        _cabi.check(lib.rbd_integrate_contact_vjp(h, dt_, B, p(qt), p(vt), p(stj), p(tq), 0, 0, ctypes.byref(c), DT, steps, p(qtb), p(vtb),
                                                  p(stb), None, p(qc), p(vb), p(sb), p(tb), stream()))

    def forward_contact():
        st.q.copy_(q0); st.v.copy_(v0); s.zero_()
        _cabi.check(lib.rbd_integrate_contact(h, dt_, B, B, p(st.q), p(st.v), p(s), p(tq), 0, 0, ctypes.byref(c), DT, steps, None, None,
                                              None, stream()))

    def backward_plain():
        _cabi.check(lib.rbd_integrate_vjp(h, dt_, B, p(qt), p(vt), p(tq), 0, 0, DT, steps, p(qtb), p(vtb), None, p(qc), p(vb), p(tb),
                                          stream()))
    paths = {"a_contact_vjp": backward_contact, "b_contact_forward": forward_contact, "c_vjp_no_contact": backward_plain}
    for _ in range(2):
        for f in paths.values():
            f()
    torch.cuda.synchronize()
    t = {k: [] for k in paths}
    for _ in range(3):
        for k, f in paths.items():
            t[k].append(event_ms(f, reps))
    ms = {k: round(min(v) / steps, 4) for k, v in t.items()}
    backward_contact()
    torch.cuda.synchronize()
    finite = bool(torch.isfinite(qc).all() and torch.isfinite(vb).all() and torch.isfinite(sb).all() and torch.isfinite(tb).all())
    rate = lambda k: round(B / (ms[k] * 1e-3) / 1e6, 3)      # noqa: E731
    return {"dtype": str(dtype).replace("torch.", ""), "B": B, "steps": steps, "contact_points": cd.npoints, "ms_per_step": ms,
            "M_sample_steps_per_s": {k: rate(k) for k in ms},
            "backward_over_forward_contact": round(ms["a_contact_vjp"] / ms["b_contact_forward"], 3),
            "backward_over_backward_no_contact": round(ms["a_contact_vjp"] / ms["c_vjp_no_contact"], 3),
            "feet_on_floor_share": round(float((stj[-1].abs().reshape(-1, 3, B).sum(1) > 0).any(0).float().mean()), 3),
            "gradients_finite": finite}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_contact_vjp.py needs a CUDA device")
    rng = np.random.default_rng(2026)
    name, power = card()
    mech = atlas_on_floor()
    cd = rbd.contact_desc(mech)
    rows = [case(mech, cd, 1 << 20, torch.float32, args.steps, args.reps, rng),
            case(mech, cd, 1 << 16, torch.float64, args.steps, args.reps, rng)]
    print(json.dumps({"tool": "time_contact_vjp", "gpu": name, "power_limit": power, "results": rows}), flush=True)


if __name__ == "__main__":
    main()
