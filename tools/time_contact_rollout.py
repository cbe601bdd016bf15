"""Times the contact rollout (rbd_integrate_contact) and prints one JSON line.

Case: floating Atlas with four contact points per foot on a floor, standing (about a third of the samples have a foot on the
floor), constant torques, fp32 at 2^20 and fp64 at 2^16.  Three paths alternate in one process, timed by CUDA events over repeated
calls after a warm-up, best of three windows, in ms per RK4 step:
  (a) rbd_integrate_contact                                       the fused contact pass + forward dynamics per stage
  (b) rbd_integrate on the same tree without contact              the specialised forward-dynamics kernels
  (c) 4 x (rbd_contact_dynamics + rbd_dynamics with wrenches)     the per-stage work the fused kernel replaces, without the
                                                                  RK4 elementwise kernels
A torch.profiler run splits one call of (a) into the fused kernel and the elementwise kernels (RK4 stage / finishing maps and the
contact-state update), so that (a) can be set against (c) plus the elementwise kernels.  The error is against the fp64 oracle
integrator (tests/contact_oracle.py) on strided samples.  The card's name and power limit are read in the same run.
Usage: python tools/time_contact_rollout.py [--steps N] [--reps N]
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
from oracle import Oracle  # noqa: E402
from rigidbodydynamics.jl_b200 import _cabi  # noqa: E402
from rigidbodydynamics.jl_b200.state import _DT  # noqa: E402
from tests.contact_oracle import integrate_contact  # noqa: E402
from tools.time_loops import card, event_ms  # noqa: E402

DT = 1e-3


def atlas_on_floor():
    mech = rbd.load_model("atlas", floating=True)
    model = rbd.SoftContactModel(rbd.hunt_crossley_hertz(), rbd.ViscoelasticCoulombModel(0.8, 20e3, 100.0))
    for foot in ("l_foot", "r_foot"):
        body = mech.findbody(foot)
        for x in (-0.08, 0.17):
            for y in (-0.06, 0.06):
                rbd.add_contact_point(body, rbd.ContactPoint(np.array([x, y, -0.08]), model))
    rbd.add_environment_primitive(mech, rbd.HalfSpace3D(np.zeros(3), [0, 0, 1.0]))
    return mech


def standing(mech, B, rng):
    nq, nv = mech.num_positions(), mech.num_velocities()
    q = np.zeros((nq, B))
    q[:4] = np.array([[1.0], [0], [0], [0]]) + 0.05 * rng.standard_normal((4, B)); q[:4] /= np.linalg.norm(q[:4], axis=0)
    q[4:6] = rng.standard_normal((2, B)); q[6] = 0.93 + 0.03 * rng.standard_normal(B)
    q[7:] = 0.1 * rng.standard_normal((nq - 7, B))
    return q, 0.2 * rng.random((nv, B)), rng.random((nv, B)) - 0.5


def case(mech, cd, B, dtype, steps, reps, rng):
    q, v, tau = standing(mech, B, rng)
    st = rbd.MechanismState(mech, B, dtype)
    nq, nv, nb, ns = st.nq, st.nv, len(mech.joints), cd.nstates
    q0, v0 = torch.from_numpy(q).to(dtype).cuda(), torch.from_numpy(v).to(dtype).cuda()
    tq = torch.from_numpy(tau).to(dtype).cuda()
    s0 = torch.zeros((ns, B), dtype=dtype, device="cuda")
    s = s0.clone()
    wr, sd = torch.empty((6 * nb, B), dtype=dtype, device="cuda"), torch.empty_like(s)
    vd = torch.empty((nv, B), dtype=dtype, device="cuda")
    lib = rbd.load_library()
    c, keep = cd.c_struct()
    h, dt_ = st.handle.ptr, _DT[dtype]
    stream = lambda: torch.cuda.current_stream().cuda_stream    # noqa: E731

    def fused():
        st.q.copy_(q0); st.v.copy_(v0); s.copy_(s0)
        _cabi.check(lib.rbd_integrate_contact(h, dt_, B, B, st.q.data_ptr(), st.v.data_ptr(), s.data_ptr(), tq.data_ptr(), 0, 0,
                                              ctypes.byref(c), DT, steps, None, None, None, stream()))

    def plain():
        st.q.copy_(q0); st.v.copy_(v0)
        _cabi.check(lib.rbd_integrate(h, dt_, B, B, st.q.data_ptr(), st.v.data_ptr(), tq.data_ptr(), DT, steps, stream()))

    def unfused():
        for _ in range(4 * steps):
            _cabi.check(lib.rbd_contact_dynamics(h, dt_, B, B, st.q.data_ptr(), st.v.data_ptr(), ctypes.byref(c), s.data_ptr(),
                                                 sd.data_ptr(), wr.data_ptr(), stream()))
            _cabi.check(lib.rbd_dynamics(h, dt_, B, B, st.q.data_ptr(), st.v.data_ptr(), tq.data_ptr(), wr.data_ptr(), vd.data_ptr(),
                                         None, stream()))
    paths = {"a_integrate_contact": fused, "b_integrate_no_contact": plain, "c_unfused_stage_work": unfused}
    for _ in range(2):
        for f in paths.values():
            f()
    torch.cuda.synchronize()
    t = {k: [] for k in paths}
    for _ in range(3):
        for k, f in paths.items():
            t[k].append(event_ms(f, reps))
    ms = {k: round(min(v) / steps, 4) for k, v in t.items()}
    # split of one fused call: the contact forward-dynamics kernel vs the elementwise RK4 kernels
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fused()
        torch.cuda.synchronize()
    split = {"aba_contact_kernel": 0.0, "elementwise": 0.0}
    for ev in prof.key_averages():
        us = getattr(ev, "device_time_total", None)
        if us is None:
            us = ev.cuda_time_total
        if us > 0 and ("integrate_" in ev.key or "contact_finish" in ev.key):
            split["elementwise"] += us
        elif us > 0 and "aba_contact_kernel" in ev.key:
            split["aba_contact_kernel"] += us
    split = {k: round(v / 1e3 / steps, 4) for k, v in split.items()}
    # accuracy: the last fused run against the fp64 oracle on strided samples
    fused()
    idx = np.arange(0, B, max(1, B // 48))
    rd = lambda a: a[:, idx].astype(np.float32).astype(np.float64) if dtype == torch.float32 else a[:, idx]    # noqa: E731
    qr, vr, sr = integrate_contact(Oracle(mech.flatten()), rd(q), rd(v), np.zeros((ns, idx.size)), cd, rd(tau), dt=DT, nsteps=steps)
    qg, vg = st.q[:, idx].double().cpu().numpy(), st.v[:, idx].double().cpu().numpy()
    qg[:4] *= np.sign((qg[:4] * qr[:4]).sum(0))
    err = lambda a, b: float((np.abs(a - b).max(0) / np.maximum(1.0, np.abs(b).max(0))).max())    # noqa: E731
    return {"dtype": str(dtype).replace("torch.", ""), "B": B, "steps": steps, "contact_points": cd.npoints, "contact_states": ns,
            "ms_per_step": ms, "fused_call_split_ms_per_step": split,
            "c_plus_elementwise_ms_per_step": round(ms["c_unfused_stage_work"] + split["elementwise"], 4),
            "fused_speedup_vs_unfused": round((ms["c_unfused_stage_work"] + split["elementwise"]) / ms["a_integrate_contact"], 3),
            "feet_on_floor_share": round(float((s.abs().reshape(-1, 3, B).sum(1) > 0).any(0).float().mean()), 3),
            "err_vs_fp64_oracle": {"q": err(qg, qr), "v": err(vg, vr), "s": err(s[:, idx].double().cpu().numpy(), sr)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_contact_rollout.py needs a CUDA device")
    rng = np.random.default_rng(2026)
    name, power = card()
    mech = atlas_on_floor()
    cd = rbd.contact_desc(mech)
    rows = [case(mech, cd, 1 << 20, torch.float32, args.steps, args.reps, rng),
            case(mech, cd, 1 << 16, torch.float64, args.steps, args.reps, rng)]
    print(json.dumps({"tool": "time_contact_rollout", "gpu": name, "power_limit": power, "results": rows}), flush=True)


if __name__ == "__main__":
    main()
