"""Times the loop rollout (rbd_integrate_loops) and prints one JSON line.

Cases: the four-bar linkage (fp64 and fp32 at 2^20), Atlas in double support (both feet welded: fp32 at 2^20, fp64 at 2^16) and
Atlas in single support (left foot welded, 4 contact points on the right foot over a floor: fp32 at 2^20), constant torques.  Two
paths alternate in one process, timed by CUDA events over repeated calls after a warm-up, best of three windows:
  (a) rbd_integrate_loops                  ms per RK4 step and sample-steps/s
  (b) 4 x rbd_dynamics_loops               the KKT solve a step evaluates four times, as single calls (no contact), same states
The card's name and power limit are read in the same run.
Usage: python tools/time_loops_rollout.py [--steps N] [--reps N]
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
from rigidbodydynamics.jl_b200.spatial import Transform3D  # noqa: E402
from tests.loops_oracle import FOUR_BAR_Q0, atlas_double_support, four_bar  # noqa: E402
from tools.time_loops import card, event_ms  # noqa: E402

DT = 1e-3


def atlas_single_support():
    mech = rbd.load_model("atlas", floating=True)
    mech.attach(mech.root_body, mech.findbody("l_foot"), rbd.Joint("l_foot_weld", rbd.Fixed()),
                joint_pose=Transform3D(trans=(0.0, 0.12, 0.0)), successor_pose=Transform3D.identity())
    model = rbd.SoftContactModel(rbd.hunt_crossley_hertz(), rbd.ViscoelasticCoulombModel(0.8, 20e3, 100.0))
    for x in (-0.08, 0.17):
        for y in (-0.06, 0.06):
            rbd.add_contact_point(mech.findbody("r_foot"), rbd.ContactPoint(np.array([x, y, -0.08]), model))
    rbd.add_environment_primitive(mech, rbd.HalfSpace3D(np.zeros(3), [0, 0, 1.0]))
    return mech


def states(name, mech, B, rng):
    nq, nv = mech.num_positions(), mech.num_velocities()
    if name == "four_bar":
        q = FOUR_BAR_Q0[:, None] + 0.2 * rng.standard_normal((3, B))
        return q, rng.standard_normal((3, B)), rng.standard_normal((3, B))
    q = np.zeros((nq, B))
    q[:4] = np.array([[1.0], [0], [0], [0]]) + 0.05 * rng.standard_normal((4, B)); q[:4] /= np.linalg.norm(q[:4], axis=0)
    q[4:6] = 0.02 * rng.standard_normal((2, B)); q[6] = 0.93 + 0.03 * rng.standard_normal(B)
    q[7:] = 0.1 * rng.standard_normal((nq - 7, B))
    return q, 0.2 * rng.random((nv, B)), rng.random((nv, B)) - 0.5


def case(name, mech, B, dtype, steps, reps, rng):
    q, v, tau = states(name, mech, B, rng)
    st = rbd.MechanismState(mech, B, dtype)
    cd = rbd.contact_desc(mech)
    ns = cd.nstates
    q0, v0 = torch.from_numpy(q).to(dtype).cuda(), torch.from_numpy(v).to(dtype).cuda()
    tq = torch.from_numpy(tau).to(dtype).cuda()
    s0 = torch.zeros((ns, B), dtype=dtype, device="cuda")
    s = s0.clone()
    vd = torch.empty((st.nv, B), dtype=dtype, device="cuda")
    lib = rbd.load_library()
    lst, keep = rbd.loop_desc(mech).c_struct()
    cst, keep2 = cd.c_struct()
    h, dt_ = st.handle.ptr, _DT[dtype]
    stream = lambda: torch.cuda.current_stream().cuda_stream    # noqa: E731

    def rollout():
        st.q.copy_(q0); st.v.copy_(v0); s.copy_(s0)
        _cabi.check(lib.rbd_integrate_loops(h, dt_, B, B, st.q.data_ptr(), st.v.data_ptr(), s.data_ptr() if ns else None, tq.data_ptr(),
                                            0, 0, ctypes.byref(lst), ctypes.byref(cst) if ns else None, DT, steps, None, None, None,
                                            stream()))

    def single():
        st.q.copy_(q0); st.v.copy_(v0)
        for _ in range(4 * steps):
            _cabi.check(lib.rbd_dynamics_loops(h, dt_, B, B, st.q.data_ptr(), st.v.data_ptr(), tq.data_ptr(), None, ctypes.byref(lst),
                                               vd.data_ptr(), None, None, None, None, stream()))
    paths = {"a_integrate_loops": rollout, "b_4x_dynamics_loops": single}
    for f in paths.values():
        f()
    torch.cuda.synchronize()
    t = {k: [] for k in paths}
    for _ in range(3):
        for k, f in paths.items():
            t[k].append(event_ms(f, reps))
    ms = {k: round(min(v) / steps, 3) for k, v in t.items()}
    rollout()
    torch.cuda.synchronize()
    finite = bool(torch.isfinite(st.q).all()) and bool(torch.isfinite(st.v).all())
    return {"case": name, "dtype": str(dtype).replace("torch.", ""), "B": B, "steps": steps, "constraints": int(rbd.num_constraints(mech)),
            "contact_points": cd.npoints, "ms_per_step": ms,
            "sample_steps_per_s": round(B / (ms["a_integrate_loops"] * 1e-3), 1),
            "rollout_vs_4x_single": round(ms["a_integrate_loops"] / ms["b_4x_dynamics_loops"], 3), "finite": finite}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_loops_rollout.py needs a CUDA device")
    rng = np.random.default_rng(2026)
    name, power = card()
    fb, ds, ss = four_bar(), atlas_double_support(), atlas_single_support()
    rows = [case("four_bar", fb, 1 << 20, torch.float64, args.steps, args.reps, rng),
            case("four_bar", fb, 1 << 20, torch.float32, args.steps, args.reps, rng),
            case("atlas_double_support", ds, 1 << 20, torch.float32, args.steps, args.reps, rng),
            case("atlas_double_support", ds, 1 << 16, torch.float64, args.steps, args.reps, rng),
            case("atlas_single_support_contact", ss, 1 << 20, torch.float32, args.steps, args.reps, rng)]
    print(json.dumps({"tool": "time_loops_rollout", "gpu": name, "power_limit": power, "results": rows}), flush=True)


if __name__ == "__main__":
    main()
