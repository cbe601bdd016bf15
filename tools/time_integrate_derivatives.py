"""Times rbd_integrate_derivatives (the Jacobians A_s, B_s of every recorded RK4 step) against the ways a user gets them without it,
and prints one JSON line.

Cases: floating Atlas (nv = 36), fp64 and fp32, at a large batch (4096 samples x 4 steps) and an MPC shape (16 samples x 100 steps),
torques per step.  Baselines, timed in the same process with alternating order by CUDA events (best of three windows):
  vjp        rbd_integrate_vjp on the (step, sample) pairs as one-step trajectories, replicated 2nv times with one seed per output
             row: velocity rows one-hot in v̄, configuration rows one-hot in q̄ (configuration coordinates).  Its agreement with the
             new entry is checked on the same run: v̄ = e_r gives row nv + r of [A B]; q̄ = g gives (N(q1)^T g)^T [A B], with N(q1)^T g
             from a zero-step VJP.
  fd         (fp64 only) one batched rbd_integrate over 2 x 3nv perturbed copies of every pair, the cost of central differences
             (the perturbations are random; only the time is reported)
  deriv4     four rbd_dynamics_derivatives_ext calls (with ∂v̇/∂τ) over the pairs: the dense Jacobians alone, a floor
The card's name and power limit are read in the same run.
Usage: python tools/time_integrate_derivatives.py [--reps N]
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
from tools.time_loops import card, event_ms  # noqa: E402

DT = 1e-3


def case(mech, B, n, dtype, reps, rng):
    st = rbd.MechanismState(mech, B, dtype)
    rbd.rand_(st, rng)
    nq, nv = st.nq, st.nv
    N = n * B
    tau = torch.from_numpy(rng.standard_normal((n, nv, B))).to(dtype).cuda()
    qt, vt = rbd.simulate_trajectory_(st, n, tau, dt=DT)
    A = torch.empty((n, 4 * nv * nv, B), dtype=dtype, device="cuda")
    Bm = torch.empty((n, 2 * nv * nv, B), dtype=dtype, device="cuda")
    lib = rbd.load_library()
    from rigidbodydynamics.jl_b200.state import _DT
    stream = lambda: torch.cuda.current_stream().cuda_stream

    def new():
        rbd.autodiff.integrate_derivatives_(mech, qt, vt, tau, dt=DT, A_out=A, B_out=Bm)

    # the pairs as one-step trajectories [2, rows, N] (column s B + b), replicated 2nv times (column r N + s B + b)
    pairs = lambda x: torch.stack([x[:-1].permute(1, 0, 2).reshape(x.shape[1], N), x[1:].permute(1, 0, 2).reshape(x.shape[1], N)])
    R = 2 * nv
    qp = pairs(qt).repeat(1, 1, R).contiguous()
    vp = pairs(vt).repeat(1, 1, R).contiguous()
    tp = tau.permute(1, 0, 2).reshape(nv, N).repeat(1, R).contiguous()
    qtb, vtb = torch.zeros_like(qp), torch.zeros_like(vp)
    for r in range(nv):
        vtb[1, r, r * N:(r + 1) * N] = 1
        qtb[1, r, (nv + r) * N:(nv + r + 1) * N] = 1       # configuration coordinate r (nv <= nq)
    q0t, v0b, tb = torch.empty((nv, R * N), dtype=dtype, device="cuda"), torch.empty((nv, R * N), dtype=dtype, device="cuda"), None
    tb = torch.zeros_like(tp)

    def vjp():
        tb.zero_()
        rbd.integrate_vjp_(mech, qp, vp, tp, dt=DT, q_traj_bar=qtb, v_traj_bar=vtb, q0_bar_tan=q0t, v0_bar=v0b, tau_bar=tb)

    # four dynamics-Jacobian calls over the pairs
    q0p, v0p, t0p = qp[0, :, :N].contiguous(), vp[0, :, :N].contiguous(), tp[:, :N].contiguous()
    vd = torch.empty((nv, N), dtype=dtype, device="cuda")
    Dq, Dv, Dt = (torch.empty((nv * nv, N), dtype=dtype, device="cuda") for _ in range(3))

    def deriv4():
        for _ in range(4):
            rbd._cabi.check(lib.rbd_dynamics_derivatives_ext(st.handle.ptr, _DT[dtype], N, N, q0p.data_ptr(), v0p.data_ptr(),
                                                             t0p.data_ptr(), None, vd.data_ptr(), Dq.data_ptr(), Dv.data_ptr(),
                                                             Dt.data_ptr(), stream()))
    fns = {"new": new, "vjp": vjp, "deriv4": deriv4}
    if dtype == torch.float64:
        M = 6 * nv * N
        qf = q0p.repeat(1, 6 * nv) + 1e-6 * torch.randn((nq, M), dtype=dtype, device="cuda")
        vf = v0p.repeat(1, 6 * nv) + 1e-6 * torch.randn((nv, M), dtype=dtype, device="cuda")
        tf = t0p.repeat(1, 6 * nv).contiguous()
        qw, vw = torch.empty_like(qf), torch.empty_like(vf)

        def fd():
            qw.copy_(qf); vw.copy_(vf)
            rbd._cabi.check(lib.rbd_integrate(st.handle.ptr, _DT[dtype], M, M, qw.data_ptr(), vw.data_ptr(), tf.data_ptr(), DT, 1,
                                              stream()))
        fns["fd"] = fd
    for f in fns.values():
        f(); f()
    torch.cuda.synchronize()
    t = {k: [] for k in fns}
    order = list(fns)
    for w in range(3):
        for k in (order if w % 2 == 0 else order[::-1]):
            t[k].append(event_ms(fns[k], reps))
    out = {k: round(min(v), 4) for k, v in t.items()}
    out.update({f"speedup_vs_{k}": round(min(t[k]) / min(t["new"]), 2) for k in fns if k != "new"})
    # agreement of the VJP composition with the new entry
    new(); vjp()
    torch.cuda.synchronize()
    Av = A.view(n, 2 * nv, 2 * nv, B).transpose(1, 2)
    Bv = Bm.view(n, nv, 2 * nv, B).transpose(1, 2)
    AB = torch.cat([Av, Bv], 2).permute(1, 2, 0, 3).reshape(2 * nv, 3 * nv, N)      # [row, column, pair]
    rows = torch.cat([q0t, v0b, tb]).view(3 * nv, R, N)                              # [column, seed, pair]
    ref_v = rows[:, :nv].permute(1, 0, 2)                                          # seeds r < nv: velocity row r
    err = ((AB[nv:] - ref_v).abs().amax((0, 1)) / AB[nv:].abs().amax((0, 1)).clamp(min=1)).max().item()
    yq = torch.empty((nv, nv * N), dtype=dtype, device="cuda")
    rbd.integrate_vjp_(mech, qp[1:, :, nv * N:].contiguous(), vp[1:, :, nv * N:].contiguous(), None, dt=DT,
                       q_traj_bar=qtb[1:, :, nv * N:].contiguous(), q0_bar_tan=yq)
    yq = yq.view(nv, nv, N)                                                        # [tangent row, seed, pair]
    lhs = torch.einsum("isn,icn->scn", yq, AB[:nv])
    ref_q = rows[:, nv:].permute(1, 0, 2)
    err = max(err, ((lhs - ref_q).abs().amax((0, 1)) / ref_q.abs().amax((0, 1)).clamp(min=1)).max().item())
    out["vjp_agreement_rel_err"] = float(f"{err:.3g}")
    out["ms"] = "per call (all steps and samples)"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    name, power = card()
    mech = rbd.load_model("atlas", floating=True)
    rng = np.random.default_rng(0)
    res = {"card": name, "power_limit": power}
    for dtype in (torch.float64, torch.float32):
        for label, B, n in (("large_4096x4", 4096, 4), ("mpc_16x100", 16, 100)):
            res[f"{label}_{str(dtype)[6:]}"] = case(mech, B, n, dtype, a.reps, rng)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
