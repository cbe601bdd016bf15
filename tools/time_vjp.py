"""Times the reverse-mode products rbd_dynamics_vjp / rbd_inverse_dynamics_vjp and prints one JSON line.

Cases: floating Atlas (fp32 at 2^20, fp64 at 2^16) and the 7-DoF iiwa14 arm (fp32 at 2^20).  In each case four things are timed
alternately in the same process: the forward VJP, the inverse-dynamics VJP, rbd_dynamics (forward dynamics) and the full-Jacobian
route (rbd_dynamics_derivatives plus the batched contraction of both Jacobians with ν̄).  Kernel time by CUDA events over repeated
calls after a warm-up, best of three windows.  The error is the max relative error against the fp64 oracle's dual-number Jacobians
(contracted) and its mass matrix on 512 strided samples.  The card's name and power limit are read in the same run.
Usage: python tools/time_vjp.py [--reps N]
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
from oracle import Oracle  # noqa: E402
from tests.util import oracle_dynamics_derivatives, rel_err  # noqa: E402
from tools.time_loops import card, event_ms  # noqa: E402


def case(name, mech, B, dtype, reps, rng):
    st = rbd.MechanismState(mech, B, dtype)
    rbd.rand_(st, rng)
    nv = st.nv
    T = lambda a: torch.from_numpy(a).to(dtype).cuda()
    tau, nu = T(rng.random((nv, B))), T(rng.standard_normal((nv, B)))
    res = rbd.DynamicsResult(mech, B, dtype)
    rbd.dynamics_(res, st, tau, want_qd=False)
    vd = res.vd.clone()
    e = lambda rows: torch.empty((rows, B), dtype=dtype, device="cuda")
    qb, vb, tb, ab = e(nv), e(nv), e(nv), e(nv)
    dq, dv = e(nv * nv), e(nv * nv)
    fd = lambda: rbd.dynamics_vjp_(st, vd, nu, tau, q_bar_tan=qb, v_bar=vb, tau_bar=tb)
    idv = lambda: rbd.inverse_dynamics_vjp_(st, vd, nu, q_bar_tan=qb, v_bar=vb, vd_bar=ab)
    fwd = lambda: rbd.dynamics_(res, st, tau, want_qd=False)

    def full():
        rbd.dynamics_derivatives_(dq, dv, res, st, tau)
        torch.einsum("jib,ib->jb", dq.view(nv, nv, B), nu)
        torch.einsum("jib,ib->jb", dv.view(nv, nv, B), nu)
    fns = {"dynamics_vjp": fd, "inverse_dynamics_vjp": idv, "rbd_dynamics": fwd, "full_jacobian_route": full}
    for _ in range(3):
        for f in fns.values():
            f()
    torch.cuda.synchronize()
    t = {k: [] for k in fns}
    for _ in range(3):
        for k, f in fns.items():
            t[k].append(event_ms(f, reps))
    # accuracy on 512 strided samples against the fp64 oracle
    idv()
    fd()
    torch.cuda.synchronize()
    idx = torch.arange(5, B, max(1, B // 512), device="cuda")[:512]
    g = lambda x: x[:, idx].double().cpu().numpy()
    q, v, ta, n = g(st.q), g(st.v), g(tau), g(nu)
    o = Oracle(mech.flatten())
    rq, rv = oracle_dynamics_derivatives(o, mech, q, v, ta)
    c = lambda J: np.einsum("jib,ib->jb", J.reshape(nv, nv, -1), n)
    M = o.mass_matrix(q).reshape(nv, nv, -1)
    err = {"dynamics_vjp_q_bar_tan": rel_err(g(qb), c(rq)), "dynamics_vjp_v_bar": rel_err(g(vb), c(rv)),
           "dynamics_vjp_tau_bar": rel_err(g(tb), np.stack([np.linalg.solve(M[:, :, b], n[:, b]) for b in range(n.shape[1])], 1)),
           "inverse_dynamics_vjp_vd_bar": rel_err(g(ab), np.einsum("ijb,jb->ib", M, n))}
    row = {"case": name, "dtype": str(dtype).replace("torch.", ""), "B": B, "nv": nv}
    for k, ts in t.items():
        ms = min(ts)
        row[k + "_ms"] = round(ms, 4)
        row[k + "_M_per_s"] = round(B / ms / 1e3, 2)
    row["max_rel_err_vs_oracle"] = {k: float(f"{x:.3g}") for k, x in err.items()}
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_vjp.py needs a CUDA device")
    rng = np.random.default_rng(2026)
    name, power = card()
    atlas, arm = rbd.load_model("atlas", floating=True), rbd.load_model("iiwa14", floating=False)
    rows = [case("atlas", atlas, 1 << 20, torch.float32, args.reps, rng),
            case("atlas", atlas, 1 << 16, torch.float64, args.reps, rng),
            case("iiwa14", arm, 1 << 20, torch.float32, args.reps, rng)]
    print(json.dumps({"tool": "time_vjp", "gpu": name, "power_limit": power, "results": rows}), flush=True)


if __name__ == "__main__":
    main()
