"""Workload for compute-sanitizer: every kernel family once, at batch sizes that take the production paths (model-specialised
kernels at 2^16; generic kernels at 257)."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import rigidbodydynamics.jl_b200 as rbd  # noqa: E402

rng = np.random.default_rng(0)
mech = rbd.load_model("atlas", floating=True)
for dtype in (torch.float32, torch.float64):
    for B in (257, 1 << 16):
        st = rbd.MechanismState(mech, B, dtype)
        rbd.rand_(st, rng)
        tau = torch.rand((st.nv, B), dtype=dtype, device="cuda")
        wext = torch.rand((6 * len(mech.joints), B), dtype=dtype, device="cuda")
        res = rbd.DynamicsResult(mech, B, dtype)
        rbd.dynamics_(res, st, tau)
        rbd.dynamics_(res, st, tau, wext)
        out = torch.empty_like(tau)
        rbd.inverse_dynamics_(out, st, tau)
        rbd.inverse_dynamics_(out, st, tau, wext)
        rbd.dynamics_bias_(out, st)
        # round 2: specialised mass matrix (2^16) / generic (257), analytic Jacobians (specialised and table-driven solve kernels),
        # per-body outputs, soft contact
        M = torch.empty((st.nv * st.nv, B), dtype=dtype, device="cuda")
        rbd.mass_matrix_(M, st)
        rbd.mass_matrix_(M, st, uplo="L")
        nb6 = 6 * len(mech.joints)
        rbd.inverse_dynamics_(out, st, tau, jointwrenchesout=torch.empty((nb6, B), dtype=dtype, device="cuda"),
                              accelerations=torch.empty((nb6, B), dtype=dtype, device="cuda"))
        Bj = min(B, 4096)
        stj = rbd.MechanismState(mech, Bj, dtype)
        stj.q.copy_(st.q[:, :Bj]); stj.v.copy_(st.v[:, :Bj])
        dq = torch.empty((st.nv * st.nv, Bj), dtype=dtype, device="cuda"); dv = torch.empty_like(dq)
        rbd.dynamics_derivatives_(dq, dv, rbd.DynamicsResult(mech, Bj, dtype), stj, tau[:, :Bj].contiguous())
        if B == 257:
            os.environ["RBD_DERIV_JIT"] = "0"
            rbd.dynamics_derivatives_(dq, dv, rbd.DynamicsResult(mech, Bj, dtype), stj, tau[:, :Bj].contiguous())
            os.environ["RBD_DERIV_GLOBAL_FACTOR"] = "1"
            rbd.dynamics_derivatives_(dq, dv, rbd.DynamicsResult(mech, Bj, dtype), stj, tau[:, :Bj].contiguous())
            del os.environ["RBD_DERIV_JIT"], os.environ["RBD_DERIV_GLOBAL_FACTOR"]
            cm = rbd.load_model("atlas", floating=True)
            foot = cm.findbody("r_foot")
            rbd.add_contact_point(foot, rbd.ContactPoint([0.1, 0.0, -0.08], rbd.SoftContactModel(rbd.hunt_crossley_hertz(), rbd.ViscoelasticCoulombModel(0.8, 20e3, 100.0))))
            rbd.add_environment_primitive(cm, rbd.HalfSpace3D([0.0, 0.0, 0.0], [0.0, 0.0, 1.0]))
            cst = rbd.MechanismState(cm, B, dtype)
            cst.q.copy_(st.q); cst.v.copy_(st.v)
            cw = torch.empty((nb6, B), dtype=dtype, device="cuda")
            cs = torch.zeros((rbd.num_contact_states(cm), B), dtype=dtype, device="cuda")
            rbd.contact_dynamics_(cst, cw, cs, torch.empty_like(cs))
        if B == 257:
            rbd.mass_matrix(st)
            p = rbd.path(mech, mech.findbody("r_foot"), mech.findbody("l_hand"))
            outs = {k: torch.empty((r, B), dtype=dtype, device="cuda") for k, r in
                    (("transforms_to_root", 12 * len(mech.joints)), ("center_of_mass", 3), ("kinetic_energy", 1),
                     ("gravitational_potential_energy", 1), ("momentum", 6), ("momentum_rate_bias", 6),
                     ("momentum_matrix", 6 * st.nv), ("geometric_jacobian", 6 * st.nv))}
            rbd.kinematics_(st, p, **outs)
            rbd.simulate_(st, 2e-4, tau, dt=1e-4)
        torch.cuda.synchronize()
        print("ok", dtype, B, rbd.launch_info().kernels_launched)
