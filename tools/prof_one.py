"""Run ONE fp32 forward-dynamics call (batch from argv, default 2^18) -- the target of an ncu capture.
    prof_one.py [batch] [atlas|valkyrie|iiwa14|chainN] [dynamics|id]"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import rigidbodydynamics.jl_b200 as rbd

B = int(sys.argv[1]) if len(sys.argv) > 1 else 1 << 18
name = sys.argv[2] if len(sys.argv) > 2 else "atlas"
algo = sys.argv[3] if len(sys.argv) > 3 else "dynamics"
if name.startswith("chain"):
    n = int(name[5:])
    mech = rbd.rand_chain_mechanism(np.random.default_rng(n), [rbd.Revolute] * n)
else:
    mech = rbd.load_model(name, floating=(name != "iiwa14"))
st = rbd.MechanismState(mech, B, torch.float32)
rbd.rand_(st, np.random.default_rng(1))
x = torch.rand((st.nv, B), dtype=torch.float32, device="cuda")
res = rbd.DynamicsResult(mech, B, torch.float32)
out = torch.empty_like(x)
for _ in range(2):
    if algo == "dynamics":
        rbd.dynamics_(res, st, x, want_qd=False)
    else:
        rbd.inverse_dynamics_(out, st, x)
torch.cuda.synchronize()
