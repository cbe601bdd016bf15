"""The launch record (rbd_get_launch_info) describes the most recent C-ABI call on this thread: every entry point resets it, and
every kernel the call enqueues -- through nested calls, on every RK4 step and on every chunk -- adds to its count."""
import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from tests.loops_oracle import FOUR_BAR_Q0, four_bar

B = 64


def _atlas_state(batch, seed):
    import torch
    st = rbd.MechanismState(rbd.load_model("atlas", floating=True), batch, torch.float64)
    rbd.rand_(st, np.random.default_rng(seed))
    return st


def _many_launches():
    """A call that enqueues many kernels (RK4 steps), so that a record it leaves behind would show in the next call's."""
    rbd.simulate_(_atlas_state(B, 0), 2e-4, dt=1e-4)
    assert rbd.launch_info().kernels_launched > 2


def _one_generic_launch():
    info = rbd.launch_info()
    return info.kernels_launched, info.specialised


@pytest.mark.gpu
def test_loops_and_vjp_entry_points_reset_the_record(built):
    import torch
    m = four_bar()
    rng = np.random.default_rng(1)
    st = rbd.MechanismState(m, B, torch.float64)
    st.q.copy_(torch.from_numpy(FOUR_BAR_Q0[:, None] + 0.2 * rng.standard_normal((3, B))))
    st.v.copy_(torch.from_numpy(rng.standard_normal((3, B))))
    res = rbd.DynamicsResult(m, B, torch.float64)
    _many_launches()
    rbd.dynamics_loops_(res, st)
    assert _one_generic_launch() == (1, 0)

    st = _atlas_state(B, 2)
    res = rbd.DynamicsResult(st.mechanism, B, torch.float64)
    rbd.dynamics_(res, st)
    bar = torch.rand_like(res.vd)
    out = torch.empty_like(res.vd)
    _many_launches()
    rbd.dynamics_vjp_(st, res.vd, bar, v_bar=out)
    assert _one_generic_launch() == (1, 0)
    _many_launches()
    rbd.inverse_dynamics_vjp_(st, res.vd, bar, v_bar=out)
    assert _one_generic_launch() == (1, 0)


@pytest.mark.gpu
def test_integrate_vjp_counts_every_step(built):
    import torch
    counts = []
    for nsteps in (1, 2, 3):
        st = _atlas_state(B, 3)
        q_traj, v_traj = rbd.simulate_trajectory_(st, nsteps)
        v0_bar = torch.empty((st.nv, B), dtype=torch.float64, device="cuda")
        rbd.integrate_vjp_(st.mechanism, q_traj, v_traj, dt=1e-4, v_traj_bar=torch.ones_like(v_traj), v0_bar=v0_bar)
        counts.append(rbd.launch_info().kernels_launched)
    # the kernel that carries q̄ across a step boundary runs between steps, so the count is linear from one step on
    assert counts[2] - counts[1] == counts[1] - counts[0] > 0, counts


@pytest.mark.gpu
def test_derivatives_count_every_chunk(built, monkeypatch):
    import torch

    def launches(batch):
        st = _atlas_state(batch, 4)
        res = rbd.DynamicsResult(st.mechanism, batch, torch.float64)
        dq = torch.empty((st.nv * st.nv, batch), dtype=torch.float64, device="cuda")
        rbd.dynamics_derivatives_(dq, torch.empty_like(dq), res, st)
        return rbd.launch_info().kernels_launched

    monkeypatch.delenv("RBD_DERIV_SCRATCH_MB", raising=False)
    one_chunk = launches(128)
    monkeypatch.setenv("RBD_DERIV_SCRATCH_MB", "1")     # Atlas fp64 then runs in chunks of 128 samples (the smallest chunk)
    assert launches(256) == 2 * one_chunk
