"""The argument checks of the four rollout VJP entry points (rbd_integrate_vjp, rbd_integrate_contact_vjp, rbd_integrate_pd_vjp,
rbd_integrate_task_pd_vjp), as one table: argument cell x entry point -> status.

Every cell is a call with one bad argument (or an empty batch) that returns before the first CUDA call: the pointers are fake and
never dereferenced, so the table runs with or without a GPU.  A `None` entry marks a cell that does not apply to that entry point
(it has no such argument).  The closed-loop entry points get the contact descriptor too, so the contact cells apply to them.
"""
import ctypes
import math

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from rigidbodydynamics.jl_b200 import _cabi
from rigidbodydynamics.jl_b200.kinematics import TaskFrame, task_desc
from rigidbodydynamics.jl_b200.pd import _RbdPdBar, _RbdPdDesc, _RbdTaskPdBar, _RbdTaskPdDesc

OK, EINVAL, EDIM, EUNSUP = _cabi.RBD_OK, _cabi.RBD_EINVAL, _cabi.RBD_EDIM, _cabi.RBD_EUNSUPPORTED
FAKE = 64                      # never dereferenced by the checks
ENTRY = ("integrate", "contact", "pd", "task")
EMPTY = dict(B=0, q=None, v=None, s=None)

# (cell, arguments that differ from a valid call, expected status per entry point in ENTRY order)
CELLS = [
    ("null_model",         dict(model=None),                     (EINVAL, EINVAL, EINVAL, EINVAL)),
    ("dtype_dual",         dict(dtype=_cabi.RBD_DUAL64X6),       (EUNSUP, EUNSUP, EUNSUP, EUNSUP)),
    ("dtype_7",            dict(dtype=7),                        (EINVAL, EINVAL, EINVAL, EINVAL)),
    ("B_negative",         dict(B=-1),                           (EDIM, EDIM, EDIM, EDIM)),
    ("nsteps_negative",    dict(n=-1),                           (EINVAL, EINVAL, EINVAL, EINVAL)),
    ("dt_zero",            dict(dt=0.0),                         (EINVAL, EINVAL, EINVAL, EINVAL)),
    ("dt_negative",        dict(dt=-1e-3),                       (EINVAL, EINVAL, EINVAL, EINVAL)),
    ("dt_nan",             dict(dt=math.nan),                    (EINVAL, EINVAL, EINVAL, EINVAL)),
    ("step_stride",        dict(step=-1),                        (EINVAL, EINVAL, EINVAL, EINVAL)),
    ("stage_stride",       dict(stage=-4),                       (EINVAL, EINVAL, EINVAL, EINVAL)),
    ("tau_bar_without_tau", dict(tau=None, tau_bar=FAKE),        (EINVAL, EINVAL, EINVAL, EINVAL)),
    ("null_q_traj",        dict(q=None),                         (EINVAL, EINVAL, EINVAL, EINVAL)),
    ("null_v_traj",        dict(v=None),                         (EINVAL, EINVAL, EINVAL, EINVAL)),
    ("null_q_traj_no_step", dict(q=None, n=0),                   (EINVAL, EINVAL, EINVAL, EINVAL)),
    ("empty_batch",        EMPTY,                                (OK, OK, OK, OK)),
    ("null_s_with_pairs",  dict(s=None),                         (None, EINVAL, EINVAL, EINVAL)),
    ("contact_bad_body",   dict(contact="bad_body"),             (None, EINVAL, EINVAL, EINVAL)),
    ("contact_too_many_points", dict(contact="many"),            (None, EUNSUP, EUNSUP, EUNSUP)),
    # the argument that names the entry point: contact, controller (refused also when there is nothing to compute)
    ("null_descriptor",    dict(desc=None),                      (None, EINVAL, EINVAL, EINVAL)),
    ("null_descriptor_empty_batch", dict(desc=None, **EMPTY),    (OK, EINVAL, EINVAL, EINVAL)),
    # the controller: rbd_integrate_pd's / rbd_integrate_task_pd's checks with leading dimension B
    ("controller_unknown_mode", dict(desc="bad_mode"),           (None, None, EINVAL, EINVAL)),
    ("controller_gain_ld", dict(desc="gain_ld"),                 (None, None, EINVAL, EINVAL)),
    ("joint_term_gain_ld", dict(desc="joint_gain_ld"),           (None, None, None, EINVAL)),
    # the adjoint of an array the controller does not have
    ("bar_v_ref_without_v_ref", dict(bar="v_ref"),               (None, None, EINVAL, None)),
    ("bar_vd_ref_without_vd_ref", dict(bar="vd_ref"),            (None, None, EINVAL, None)),
    ("bar_xd_ref_without_xd_ref", dict(bar="xd_ref"),            (None, None, None, EINVAL)),
    ("bar_joint_without_joint", dict(bar="joint"),               (None, None, None, EINVAL)),
    ("bar_joint_v_ref_without_v_ref", dict(desc="joint", bar="joint_v_ref"), (None, None, None, EINVAL)),
    # computed-torque mode runs the inverse-dynamics VJP: a model beyond its limits is refused, even with nothing to compute
    ("computed_torque_model_limits", dict(model="big", desc="ct"), (None, None, EUNSUP, EUNSUP)),
    ("computed_torque_model_limits_empty_batch", dict(model="big", desc="ct", **EMPTY), (None, None, EUNSUP, EUNSUP)),
]

_CASES = [pytest.param(cell, over, entry, want[i], id=f"{cell}-{entry}")
          for cell, over, want in CELLS for i, entry in enumerate(ENTRY) if want[i] is not None]


def _pd(**kw):
    f = dict(mode=0, kp=FAKE, kd=FAKE, gain_ld=0, q_ref=FAKE, v_ref=None, vd_ref=None, q_ref_step_stride=0, v_ref_step_stride=0,
             effort_lo=None, effort_hi=None)
    f.update(kw)
    return _RbdPdDesc(**f)


def _task(mech, keep, joint=None, **kw):
    td, k = task_desc(mech, [TaskFrame(mech.joints[-1].successor, None, None)])
    kind = np.zeros(1, np.int32)
    keep += [td, k, kind, joint]
    f = dict(mode=0, tasks=td, kind=kind.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), kp=FAKE, kd=FAKE, gain_ld=0, x_ref=FAKE,
             x_ref_step_stride=0, xd_ref=None, xd_ref_step_stride=0, joint=None if joint is None else ctypes.pointer(joint),
             effort_lo=None, effort_hi=None)
    f.update(kw)
    return _RbdTaskPdDesc(**f)


@pytest.fixture(scope="module")
def setup(built):
    lib = rbd.load_library()
    mech = rbd.load_model("iiwa14")
    # 21 floating joints: beyond the inverse-dynamics VJP's mass-matrix limit
    big = rbd.rand_chain_mechanism(np.random.default_rng(2), [rbd.QuaternionFloating] * 21)
    handles = {"iiwa14": _cabi.ModelHandle(mech.flatten()), "big": _cabi.ModelHandle(big.flatten())}
    one = lambda *row: np.asarray([row], float)                        # noqa: E731
    cd = rbd.ContactDesc(np.asarray([3], np.int32), one(0.0, 0.0, 0.1), one(50e3, 15e3, 1.5), one(0.8, 20e3, 100.0),
                         one(0.0, 0.0, 0.0, 0.0, 0.0, 1.0))
    assert cd.nstates > 0
    bad = rbd.ContactDesc(np.asarray([99], np.int32), cd.location, cd.normal_model, cd.friction_model, cd.halfspace)
    many = rbd.ContactDesc(np.zeros(33, np.int32), np.zeros((33, 3)), np.ones((33, 3)), np.ones((33, 3)), cd.halfspace)
    keep = []
    contacts = {}
    for name, c in (("ok", cd), ("bad_body", bad), ("many", many)):
        st, k = c.c_struct()
        keep += [st, k]
        contacts[name] = ctypes.byref(st)
    descs = {
        "pd": {"ok": _pd(), "bad_mode": _pd(mode=2), "gain_ld": _pd(gain_ld=3), "ct": _pd(mode=1)},
        "task": {"ok": _task(mech, keep), "bad_mode": _task(mech, keep, mode=3), "gain_ld": _task(mech, keep, gain_ld=3),
                 "joint_gain_ld": _task(mech, keep, _pd(gain_ld=3)), "joint": _task(mech, keep, _pd()), "ct": _task(big, keep, mode=1)},
    }
    jb = _RbdPdBar(None, None, None, FAKE, None)
    bars = {"pd": {"v_ref": _RbdPdBar(None, None, None, FAKE, None), "vd_ref": _RbdPdBar(None, None, None, None, FAKE)},
            "task": {"xd_ref": _RbdTaskPdBar(None, None, None, FAKE, None),
                     "joint": _RbdTaskPdBar(None, None, None, None, ctypes.pointer(_RbdPdBar(FAKE, None, None, None, None))),
                     "joint_v_ref": _RbdTaskPdBar(None, None, None, None, ctypes.pointer(jb))}}
    yield lib, handles, contacts, descs, bars
    del keep
    for h in handles.values():
        h.close()


def _call(setup, entry, model="iiwa14", dtype=_cabi.RBD_F64, B=4, q=FAKE, v=FAKE, s=FAKE, tau=FAKE, tau_bar=None, step=0, stage=0,
          dt=1e-3, n=1, contact="ok", desc="ok", bar=None):
    lib, handles, contacts, descs, bars = setup
    h = None if model is None else handles[model].ptr
    c = contacts[contact]
    if entry == "integrate":
        return lib.rbd_integrate_vjp(h, dtype, B, q, v, tau, step, stage, dt, n, None, None, None, None, None, tau_bar, None)
    if entry == "contact":
        return lib.rbd_integrate_contact_vjp(h, dtype, B, q, v, s, tau, step, stage, None if desc is None else c, dt, n, None, None, None,
                                             None, None, None, None, tau_bar, None)
    d = None if desc is None else ctypes.byref(descs[entry][desc])
    b = None if bar is None else ctypes.byref(bars[entry][bar])
    fn = lib.rbd_integrate_pd_vjp if entry == "pd" else lib.rbd_integrate_task_pd_vjp
    return fn(h, dtype, B, q, v, s, tau, step, stage, d, c, dt, n, None, None, None, None, None, None, None, tau_bar, b, None)


@pytest.mark.parametrize("cell,over,entry,want", _CASES)
def test_rollout_vjp_argument_status(setup, cell, over, entry, want):
    assert _call(setup, entry, **over) == want, setup[0].rbd_last_error()
