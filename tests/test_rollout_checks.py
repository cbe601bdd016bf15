"""The argument checks of the six RK4 rollout entry points (rbd_integrate, rbd_integrate_schedule, rbd_integrate_trajectory,
rbd_integrate_contact, rbd_integrate_loops, rbd_integrate_pd), as one table: argument cell x entry point -> status.

Every cell is a call with one bad argument (or an empty batch) that returns before the first CUDA call: the pointers are fake and
never dereferenced, so the table runs with or without a GPU.  A `None` entry marks a cell that does not apply to that entry point
(it has no such argument).
"""
import ctypes
import math

import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from rigidbodydynamics.jl_b200 import _cabi

OK, EINVAL, EDIM, EUNSUP = _cabi.RBD_OK, _cabi.RBD_EINVAL, _cabi.RBD_EDIM, _cabi.RBD_EUNSUPPORTED
FAKE = 64                      # never dereferenced by the checks
ENTRY = ("integrate", "schedule", "trajectory", "contact", "loops", "pd")


class _PdDesc(ctypes.Structure):
    _fields_ = [("mode", ctypes.c_int32), ("kp", ctypes.c_void_p), ("kd", ctypes.c_void_p), ("gain_ld", ctypes.c_int64),
                ("q_ref", ctypes.c_void_p), ("v_ref", ctypes.c_void_p), ("vd_ref", ctypes.c_void_p),
                ("q_ref_step_stride", ctypes.c_int64), ("v_ref_step_stride", ctypes.c_int64),
                ("effort_lo", ctypes.POINTER(ctypes.c_double)), ("effort_hi", ctypes.POINTER(ctypes.c_double))]


# (cell, arguments that differ from a valid call, expected status per entry point in ENTRY order)
CELLS = [
    ("null_model",         dict(model=None),                     (EINVAL, EINVAL, EINVAL, EINVAL, EINVAL, EINVAL)),
    ("dtype_dual",         dict(dtype=_cabi.RBD_DUAL64X6),       (EUNSUP, EUNSUP, EUNSUP, EUNSUP, EUNSUP, EUNSUP)),
    ("dtype_7",            dict(dtype=7),                        (EINVAL, EINVAL, EINVAL, EUNSUP, EUNSUP, EUNSUP)),
    ("B_gt_ld",            dict(B=8, ld=4),                      (EDIM, EDIM, EDIM, EDIM, EDIM, EDIM)),
    ("nsteps_negative",    dict(n=-1),                           (EINVAL, EINVAL, EINVAL, EINVAL, EINVAL, EINVAL)),
    ("dt_zero",            dict(dt=0.0),                         (EINVAL, EINVAL, EINVAL, EINVAL, EINVAL, EINVAL)),
    ("dt_negative",        dict(dt=-1e-3),                       (EINVAL, EINVAL, EINVAL, EINVAL, EINVAL, EINVAL)),
    ("dt_nan",             dict(dt=math.nan),                    (EINVAL, EINVAL, EINVAL, EINVAL, EINVAL, EINVAL)),
    ("step_stride",        dict(step=-1),                        (None, EINVAL, EINVAL, EINVAL, EINVAL, EINVAL)),
    ("stage_stride",       dict(stage=-4),                       (None, EINVAL, EINVAL, EINVAL, EINVAL, EINVAL)),
    ("null_q",             dict(q=None),                         (EINVAL, EINVAL, EINVAL, EINVAL, EINVAL, EINVAL)),
    ("null_v",             dict(v=None),                         (EINVAL, EINVAL, EINVAL, EINVAL, EINVAL, EINVAL)),
    # no step: the tree rollout reads nothing; the trajectory records block 0; the others check their state anyway
    ("null_q_no_step",     dict(q=None, n=0),                    (OK, OK, EINVAL, EINVAL, EINVAL, EINVAL)),
    ("null_v_no_step",     dict(v=None, n=0),                    (OK, OK, EINVAL, EINVAL, EINVAL, EINVAL)),
    ("empty_batch",        dict(B=0, ld=0, q=None, v=None, s=None, traj=(None, None, None)), (OK, OK, OK, OK, OK, OK)),
    ("traj_q_only",        dict(traj=(FAKE, None, FAKE)),        (None, None, EINVAL, EINVAL, EINVAL, EINVAL)),
    ("traj_v_only",        dict(traj=(None, FAKE, FAKE)),        (None, None, EINVAL, EINVAL, EINVAL, EINVAL)),
    ("traj_without_s",     dict(traj=(FAKE, FAKE, None)),        (None, None, None, EINVAL, EINVAL, EINVAL)),
    # an empty batch: the trajectory rollout looks at no pointer, the others still refuse a partial set
    ("empty_batch_traj_q_only", dict(B=0, ld=0, q=None, v=None, s=None, traj=(FAKE, None, FAKE)),
     (None, None, OK, EINVAL, EINVAL, EINVAL)),
    ("null_s_with_pairs",  dict(s=None),                         (None, None, None, EINVAL, EINVAL, EINVAL)),
    # the argument that names the entry point: trajectories, contact, loops, controller
    ("null_descriptor",    dict(desc=None),                      (None, None, EINVAL, EINVAL, EINVAL, EINVAL)),
]

_CASES = [pytest.param(cell, over, entry, want[i], id=f"{cell}-{entry}")
          for cell, over, want in CELLS for i, entry in enumerate(ENTRY) if want[i] is not None]


@pytest.fixture(scope="module")
def setup(built):
    lib = rbd.load_library()
    mech = rbd.load_model("iiwa14")
    h = _cabi.ModelHandle(mech.flatten())
    one = lambda *row: np.asarray([row], float)                        # noqa: E731
    cd = rbd.ContactDesc(np.asarray([3], np.int32), one(0.0, 0.0, 0.1), one(50e3, 15e3, 1.5), one(0.8, 20e3, 100.0),
                         one(0.0, 0.0, 0.0, 0.0, 0.0, 1.0))
    assert cd.nstates > 0
    cst, keep_c = cd.c_struct()
    lst, keep_l = rbd.loop_desc(mech).c_struct()                       # a tree: no loop joints
    pd = _PdDesc(0, FAKE, FAKE, 0, FAKE, None, None, 0, 0, None, None)
    yield lib, h, ctypes.byref(cst), ctypes.byref(lst), ctypes.byref(pd)
    del keep_c, keep_l
    h.close()


def _call(setup, entry, model=..., dtype=_cabi.RBD_F64, B=4, ld=4, q=FAKE, v=FAKE, s=FAKE, step=0, stage=0, dt=1e-3, n=1,
          traj=..., desc=...):
    lib, h, contact, loops, pd = setup
    model = h.ptr if model is ... else model
    if traj is ...:
        traj = (FAKE, FAKE, FAKE) if entry == "trajectory" else (None, None, None)
    if entry == "integrate":
        return lib.rbd_integrate(model, dtype, B, ld, q, v, None, dt, n, None)
    if entry == "schedule":
        return lib.rbd_integrate_schedule(model, dtype, B, ld, q, v, None, step, stage, dt, n, None)
    if entry == "trajectory":
        qt, vt = (None, None) if desc is None else traj[:2]
        return lib.rbd_integrate_trajectory(model, dtype, B, ld, q, v, None, step, stage, dt, n, qt, vt, None)
    if entry == "contact":
        return lib.rbd_integrate_contact(model, dtype, B, ld, q, v, s, None, step, stage, contact if desc is ... else desc, dt, n,
                                         *traj, None)
    if entry == "loops":
        return lib.rbd_integrate_loops(model, dtype, B, ld, q, v, s, None, step, stage, loops if desc is ... else desc, contact, dt, n,
                                       *traj, None)
    return lib.rbd_integrate_pd(model, dtype, B, ld, q, v, s, None, step, stage, pd if desc is ... else desc, None, contact, dt, n,
                                *traj, None)


@pytest.mark.parametrize("cell,over,entry,want", _CASES)
def test_rollout_argument_status(setup, cell, over, entry, want):
    assert _call(setup, entry, **over) == want, setup[0].rbd_last_error()
