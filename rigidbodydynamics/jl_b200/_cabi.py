"""ctypes binding of ``librbd_b200.so`` -- the C ABI declared in ``include/rbd_b200.h``.

This is the same boundary the Julia shim ``ccall``s (``julia/RBDB200.jl``, ``INTEGRATION.md``).  There is NO
fallback: if the shared library is missing or a call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_double, c_float, c_int32, c_int64, c_void_p

import numpy as np

RBD_MAX_BODIES = 64
RBD_MAX_LOOP_JOINTS, RBD_MAX_CONSTRAINTS = 16, 96
RBD_MAX_TASKS = 32

RBD_OK, RBD_EINVAL, RBD_EDIM, RBD_ELOOP, RBD_ESTALE, RBD_ECUDA, RBD_EUNSUPPORTED, RBD_ENOMEM = range(8)
RBD_F32, RBD_F64, RBD_DUAL64X6 = 0, 1, 2
RBD_SPEC_DYNAMICS, RBD_SPEC_DYNAMICS_QDOT, RBD_SPEC_DYNAMICS_NOTAU, RBD_SPEC_INVERSE_DYNAMICS, RBD_SPEC_DYNAMICS_BIAS = 1, 2, 4, 8, 16
RBD_SPEC_DYNAMICS_GATHER = 32
RBD_SPEC_MASS_MATRIX, RBD_SPEC_MASS_MATRIX_LOWER = 64, 128
RBD_SPEC_ALL = 63

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "librbd_b200.so")


class RbdModelDesc(Structure):
    _fields_ = [
        ("nb", c_int32),
        ("num_non_tree_joints", c_int32),
        ("parent", POINTER(c_int32)),
        ("jtype", POINTER(c_int32)),
        ("X_tree", POINTER(c_double)),
        ("jparam", POINTER(c_double)),
        ("inertia", POINTER(c_double)),
        ("gravity", c_double * 3),
        ("modcount", c_int64),
    ]


class RbdModelInfo(Structure):
    _fields_ = [
        ("nb", c_int32), ("nq", c_int32), ("nv", c_int32),
        ("stash_rows", c_int32), ("max_branch_depth", c_int32), ("general_path", c_int32),
        ("modcount", c_int64),
        ("qstart", c_int32 * RBD_MAX_BODIES),
        ("vstart", c_int32 * RBD_MAX_BODIES),
        ("eval_order", c_int32 * RBD_MAX_BODIES),
    ]


class RbdLaunchInfo(Structure):
    _fields_ = [
        ("kernels_launched", c_int32), ("grid", c_int32), ("block", c_int32),
        ("smem_bytes", c_int32), ("blocks_per_sm", c_int32), ("last_kernel_ms", c_float), ("specialised", c_int32),
    ]


class RbdKinematicsOut(Structure):
    _fields_ = [(n, c_void_p) for n in ("transforms_to_root", "center_of_mass", "kinetic_energy",
                                        "gravitational_potential_energy", "momentum", "momentum_rate_bias",
                                        "momentum_matrix", "geometric_jacobian")]


TASK_OUTPUTS = ("transform", "point", "twist", "point_velocity", "geometric_jacobian", "point_jacobian", "acceleration",
                "point_acceleration")


class RbdTaskDesc(Structure):
    _fields_ = [("ntasks", c_int32), ("body", POINTER(c_int32)), ("base", POINTER(c_int32)), ("frame", POINTER(c_int32)),
                ("point", POINTER(c_double))]


class RbdTaskOut(Structure):
    _fields_ = [(n, c_void_p) for n in TASK_OUTPUTS]


class RbdError(RuntimeError):
    """Raised for any non-zero rbd_status.  ``status`` carries the code so callers can map it to the reference's
    exception types (DimensionMismatch, ModificationCountMismatch, ...)."""

    def __init__(self, status: int, message: str):
        super().__init__(f"rbd_b200 status {status}: {message}")
        self.status = status


def make_desc(desc, num_non_tree_joints: int = 0):
    """Build the C struct for a ``ModelDesc``; returns (struct, keepalive arrays)."""
    parent = np.ascontiguousarray(desc.parent, np.int32)
    jtype = np.ascontiguousarray(desc.jtype, np.int32)
    X = np.ascontiguousarray(desc.X_tree, np.float64)
    jp = np.ascontiguousarray(desc.jparam, np.float64)
    inr = np.ascontiguousarray(desc.inertia, np.float64)
    d = RbdModelDesc()
    d.nb = int(desc.nb)
    d.num_non_tree_joints = int(num_non_tree_joints)
    d.parent = parent.ctypes.data_as(POINTER(c_int32))
    d.jtype = jtype.ctypes.data_as(POINTER(c_int32))
    d.X_tree = X.ctypes.data_as(POINTER(c_double))
    d.jparam = jp.ctypes.data_as(POINTER(c_double))
    d.inertia = inr.ctypes.data_as(POINTER(c_double))
    for k in range(3):
        d.gravity[k] = float(desc.gravity[k])
    d.modcount = int(desc.modcount)
    return d, (parent, jtype, X, jp, inr)


_lib = None

# (name, restype, argtypes) of every symbol include/rbd_b200.h declares
_vp, _i32, _i64 = c_void_p, c_int32, c_int64
SYMBOLS = {
    "rbd_version": (c_int32, []),
    "rbd_last_error": (c_char_p, []),
    "rbd_status_string": (c_char_p, [_i32]),
    "rbd_model_create": (c_int32, [POINTER(RbdModelDesc), POINTER(_vp)]),
    "rbd_model_destroy": (c_int32, [_vp]),
    "rbd_model_get_info": (c_int32, [_vp, POINTER(RbdModelInfo)]),
    "rbd_model_check_modcount": (c_int32, [_vp, _i64]),
    "rbd_get_launch_info": (c_int32, [POINTER(RbdLaunchInfo)]),
    "rbd_model_precompile": (c_int32, [_vp, _i32, _i32, _i32]),
    "rbd_dynamics": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "rbd_dynamics_gather": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, _i32, POINTER(_vp), _vp, _i64, _i64, _vp]),
    "rbd_inverse_dynamics": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp]),
    "rbd_inverse_dynamics_bodies": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "rbd_contact_dynamics": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "rbd_dynamics_loops": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "rbd_dynamics_result": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "rbd_dynamics_derivatives": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "rbd_model_precompile_derivatives": (c_int32, [_vp, _i32]),
    "rbd_dynamics_derivatives_ext": (c_int32, [_vp, _i32, _i64, _i64] + [_vp] * 9),
    "rbd_inverse_dynamics_derivatives": (c_int32, [_vp, _i32, _i64, _i64] + [_vp] * 9),
    "rbd_model_precompile_derivatives_ext": (c_int32, [_vp, _i32, _i32]),
    "rbd_dynamics_vjp": (c_int32, [_vp, _i32, _i64, _i64] + [_vp] * 12),
    "rbd_inverse_dynamics_vjp": (c_int32, [_vp, _i32, _i64, _i64] + [_vp] * 11),
    "rbd_dynamics_bias": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, _vp, _vp]),
    "rbd_mass_matrix": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp]),
    "rbd_mass_matrix_uplo": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _i32, _vp]),
    "rbd_integrate": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, c_double, _i32, _vp]),
    "rbd_integrate_schedule": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, _i64, _i64, c_double, _i32, _vp]),
    "rbd_integrate_trajectory": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, _i64, _i64, c_double, _i32, _vp, _vp, _vp]),
    "rbd_integrate_vjp": (c_int32, [_vp, _i32, _i64, _vp, _vp, _vp, _i64, _i64, c_double, _i32] + [_vp] * 7),
    "rbd_integrate_contact": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, _vp, _i64, _i64, _vp, c_double, _i32, _vp, _vp, _vp, _vp]),
    "rbd_integrate_loops": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp, c_double, _i32, _vp, _vp, _vp, _vp]),
    "rbd_integrate_pd": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, c_double, _i32, _vp, _vp, _vp, _vp]),
    "rbd_integrate_task_pd": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, c_double, _i32, _vp, _vp, _vp, _vp]),
    "rbd_task_pd_torques": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, _vp, _i32, _vp, _vp]),
    "rbd_integrate_contact_vjp":(c_int32, [_vp, _i32, _i64, _vp, _vp, _vp, _vp, _i64, _i64, _vp, c_double, _i32] + [_vp] * 9),
    "rbd_integrate_pd_vjp":   (c_int32, [_vp, _i32, _i64, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp, c_double, _i32] + [_vp] * 10),
    "rbd_integrate_task_pd_vjp": (c_int32, [_vp, _i32, _i64, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp, c_double, _i32] + [_vp] * 10),
    "rbd_task_pd_torques_vjp": (c_int32, [_vp, _i32, _i64, _vp, _vp, _vp, _vp, _i32] + [_vp] * 7),
    "rbd_kinematics": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, POINTER(RbdKinematicsOut), _vp]),
    "rbd_kinematics_vjp": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, POINTER(RbdKinematicsOut)] + [_vp] * 4),
    "rbd_task_kinematics": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, POINTER(RbdTaskDesc), POINTER(RbdTaskOut), _vp]),
    "rbd_task_kinematics_vjp": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, POINTER(RbdTaskDesc), POINTER(RbdTaskOut)] + [_vp] * 5),
    "rbd_dynamics_host": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp]),
    "rbd_inverse_dynamics_host": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, _vp, _vp]),
    "rbd_dynamics_bias_host": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, _vp]),
    "rbd_mass_matrix_host": (c_int32, [_vp, _i32, _i64, _i64, _vp, _vp]),
}


def load_library(path: str = LIB_PATH):
    """Load librbd_b200.so (built in-tree by ``__graft_entry__.build()`` / ``csrc/Makefile``).  Fails loudly."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(path):
        raise ImportError(f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          f"(there is no CPU fallback)")
    lib = ctypes.CDLL(path)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status: int):
    if status != RBD_OK:
        msg = load_library().rbd_last_error()
        raise RbdError(status, msg.decode() if msg else "unknown error")


class ModelHandle:
    """Owns one ``rbd_model*``."""

    def __init__(self, desc, num_non_tree_joints: int = 0):
        lib = load_library()
        cdesc, keep = make_desc(desc, num_non_tree_joints)
        h = c_void_p()
        check(lib.rbd_model_create(ctypes.byref(cdesc), ctypes.byref(h)))
        self._h = h
        self._lib = lib
        info = RbdModelInfo()
        check(lib.rbd_model_get_info(h, ctypes.byref(info)))
        self.info = info

    @property
    def ptr(self):
        return self._h

    def check_modcount(self, modcount: int):
        check(self._lib.rbd_model_check_modcount(self._h, int(modcount)))

    def precompile(self, dtype: int = RBD_F32, what: int = RBD_SPEC_ALL, load: bool = False):
        """rbd_model_precompile: generate + NVRTC-compile the model-specialised kernels into the cubin cache (no GPU needed
        unless ``load``)."""
        check(self._lib.rbd_model_precompile(self._h, int(dtype), int(what), 1 if load else 0))

    def precompile_derivatives(self, dtype: int = RBD_F64, with_dtau: bool = False):
        """rbd_model_precompile_derivatives: the model-specialised solve kernel of rbd_dynamics_derivatives into the cubin cache.
        ``with_dtau``: the variant that also solves d v̇ / d tau (rbd_model_precompile_derivatives_ext)."""
        if with_dtau:
            check(self._lib.rbd_model_precompile_derivatives_ext(self._h, int(dtype), 1))
        else:
            check(self._lib.rbd_model_precompile_derivatives(self._h, int(dtype)))

    def close(self):
        if getattr(self, "_h", None):
            self._lib.rbd_model_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def launch_info() -> RbdLaunchInfo:
    info = RbdLaunchInfo()
    check(load_library().rbd_get_launch_info(ctypes.byref(info)))
    return info
