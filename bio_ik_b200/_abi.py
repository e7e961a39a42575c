"""ctypes mirror of include/bioik_b200.h (the C ABI of libbioik_b200.so).

Only POD tables cross the boundary; numpy arrays are kept alive by the owning
Python objects for as long as the C structs point into them.
"""
import ctypes as C
import os

import numpy as np

GOAL_NPARAM = 12

# status codes
OK, E_INVALID, E_UNSUPPORTED_GOAL, E_UNSUPPORTED_JOINT, E_CUDA, E_NO_PROBLEM, E_LIMIT = range(7)

# joint types (moveit::core::JointModel::JointType subset, src/forward_kinematics.h:78-139)
JOINT_FIXED, JOINT_REVOLUTE, JOINT_PRISMATIC, JOINT_FLOATING, JOINT_PLANAR = range(5)
OPT_REFERENCE_STALE_TIPS = 1
OPT_ISLAND_STREAM_STRIDE = 2  # islands of a query start i * value solver steps into the shared random streams (0: clones, as in the reference)
JOINT_VARS = {JOINT_FIXED: 0, JOINT_REVOLUTE: 1, JOINT_PRISMATIC: 1, JOINT_FLOATING: 7, JOINT_PLANAR: 3}

# goal types (include/bio_ik/goal_types.h)
(GOAL_POSITION, GOAL_ORIENTATION, GOAL_POSE, GOAL_LOOK_AT, GOAL_MAX_DISTANCE, GOAL_MIN_DISTANCE, GOAL_LINE,
 GOAL_PLANE, GOAL_AVOID_JOINT_LIMITS, GOAL_CENTER_JOINTS, GOAL_REGULARIZATION, GOAL_MINIMAL_DISPLACEMENT,
 GOAL_JOINT_VARIABLE, GOAL_SIDE, GOAL_DIRECTION, GOAL_CONE, GOAL_BALANCE) = range(1, 18)

c_double_p = C.POINTER(C.c_double)
c_int32_p = C.POINTER(C.c_int32)
c_uint32_p = C.POINTER(C.c_uint32)
c_int64_p = C.POINTER(C.c_int64)


class BioikRobot(C.Structure):
    _fields_ = [
        ("n_links", C.c_int32), ("n_vars", C.c_int32),
        ("link_parent", c_int32_p), ("joint_type", c_int32_p), ("joint_first_var", c_int32_p),
        ("link_origin", c_double_p), ("joint_axis", c_double_p),
        ("joint_mimic", c_int32_p), ("joint_mimic_factor", c_double_p), ("joint_mimic_offset", c_double_p),
        ("var_min", c_double_p), ("var_max", c_double_p), ("var_bounded", c_int32_p), ("var_max_velocity", c_double_p),
        ("link_mass", c_double_p), ("link_com", c_double_p),
    ]


class BioikGoal(C.Structure):
    _fields_ = [
        ("type", C.c_int32), ("tip", C.c_int32), ("secondary", C.c_int32), ("var", C.c_int32),
        ("weight", C.c_double), ("p", C.c_double * GOAL_NPARAM),
    ]


class BioikProblem(C.Structure):
    _fields_ = [
        ("n_tips", C.c_int32), ("tip_links", c_int32_p),
        ("n_active", C.c_int32), ("active_vars", c_int32_p),
        ("n_goals", C.c_int32), ("goals", C.POINTER(BioikGoal)),
        ("dpos", C.c_double), ("drot", C.c_double), ("dtwist", C.c_double),
    ]


class BioikSolverCfg(C.Structure):
    _fields_ = [
        ("population", C.c_int32), ("generations", C.c_int32), ("memetic", C.c_int32), ("memetic_iters", C.c_int32),
        ("table_seed", C.c_uint32), ("device", C.c_int32),
    ]


def dptr(a):
    """double* into a C-contiguous float64 numpy array (None -> NULL)."""
    if a is None:
        return None
    assert a.dtype == np.float64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(c_double_p)


def iptr(a):
    if a is None:
        return None
    assert a.dtype == np.int32 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(c_int32_p)


def uptr(a):
    if a is None:
        return None
    assert a.dtype == np.uint32 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(c_uint32_p)


REPO_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.environ.get("BIOIK_LIB") or os.path.join(REPO_ROOT, "bio_ik_b200", "csrc", "libbioik_b200.so")  # BIOIK_LIB: alternative build (experiments)

# every symbol include/bioik_b200.h declares
ABI_SYMBOLS = [
    "bioik_create", "bioik_destroy", "bioik_set_problem", "bioik_solve_batch", "bioik_solve_batch_device",
    "bioik_synchronize", "bioik_fk_batch", "bioik_approx_batch", "bioik_approx_fitness_batch",
    "bioik_solve_batch_trace", "bioik_solve_islands", "bioik_begin", "bioik_step", "bioik_get_solution", "bioik_pack_results_device", "bioik_kernel_name", "bioik_set_option", "bioik_cancel", "bioik_launch_count", "bioik_kernel_time", "bioik_last_error", "bioik_abi_version",
]

_lib = None


def load_library(path=None):
    """dlopen libbioik_b200.so and declare the prototypes.  Fails loudly if the
    CUDA extension has not been built (there is no CPU fallback)."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise RuntimeError(
            f"{p} not found: build the sm_90a extension first (python -c 'import __graft_entry__ as g; g.build()'). "
            "bio_ik_b200 has no CPU fallback.")
    lib = C.CDLL(p)
    ctx_p = C.c_void_p
    lib.bioik_create.argtypes = [C.POINTER(BioikRobot), C.POINTER(BioikSolverCfg), C.POINTER(ctx_p)]
    lib.bioik_create.restype = C.c_int
    lib.bioik_destroy.argtypes = [ctx_p]
    lib.bioik_destroy.restype = None
    lib.bioik_set_problem.argtypes = [ctx_p, C.POINTER(BioikProblem)]
    lib.bioik_set_problem.restype = C.c_int
    lib.bioik_solve_batch.argtypes = [ctx_p, C.c_int32, c_double_p, c_double_p, c_uint32_p, C.c_int32, C.c_int32,
                                      c_double_p, c_double_p, c_int32_p, c_int32_p]
    lib.bioik_solve_batch.restype = C.c_int
    lib.bioik_solve_batch_device.argtypes = [ctx_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.bioik_solve_batch_device.restype = C.c_int
    lib.bioik_synchronize.argtypes = [ctx_p]
    lib.bioik_synchronize.restype = C.c_int
    lib.bioik_fk_batch.argtypes = [ctx_p, C.c_int32, c_double_p, c_double_p]
    lib.bioik_fk_batch.restype = C.c_int
    lib.bioik_approx_batch.argtypes = [ctx_p, C.c_int32, c_double_p, c_double_p]
    lib.bioik_approx_batch.restype = C.c_int
    lib.bioik_approx_fitness_batch.argtypes = [ctx_p, C.c_int32, C.c_int32, c_double_p, c_double_p, c_double_p,
                                               c_double_p, c_double_p, c_double_p]
    lib.bioik_approx_fitness_batch.restype = C.c_int
    lib.bioik_solve_batch_trace.argtypes = [ctx_p, C.c_int32, c_double_p, c_double_p, c_uint32_p, C.c_int32,
                                            c_double_p, c_double_p, c_double_p, c_double_p, c_double_p]
    lib.bioik_solve_batch_trace.restype = C.c_int
    lib.bioik_solve_islands.argtypes = [ctx_p, C.c_int32, C.c_int32, c_double_p, c_double_p, c_uint32_p, C.c_int32, C.c_int32, C.c_int32,
                                        c_double_p, c_double_p, c_int32_p, c_int32_p, c_int32_p]
    lib.bioik_solve_islands.restype = C.c_int
    lib.bioik_begin.argtypes = [ctx_p, C.c_int32, C.c_int32, c_double_p, c_double_p, c_uint32_p, C.c_int32, C.c_int32]
    lib.bioik_begin.restype = C.c_int
    lib.bioik_step.argtypes = [ctx_p, C.c_int32, c_int32_p]
    lib.bioik_step.restype = C.c_int
    lib.bioik_get_solution.argtypes = [ctx_p, C.c_int32, c_double_p, c_double_p, c_int32_p, c_int32_p, c_int32_p]
    lib.bioik_get_solution.restype = C.c_int
    lib.bioik_pack_results_device.argtypes = [ctx_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.bioik_pack_results_device.restype = C.c_int
    lib.bioik_kernel_name.argtypes = [ctx_p]
    lib.bioik_kernel_name.restype = C.c_char_p
    lib.bioik_cancel.argtypes = [ctx_p]
    lib.bioik_cancel.restype = C.c_int
    lib.bioik_set_option.argtypes = [ctx_p, C.c_int32, C.c_int32]
    lib.bioik_set_option.restype = C.c_int
    lib.bioik_launch_count.argtypes = [ctx_p]
    lib.bioik_launch_count.restype = C.c_int64
    lib.bioik_kernel_time.argtypes = [ctx_p, C.c_int32, c_double_p, c_int64_p, c_double_p, c_int64_p]
    lib.bioik_kernel_time.restype = C.c_int
    lib.bioik_last_error.argtypes = [ctx_p]
    lib.bioik_last_error.restype = C.c_char_p
    lib.bioik_abi_version.argtypes = []
    lib.bioik_abi_version.restype = C.c_int
    if path is None:
        _lib = lib
    return lib
