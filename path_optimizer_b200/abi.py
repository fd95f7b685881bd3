"""ctypes / numpy mirrors of the POD records in ``include/pqp.h``.

Pure host-side definitions (no CUDA, no oracle).  Field order and types must match
``include/pqp.h`` exactly; ``tests/test_abi.py`` checks sizes against the compiled library.
"""
import ctypes as C

import numpy as np

# PathOptimizationNS::State (reference include/path_optimizer/data_struct/data_struct.hpp:13-30)
STATE_DTYPE = np.dtype([(f, "<f8") for f in ("x", "y", "z", "k", "s", "v", "a")])
# CoveringCircleBounds ub/lb per circle (data_struct.hpp:72-91)
BOUNDS_DTYPE = np.dtype([(f, "<f8") for f in (
    "c0_ub", "c0_lb", "c1_ub", "c1_lb", "c2_ub", "c2_lb", "c3_ub", "c3_lb")])

FORM_KP, FORM_K, FORM_KPC = 0, 1, 2
FORMULATIONS = {"KP": FORM_KP, "K": FORM_K, "KPC": FORM_KPC}

SOLVED = 1
SOLVED_INACCURATE = 2
MAX_ITER_REACHED = -2
PRIMAL_INFEASIBLE = -3
DUAL_INFEASIBLE = -4
NON_CVX = -7
UNSOLVED = -10
INVALID_PROBLEM = -100

OK, ERR_ARG, ERR_CAPACITY, ERR_CUDA, ERR_UNSUPPORTED = 0, 1, 2, 3, 4


class Params(C.Structure):
    """``pqp_params``: snapshot of the reference's gflags + OSQP settings."""
    _fields_ = [
        ("car_width", C.c_double), ("car_length", C.c_double), ("safety_margin", C.c_double),
        ("wheel_base", C.c_double), ("rear_axle_to_center", C.c_double),
        ("max_steering_angle", C.c_double), ("mu", C.c_double), ("max_curvature_rate", C.c_double),
        ("circle_radius", C.c_double),
        ("d1", C.c_double), ("d2", C.c_double), ("d3", C.c_double), ("d4", C.c_double),
        ("K_curvature_weight", C.c_double), ("K_curvature_rate_weight", C.c_double),
        ("K_deviation_weight", C.c_double),
        ("KP_curvature_weight", C.c_double), ("KP_curvature_rate_weight", C.c_double),
        ("KP_deviation_weight", C.c_double), ("KP_slack_weight", C.c_double),
        ("expected_safety_margin", C.c_double),
        ("constraint_end_heading", C.c_int32),
        ("rho", C.c_double), ("sigma", C.c_double), ("alpha", C.c_double),
        ("eps_abs", C.c_double), ("eps_rel", C.c_double),
        ("eps_prim_inf", C.c_double), ("eps_dual_inf", C.c_double),
        ("max_iter", C.c_int32), ("scaling", C.c_int32), ("check_termination", C.c_int32),
        ("adaptive_rho", C.c_int32), ("adaptive_rho_interval", C.c_int32),
        ("adaptive_rho_tolerance", C.c_double),
        ("reserved_", C.c_int32 * 3),
    ]

    def copy(self):
        other = Params()
        C.memmove(C.byref(other), C.byref(self), C.sizeof(Params))
        return other


class Stats(C.Structure):
    """``pqp_stats``."""
    _fields_ = [
        ("h2d_ms", C.c_float), ("kernel_ms", C.c_float), ("d2h_ms", C.c_float),
        ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64),
        ("kernel_launches", C.c_int32), ("max_iters", C.c_int32),
        ("total_iters", C.c_int64), ("n_solved", C.c_int32), ("reserved_", C.c_int32),
    ]


class DistanceMap(C.Structure):
    """``pqp_distance_map`` (include/pqp_env.h)."""
    _fields_ = [("distance", C.c_void_p), ("rows", C.c_int32), ("cols", C.c_int32),
                ("resolution", C.c_double), ("center_x", C.c_double), ("center_y", C.c_double)]


class OccupancyMap(C.Structure):
    """``pqp_occupancy_map`` (include/pqp_env.h)."""
    _fields_ = [("cells", C.c_void_p), ("rows", C.c_int32), ("cols", C.c_int32),
                ("resolution", C.c_double), ("center_x", C.c_double), ("center_y", C.c_double)]


def ptr(arr, ctype=C.c_void_p):
    """Raw pointer of a C-contiguous numpy array (or None)."""
    if arr is None:
        return None
    assert arr.flags["C_CONTIGUOUS"]
    return arr.ctypes.data_as(ctype)
