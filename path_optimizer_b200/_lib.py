"""ctypes binding of libpqp.so (include/pqp.h).  Fails loudly when the library is missing: the
product has no CPU fallback."""
import ctypes as C
import os

from .abi import DistanceMap, Params, Stats

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PQP_LIB") or os.path.join(_HERE, "libpqp.so")   # PQP_LIB: A/B builds of the same ABI

# every symbol include/pqp.h declares
SYMBOLS = ["pqp_params_default", "pqp_params_update_config", "pqp_keep_control_steps", "pqp_problem_size",
           "pqp_create", "pqp_destroy", "pqp_set_params", "pqp_solve_batch", "pqp_solve_batch_device",
           "pqp_solve_batch_device_classes", "pqp_last_error", "pqp_version", "pqp_max_points", "pqp_max_points_keep",
           "pqp_class_info", "pqp_class_info_kpc", "pqp_class_info_form", "pqp_set_order_hint", "pqp_class_name", "pqp_device_class_info",
           "pqp_solve_batch_device_dispatch", "pqp_class_table"]
# ... and include/pqp_env.h
ENV_SYMBOLS = ["pqp_update_limits", "pqp_update_limits_device", "pqp_set_map", "pqp_map_distance", "pqp_spline_fit", "pqp_spline_eval", "pqp_update_bounds_batch",
               "pqp_check_states", "pqp_finish_raw_batch", "pqp_densify_batch", "pqp_plan_batch", "pqp_plan_batch_device",
               "pqp_set_maps", "pqp_plan_batch_maps", "pqp_plan_batch_device_maps"]
# ... and include/pqp_multi.h
MULTI_SYMBOLS = ["pqp_nccl_unique_id", "pqp_comm_init_rank", "pqp_allgather", "pqp_comm_destroy", "pqp_multi_create",
                 "pqp_multi_destroy", "pqp_multi_devices", "pqp_multi_solve_batch", "pqp_multi_gathered",
                 "pqp_multi_gather_rows", "pqp_multi_shard"]
SYMBOLS = SYMBOLS + ENV_SYMBOLS + MULTI_SYMBOLS

_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -m path_optimizer_b200.build` "
            "(nvcc, sm_90a).  There is no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    L.pqp_params_default.argtypes = [C.POINTER(Params)]
    L.pqp_params_update_config.argtypes = [C.POINTER(Params)]
    L.pqp_keep_control_steps.argtypes = [C.c_int, vp, C.c_int]
    L.pqp_problem_size.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.pqp_create.argtypes = [C.POINTER(vp), C.POINTER(Params), C.c_int, C.c_int, C.c_int]
    L.pqp_destroy.argtypes = [vp]
    L.pqp_destroy.restype = None
    L.pqp_set_params.argtypes = [vp, C.POINTER(Params)]
    L.pqp_solve_batch.argtypes = [vp, C.c_int, C.c_int] + [vp] * 11 + [C.POINTER(Stats)]
    L.pqp_solve_batch_device.argtypes = [vp] + [C.c_int] * 6 + [vp] * 13 + [C.POINTER(Stats)]
    L.pqp_last_error.restype = C.c_char_p
    L.pqp_version.restype = C.c_char_p
    L.pqp_max_points.argtypes = [vp, C.c_int]
    L.pqp_max_points_keep.argtypes = [vp, C.c_int, C.c_int]
    L.pqp_class_info.argtypes = [C.c_int] * 3 + [C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int64)]
    L.pqp_set_order_hint.argtypes = [vp, C.c_int, vp]
    L.pqp_class_info_form.argtypes = [C.c_int] * 4 + [C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int64)]
    L.pqp_class_info_kpc.argtypes = [C.c_int] * 2 + [C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int64)]
    L.pqp_class_name.argtypes = [C.c_int]
    L.pqp_class_name.restype = C.c_char_p
    L.pqp_device_class_info.argtypes = [C.c_int] * 4 + [C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int64)]
    L.pqp_solve_batch_device_classes.argtypes = [vp] + [C.c_int] * 3 + [vp] * 15 + [C.POINTER(Stats)]
    L.pqp_solve_batch_device_dispatch.argtypes = [vp] + [C.c_int] * 6 + [vp] * 13 + [C.POINTER(Stats)]
    L.pqp_class_table.argtypes = [C.c_int, C.c_int, vp, C.c_int, C.POINTER(C.c_int)]
    # include/pqp_env.h
    L.pqp_update_limits.argtypes = [C.POINTER(Params), C.c_int, C.c_int, vp, vp, vp]
    L.pqp_update_limits_device.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, vp]
    L.pqp_set_map.argtypes = [vp, C.POINTER(DistanceMap)]
    L.pqp_map_distance.argtypes = [vp, C.c_int, vp, vp]
    L.pqp_spline_fit.argtypes = [C.c_int, vp, vp, vp]
    L.pqp_spline_eval.argtypes = [C.c_int, vp, vp, C.c_int, C.c_double]
    L.pqp_spline_eval.restype = C.c_double
    L.pqp_update_bounds_batch.argtypes = [vp, C.c_int, C.c_int] + [vp] * 8 + [C.POINTER(Stats)]
    L.pqp_check_states.argtypes = [vp, C.c_int, vp, vp]
    L.pqp_finish_raw_batch.argtypes = [vp, C.c_int, vp, vp, C.c_int, vp, vp, C.POINTER(Stats)]
    L.pqp_densify_batch.argtypes = [vp, C.c_int, vp, vp, C.c_double, C.c_int, C.c_int, vp, vp, vp, C.POINTER(Stats)]
    L.pqp_plan_batch.argtypes = ([vp, C.c_int, C.c_int, C.c_int, C.c_int] + [vp] * 8 +
                                 [C.c_double, C.c_int, C.c_int] + [vp] * 6 + [C.POINTER(Stats)])
    L.pqp_plan_batch_device.argtypes = ([vp] + [C.c_int] * 6 + [vp] * 9 + [C.c_double, C.c_int, C.c_int] + [vp] * 7 +
                                        [C.POINTER(Stats)])
    L.pqp_set_maps.argtypes = [vp, C.c_int, C.POINTER(DistanceMap)]
    L.pqp_plan_batch_maps.argtypes = ([vp, C.c_int, C.c_int, C.c_int, C.c_int] + [vp] * 9 +
                                      [C.c_double, C.c_int, C.c_int] + [vp] * 6 + [C.POINTER(Stats)])
    L.pqp_plan_batch_device_maps.argtypes = ([vp] + [C.c_int] * 6 + [vp] * 10 + [C.c_double, C.c_int, C.c_int] +
                                             [vp] * 7 + [C.POINTER(Stats)])
    # include/pqp_multi.h
    L.pqp_nccl_unique_id.argtypes = [vp]
    L.pqp_comm_init_rank.argtypes = [vp, C.c_int, C.c_int, vp]
    L.pqp_allgather.argtypes = [vp, vp, vp, C.c_int64, vp]
    L.pqp_comm_destroy.argtypes = [vp]
    L.pqp_multi_create.argtypes = [C.POINTER(vp), C.POINTER(Params), C.c_int, vp, C.c_int, C.c_int]
    L.pqp_multi_destroy.argtypes = [vp]
    L.pqp_multi_destroy.restype = None
    L.pqp_multi_devices.argtypes = [vp]
    L.pqp_multi_solve_batch.argtypes = [vp, C.c_int, C.c_int] + [vp] * 9 + [C.c_int, C.POINTER(Stats)]
    L.pqp_multi_gathered.argtypes = [vp, C.c_int]
    L.pqp_multi_gathered.restype = vp
    L.pqp_multi_gather_rows.argtypes = [vp]
    L.pqp_multi_gather_rows.restype = C.c_int64
    L.pqp_multi_shard.argtypes = [vp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int64)]
    _lib = L
    return L


def last_error():
    return load().pqp_last_error().decode()
