"""ctypes loader for the CPU warp-emulator build of the product's solver source (TEST HARNESS).

Builds tests/emu/libkp_emu.so from tests/emu/kp_emu.cpp with plain g++ (-DPQP_HOST_EMU) and runs
the SAME pqp_kp_core.cuh that nvcc compiles for sm_90a, one host thread per lane.  Used by the
CPU test-suite to check the kernel logic against the oracle without a GPU; never used by the product.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from path_optimizer_b200.abi import BOUNDS_DTYPE, STATE_DTYPE, DistanceMap, Params, ptr

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "libkp_emu.so")
_ENV_LIB = os.path.join(_HERE, "libenv_emu.so")
_CSRC = os.path.join(os.path.dirname(os.path.dirname(_HERE)), "path_optimizer_b200", "csrc")


def build():
    srcs = [os.path.join(_HERE, "kp_emu.cpp")] + [os.path.join(_CSRC, f) for f in os.listdir(_CSRC)
                                                  if f.endswith((".cuh", ".h"))]
    if (not os.path.exists(_LIB)) or any(os.path.getmtime(s) > os.path.getmtime(_LIB) for s in srcs):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++",
                        os.path.join(_HERE, "kp_emu.cpp"), "-o", _LIB, "-lpthread"], check=True)
    env_src = os.path.join(_HERE, "env_emu.cpp")
    if (not os.path.exists(_ENV_LIB)) or any(os.path.getmtime(s) > os.path.getmtime(_ENV_LIB) for s in srcs + [env_src]):
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", env_src, "-o", _ENV_LIB],
                       check=True)
    return _LIB


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.kp_emu_solve_batch.argtypes = [C.POINTER(Params), C.c_int] + [C.c_void_p] * 10 + [C.c_int, C.c_int, C.c_int]
        _lib.kp_emu_solve_batch.restype = C.c_int
        _lib.kp_emu_set_limits.argtypes = [C.c_void_p, C.c_void_p]
        _lib.kp_emu_set_limits.restype = None
        _lib.gen_emu_solve_batch.argtypes = [C.POINTER(Params), C.c_int, C.c_int] + [C.c_void_p] * 12
        _lib.gen_emu_solve_batch.restype = C.c_int
    return _lib


def solve_batch(params, batch, smem_bytes=227 * 1024, variant=0, nwarps=4, max_k=None, max_kp=None):
    """variant 0 = one-warp generic core (pqp_kp_core.cuh); 5..7 = Kp3<17,6,4>, <23,7,4>, <27,7,8>; 8, 9 = the 34-separator eight-warp classes Kp3<17,6,8,34>, <23,7,8,34>;
    10, 11, 12 = the long-path classes Kp3<37,7,13,34>, <37,7,12,34>, <27,7,10,34>;
    20, 21 = the "KPC" classes Kp3<23,7,4,17,KPC>, <23,7,8,34,KPC> (need max_k / max_kp)."""
    B = len(batch["n_points"])
    total = int(batch["offsets"][-1])
    ref = np.ascontiguousarray(batch["ref"], dtype=STATE_DTYPE)
    bounds = np.ascontiguousarray(batch["bounds"], dtype=BOUNDS_DTYPE)
    out = np.zeros(total, dtype=STATE_DTYPE)
    frenet = np.zeros((total, 3))
    status = np.zeros(B, dtype=np.int32)
    iters = np.zeros(B, dtype=np.int32)
    if max_k is not None:
        max_k = np.ascontiguousarray(max_k, dtype=np.float64)
        max_kp = np.ascontiguousarray(max_kp, dtype=np.float64)
    lib().kp_emu_set_limits(ptr(max_k), ptr(max_kp))
    lib().kp_emu_solve_batch(C.byref(params), B, ptr(batch["n_points"]), ptr(batch["offsets"]), ptr(ref),
                             ptr(bounds), ptr(batch["x0"]), ptr(batch["end_heading"]), ptr(out),
                             ptr(frenet), ptr(status), ptr(iters), smem_bytes, variant, nwarps)
    return dict(states=out, frenet=frenet, status=status, iters=iters)


def solve_batch_generic(params, formulation, batch, max_k=None, max_kp=None):
    """The generic banded kernel source (pqp_gen_core.cuh) + the host assembly (pqp_forms.h) for the
    "K" (formulation 1) and "KPC" (2) formulations, under the warp emulator."""
    B = len(batch["n_points"])
    total = int(batch["offsets"][-1])
    ref = np.ascontiguousarray(batch["ref"], dtype=STATE_DTYPE)
    bounds = np.ascontiguousarray(batch["bounds"], dtype=BOUNDS_DTYPE)
    out = np.zeros(total, dtype=STATE_DTYPE)
    frenet = np.zeros((total, 3))
    status = np.zeros(B, dtype=np.int32)
    iters = np.zeros(B, dtype=np.int32)
    lib().gen_emu_solve_batch(C.byref(params), int(formulation), B, ptr(batch["n_points"]), ptr(batch["offsets"]), ptr(ref),
                              ptr(bounds), ptr(batch["x0"]), ptr(batch["end_heading"]), ptr(max_k), ptr(max_kp), ptr(out),
                              ptr(frenet), ptr(status), ptr(iters))
    return dict(states=out, frenet=frenet, status=status, iters=iters)


# ---------------------------------------------------------------------------------------------
# stages either side of the QP: pqp_env_core.cuh through env_emu.cpp
# ---------------------------------------------------------------------------------------------
_env = None


def env_lib():
    global _env
    if _env is None:
        build()
        L = C.CDLL(_ENV_LIB)
        vp, dm, pp = C.c_void_p, C.POINTER(DistanceMap), C.POINTER(Params)
        L.env_emu_map_distance.argtypes = [dm, C.c_int, vp, vp]
        L.env_emu_update_bounds.argtypes = [pp, dm, C.c_int, C.c_int] + [vp] * 8
        L.env_emu_check_states.argtypes = [pp, dm, C.c_int, vp, vp]
        L.env_emu_finish_raw.argtypes = [pp, dm, C.c_int, vp, vp, C.c_int, vp, vp]
        L.env_emu_densify.argtypes = [pp, dm, C.c_int, vp, vp, C.c_double, C.c_int, C.c_int, vp, vp, vp]
        for f in (L.env_emu_map_distance, L.env_emu_update_bounds, L.env_emu_check_states, L.env_emu_finish_raw,
                  L.env_emu_densify):
            f.restype = None
        _env = L
    return _env


def _dm(m):
    dist = np.ascontiguousarray(m["distance"], dtype=np.float32)
    return DistanceMap(ptr(dist), dist.shape[0], dist.shape[1], float(m["resolution"]), float(m["center_x"]),
                       float(m["center_y"])), dist


def map_distance(m, xy):
    dm, _keep = _dm(m)
    xy = np.ascontiguousarray(xy, dtype=np.float64).reshape(-1, 2)
    out = np.zeros(len(xy))
    env_lib().env_emu_map_distance(C.byref(dm), len(xy), ptr(xy), ptr(out))
    return out


def update_bounds(params, m, batch, mode=1, splines=None):
    dm, _keep = _dm(m)
    n_points = np.ascontiguousarray(batch["n_points"], dtype=np.int32)
    ref = np.ascontiguousarray(batch["ref"], dtype=STATE_DTYPE)
    bounds = np.zeros(len(ref), dtype=BOUNDS_DTYPE)
    n_valid = np.zeros(len(n_points), dtype=np.int32)
    nk = kn = xc = yc = None
    if splines is not None:
        nk = np.ascontiguousarray(splines["n_knots"], dtype=np.int32)
        kn = np.ascontiguousarray(splines["knots"], dtype=np.float64)
        xc = np.ascontiguousarray(splines["x_coef"], dtype=np.float64)
        yc = np.ascontiguousarray(splines["y_coef"], dtype=np.float64)
    env_lib().env_emu_update_bounds(C.byref(params), C.byref(dm), int(mode), len(n_points), ptr(n_points), ptr(ref),
                                    ptr(nk), ptr(kn), ptr(xc), ptr(yc), ptr(bounds), ptr(n_valid))
    return dict(bounds=bounds, n_valid=n_valid)


def check_states(params, m, states):
    dm, _keep = _dm(m)
    states = np.ascontiguousarray(states, dtype=STATE_DTYPE)
    ok = np.zeros(len(states), dtype=np.int32)
    env_lib().env_emu_check_states(C.byref(params), C.byref(dm), len(states), ptr(states), ptr(ok))
    return ok


def finish_raw(params, m, n_points, paths, collision_check=True):
    dm, _keep = _dm(m)
    n_points = np.ascontiguousarray(n_points, dtype=np.int32)
    paths = np.array(paths, dtype=STATE_DTYPE)
    n_kept = np.zeros(len(n_points), dtype=np.int32)
    ok = np.zeros(len(n_points), dtype=np.int32)
    env_lib().env_emu_finish_raw(C.byref(params), C.byref(dm), len(n_points), ptr(n_points), ptr(paths),
                                 int(collision_check), ptr(n_kept), ptr(ok))
    return dict(states=paths, n_kept=n_kept, ok=ok)


def densify(params, m, n_points, paths, output_spacing=0.3, collision_check=True, max_out=512):
    dm, _keep = _dm(m)
    n_points = np.ascontiguousarray(n_points, dtype=np.int32)
    paths = np.ascontiguousarray(paths, dtype=STATE_DTYPE)
    B = len(n_points)
    out = np.zeros((B, max_out), dtype=STATE_DTYPE)
    n_out = np.zeros(B, dtype=np.int32)
    ok = np.zeros(B, dtype=np.int32)
    env_lib().env_emu_densify(C.byref(params), C.byref(dm), B, ptr(n_points), ptr(paths), float(output_spacing),
                              int(collision_check), int(max_out), ptr(out), ptr(n_out), ptr(ok))
    return dict(states=out, n_out=n_out, ok=ok)
