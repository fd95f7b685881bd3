"""ctypes loader for the map-indexed emulator drivers (TEST HARNESS): tests/emu/env_maps_emu.cpp, compiled with plain
g++ (-DPQP_HOST_EMU) on first use into a temporary directory, runs the stages either side of the QP over a map set and a
per-path index exactly as the kernels of pqp_env.cu look a path's map up (pqp::map_of).  Never used by the product."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

from path_optimizer_b200.abi import BOUNDS_DTYPE, STATE_DTYPE, DistanceMap, Params, ptr

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "env_maps_emu.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="pqp_maps_emu_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libenv_maps_emu.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", _SRC, "-o", so], check=True)
        L = C.CDLL(so)
        vp, dm, pp = C.c_void_p, C.POINTER(DistanceMap), C.POINTER(Params)
        L.env_emu_update_bounds_maps.argtypes = [pp, dm, C.c_int, vp, C.c_int, C.c_int] + [vp] * 8
        L.env_emu_finish_raw_maps.argtypes = [pp, dm, C.c_int, vp, C.c_int, vp, vp, C.c_int, vp, vp]
        L.env_emu_densify_maps.argtypes = [pp, dm, C.c_int, vp, C.c_int, vp, vp, C.c_double, C.c_int, C.c_int, vp, vp, vp]
        for f in (L.env_emu_update_bounds_maps, L.env_emu_finish_raw_maps, L.env_emu_densify_maps):
            f.restype = None
        _lib = L
    return _lib


def _dms(maps):
    dists = [np.ascontiguousarray(m["distance"], dtype=np.float32) for m in maps]
    arr = (DistanceMap * len(maps))(*[DistanceMap(ptr(d), d.shape[0], d.shape[1], float(m["resolution"]),
                                                  float(m["center_x"]), float(m["center_y"])) for m, d in zip(maps, dists)])
    return arr, dists


def _index(map_index, B):
    return None if map_index is None else np.ascontiguousarray(map_index, dtype=np.int32).reshape(B)


def update_bounds_maps(params, maps, map_index, batch, mode=1, splines=None):
    dms, _keep = _dms(maps)
    n_points = np.ascontiguousarray(batch["n_points"], dtype=np.int32)
    mi = _index(map_index, len(n_points))
    ref = np.ascontiguousarray(batch["ref"], dtype=STATE_DTYPE)
    bounds = np.zeros(len(ref), dtype=BOUNDS_DTYPE)
    n_valid = np.zeros(len(n_points), dtype=np.int32)
    nk = kn = xc = yc = None
    if splines is not None:
        nk = np.ascontiguousarray(splines["n_knots"], dtype=np.int32)
        kn = np.ascontiguousarray(splines["knots"], dtype=np.float64)
        xc = np.ascontiguousarray(splines["x_coef"], dtype=np.float64)
        yc = np.ascontiguousarray(splines["y_coef"], dtype=np.float64)
    lib().env_emu_update_bounds_maps(C.byref(params), dms, len(maps), ptr(mi), int(mode), len(n_points),
                                         ptr(n_points), ptr(ref), ptr(nk), ptr(kn), ptr(xc), ptr(yc), ptr(bounds),
                                         ptr(n_valid))
    return dict(bounds=bounds, n_valid=n_valid)


def finish_raw_maps(params, maps, map_index, n_points, paths, collision_check=True):
    dms, _keep = _dms(maps)
    n_points = np.ascontiguousarray(n_points, dtype=np.int32)
    mi = _index(map_index, len(n_points))
    paths = np.array(paths, dtype=STATE_DTYPE)
    n_kept = np.zeros(len(n_points), dtype=np.int32)
    ok = np.zeros(len(n_points), dtype=np.int32)
    lib().env_emu_finish_raw_maps(C.byref(params), dms, len(maps), ptr(mi), len(n_points), ptr(n_points), ptr(paths),
                                      int(collision_check), ptr(n_kept), ptr(ok))
    return dict(states=paths, n_kept=n_kept, ok=ok)


def densify_maps(params, maps, map_index, n_points, paths, output_spacing=0.3, collision_check=True, max_out=512):
    dms, _keep = _dms(maps)
    n_points = np.ascontiguousarray(n_points, dtype=np.int32)
    B = len(n_points)
    mi = _index(map_index, B)
    paths = np.ascontiguousarray(paths, dtype=STATE_DTYPE)
    out = np.zeros((B, max_out), dtype=STATE_DTYPE)
    n_out = np.zeros(B, dtype=np.int32)
    ok = np.zeros(B, dtype=np.int32)
    lib().env_emu_densify_maps(C.byref(params), dms, len(maps), ptr(mi), B, ptr(n_points), ptr(paths),
                                   float(output_spacing), int(collision_check), int(max_out), ptr(out), ptr(n_out),
                                   ptr(ok))
    return dict(states=out, n_out=n_out, ok=ok)
