"""ctypes loader for the parameter-set-indexed emulator drivers and the (set, class) segment sort (TEST HARNESS):
tests/emu/env_sets_emu.cpp, compiled with plain g++ (-DPQP_HOST_EMU) on first use into a temporary directory.  Never
used by the product."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

from path_optimizer_b200.abi import BOUNDS_DTYPE, STATE_DTYPE, DistanceMap, Params, ptr

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "env_sets_emu.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="pqp_sets_emu_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libenv_sets_emu.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", _SRC, "-o", so], check=True)
        L = C.CDLL(so)
        vp, dm, pp = C.c_void_p, C.POINTER(DistanceMap), C.POINTER(Params)
        L.env_emu_update_bounds_sets.argtypes = [pp, C.c_int, vp, dm, C.c_int, vp, C.c_int, C.c_int] + [vp] * 8
        L.env_emu_finish_raw_sets.argtypes = [pp, C.c_int, vp, dm, C.c_int, vp, C.c_int, vp, vp, C.c_int, vp, vp]
        L.env_emu_densify_sets.argtypes = ([pp, C.c_int, vp, dm, C.c_int, vp, C.c_int, vp, vp, C.c_double, C.c_int,
                                            C.c_int, vp, vp, vp])
        L.sets_dispatch_emu.argtypes = [vp] + [C.c_int] * 6 + [vp] * 4 + [C.c_int] * 3 + [vp, vp]
        for f in (L.env_emu_update_bounds_sets, L.env_emu_finish_raw_sets, L.env_emu_densify_sets, L.sets_dispatch_emu):
            f.restype = None
        _lib = L
    return _lib


def _sets(sets):
    return (Params * len(sets))(*sets)


def _dms(maps):
    dists = [np.ascontiguousarray(m["distance"], dtype=np.float32) for m in maps]
    arr = (DistanceMap * len(maps))(*[DistanceMap(ptr(d), d.shape[0], d.shape[1], float(m["resolution"]),
                                                  float(m["center_x"]), float(m["center_y"])) for m, d in zip(maps, dists)])
    return arr, dists


def _index(index, B):
    return None if index is None else np.ascontiguousarray(index, dtype=np.int32).reshape(B)


def update_bounds_sets(sets, set_index, maps, map_index, batch, mode=1, splines=None):
    dms, _keep = _dms(maps)
    n_points = np.ascontiguousarray(batch["n_points"], dtype=np.int32)
    B = len(n_points)
    si, mi = _index(set_index, B), _index(map_index, B)
    ref = np.ascontiguousarray(batch["ref"], dtype=STATE_DTYPE)
    bounds = np.zeros(len(ref), dtype=BOUNDS_DTYPE)
    n_valid = np.zeros(B, dtype=np.int32)
    nk = kn = xc = yc = None
    if splines is not None:
        nk = np.ascontiguousarray(splines["n_knots"], dtype=np.int32)
        kn = np.ascontiguousarray(splines["knots"], dtype=np.float64)
        xc = np.ascontiguousarray(splines["x_coef"], dtype=np.float64)
        yc = np.ascontiguousarray(splines["y_coef"], dtype=np.float64)
    lib().env_emu_update_bounds_sets(_sets(sets), len(sets), ptr(si), dms, len(maps), ptr(mi), int(mode), B,
                                     ptr(n_points), ptr(ref), ptr(nk), ptr(kn), ptr(xc), ptr(yc), ptr(bounds), ptr(n_valid))
    return dict(bounds=bounds, n_valid=n_valid)


def finish_raw_sets(sets, set_index, maps, map_index, n_points, paths, collision_check=True):
    dms, _keep = _dms(maps)
    n_points = np.ascontiguousarray(n_points, dtype=np.int32)
    B = len(n_points)
    si, mi = _index(set_index, B), _index(map_index, B)
    paths = np.array(paths, dtype=STATE_DTYPE)
    n_kept = np.zeros(B, dtype=np.int32)
    ok = np.zeros(B, dtype=np.int32)
    lib().env_emu_finish_raw_sets(_sets(sets), len(sets), ptr(si), dms, len(maps), ptr(mi), B, ptr(n_points), ptr(paths),
                                  int(collision_check), ptr(n_kept), ptr(ok))
    return dict(states=paths, n_kept=n_kept, ok=ok)


def densify_sets(sets, set_index, maps, map_index, n_points, paths, output_spacing=0.3, collision_check=True,
                 max_out=512):
    dms, _keep = _dms(maps)
    n_points = np.ascontiguousarray(n_points, dtype=np.int32)
    B = len(n_points)
    si, mi = _index(set_index, B), _index(map_index, B)
    paths = np.ascontiguousarray(paths, dtype=STATE_DTYPE)
    out = np.zeros((B, max_out), dtype=STATE_DTYPE)
    n_out = np.zeros(B, dtype=np.int32)
    ok = np.zeros(B, dtype=np.int32)
    lib().env_emu_densify_sets(_sets(sets), len(sets), ptr(si), dms, len(maps), ptr(mi), B, ptr(n_points), ptr(paths),
                               float(output_spacing), int(collision_check), int(max_out), ptr(out), ptr(n_out), ptr(ok))
    return dict(states=out, n_out=n_out, ok=ok)


def sort(table, ncols, formulation, v0, nv, n_sets, batch, set_index, max_n=0, min_keep=0, max_keep=0):
    """(order [n_sets, nv, B], key [B]) of the dispatch's (set, class) segment sort."""
    n_points = np.ascontiguousarray(batch["n_points"], dtype=np.int32)
    B = len(n_points)
    offsets = np.ascontiguousarray(batch["offsets"], dtype=np.int32)
    ref = np.ascontiguousarray(batch["ref"], dtype=STATE_DTYPE)
    si = _index(set_index, B)
    table = np.ascontiguousarray(table, dtype=np.int8)
    order = np.zeros(n_sets * nv * B, dtype=np.int32)
    key = np.zeros(B, dtype=np.int32)
    lib().sets_dispatch_emu(ptr(table), int(ncols), int(formulation), int(v0), int(nv), int(n_sets), B, ptr(n_points),
                            ptr(offsets), ptr(ref), ptr(si), int(max_n), int(min_keep), int(max_keep), ptr(order), ptr(key))
    return order.reshape(n_sets, nv, B), key
