"""ctypes loader for the TENSION smoothing emulator (TEST HARNESS): tests/emu/tension_emu.cpp, compiled with plain g++
(-DPQP_HOST_EMU) on first use into a temporary directory, runs the per-thread functions of
pqp_smooth_reference_tension_device (csrc/pqp_smooth_core.cuh) on one polyline and map, and the width-9 generic core
(csrc/pqp_gen_core.cuh) on its QP with one host thread per lane.  Never used by the product."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

from path_optimizer_b200.abi import STATE_DTYPE, DistanceMap, ptr

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "tension_emu.cpp")
_lib = None
PARTNERS = 6


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="pqp_tension_emu_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libtension_emu.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", _SRC, "-o", so,
                        "-lpthread"], check=True)
        L = C.CDLL(so)
        vp, d_, i_ = C.c_void_p, C.c_double, C.c_int
        L.tension_emu_stage.argtypes = [i_, vp, vp, C.POINTER(DistanceMap), d_, d_, d_, i_, i_] + [vp] * 15
        L.tension_emu_stage.restype = i_
        L.tension_emu_solve.argtypes = [vp, i_, i_] + [vp] * 15
        L.tension_emu_solve.restype = i_
        _lib = L
    return _lib


def stage(px, py, dmap, weights=(0.0, 1.0, 50.0), max_raw=4096, max_points=277):
    """One polyline on the distance map `dmap` (None: a map index outside the set): dict(reason, N, stations
    (STATE_DTYPE), clearance, and the band-order QP: A_col [m][4], A_val, l, u, Pd, Po_idx [n][6], Po_val, csc_ptr,
    csc_row, csc_val, sep)."""
    f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)   # noqa: E731
    px, py = f64(px), f64(py)
    Nm = int(max_points)
    st = np.zeros(Nm, dtype=STATE_DTYPE)
    clear = np.zeros(Nm)
    n = m = 3 * Nm
    A_col, A_val = np.zeros((m, 4), dtype=np.int32), np.zeros((m, 4))
    l, u, Pd = np.zeros(m), np.zeros(m), np.zeros(n)
    Po_idx, Po_val = np.zeros((n, PARTNERS), dtype=np.int32), np.zeros((n, PARTNERS))
    cp, cr, cv = np.zeros(n + 1, dtype=np.int32), np.zeros(5 * Nm, dtype=np.int32), np.zeros(5 * Nm)
    sep = np.zeros(32, dtype=np.int32)
    N, M = C.c_int(0), C.c_int(0)
    keep = None
    dm = None
    if dmap is not None:
        keep = np.ascontiguousarray(dmap["distance"], dtype=np.float32)
        dm = C.byref(DistanceMap(ptr(keep), keep.shape[0], keep.shape[1], float(dmap["resolution"]),
                                 float(dmap["center_x"]), float(dmap["center_y"])))
    p = lambda a: a.ctypes.data  # noqa: E731
    reason = lib().tension_emu_stage(len(px), p(px), p(py), dm, *map(float, weights), int(max_raw), Nm, C.byref(N),
                                     p(st), p(clear), p(A_col), p(A_val), p(l), p(u), p(Pd), p(Po_idx), p(Po_val),
                                     p(cp), p(cr), p(cv), p(sep), C.byref(M))
    del keep
    N = N.value
    k = 3 * N
    nnz = int(cp[k]) if N else 0
    return dict(reason=reason, N=N, stations=st[:N], clearance=clear[:N], A_col=A_col[:k], A_val=A_val[:k], l=l[:k],
                u=u[:k], Pd=Pd[:k], Po_idx=Po_idx[:k], Po_val=Po_val[:k], csc_ptr=cp[:k + 1] if N else cp[:0],
                csc_row=cr[:nnz], csc_val=cv[:nnz], sep=sep[:M.value])


def solve(params, g):
    """The width-9 generic core on the QP of stage(): dict(status, iters, frenet [N][3] = (x_i, y_i, d_i))."""
    N = g["N"]
    frenet = np.zeros((N, 3))
    status, iters = C.c_int32(0), C.c_int32(0)
    c = lambda a: np.ascontiguousarray(a)   # noqa: E731
    arrs = [c(g[k]) for k in ("A_col", "A_val", "l", "u", "Pd", "Po_idx", "Po_val", "csc_ptr", "csc_row", "csc_val",
                              "sep", "stations")]
    lib().tension_emu_solve(C.byref(params), N, len(g["sep"]), *[a.ctypes.data for a in arrs], frenet.ctypes.data,
                            C.byref(status), C.byref(iters))
    return dict(status=status.value, iters=iters.value, frenet=frenet)
