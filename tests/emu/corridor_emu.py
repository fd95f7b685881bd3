"""ctypes loader for the corridor emulator (TEST HARNESS): tests/emu/corridor_emu.cpp, compiled with plain g++
(-DPQP_HOST_EMU) on first use into a temporary directory, runs the per-thread functions of pqp_post_smooth_device's
search kernel (csrc/pqp_corridor_core.cuh) on one path.  Never used by the product."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

from path_optimizer_b200.abi import STATE_DTYPE

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "corridor_emu.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="pqp_corridor_emu_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libcorridor_emu.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", _SRC, "-o", so], check=True)
        L = C.CDLL(so)
        vp, d_, i_ = C.c_void_p, C.c_double, C.c_int
        L.corridor_emu.argtypes = ([i_, vp, vp, vp, d_, vp, vp, i_, i_, d_, d_, d_, d_, d_, d_, i_] + [vp] * 15)
        L.corridor_emu.restype = i_
        _lib = L
    return _lib


def search(knots, x_coef, y_coef, max_s, start, m, range_=10.0, spacing=0.6, ds_long=1.5, max_layers=400):
    """One path: dict(reason, s, bounds [R][2], chain, vehicle_l, A_col [m][4], A_val, l, u, csc_ptr, csc_row, csc_val,
    sep)."""
    f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)   # noqa: E731
    kn, xc, yc = f64(knots), f64(x_coef).reshape(-1), f64(y_coef).reshape(-1)
    st = np.ascontiguousarray(np.array([start], dtype=STATE_DTYPE))
    dist = np.ascontiguousarray(m["distance"], dtype=np.float32)
    Lm = int(max_layers)
    s, lo, hi = np.zeros(Lm), np.zeros(Lm), np.zeros(Lm)
    chain = np.zeros(Lm, dtype=np.int32)
    A_col, A_val = np.zeros((3 * Lm, 4), dtype=np.int32), np.zeros((3 * Lm, 4))
    l, u = np.zeros(3 * Lm), np.zeros(3 * Lm)
    cp, cr, cv = np.zeros(3 * Lm + 1, dtype=np.int32), np.zeros(7 * Lm, dtype=np.int32), np.zeros(7 * Lm)
    sep = np.zeros(32, dtype=np.int32)
    R, M, vl = C.c_int(0), C.c_int(0), C.c_double(np.nan)
    p = lambda a: a.ctypes.data  # noqa: E731
    reason = lib().corridor_emu(len(kn), p(kn), p(xc), p(yc), float(max_s), p(st), p(dist), dist.shape[0], dist.shape[1],
                                float(m["resolution"]), float(m["center_x"]), float(m["center_y"]), float(range_),
                                float(spacing), float(ds_long), Lm, C.byref(R), p(s), p(lo), p(hi), p(chain),
                                C.byref(vl), p(A_col), p(A_val), p(l), p(u), p(cp), p(cr), p(cv), p(sep), C.byref(M))
    R, mm = R.value, 3 * R.value - 2
    return dict(reason=reason, s=list(s[:R]), bounds=list(zip(lo[:R], hi[:R])), chain=list(chain[:R]), vehicle_l=vl.value,
                A_col=A_col[:max(mm, 0)], A_val=A_val[:max(mm, 0)], l=l[:max(mm, 0)], u=u[:max(mm, 0)],
                csc_ptr=cp[:3 * R + 1] if R else cp[:0], csc_row=cr[:max(7 * R - 6, 0)], csc_val=cv[:max(7 * R - 6, 0)],
                sep=list(sep[:M.value]))
