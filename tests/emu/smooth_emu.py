"""ctypes loader for the smoothing emulator (TEST HARNESS): tests/emu/smooth_emu.cpp, compiled with plain g++
(-DPQP_HOST_EMU) on first use into a temporary directory, runs the per-thread functions of pqp_smooth_reference_device
(csrc/pqp_smooth_core.cuh) on one polyline, and the width-4 generic core (csrc/pqp_gen_core.cuh) on its QP with one
host thread per lane.  Never used by the product."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

from path_optimizer_b200.abi import STATE_DTYPE

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "smooth_emu.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="pqp_smooth_emu_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libsmooth_emu.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", _SRC, "-o", so,
                        "-lpthread"], check=True)
        L = C.CDLL(so)
        vp, d_, i_ = C.c_void_p, C.c_double, C.c_int
        L.smooth_emu_stage.argtypes = [i_, vp, vp, d_, d_, d_, i_, i_] + [vp] * 22
        L.smooth_emu_stage.restype = i_
        L.smooth_emu_solve.argtypes = [vp, i_, i_] + [vp] * 16
        L.smooth_emu_solve.restype = i_
        _lib = L
    return _lib


def stage(px, py, weights=(0.005, 1.0, 10.0), max_raw=4096, max_points=512):
    """One polyline: dict(reason, t, x, y, s, xc, yc, stations (STATE_DTYPE), and the band-order QP: A_col [m][4], A_val,
    l, u, Pd, q, Po_idx [n][2], Po_val, csc_ptr, csc_row, csc_val, sep)."""
    f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)   # noqa: E731
    px, py = f64(px), f64(py)
    Km, Nm = int(max_raw), int(max_points)
    t, x, y, s = (np.zeros(Km + 1) for _ in range(4))
    xc, yc = np.zeros((Km, 4)), np.zeros((Km, 4))
    st = np.zeros(Nm, dtype=STATE_DTYPE)
    n, m = 4 * Nm, 3 * Nm
    A_col, A_val = np.zeros((m, 4), dtype=np.int32), np.zeros((m, 4))
    l, u, Pd, q = np.zeros(m), np.zeros(m), np.zeros(n), np.zeros(n)
    Po_idx, Po_val = np.zeros((n, 2), dtype=np.int32), np.zeros((n, 2))
    cp, cr, cv = np.zeros(n + 1, dtype=np.int32), np.zeros(9 * Nm, dtype=np.int32), np.zeros(9 * Nm)
    sep = np.zeros(32, dtype=np.int32)
    K, N, M = C.c_int(0), C.c_int(0), C.c_int(0)
    p = lambda a: a.ctypes.data  # noqa: E731
    reason = lib().smooth_emu_stage(len(px), p(px), p(py), *map(float, weights), Km, Nm, C.byref(K), p(t), p(x), p(y),
                                    p(s), p(xc), p(yc), C.byref(N), p(st), p(A_col), p(A_val), p(l), p(u), p(Pd), p(q),
                                    p(Po_idx), p(Po_val), p(cp), p(cr), p(cv), p(sep), C.byref(M))
    K, N = K.value, N.value
    nn, mm = max(4 * N - 1, 0), max(3 * N - 1, 0)
    return dict(reason=reason, t=t[:K], x=x[:K], y=y[:K], s=s[:K], xc=xc[:K], yc=yc[:K], stations=st[:N], N=N,
                A_col=A_col[:mm], A_val=A_val[:mm], l=l[:mm], u=u[:mm], Pd=Pd[:nn], q=q[:nn], Po_idx=Po_idx[:nn],
                Po_val=Po_val[:nn], csc_ptr=cp[:nn + 1] if N else cp[:0], csc_row=cr[:max(9 * N - 7, 0)],
                csc_val=cv[:max(9 * N - 7, 0)], sep=sep[:M.value])


def solve(params, g):
    """The width-4 generic core on the QP of stage(): dict(status, iters, frenet [N][3] = (x_i, y_i, theta_i))."""
    N = g["N"]
    frenet = np.zeros((N, 3))
    status, iters = C.c_int32(0), C.c_int32(0)
    c = lambda a: np.ascontiguousarray(a)   # noqa: E731
    arrs = [c(g[k]) for k in ("A_col", "A_val", "l", "u", "Pd", "q", "Po_idx", "Po_val", "csc_ptr", "csc_row",
                              "csc_val", "sep", "stations")]
    lib().smooth_emu_solve(C.byref(params), N, len(g["sep"]), *[a.ctypes.data for a in arrs], frenet.ctypes.data,
                           C.byref(status), C.byref(iters))
    return dict(status=status.value, iters=iters.value, frenet=frenet)
