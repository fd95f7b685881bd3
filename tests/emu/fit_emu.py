"""ctypes loader for the spline-fit emulator (TEST HARNESS): tests/emu/fit_emu.cpp, compiled with plain g++
(-DPQP_HOST_EMU) on first use into a temporary directory, runs the per-thread functions of pqp_fit_splines_device
(csrc/pqp_env_core.cuh) over a batch.  Never used by the product."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

from path_optimizer_b200.abi import STATE_DTYPE

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "fit_emu.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="pqp_fit_emu_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libfit_emu.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", _SRC, "-o", so], check=True)
        L = C.CDLL(so)
        L.fit_emu.argtypes = [C.c_int] + [C.c_void_p] * 6
        L.fit_emu.restype = None
        _lib = L
    return _lib


def fit_splines(offsets, ref):
    """What pqp_fit_splines_device writes for a batch: dict(knots [T], x_coef [T, 4], y_coef [T, 4], ok int32 [B])."""
    off = np.ascontiguousarray(offsets, dtype=np.int32)
    ref = np.ascontiguousarray(ref, dtype=STATE_DTYPE)
    B, T = len(off) - 1, len(ref)
    knots, xc, yc = np.zeros(T), np.zeros((T, 4)), np.zeros((T, 4))
    ok = np.zeros(B, dtype=np.int32)
    lib().fit_emu(B, off.ctypes.data, ref.ctypes.data, knots.ctypes.data, xc.ctypes.data, yc.ctypes.data, ok.ctypes.data)
    return dict(knots=knots, x_coef=xc, y_coef=yc, ok=ok)
