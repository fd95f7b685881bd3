"""ctypes loader for the distance-transform emulator (TEST HARNESS): tests/emu/edt_emu.cpp, compiled with plain g++
(-DPQP_HOST_EMU) on first use into a temporary directory, runs the per-thread functions of csrc/pqp_edt_core.cuh in the
kernels' scratch layout.  Never used by the product."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "edt_emu.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="pqp_edt_emu_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libedt_emu.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", _SRC, "-o", so], check=True)
        L = C.CDLL(so)
        L.edt_emu.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_void_p]
        L.edt_emu.restype = None
        _lib = L
    return _lib


def distance_map(occupancy, resolution):
    """The layer pqp_set_maps_occupancy builds from `occupancy` uint8 [rows, cols] (0 = obstacle): float32 [rows, cols]."""
    occ = np.ascontiguousarray(occupancy, dtype=np.uint8)
    out = np.empty(occ.shape, dtype=np.float32)
    lib().edt_emu(occ.ctypes.data, occ.shape[0], occ.shape[1], float(resolution), out.ctypes.data)
    return out
