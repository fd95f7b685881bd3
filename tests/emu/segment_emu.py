"""ctypes loader for the segmentation emulator (TEST HARNESS): tests/emu/segment_emu.cpp, compiled with plain g++
(-DPQP_HOST_EMU) on first use into a temporary directory, runs the per-thread functions of
pqp_segment_reference_device (csrc/pqp_segment_core.cuh) over a batch.  Never used by the product."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

from path_optimizer_b200.abi import STATE_DTYPE

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "segment_emu.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="pqp_segment_emu_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libsegment_emu.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", _SRC, "-o", so], check=True)
        L = C.CDLL(so)
        vp = C.c_void_p
        L.segment_emu.argtypes = ([C.c_int] + [vp] * 7 + [C.c_double, C.c_double, C.c_int, C.c_double, C.c_int, C.c_int]
                                  + [vp] * 8)
        L.segment_emu.restype = None
        _lib = L
    return _lib


def segment(splines, max_s, start, goal, capacity, max_n=1 << 30, ds_small=0.15, ds_large=0.3, dynamic=True,
            search_ds=0.5):
    """What pqp_segment_reference_device writes for a batch: dict(n_points, offsets, ref [offsets[B]] records, x0 [B, 3],
    end_heading, ok) plus reason and cut_s.  start / goal: STATE_DTYPE records [B]."""
    ko = np.ascontiguousarray(splines["knot_offsets"], dtype=np.int32)
    kn = np.ascontiguousarray(splines["knots"], dtype=np.float64)
    xc = np.ascontiguousarray(splines["x_coef"], dtype=np.float64)
    yc = np.ascontiguousarray(splines["y_coef"], dtype=np.float64)
    ms = np.ascontiguousarray(max_s, dtype=np.float64)
    st = np.ascontiguousarray(start, dtype=STATE_DTYPE)
    gl = np.ascontiguousarray(goal, dtype=STATE_DTYPE)
    B = len(ms)
    n = np.zeros(B, dtype=np.int32)
    off = np.zeros(B + 1, dtype=np.int32)
    ref = np.zeros(max(int(capacity), 1), dtype=STATE_DTYPE)
    x0, end = np.zeros((B, 3)), np.zeros(B)
    ok, reason, cut = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32), np.zeros(B)
    p = lambda a: a.ctypes.data  # noqa: E731
    lib().segment_emu(B, p(ko), p(kn), p(xc), p(yc), p(ms), p(st), p(gl), float(ds_small), float(ds_large),
                      int(bool(dynamic)), float(search_ds), int(max_n), int(capacity), p(n), p(off), p(ref), p(x0),
                      p(end), p(ok), p(reason), p(cut))
    return dict(n_points=n, offsets=off, ref=ref[:off[-1]], x0=x0, end_heading=end, ok=ok, reason=reason, cut_s=cut)
