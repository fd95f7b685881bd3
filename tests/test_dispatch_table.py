"""CPU test of the device dispatch's per-path class selection (pqp_dispatch.h): keep_control_steps from the reference
states, the caller's bounds, and the lookup in the class table the library builds with its own selection.  The same
source that nvcc compiles into the dispatch kernel is compiled here with g++ (tests/emu/dispatch_emu.cpp) and must
agree with pqp_keep_control_steps + pqp_class_info_form for every length up to two stations past the table, at every
station spacing of the shape sweep and at keep > 10, for all three formulations."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from path_optimizer_b200 import _lib, synth
from path_optimizer_b200.abi import ERR_CAPACITY, STATE_DTYPE
from tests import shapes

HERE = os.path.dirname(os.path.abspath(__file__))
FORMS = {"KP": shapes.KP, "K": shapes.K, "KPC": shapes.KPC}
KEEP_OVER_10 = 0.05     # station spacing that gives keep_control_steps > 10


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("dispatch_emu") / "libdispatch_emu.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", os.path.join(HERE, "emu", "dispatch_emu.cpp"), "-o", so],
                   check=True)
    L = C.CDLL(so)
    L.dispatch_emu_class.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.POINTER(C.c_int)]
    L.dispatch_emu_class.restype = C.c_int
    return L


def class_table(form):
    L = _lib.load()
    ncols = C.c_int()
    assert L.pqp_class_table(form, 0, None, 0, C.byref(ncols)) == 0
    tab = np.zeros(11 * ncols.value, dtype=np.int8)
    assert L.pqp_class_table(form, 0, tab.ctypes.data_as(C.c_void_p), len(tab) - 1, C.byref(ncols)) == ERR_CAPACITY
    assert L.pqp_class_table(form, 0, tab.ctypes.data_as(C.c_void_p), len(tab), C.byref(ncols)) == 0
    return tab, ncols.value


def _ref(n, ds):
    ref = np.zeros(max(n, 1), dtype=STATE_DTYPE)
    ref["s"][:n] = synth._accumulate_s(n, ds)
    return ref


def _emu(H, tab, ncols, form, ref, n, max_n=0, min_keep=0, max_keep=0):
    keep = C.c_int()
    v = H.dispatch_emu_class(tab.ctypes.data_as(C.c_void_p), ncols, form, ref.ctypes.data_as(C.c_void_p), n, max_n,
                             min_keep, max_keep, C.byref(keep))
    return v, keep.value


@pytest.mark.parametrize("name", list(FORMS))
def test_selection_matches_host(harness, name):
    form = FORMS[name]
    L = _lib.load()
    tab, ncols = class_table(form)
    limit = ncols - 2
    # the table ends one station past the longest path any class of the formulation takes
    assert limit == max(shapes.max_points(form, k) for k in ((1, 2, 3, 4, 5, 7, 10) if form == shapes.KP else (1,)))
    keeps_seen, classes_seen = set(), set()
    for ds in shapes.SPACINGS + (KEEP_OVER_10,):
        for n in range(0, limit + 3):
            ref = _ref(n, ds)
            keep = L.pqp_keep_control_steps(form, ref.ctypes.data_as(C.c_void_p), n)
            v, t, s = C.c_int(), C.c_int(), C.c_int64()
            L.pqp_class_info_form(form, n, keep, 0, C.byref(v), C.byref(t), C.byref(s))
            got, got_keep = _emu(harness, tab, ncols, form, ref, n)
            assert (got, got_keep) == (v.value, keep), (name, ds, n, got, v.value, got_keep, keep)
            keeps_seen.add(keep)
            classes_seen.add(got)
    if form == shapes.KP:
        assert {1, 2, 3, 4, 5, 7, 10} <= keeps_seen and max(keeps_seen) > 10
    assert {_lib.load().pqp_class_name(c).decode() for c in classes_seen} >= set(shapes.CLASSES[form])


def test_bounds_reject(harness):
    """A path outside the stated bounds gets no class (-1: PQP_INVALID_PROBLEM); 0 means unknown."""
    tab, ncols = class_table(shapes.KP)
    ref = _ref(120, 0.3)                                      # keep 3
    assert _emu(harness, tab, ncols, shapes.KP, ref, 120)[0] >= 0
    assert _emu(harness, tab, ncols, shapes.KP, ref, 120, max_n=119)[0] == -1
    assert _emu(harness, tab, ncols, shapes.KP, ref, 120, max_n=120)[0] >= 0
    assert _emu(harness, tab, ncols, shapes.KP, ref, 120, min_keep=4)[0] == -1
    assert _emu(harness, tab, ncols, shapes.KP, ref, 120, max_keep=2)[0] == -1
    assert _emu(harness, tab, ncols, shapes.KP, ref, 120, min_keep=3, max_keep=3)[0] >= 0
    # keep bounds do not apply to K and KPC (their keep is fixed)
    for form in (shapes.K, shapes.KPC):
        t, nc = class_table(form)
        assert _emu(harness, t, nc, form, ref, 120, min_keep=5, max_keep=6)[0] >= 0
