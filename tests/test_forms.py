"""CPU tests of one batch over several formulations ("KP", "K", "KPC" per path): the per-path-formulation dispatch of
pqp_dispatch.h (pqp::dispatch_key_forms and the sort built on it, compiled with g++ from tests/emu/forms_emu.cpp)
against the host selection (pqp_keep_control_steps + pqp_class_info_form), the argument checks of the four _forms
entries, and the C++ driver against the headers."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from path_optimizer_b200 import _lib, synth
from path_optimizer_b200.abi import ERR_ARG, STATE_DTYPE
from tests import shapes

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FORMS = (shapes.KP, shapes.K, shapes.KPC)
ALL = 7


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("forms_emu") / "libforms_emu.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", os.path.join(HERE, "emu", "forms_emu.cpp"), "-o", so],
                   check=True)
    L = C.CDLL(so)
    vp = C.c_void_p
    L.forms_emu_key.argtypes = [vp, vp, vp] + [C.c_int] * 10
    L.forms_emu_key.restype = C.c_int
    L.forms_dispatch_emu.argtypes = [vp, vp, vp] + [C.c_int] * 5 + [vp] * 5 + [C.c_int] * 2 + [vp] * 2
    L.forms_dispatch_emu.restype = None
    return L


def _class_table(form):
    L = _lib.load()
    ncols = C.c_int()
    assert L.pqp_class_table(form, 0, None, 0, C.byref(ncols)) == 0
    tab = np.zeros(11 * ncols.value, dtype=np.int8)
    assert L.pqp_class_table(form, 0, tab.ctypes.data_as(C.c_void_p), len(tab), C.byref(ncols)) == 0
    return tab, ncols.value


class Tables:
    """The three class tables as the library builds them, in the argument shape of forms_emu.cpp."""

    def __init__(self, max_n=(0, 0, 0)):
        self.tabs = [_class_table(f) for f in FORMS]
        self.ptrs = (C.c_void_p * 3)(*[t.ctypes.data_as(C.c_void_p).value for t, _ in self.tabs])
        self.ncols = (C.c_int * 3)(*[n for _, n in self.tabs])
        self.max_n = (C.c_int * 3)(*max_n)
        self.stride = max(n for _, n in self.tabs)
        self.n_variants = len(shapes.compiled_classes())

    def key(self, H, form, n, keep, form_mask=ALL, set_=0, n_sets=1, min_keep=0, max_keep=0):
        return H.forms_emu_key(self.ptrs, self.ncols, self.max_n, form_mask, form, set_, n_sets, n, keep, min_keep,
                               max_keep, self.n_variants, self.stride)


def _host_class(form, n, keep):
    L = _lib.load()
    v, t, s = C.c_int(), C.c_int(), C.c_int64()
    L.pqp_class_info_form(form, n, keep, 0, C.byref(v), C.byref(t), C.byref(s))
    return v.value


@pytest.mark.parametrize("form", FORMS)
def test_mixed_key_picks_the_host_class(harness, form):
    """Every length from 0 to one past the formulation's table and keep 1..11: the key's class is class_for's."""
    T = Tables()
    ncols = T.tabs[form][1]
    seen = set()
    for keep in range(1, 12):
        for n in range(0, ncols):
            k = T.key(harness, form, n, keep, set_=2, n_sets=3)
            assert k >= 0, (form, n, keep)
            seg, bucket = divmod(k, T.stride)
            s, v = divmod(seg, T.n_variants)
            assert (s, v) == (2, _host_class(form, n, keep)), (form, n, keep, s, v)
            assert bucket == T.stride - 1 - min(n, T.stride - 1)
            seen.add(v)
    assert {_lib.load().pqp_class_name(v).decode() for v in seen} >= set(shapes.CLASSES[form])


def test_unknown_and_out_of_mask_forms_and_sets_get_no_key(harness):
    T = Tables()
    for f in (-1, 3, 7, -100):
        assert T.key(harness, f, 100, 3) == -1
    for f in FORMS:
        assert T.key(harness, f, 100, 3, form_mask=ALL & ~(1 << f)) == -1
        assert T.key(harness, f, 100, 3, form_mask=1 << f) >= 0
        assert T.key(harness, f, 100, 3, set_=-1, n_sets=4) == -1
        assert T.key(harness, f, 100, 3, set_=4, n_sets=4) == -1
        assert T.key(harness, f, 100, 3, set_=3, n_sets=4) >= 0
    # bounds per formulation: max_n[f] for the paths of f only; keep bounds on "KP" only
    B = Tables(max_n=(100, 300, 50))
    assert B.key(harness, shapes.KP, 101, 3) == -1 and B.key(harness, shapes.KP, 100, 3) >= 0
    assert B.key(harness, shapes.K, 300, 1) >= 0 and B.key(harness, shapes.K, 301, 1) == -1
    assert B.key(harness, shapes.KPC, 51, 4) == -1 and B.key(harness, shapes.KPC, 50, 4) >= 0
    assert T.key(harness, shapes.KP, 100, 3, min_keep=4) == -1
    assert T.key(harness, shapes.K, 100, 1, min_keep=4, max_keep=5) >= 0


def _mixed_batch(seed=5):
    rng = np.random.default_rng(seed)
    lens = rng.integers(2, 420, 120).astype(np.int32)
    lens[:4] = [2, 257, 417, 1000]   # past the "KPC" and "K" limits, and past every table
    b = synth.curvy_corridors(len(lens), n_points=lens)
    for i in range(0, len(lens), 5):   # some paths at 0.15 m spacing: keep 7..8 ("KP")
        o, n = b["offsets"][i], b["n_points"][i]
        b["ref"]["s"][o:o + n] = np.arange(n) * 0.15
    forms = (np.arange(len(lens)) % 5 - 1).astype(np.int32)   # -1, 0, 1, 2, 3: two of five are no formulation
    rng.shuffle(forms)
    return b, forms


@pytest.mark.parametrize("n_sets,mask", [(1, ALL), (4, ALL), (3, (1 << shapes.KP) | (1 << shapes.KPC))])
def test_segments_per_set_and_class_longest_first(harness, n_sets, mask):
    T = Tables()
    b, forms = _mixed_batch()
    B = len(forms)
    si = None if n_sets == 1 else (np.arange(B) % (n_sets + 1)).astype(np.int32)   # n_sets is out of range
    order = np.zeros(n_sets * T.n_variants * B, dtype=np.int32)
    key = np.zeros(B, dtype=np.int32)
    p = lambda a: None if a is None else np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)  # noqa: E731
    ref = np.ascontiguousarray(b["ref"], dtype=STATE_DTYPE)
    n_points = np.ascontiguousarray(b["n_points"], dtype=np.int32)
    offsets = np.ascontiguousarray(b["offsets"], dtype=np.int32)
    harness.forms_dispatch_emu(T.ptrs, T.ncols, T.max_n, mask, T.n_variants, T.stride, n_sets, B, p(n_points), p(offsets),
                               p(ref), p(si), p(forms), 0, 0, p(order), p(key))
    order = order.reshape(n_sets, T.n_variants, B)
    seen = {}
    for s in range(n_sets):
        for v in range(T.n_variants):
            seg = order[s, v]
            entries = seg[seg != B]
            assert (seg[len(entries):] == B).all()
            assert (np.diff(np.minimum(n_points[entries], T.stride - 1)) <= 0).all(), (s, v)
            for i in entries:
                assert int(i) not in seen
                seen[int(i)] = (s, v)
    L = _lib.load()
    for i in range(B):
        f, s = int(forms[i]), 0 if si is None else int(si[i])
        if not (0 <= f <= 2 and (mask >> f) & 1 and 0 <= s < n_sets):
            assert i not in seen and key[i] == -1, i
            continue
        r = ref[offsets[i]:offsets[i + 1]]
        keep = L.pqp_keep_control_steps(f, r.ctypes.data_as(C.c_void_p), int(n_points[i]))
        assert seen.get(i) == (s, _host_class(f, int(n_points[i]), keep)), i


# ---- the ABI -------------------------------------------------------------------------------------------------------

def test_abi_exports_the_four_entries():
    L = _lib.load()
    for name in ("pqp_solve_batch_forms", "pqp_solve_batch_device_dispatch_forms", "pqp_plan_batch_forms",
                 "pqp_plan_batch_device_forms"):
        assert hasattr(L, name) and name in _lib.SYMBOLS
    hdr = open(os.path.join(ROOT, "include", "pqp.h")).read() + open(os.path.join(ROOT, "include", "pqp_env.h")).read()
    for name in ("pqp_solve_batch_forms", "pqp_solve_batch_device_dispatch_forms", "pqp_plan_batch_forms",
                 "pqp_plan_batch_device_forms"):
        assert f"int {name}(" in hdr


def test_entries_refuse_bad_arguments():
    L = _lib.load()
    # no handle
    assert L.pqp_solve_batch_forms(None, 1, *([None] * 13), None) == ERR_ARG
    assert L.pqp_solve_batch_device_dispatch_forms(None, 1, 2, 0, 0, 0, 0, 0, *([None] * 15), None) == ERR_ARG
    assert L.pqp_plan_batch_forms(None, 1, 0, 1, *([None] * 11), 0.3, 1, 16, *([None] * 6), None) == ERR_ARG
    assert L.pqp_plan_batch_device_forms(None, 1, 0, 1, 2, 0, 0, 0, *([None] * 12), 0.3, 1, 16, *([None] * 7),
                                         None) == ERR_ARG


def test_cpp_driver_compiles(tmp_path):
    exe = str(tmp_path / "planner_forms_driver")
    lib = os.path.join(ROOT, "path_optimizer_b200")
    subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", os.path.join(HERE, "cpp", "planner_forms_driver.cpp"),
                    "-o", exe, "-L" + lib, "-lpqp", "-Wl,-rpath," + lib], check=True)
    # and the solver mirror's overload, from a translation unit of its own
    src = tmp_path / "solver_forms.cpp"
    src.write_text('#include "pqp_solver.hpp"\n'
                   "bool run(pqp::BatchPathSolver &s, const std::vector<int32_t> &n, const std::vector<pqp::State> &r,\n"
                   "         const std::vector<pqp::CoveringCircleBounds> &b, const std::vector<pqp::VehicleStateView> &v,\n"
                   "         pqp::BatchPathSolver::Result *out) {\n"
                   '    return s.solve(n, r, b, v, {}, std::vector<std::string>(n.size(), "KPC"), out);\n'
                   "}\n")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"),
                    str(src)], check=True)
