"""CPU tests of the kernel-class selection (host logic of libpqp.so, no device): every BASELINE path length maps
onto a thread-per-station class, the single class of the device entry point takes every path inside the caller's
bounds, and the documented length limits hold."""
import ctypes as C

import pytest

from path_optimizer_b200 import _lib


def _class(n, keep):
    L = _lib.load()
    v, t, s = C.c_int(), C.c_int(), C.c_int64()
    rc = L.pqp_class_info(n, keep, 0, C.byref(v), C.byref(t), C.byref(s))
    return rc, L.pqp_class_name(v.value).decode(), t.value, s.value


def test_every_baseline_length_runs_thread_per_station():
    """Configs 2-5 use 0.3 m stations (keep_control_steps 3) and 50..400 stations: none of them may fall back to the
    one-warp kernel."""
    for keep in (3, 4):
        for n in range(2, 409):
            rc, name, threads, smem = _class(n, keep)
            assert rc == 0 and name.startswith("pqp_kp3_solve_kernel"), (n, keep, name)
            assert threads >= n and smem <= 232448
    assert _class(100, 3)[1] == "pqp_kp3_solve_kernel<17,6,4,17>"
    assert _class(200, 3)[1] == "pqp_kp3_solve_kernel<17,6,8,34>"
    assert _class(300, 3)[1] == "pqp_kp3_solve_kernel<27,7,10,34>"
    assert _class(350, 3)[1] == "pqp_kp3_solve_kernel<37,7,12,34>"
    assert _class(400, 3)[1] == "pqp_kp3_solve_kernel<37,7,13,34>"


def test_long_and_dense_station_paths_fall_back_then_fail():
    assert _class(412, 3)[1] == "pqp_kp_solve_kernel"          # one-warp kernel beyond the 13-warp class
    assert _class(415, 3)[0] != 0                              # too long for one SM: PQP_INVALID_PROBLEM
    assert _class(300, 8)[1] == "pqp_kp_solve_kernel"          # 0.15 m stations (keep 8): one-warp kernel
    assert _class(322, 8)[0] != 0


@pytest.mark.parametrize("hint", [(100, 3, 3), (128, 3, 4), (150, 3, 4), (200, 3, 3), (256, 3, 4), (400, 3, 3), (408, 3, 4)])
def test_device_class_covers_its_bounds(hint):
    """pqp_device_class_info returns PQP_ERR_ARG when a (n, keep) inside the bounds would fail the kernel's own
    fits / shared-memory check."""
    L = _lib.load()
    v, t, s = C.c_int(), C.c_int(), C.c_int64()
    assert L.pqp_device_class_info(hint[0], hint[1], hint[2], 0, C.byref(v), C.byref(t), C.byref(s)) == 0
    assert t.value >= hint[0] or t.value == 32
    assert s.value <= 232448


def test_shape_sweeps_reach_every_class():
    """The GPU shape sweep (test_gpu_shapes.py) runs every length at the keep values of its station spacings: together
    they reach every class each formulation selects, and every compiled class is either selected or listed as not
    selected.  The emulator runs each compiled class under the name the library reports for it."""
    from tests import shapes
    from tests.emu import emu
    assert shapes.kp_keeps() == [1, 2, 3, 4, 5, 7, 8, 10]
    for form, keeps in ((shapes.KP, shapes.kp_keeps()), (shapes.K, [1]), (shapes.KPC, [4])):
        reached = set()
        for keep in keeps:
            reached |= set(shapes.class_ranges(form, keep))
        assert reached == set(shapes.CLASSES[form]), (form, sorted(reached ^ set(shapes.CLASSES[form])))
    compiled = shapes.compiled_classes()
    assert sorted(compiled) == sorted(sum(shapes.CLASSES.values(), []) + shapes.UNSELECTED)
    assert set(emu.VARIANTS) == set(compiled)


def test_device_class_refuses_bounds_no_single_class_takes():
    L = _lib.load()
    v, t, s = C.c_int(), C.c_int(), C.c_int64()
    assert L.pqp_device_class_info(400, 1, 4, 0, C.byref(v), C.byref(t), C.byref(s)) != 0
