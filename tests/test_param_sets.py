"""CPU tests of one batch over several parameter sets: the set-indexed emulator drivers (the kernels' lookup
pqp::param_of on a parameter table, tests/emu/env_sets_emu.cpp) against the map-indexed drivers run with each set's
params and against the oracle with each path's own params; the device dispatch's (set, class) segment sort against the
host selection; the argument checks of the new entries.

Bounds, cuts and flags are compared exactly against the drivers and the oracle (simple bounds; improved bounds to 1e-9,
as tests/test_env_oracle.py); tail states exactly against the drivers and to 1e-9 against the oracle."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from oracle import oracle
from path_optimizer_b200 import _lib, planner, synth
from path_optimizer_b200.abi import ERR_ARG, FORMULATIONS, Params
from tests.emu import maps_emu, sets_emu

S, N_MAPS, N_CAND, N = 6, 3, 8, 120
WILD = dict(y_range=(-3.0, 3.0), heading_range=0.05, curvature_amp=0.02)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _config1_map():
    g = np.load(os.path.join(ROOT, "tests", "golden", "config1_benchmark_map.npz"))
    return dict(distance=g["map_distance"], rows=int(g["image_shape"][0]), cols=int(g["image_shape"][1]),
                resolution=float(g["map_geo"][0]), center_x=float(g["map_geo"][1]), center_y=float(g["map_geo"][2]))


@pytest.fixture(scope="module")
def scene():
    maps, b, mi = synth.multi_map_batch(N_MAPS, N_CAND, n=N, first_maps=[_config1_map()], order="interleaved", **WILD)
    pi = (np.arange(len(mi)) % S).astype(np.int32)
    np.random.default_rng(7).shuffle(pi)
    return maps, b, mi, pi, synth.param_sets(S, seed=11)


def test_param_sets_differ_in_every_group(scene):
    sets = scene[4]
    f = lambda name: {round(getattr(p, name), 12) for p in sets}   # noqa: E731
    for name in ("circle_radius", "d1", "wheel_base", "max_steering_angle", "KP_deviation_weight", "K_curvature_weight",
                 "expected_safety_margin", "mu", "max_curvature_rate", "eps_abs", "max_iter", "adaptive_rho_interval",
                 "constraint_end_heading"):
        assert len(f(name)) > 1, name
    assert 0 in f("constraint_end_heading") and 100 in f("adaptive_rho_interval")


@pytest.mark.parametrize("mode", [planner.BOUNDS_SIMPLE, planner.BOUNDS_IMPROVED])
def test_bounds_sets_match_drivers_and_oracle(scene, mode):
    maps, b, mi, pi, sets = scene
    spl = planner.reference_splines(b) if mode == planner.BOUNDS_IMPROVED else None
    got = sets_emu.update_bounds_sets(sets, pi, maps, mi, b, mode=mode, splines=spl)
    G = got["bounds"].view(np.float64).reshape(-1, 8)
    radii = set()
    for k in range(S):
        idx = np.flatnonzero(pi == k)
        sub = synth.take_paths(b, idx)
        sspl = planner.reference_splines(sub) if spl is not None else None
        want = maps_emu.update_bounds_maps(sets[k], maps, mi[idx], sub, mode=mode, splines=sspl)
        W = want["bounds"].view(np.float64).reshape(-1, 8)
        for j, i in enumerate(idx):
            assert got["n_valid"][i] == want["n_valid"][j]
            g, w = slice(b["offsets"][i], b["offsets"][i + 1]), slice(sub["offsets"][j], sub["offsets"][j + 1])
            nv = want["n_valid"][j]
            assert G[g][:nv].tobytes() == W[w][:nv].tobytes(), (k, i)
        for j, i in enumerate(idx[:2]):
            one = synth.take_paths(b, [i])
            o = oracle.update_bounds(sets[k], maps[mi[i]], one, mode=mode,
                                     splines=planner.reference_splines(one) if spl is not None else None)
            nv = o["n_valid"][0]
            assert got["n_valid"][i] == nv
            Og = G[b["offsets"][i]:b["offsets"][i] + nv]
            Ow = o["bounds"][:nv].view(np.float64).reshape(-1, 8)
            if mode == planner.BOUNDS_SIMPLE:
                assert Og.tobytes() == Ow.tobytes(), (k, i)
            else:
                assert np.abs(Og - Ow).max(initial=0.0) <= 1e-9, (k, i)
        radii.add(round(sets[k].circle_radius, 9))
    assert len(radii) >= 4


@pytest.mark.parametrize("tail", ["raw", "densify"])
def test_tails_sets_match_drivers_and_oracle(scene, tail):
    maps, b, mi, pi, sets = scene
    if tail == "raw":
        got = sets_emu.finish_raw_sets(sets, pi, maps, mi, b["n_points"], b["ref"])
    else:
        got = sets_emu.densify_sets(sets, pi, maps, mi, b["n_points"], b["ref"], max_out=512)
    cut = "n_kept" if tail == "raw" else "n_out"
    for k in range(S):
        idx = np.flatnonzero(pi == k)
        sub = synth.take_paths(b, idx)
        if tail == "raw":
            want = maps_emu.finish_raw_maps(sets[k], maps, mi[idx], sub["n_points"], sub["ref"])
        else:
            want = maps_emu.densify_maps(sets[k], maps, mi[idx], sub["n_points"], sub["ref"], max_out=512)
        for j, i in enumerate(idx):
            assert got[cut][i] == want[cut][j] and got["ok"][i] == want["ok"][j], (k, i)
            if tail == "raw":
                assert (got["states"][b["offsets"][i]:b["offsets"][i + 1]].tobytes()
                        == want["states"][sub["offsets"][j]:sub["offsets"][j + 1]].tobytes())
            else:
                assert got["states"][i, :got[cut][i]].tobytes() == want["states"][j, :want[cut][j]].tobytes()
        i = idx[0]
        one = synth.take_paths(b, [i])
        if tail == "raw":
            o = oracle.finish_raw(sets[k], maps[mi[i]], one["n_points"], one["ref"])
            assert (o["n_kept"][0], o["ok"][0]) == (got["n_kept"][i], got["ok"][i])
            gs = got["states"]["s"][b["offsets"][i]:b["offsets"][i + 1]]
            assert np.abs(o["states"]["s"] - gs).max(initial=0.0) <= 1e-9
        else:
            o = oracle.densify(sets[k], maps[mi[i]], one["n_points"], one["ref"], max_out=512)
            c = o["n_out"][0]
            assert (c, o["ok"][0]) == (got["n_out"][i], got["ok"][i])
            for f in "xyzks":
                assert np.abs(got["states"][f][i, :c] - o["states"][f][0, :c]).max(initial=0.0) <= 1e-9


def test_out_of_range_set_touches_only_its_path(scene):
    maps, b, mi, pi, sets = scene
    bad = pi.copy()
    bad[2], bad[5] = -1, S
    ok_b = sets_emu.update_bounds_sets(sets, pi, maps, mi, b)
    bd_b = sets_emu.update_bounds_sets(sets, bad, maps, mi, b)
    ok_t = sets_emu.finish_raw_sets(sets, pi, maps, mi, b["n_points"], b["ref"])
    bd_t = sets_emu.finish_raw_sets(sets, bad, maps, mi, b["n_points"], b["ref"])
    for i in range(len(bad)):
        if i in (2, 5):
            assert bd_b["n_valid"][i] == 0 and bd_t["n_kept"][i] == 0 and bd_t["ok"][i] == 0
            continue
        assert bd_b["n_valid"][i] == ok_b["n_valid"][i] and bd_t["n_kept"][i] == ok_t["n_kept"][i]
        o = slice(b["offsets"][i], b["offsets"][i + 1])
        assert bd_b["bounds"][o][:ok_b["n_valid"][i]].tobytes() == ok_b["bounds"][o][:ok_b["n_valid"][i]].tobytes()
    # without a collision check the tail reads no set: an out-of-range index changes nothing
    a = sets_emu.finish_raw_sets(sets, bad, maps, mi, b["n_points"], b["ref"], collision_check=False)
    w = sets_emu.finish_raw_sets(sets, pi, maps, mi, b["n_points"], b["ref"], collision_check=False)
    assert a["n_kept"].tolist() == w["n_kept"].tolist() and a["states"].tobytes() == w["states"].tobytes()


# ---- the dispatch's (set, class) segment sort ------------------------------------------------------------------------

def _class_table(form):
    L = _lib.load()
    ncols = C.c_int()
    assert L.pqp_class_table(form, 0, None, 0, C.byref(ncols)) == 0
    tab = np.zeros(11 * ncols.value, dtype=np.int8)
    assert L.pqp_class_table(form, 0, tab.ctypes.data_as(C.c_void_p), len(tab), C.byref(ncols)) == 0
    return tab, ncols.value


def _form_classes(form):
    """[v0, v1) of the formulation's classes in the library's table (pqp_class_info_form over every length and keep)."""
    L = _lib.load()
    vs = set()
    v, t, s = C.c_int(), C.c_int(), C.c_int64()
    for keep in range(1, 12):
        for n in range(0, 420):
            L.pqp_class_info_form(form, n, keep, 0, C.byref(v), C.byref(t), C.byref(s))
            vs.add(v.value)
    return min(vs), max(vs) + 1


@pytest.mark.parametrize("form", ["KP", "KPC", "K"])
@pytest.mark.parametrize("bounds", [dict(), dict(max_n=200, min_keep=2, max_keep=4)])
def test_segment_sort_places_every_path_once(form, bounds):
    f = FORMULATIONS[form]
    tab, ncols = _class_table(f)
    v0, v1 = _form_classes(f)
    nv = v1 - v0
    lens = np.random.default_rng(3).integers(2, 420, 96).astype(np.int32)
    lens[:3] = [2, 500, 1000]   # and two paths longer than any class takes
    b = synth.curvy_corridors(len(lens), n_points=lens)
    for i in range(0, len(lens), 7):   # some paths at 0.15 m spacing: keep 7..8 (KP)
        o, n = b["offsets"][i], b["n_points"][i]
        b["ref"]["s"][o:o + n] = np.arange(n) * 0.15
    n_sets = 5
    si = (np.arange(len(lens)) % (n_sets + 2) - 1).astype(np.int32)   # -1 and n_sets are out of range
    order, key = sets_emu.sort(tab, ncols, f, v0, nv, n_sets, b, si, **bounds)
    L = _lib.load()
    seen = {}
    for s in range(n_sets):
        for c in range(nv):
            seg = order[s, c]
            entries = seg[seg != len(lens)]
            assert (seg[len(entries):] == len(lens)).all()   # the sentinel fills the tail
            # longest first (every path longer than any class takes shares the last length bucket)
            assert (np.diff(np.minimum(b["n_points"][entries], ncols - 1)) <= 0).all(), (s, c)
            for i in entries:
                assert i not in seen
                seen[int(i)] = (s, c)
    for i in range(len(lens)):
        n = int(b["n_points"][i])
        ref = b["ref"][b["offsets"][i]:b["offsets"][i + 1]]
        keep = L.pqp_keep_control_steps(f, ref.ctypes.data_as(C.c_void_p), n)
        v, t, sm = C.c_int(), C.c_int(), C.c_int64()
        L.pqp_class_info_form(f, n, keep, 0, C.byref(v), C.byref(t), C.byref(sm))
        inside = not ((bounds.get("max_n", 0) and n > bounds["max_n"]) or
                      (f == FORMULATIONS["KP"] and bounds and not (bounds["min_keep"] <= keep <= bounds["max_keep"])))
        if 0 <= si[i] < n_sets and inside:
            assert seen.get(i) == (si[i], v.value - v0), i
        else:
            assert i not in seen and key[i] == -1, i


# ---- argument checks -------------------------------------------------------------------------------------------------

def test_max_param_sets_is_at_least_64():
    src = open(os.path.join(ROOT, "include", "pqp.h")).read()
    assert int(re.search(r"#define PQP_MAX_PARAM_SETS (\d+)", src).group(1)) >= 64


def test_entries_refuse_bad_arguments():
    L = _lib.load()
    arr = (Params * 2)()
    assert L.pqp_set_param_sets(None, 1, arr) == ERR_ARG
    vp = [None] * 12
    assert L.pqp_solve_batch_sets(None, 0, 1, *vp, None) == ERR_ARG
    assert L.pqp_solve_batch_device_dispatch_sets(None, 0, 1, 2, 0, 0, 0, 0, *([None] * 14), None) == ERR_ARG
    assert L.pqp_plan_batch_sets(None, 0, 1, 0, 1, *([None] * 10), 0.3, 1, 16, *([None] * 6), None) == ERR_ARG
    assert L.pqp_plan_batch_device_sets(None, 0, 1, 0, 1, 2, 0, 0, *([None] * 11), 0.3, 1, 16, *([None] * 7),
                                        None) == ERR_ARG
