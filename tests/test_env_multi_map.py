"""CPU tests of planning one batch over several distance maps: the map-indexed emulator drivers (the kernels' lookup
pqp::map_of on a descriptor table, tests/emu/env_maps_emu.cpp) against the single-map drivers run per map and against the
oracle with each path's own map, on maps of different geometry with the paths of the maps interleaved.

Bounds, cuts and flags are compared exactly; re-accumulated s exactly; densified states to 1e-9 against the oracle
(floating point, as tests/test_env_oracle.py) and exactly against the single-map driver (the same code)."""
import os

import numpy as np
import pytest

from oracle import oracle
from path_optimizer_b200 import planner, synth
from tests.emu import emu, maps_emu

WILD = dict(y_range=(-3.0, 3.0), heading_range=0.05, curvature_amp=0.02)
N_MAPS, N_CAND, N = 4, 10, 120


def _config1_map():
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "config1_benchmark_map.npz"))
    return dict(distance=g["map_distance"], rows=int(g["image_shape"][0]), cols=int(g["image_shape"][1]),
                resolution=float(g["map_geo"][0]), center_x=float(g["map_geo"][1]), center_y=float(g["map_geo"][2]))


@pytest.fixture(scope="module")
def scene():
    maps, b, mi = synth.multi_map_batch(N_MAPS, N_CAND, n=N, first_maps=[_config1_map()], order="interleaved", **WILD)
    return maps, b, mi


def test_helper_builds_mixed_geometry(scene):
    maps, b, mi = scene
    assert len(maps) == N_MAPS and len(mi) == N_MAPS * N_CAND
    assert (mi[:N_MAPS] == np.arange(N_MAPS)).all()                        # interleaved
    geo = {(m["rows"], m["cols"], m["resolution"], m["center_x"], m["center_y"]) for m in maps}
    assert len(geo) >= 3                                                   # config 1, 0.2 m at 0, 0.25 m off-centre
    for m in range(N_MAPS):                                               # every line starts inside its own map
        mp = maps[m]
        st = b["ref"][b["offsets"][:-1][mi == m]]
        assert (np.abs(st["x"] - mp["center_x"]) < mp["rows"] * mp["resolution"] / 2).all()
        assert (np.abs(st["y"] - mp["center_y"]) < mp["cols"] * mp["resolution"] / 2).all()


def _per_map(fn, mi, n_maps):
    """fn(m, idx) for every map's paths."""
    for m in range(n_maps):
        fn(m, np.flatnonzero(mi == m))


@pytest.mark.parametrize("mode", [planner.BOUNDS_SIMPLE, planner.BOUNDS_IMPROVED])
def test_bounds_maps_match_single_map_and_oracle(scene, mode):
    maps, b, mi = scene
    prm = oracle.default_params()
    spl = planner.reference_splines(b) if mode == planner.BOUNDS_IMPROVED else None
    got = maps_emu.update_bounds_maps(prm, maps, mi, b, mode=mode, splines=spl)
    G = got["bounds"].view(np.float64).reshape(-1, 8)
    seen_blocked = []

    def check(m, idx):
        sub = synth.take_paths(b, idx)
        ssp = planner.reference_splines(sub) if spl is not None else None
        one = emu.update_bounds(prm, maps[m], sub, mode=mode, splines=ssp)
        want = oracle.update_bounds(prm, maps[m], sub, mode=mode, splines=ssp)
        assert (got["n_valid"][idx] == one["n_valid"]).all() and (one["n_valid"] == want["n_valid"]).all()
        O = one["bounds"].view(np.float64).reshape(-1, 8)
        W = want["bounds"].view(np.float64).reshape(-1, 8)
        for k, i in enumerate(idx):
            nv = want["n_valid"][k]
            g = G[b["offsets"][i]:b["offsets"][i] + nv]
            assert g.tobytes() == O[sub["offsets"][k]:sub["offsets"][k] + nv].tobytes()
            assert g.tobytes() == W[sub["offsets"][k]:sub["offsets"][k] + nv].tobytes()
        seen_blocked.append((want["n_valid"] < sub["n_points"]).any())
    _per_map(check, mi, len(maps))
    assert any(seen_blocked)
    # the same batch on one map: a NULL index is map 0
    g0 = maps_emu.update_bounds_maps(prm, maps, None, b, mode=mode, splines=spl)
    w0 = emu.update_bounds(prm, maps[0], b, mode=mode, splines=spl)
    assert (g0["n_valid"] == w0["n_valid"]).all()


def _solved_like(b):
    paths = b["ref"].copy()
    paths["s"] = 0.0
    return b["n_points"], paths


def test_tails_maps_match_single_map_and_oracle(scene):
    maps, b, mi = scene
    prm = oracle.default_params()
    n_points, paths = _solved_like(b)
    raw = maps_emu.finish_raw_maps(prm, maps, mi, n_points, paths)
    free = maps_emu.finish_raw_maps(prm, maps, mi, n_points, paths, collision_check=False)
    assert (free["n_kept"] == n_points).all()
    dense = maps_emu.densify_maps(prm, maps, mi, n_points, free["states"], 0.3, True, 256)
    cut = []

    def check(m, idx):
        sub = synth.take_paths(dict(b, ref=paths), idx)
        one = emu.finish_raw(prm, maps[m], sub["n_points"], sub["ref"])
        want = oracle.finish_raw(prm, maps[m], sub["n_points"], sub["ref"])
        assert (raw["n_kept"][idx] == one["n_kept"]).all() and (one["n_kept"] == want["n_kept"]).all()
        assert (raw["ok"][idx] == one["ok"]).all() and (one["ok"] == want["ok"]).all()
        for k, i in enumerate(idx):
            s_got = raw["states"]["s"][b["offsets"][i]:b["offsets"][i + 1]]
            assert s_got.tobytes() == one["states"]["s"][sub["offsets"][k]:sub["offsets"][k + 1]].tobytes()
        src = synth.take_paths(dict(b, ref=free["states"]), idx)["ref"]
        d1 = emu.densify(prm, maps[m], sub["n_points"], src, 0.3, True, 256)
        dw = oracle.densify(prm, maps[m], sub["n_points"], src, 0.3, True, 256)
        assert (dense["n_out"][idx] == d1["n_out"]).all() and (d1["n_out"] == dw["n_out"]).all()
        assert (dense["ok"][idx] == d1["ok"]).all() and (d1["ok"] == dw["ok"]).all()
        for k, i in enumerate(idx):
            c = d1["n_out"][k]
            assert dense["states"][i, :c].tobytes() == d1["states"][k, :c].tobytes()
            for f in ("x", "y", "z", "k", "s"):
                assert np.abs(dense["states"][f][i, :c] - dw["states"][f][k, :c]).max(initial=0.0) <= 1e-9
        cut.append((want["n_kept"] < sub["n_points"]).any())
    _per_map(check, mi, len(maps))
    assert any(cut)


@pytest.mark.parametrize("bad", [-1, N_MAPS, 1 << 30])
def test_index_outside_the_set_only_touches_its_path(scene, bad):
    maps, b, mi = scene
    prm = oracle.default_params()
    n_points, paths = _solved_like(b)
    free = maps_emu.finish_raw_maps(prm, maps, mi, n_points, paths, collision_check=False)["states"]
    bad_idx = mi.copy()
    victims = [0, 5, len(mi) - 1]
    bad_idx[victims] = bad
    others = np.setdiff1d(np.arange(len(mi)), victims)
    for mode in (planner.BOUNDS_SIMPLE, planner.BOUNDS_IMPROVED):
        spl = planner.reference_splines(b) if mode == planner.BOUNDS_IMPROVED else None
        good = maps_emu.update_bounds_maps(prm, maps, mi, b, mode=mode, splines=spl)
        got = maps_emu.update_bounds_maps(prm, maps, bad_idx, b, mode=mode, splines=spl)
        assert (got["n_valid"][victims] == 0).all()
        assert (got["n_valid"][others] == good["n_valid"][others]).all()
        for i in others:
            sl = slice(b["offsets"][i], b["offsets"][i] + good["n_valid"][i])
            assert got["bounds"][sl].tobytes() == good["bounds"][sl].tobytes()
    good = maps_emu.finish_raw_maps(prm, maps, mi, n_points, paths)
    got = maps_emu.finish_raw_maps(prm, maps, bad_idx, n_points, paths)
    assert (got["n_kept"][victims] == 0).all() and (got["ok"][victims] == 0).all()
    assert (got["n_kept"][others] == good["n_kept"][others]).all() and (got["ok"][others] == good["ok"][others]).all()
    for i in victims:                                                     # left as it came in
        sl = slice(b["offsets"][i], b["offsets"][i + 1])
        assert got["states"][sl].tobytes() == paths[sl].tobytes()
    good = maps_emu.densify_maps(prm, maps, mi, n_points, free, 0.3, True, 256)
    got = maps_emu.densify_maps(prm, maps, bad_idx, n_points, free, 0.3, True, 256)
    assert (got["n_out"][victims] == 0).all() and (got["ok"][victims] == 0).all()
    assert (got["n_out"][others] == good["n_out"][others]).all()
    assert got["states"][others].tobytes() == good["states"][others].tobytes()
    # without a collision check the tails never read the map, so the index does not matter
    nc = maps_emu.finish_raw_maps(prm, maps, bad_idx, n_points, paths, collision_check=False)
    assert (nc["n_kept"] == n_points).all()


def test_single_map_drivers_agree_with_a_set_of_one():
    prm = oracle.default_params()
    field = synth.disc_field_map()
    b = synth.map_reference_paths(24, 100, **WILD)
    one = emu.update_bounds(prm, field, b)
    got = maps_emu.update_bounds_maps(prm, [field], np.zeros(24, dtype=np.int32), b)
    assert (got["n_valid"] == one["n_valid"]).all() and got["bounds"].tobytes() == one["bounds"].tobytes()
