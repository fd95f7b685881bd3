"""CPU tests of building distance maps from occupancy grids (pqp_set_maps_occupancy, pqp_set_maps_occupancy_device): the
transform of csrc/pqp_edt_core.cuh, emulated on the host (tests/emu/edt_emu.cpp), against the scipy recipe of
synth.distance_layer bit for bit, against the config-1 fixture, and within 1 ulp of OpenCV's distanceTransform (the
reference's recipe, from tests/golden/occupancy_cv2.npz); argument checks of the entries."""
import ctypes as C
import os

import numpy as np
import pytest

from path_optimizer_b200 import _lib, synth
from path_optimizer_b200.abi import ERR_ARG, OccupancyMap
from tests.emu import edt_emu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
EMPTY = np.float32(2.0 ** 64)   # cv::distanceTransform on a grid with no obstacle


def _scipy(occ, res):
    return synth.distance_layer(occ, res)


def _same(got, want):
    assert got.dtype == np.float32 and got.shape == want.shape
    bad = np.flatnonzero(got.view(np.int32) != want.view(np.int32))
    assert bad.size == 0, (bad[:5], got.flat[bad[:5]], want.flat[bad[:5]])


def random_grids(seed=0):
    """Seeded random grids: 1 x 1 up to a few hundred cells per side, obstacle densities 0.001 to 0.9 (every grid with an
    obstacle)."""
    rng = np.random.default_rng(seed)
    shapes = [(1, 1), (1, 2), (2, 1), (3, 3), (1, 57), (64, 1), (7, 300), (300, 9), (128, 128), (255, 257), (331, 190)]
    shapes += [tuple(int(v) for v in rng.integers(1, 400, 2)) for _ in range(12)]
    out = []
    for k, (r, c) in enumerate(shapes):
        p = [0.001, 0.01, 0.05, 0.2, 0.5, 0.9][k % 6]
        occ = (rng.random((r, c)) >= p).astype(np.uint8) * rng.integers(1, 256, (r, c)).astype(np.uint8)
        if (occ == 0).sum() == 0:
            occ.flat[rng.integers(0, r * c)] = 0
        out.append((occ, [0.2, 0.25, 0.05, 1.0, 0.3][k % 5]))
    return out


def edge_grids():
    """(name, occupancy, resolution) of the edge cases; the last one has no obstacle."""
    corner = np.ones((60, 45), np.uint8)
    corner[0, 0] = 0
    far_corner = np.ones((45, 60), np.uint8)
    far_corner[-1, -1] = 0
    border = np.ones((50, 41), np.uint8)
    border[0, :] = border[-1, :] = border[:, 0] = border[:, -1] = 0
    free_cols = np.ones((40, 30), np.uint8)
    free_cols[5, 3] = free_cols[30, 20] = 0           # every other column has no obstacle
    free_rows = np.ones((30, 40), np.uint8)
    free_rows[3, 5] = free_rows[20, 30] = 0           # every other row has no obstacle
    long_row = np.ones((1, 20000), np.uint8)
    long_row[0, 0] = 0                                # d2 up to 19999^2 > 2^24
    return [("corner", corner, 0.2), ("far_corner", far_corner, 0.25), ("border", border, 0.2),
            ("free_columns", free_cols, 0.2), ("free_rows", free_rows, 0.1), ("all_obstacle", np.zeros((13, 17), np.uint8), 0.2),
            ("long_row", long_row, 0.2), ("no_obstacle", np.full((19, 23), 7, np.uint8), 0.2)]


def expected(occ, res):
    """The contract: the scipy recipe, and 2^64 * resolution everywhere on a grid with no obstacle."""
    if (occ == 0).sum() == 0:
        return np.full(occ.shape, EMPTY * np.float32(res), dtype=np.float32)
    return _scipy(occ, res)


def test_emulated_transform_matches_scipy_on_random_grids():
    for occ, res in random_grids():
        _same(edt_emu.distance_map(occ, res), expected(occ, res))


@pytest.mark.parametrize("case", [c[0] for c in edge_grids()])
def test_emulated_transform_edge_cases(case):
    _, occ, res = next(c for c in edge_grids() if c[0] == case)
    got = edt_emu.distance_map(occ, res)
    _same(got, expected(occ, res))
    if case == "long_row":
        assert got[0, -1] == np.float32(19999.0) * np.float32(res) and 19999 ** 2 > 2 ** 24
    if case == "no_obstacle":
        assert (got == np.float32(1.8446744e19) * np.float32(res)).all()
    if case == "all_obstacle":
        assert (got == 0).all()


def config1_occupancy():
    g = np.load(os.path.join(GOLDEN, "config1_benchmark_map.npz"))
    dist = g["map_distance"]
    return (dist != 0).astype(np.uint8), float(g["map_geo"][0]), dist


def test_config1_layer_rebuilt_bit_for_bit():
    """The config-1 fixture's layer (made with cv2) is the exact transform of map_distance != 0 in every cell."""
    occ, res, dist = config1_occupancy()
    assert dist.size == 246015
    _same(edt_emu.distance_map(occ, res), dist)


def test_within_one_ulp_of_opencv():
    """The reference's recipe, cv::distanceTransform(L2, MASK_PRECISE), from the committed fixture: within 1 ulp of
    the transform wherever a grid has an obstacle, and exactly OpenCV's 2^64 (times the resolution) without one."""
    g = np.load(os.path.join(GOLDEN, "occupancy_cv2.npz"))
    n_empty = 0
    for k in range(int(g["n"])):
        occ, cv = g[f"occ_{k}"], g[f"cv2_{k}"]
        got = edt_emu.distance_map(occ, 1.0)
        if (occ == 0).sum() == 0:
            n_empty += 1
            _same(got, cv)
            _same(edt_emu.distance_map(occ, 0.2), cv * np.float32(0.2))
            continue
        ulp = np.abs(got.view(np.int32).astype(np.int64) - cv.view(np.int32).astype(np.int64))
        assert ulp.max() <= 1, k
        assert ((got == 0) == (cv == 0)).all(), k
    assert n_empty == 1


def _occ_array(descs):
    return (OccupancyMap * max(len(descs), 1))(*descs)


def test_entries_refuse_bad_arguments():
    L = _lib.load()
    cells = np.ones((4, 5), np.uint8)
    good = OccupancyMap(cells.ctypes.data, 4, 5, 0.2, 0.0, 0.0)
    bad = [OccupancyMap(None, 4, 5, 0.2, 0.0, 0.0), OccupancyMap(cells.ctypes.data, 0, 5, 0.2, 0.0, 0.0),
           OccupancyMap(cells.ctypes.data, 4, 0, 0.2, 0.0, 0.0), OccupancyMap(cells.ctypes.data, 4, 5, 0.0, 0.0, 0.0),
           OccupancyMap(cells.ctypes.data, 4, -1, 0.2, 0.0, 0.0), OccupancyMap(cells.ctypes.data, 4, 5, -0.2, 0.0, 0.0)]
    for d in bad:
        assert L.pqp_set_maps_occupancy(None, 2, _occ_array([good, d])) == ERR_ARG
        assert L.pqp_set_maps_occupancy_device(None, 2, _occ_array([good, d]), None) == ERR_ARG
    for n in (0, -1):
        assert L.pqp_set_maps_occupancy(None, n, _occ_array([good])) == ERR_ARG
        assert L.pqp_set_maps_occupancy_device(None, n, _occ_array([good]), None) == ERR_ARG
    assert L.pqp_set_maps_occupancy(None, 1, None) == ERR_ARG
    out = np.zeros(20, np.float32)
    for m in (-1, 0, 1):
        assert L.pqp_get_map(None, m, out.ctypes.data_as(C.c_void_p)) == ERR_ARG
