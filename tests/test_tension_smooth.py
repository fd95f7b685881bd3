"""CPU tests of the TENSION smoothing stage's restatement (tests/tension_restatement.py): its QP against dense
matrices built the reference's way (TensionSmoother::setHessianMatrix's dds / ddds blocks, setConstraintMatrix's rows,
sparseView's zeros dropped, the clearance bounds), solved by the oracle's OSQP against the independent twin
(oracle/twin.py), on the config-1 map, on that map moved to the quarter-turn poses, and under non-default weights."""
import math

import numpy as np
import pytest

from oracle import oracle as O
from oracle import smooth as S
from oracle.twin import osqp_twin
from tests import tension_restatement as T
from tests import tension_cases as tc

CASES = tc.named()
NAMES = ["config1", "u_turn", "corner", "four_far", "straight_x", "down", "pose3", "pose1", "pose13"]


def bar(w):
    """Iterates agree within 1e-9 of their scale.  Below a deviation weight of 1e-4 of the larger curvature weight (the
    default TENSION weights have none) the offsets d have no curvature of their own beyond sigma, and two correct
    restatements drift apart by up to 3e-8 m over 100 iterations (the corner at 1.3e-9 of its scale): 1e-8 there."""
    return 1e-9 if w[0] >= 1e-4 * max(w[1], w[2]) else 1e-8


def _lists(name):
    return tuple([float(v) for v in a] for a in CASES[name])


def _dense_reference_way(stations, dmap, w):
    """setHessianMatrix / setConstraintMatrix as dense numpy blocks, the clearance from oracle.map_distance."""
    N = len(stations)
    n = 3 * N
    H = np.zeros((n, n))
    dds, ddds = np.array([1.0, -2.0, 1.0]), np.array([-1.0, 3.0, -3.0, 1.0])
    for i in range(N - 2):
        for base in (0, N):
            H[base + i:base + i + 3, base + i:base + i + 3] += np.outer(dds, dds) * w[1]
            if i != N - 3:
                H[base + i:base + i + 4, base + i:base + i + 4] += np.outer(ddds, ddds) * w[2]
    H[2 * N + np.arange(N), 2 * N + np.arange(N)] = w[0]
    st = np.array(stations)
    A = np.zeros((n, n))
    idx = np.arange(N)
    A[idx, idx] = A[N + idx, N + idx] = A[2 * N + idx, 2 * N + idx] = 1.0
    theta = st[:, 2] + math.pi / 2
    A[idx, 2 * N + idx], A[N + idx, 2 * N + idx] = -np.cos(theta), -np.sin(theta)
    lo, up = np.concatenate([st[:, 0], st[:, 1], np.zeros(N)]), np.concatenate([st[:, 0], st[:, 1], np.zeros(N)])
    clear = np.minimum(O.map_distance(dmap, st[1:-1, :2]), 2.0)
    lo[2 * N + 1:3 * N - 1], up[2 * N + 1:3 * N - 1] = -clear, clear
    lo[3 * N - 1], up[3 * N - 1] = -0.5, 0.5
    return H, np.zeros(n), A, lo, up


def _check(name, dmap, w):
    prm = O.default_params()
    r = T.smooth(*_lists(name), prm, dmap, weights=w)
    assert r["reason"] == S.SM_OK and r["qp"] is not None, name
    want = _dense_reference_way(r["stations"], dmap, w)
    got = S.dense(r["qp"])
    for a, b in zip(want, got):
        assert np.array_equal(a, b), name
    # sparseView: no stored zero in P or A
    assert np.all(r["qp"]["P"][2] != 0) and np.all(r["qp"]["A"][2] != 0)
    tw = osqp_twin(prm, *want)
    x, _, info = S.osqp_solve(prm, r["qp"])
    assert (tw["status"], tw["iters"]) == (info.status, info.iters) == (r["status"], r["iters"]), name
    scale = max(1.0, float(np.max(np.abs(x))))
    assert np.max(np.abs(tw["x"] - x)) <= bar(w) * scale, name
    return r, x


@pytest.mark.parametrize("name", NAMES)
def test_qp_against_dense_and_twin(name):
    r, _ = _check(name, tc.config1_map(), T.WEIGHTS)
    assert r["status"] == S.SOLVED


@pytest.mark.parametrize("name", ["pose0", "pose3", "pose4", "pose7", "pose14"])
def test_moved_maps(name):
    """On the config-1 map moved with the polyline, the clearances equal the unmoved ones up to the lookup's
    rounding."""
    dmap = tc.pose_maps()[name]
    r, _ = _check(name, dmap, T.WEIGHTS)
    base = T.smooth(*_lists("config1"), O.default_params(), tc.config1_map())
    assert np.allclose(r["clearance"], base["clearance"], atol=1e-6)
    assert sum(c > 0 for c in r["clearance"]) == len(r["clearance"]) - 2


@pytest.mark.parametrize("w", tc.WEIGHTS[1:])
@pytest.mark.parametrize("name", ["config1", "u_turn", "corner"])
def test_weights(name, w):
    _check(name, tc.config1_map(), w)


def test_zero_curvature_weight_drops_dds():
    r = T.smooth(*_lists("config1"), O.default_params(), tc.config1_map(), weights=(0.0, 0.0, 50.0))
    P, _, _, _, _ = S.dense(r["qp"])
    N = len(r["stations"])
    # the ddds blocks alone: x_0 x_0 is 1 * 50, and the d columns of P are empty at a zero deviation weight
    assert P[0, 0] == 50.0 and not P[2 * N:, :].any()


def test_clearance_bounds():
    prm = O.default_params()
    m = tc.config1_map()
    # a station outside the map: clearance 0, its offset pinned to 0
    r = T.smooth(*_lists("u_turn"), prm, m)
    N = len(r["stations"])
    outside = [i for i in range(1, N - 1) if r["clearance"][i] == 0.0]
    assert outside
    lo, up = r["qp"]["l"], r["qp"]["u"]
    assert all(lo[2 * N + i] == 0.0 and up[2 * N + i] == 0.0 for i in outside)
    assert lo[2 * N] == up[2 * N] == 0.0 and (lo[3 * N - 1], up[3 * N - 1]) == (-0.5, 0.5)
    # interior bounds bind at a non-zero clearance below 2
    r, x = _check(tc.BINDING, m, T.WEIGHTS)
    N = len(r["stations"])
    d = x[2 * N:]
    bind = [i for i in range(1, N - 1) if 0 < r["clearance"][i] < 2 and abs(d[i]) >= r["clearance"][i] - 1e-4]
    assert bind


def test_map_refusal_and_batch():
    prm = O.default_params()
    assert T.smooth(*_lists("config1"), prm, None)["reason"] == T.SM_MAP
    # the sample refusals come before the map check
    assert T.smooth(*_lists("three"), prm, None)["reason"] == S.SM_FEW
    names, pts, off, maps, _ = tc.batch(["config1", "u_turn", "corner"])
    out = T.smooth_batch(pts, off, prm, 1 << 20, maps, map_index=[0, 5, -1])
    assert list(out["ok"]) == [1, 0, 0] and list(out["reason"][1:]) == [T.SM_MAP, T.SM_MAP]
    assert list(out["status"][1:]) == [-100, -100]
