"""CPU tests of the smoothing stage's restatement (oracle/smooth.py): its B-spline samples against scipy's BSpline on
the clamped uniform knot vector, its resampling against scipy's natural CubicSpline, and its TENSION2 QP, solved by the
oracle's OSQP, against the independent twin (oracle/twin.py) on dense matrices built the reference's way."""
import math

import numpy as np
import pytest
from scipy.interpolate import BSpline, CubicSpline

from oracle import oracle as O
from oracle import smooth as S
from oracle.twin import kkt_certificate, osqp_twin
from tests import smooth_cases as sc

CASES = sc.named()
SMOOTHED = ["config1", "straight_x", "u_turn", "corner", "four_far", "pose4", "pose13"]


def _params():
    return O.default_params()


@pytest.mark.parametrize("name", ["config1", "u_turn", "corner", "four_far", "six_close", "pose13"])
def test_bspline_against_scipy(name):
    x, y = (list(map(float, v)) for v in CASES[name])
    raw = S.b_spline(x, y)
    assert raw["reason"] == S.SM_OK
    n, p = len(x), raw["degree"]
    knots = np.concatenate([np.zeros(p + 1), np.arange(1, n - p) / (n - p), np.ones(p + 1)])
    bs = BSpline(knots, np.stack([x, y], 1), p)
    ref = bs(np.array(raw["t"]))
    scale = max(1.0, float(np.max(np.abs(ref))))
    assert np.max(np.abs(np.stack([raw["x"], raw["y"]], 1) - ref)) <= 1e-12 * scale
    # t accumulated as the reference does, s the serial sum of the sample distances
    dt = 1.0 / raw["length"]
    assert raw["t"][-1] == 1.0 and raw["t"][-2] < 1.0 and raw["t"][1] == dt
    d = np.hypot(np.diff(raw["x"]), np.diff(raw["y"]))
    assert np.allclose(raw["s"][1:], np.cumsum(d), rtol=1e-12, atol=1e-9)


def test_degree_rule_and_refusals():
    assert S.b_spline(*CASES["three"])["reason"] == S.SM_FEW
    assert S.b_spline(*CASES["four_close"])["reason"] == S.SM_DEGREE     # degree 5 >= 4 points
    assert S.b_spline(*CASES["five_close"])["reason"] == S.SM_DEGREE     # degree 5 >= 5 points
    assert S.b_spline(*CASES["six_close"])["reason"] == S.SM_OK
    assert S.b_spline(*CASES["four_far"])["degree"] == 3
    assert S.b_spline(*CASES["nan"])["reason"] == S.SM_LENGTH
    # a repeated input point is a repeated control point: the B-spline's samples still advance, and the path is kept
    assert S.smooth(*CASES["repeated"], _params())["reason"] == S.SM_OK
    tiny = S.b_spline(*CASES["tiny"])
    assert tiny["reason"] == S.SM_OK and len(tiny["s"]) == 2
    assert S.smooth(*CASES["tiny"], _params())["reason"] == S.SM_RAW_ORDER     # tk::spline needs 3 samples
    assert S.smooth(*CASES["short"], _params())["reason"] == S.SM_SHORT        # 2 stations


@pytest.mark.parametrize("name", ["config1", "u_turn", "corner"])
def test_resampling_against_cubic_spline(name):
    raw = S.b_spline(*CASES[name])
    _, _, s, st = S.segment_raw(raw)
    assert s == [float(i) for i in range(len(s))] and s[-2] < raw["s"][-1] <= s[-1]
    cx = CubicSpline(raw["s"], raw["x"], bc_type="natural")
    cy = CubicSpline(raw["s"], raw["y"], bc_type="natural")
    inner = np.array(s[:-1])
    x, y = np.array([v[0] for v in st[:-1]]), np.array([v[1] for v in st[:-1]])
    assert np.max(np.abs(x - cx(inner))) < 1e-9 and np.max(np.abs(y - cy(inner))) < 1e-9
    dx, dy, ddx, ddy = cx(inner, 1), cy(inner, 1), cx(inner, 2), cy(inner, 2)
    assert np.max(np.abs(np.array([v[2] for v in st[:-1]]) - np.arctan2(dy, dx))) < 1e-9
    k = (dx * ddy - dy * ddx) / (dx * dx + dy * dy) ** 1.5
    assert np.max(np.abs(np.array([v[3] for v in st[:-1]]) - k)) < 1e-7


def _dense_reference_way(stations, s, w=S.WEIGHTS):
    """setHessianMatrix / setGradient / setConstraintMatrix written as dense numpy blocks."""
    N = len(stations)
    n, m = 4 * N - 1, 3 * (N - 1) + 2
    X, Y, T, K = 0, N, 2 * N, 3 * N
    H = np.zeros((n, n))
    H[np.arange(N), np.arange(N)] = 2 * w[0]
    H[Y + np.arange(N), Y + np.arange(N)] = 2 * w[0]
    H[K + np.arange(N - 1), K + np.arange(N - 1)] = 2 * w[1]
    for i in range(N - 2):
        H[K + i:K + i + 2, K + i:K + i + 2] += 2 * w[2] * np.array([[1.0, -1.0], [-1.0, 1.0]])
    st = np.array(stations)
    q = np.zeros(n)
    q[:N], q[Y:Y + N] = -2 * w[0] * st[:, 0], -2 * w[0] * st[:, 1]
    A, b = np.zeros((m, n)), np.zeros(m)
    ds = np.diff(np.array(s))
    for i in range(N - 1):
        for r, base in ((i, X), (N - 1 + i, Y), (2 * N - 2 + i, T)):
            A[r, base + i + 1], A[r, base + i] = 1.0, -1.0
        A[i, T + i], A[N - 1 + i, T + i], A[2 * N - 2 + i, K + i] = ds[i] * np.sin(st[i, 2]), -ds[i] * np.cos(st[i, 2]), -ds[i]
        b[i], b[N - 1 + i], b[2 * N - 2 + i] = ds[i] * np.cos(st[i, 2]), ds[i] * np.sin(st[i, 2]), -ds[i] * st[i, 3]
    A[3 * N - 3, X], A[3 * N - 2, Y] = 1.0, 1.0
    b[3 * N - 3], b[3 * N - 2] = st[0, 0], st[0, 1]
    return H, q, A, b, b.copy()


@pytest.mark.parametrize("name", SMOOTHED)
def test_qp_against_twin(name):
    prm = _params()
    r = S.smooth(*CASES[name], prm)
    assert r["qp"] is not None
    P, q, A, l, u = _dense_reference_way(r["stations"], r["s_stations"])
    P2, q2, A2, l2, u2 = S.dense(r["qp"])
    assert np.array_equal(P, P2) and np.array_equal(q, q2) and np.array_equal(l, l2) and np.array_equal(u, u2)
    assert np.array_equal(A, A2)
    tw = osqp_twin(prm, P, q, A, l, u)
    x, _, info = S.osqp_solve(prm, r["qp"])
    assert (tw["status"], tw["iters"]) == (info.status, info.iters) == (r["status"], r["iters"])
    scale = max(1.0, float(np.max(np.abs(x))))
    assert np.max(np.abs(tw["x"] - x)) <= 1e-9 * scale
    assert r["status"] == S.SOLVED
    cert = kkt_certificate(P, q, A, l, u, tw["x"], tw["y"])
    Ax = A @ tw["x"]
    assert cert["primal"] < prm.eps_abs + prm.eps_rel * max(np.max(np.abs(Ax)), np.max(np.abs(l))) + 1e-9 * scale


def test_batch_reservation_and_outputs():
    prm = _params()
    names, pts, off = sc.batch(["config1", "four_close", "u_turn", "nan", "corner"])
    full = S.smooth_batch(pts, off, prm, capacity=1 << 20)
    assert list(full["ok"]) == [1, 0, 1, 0, 1]
    assert list(full["reason"][[1, 3]]) == [S.SM_DEGREE, S.SM_LENGTH]
    counts = np.diff(full["knot_offsets"])
    assert all(math.isnan(full["max_s"][b]) for b in (1, 3))
    cap = int(counts[0] + counts[2])
    part = S.smooth_batch(pts, off, prm, capacity=cap + 5)
    assert list(part["ok"]) == [1, 0, 1, 0, 0] and part["reason"][4] == S.SM_CAPACITY
    assert np.array_equal(part["knots"], full["knots"][:cap])
