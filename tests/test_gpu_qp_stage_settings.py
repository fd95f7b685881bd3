"""GPU tests (run with -m gpu on an H100) of the smoothing and post-smoothing QPs away from the defaults, through the
device entries: solver settings through set_params on the handle and the smoothing weights as call arguments.
PathPlanner.smooth_device (pqp_smooth_reference_device, width-4 core) is compared with oracle/smooth.py, and
PathPlanner.post_smooth_device (pqp_post_smooth_device, width-3 core) with oracle/corridor.py.  Also tested: the
largest max_points the smoothing entry accepts, solved at that cap, with ERR_CAPACITY one station above it.

Status and iterations must be exact.  Near the origin the knots must agree within 1e-8 of their column scale (1e-6 for
lopsided weights, see test_weights).  A path whose deciding
comparison in the oracle lies within 1e-9 (relative) of its threshold is a rounding coin flip; it is dropped and
counted."""
import math

import numpy as np
import pytest

from oracle import corridor as oc
from oracle import oracle as O
from oracle import smooth as S
from path_optimizer_b200 import planner
from path_optimizer_b200.abi import DUAL_INFEASIBLE, DUAL_INFEASIBLE_INACCURATE, ERR_CAPACITY
from tests import corridor_cases as cc
from tests import segment_cases
from tests import smooth_cases as sc
from tests import verdicts as V

pytestmark = pytest.mark.gpu
NEAR = 1e-9
FAR = 1e5
CAP = 65536
MAX_RAW = 4096
MAX_PTS = 200
NAMES = ["config1", "corner", "u_turn", "straight_x"] + [f"pose{k}" for k in range(24)]
WEIGHTS = [S.WEIGHTS, (0.0, 1.0, 10.0), (0.005, 0.0, 10.0), (0.005, 1.0, 0.0), (1e-6, 1.0, 10.0),
           (0.005, 1e-6, 10.0), (10.0, 1.0, 10.0), (1000.0, 1.0, 10.0), (0.005, 1000.0, 1000.0), (10.0, 1e-6, 0.0)]


def _dev():
    import torch
    return torch.device("cuda", 0)


def _np(t):
    return t.detach().cpu().numpy()


def _t(a):
    import torch
    a = np.ascontiguousarray(a)
    if a.dtype.names:
        a = a.view(np.float64).reshape(len(a), -1)
    return torch.from_numpy(a.copy()).to(_dev())


def _params(**over):
    p = O.default_params()
    for k, v in over.items():
        setattr(p, k, v)
    return p


@pytest.fixture(scope="module")
def pl():
    p = planner.PathPlanner(max_batch=256, max_total_points=CAP)
    p.set_maps([segment_cases.config1()["field"]])
    yield p
    p.close()


def _smooth(pl, pts, off, p, weights=S.WEIGHTS, max_points=MAX_PTS):
    import torch
    pl.set_params(p)
    try:
        r = pl.smooth_device(_t(pts), _t(off), MAX_RAW, max_points, capacity=CAP, weights=weights)
        torch.cuda.synchronize()
    finally:
        pl.set_params(O.default_params())
    return {k: _np(v) for k, v in r.items()}


def _compare_smooth(got, want, names, pts, off, bar=1e-8):
    """Returns (compared, dropped)."""
    done = dropped = 0
    ko_g, ko_w = got["knot_offsets"], want["knot_offsets"]
    for b, name in enumerate(names):
        if not want["qp_margin"][b] >= NEAR:
            dropped += 1
            continue
        done += 1
        assert (got["ok"][b], got["status"][b], got["iters"][b]) == (want["ok"][b], want["status"][b],
                                                                    want["iters"][b]), name
        if not want["ok"][b]:
            assert ko_g[b + 1] == ko_g[b] and np.isnan(got["max_s"][b]), name
            continue
        if np.nanmax(np.abs(pts[off[b]:off[b + 1], :2])) > FAR:
            continue
        g, w = slice(ko_g[b], ko_g[b + 1]), slice(ko_w[b], ko_w[b + 1])
        for k in ("knots", "x_coef", "y_coef"):
            a, e = got[k][g].reshape(len(got[k][g]), -1), want[k][w].reshape(len(want[k][w]), -1)
            scale = np.maximum(1.0, np.max(np.abs(e), axis=0))
            assert np.all(np.max(np.abs(a - e), axis=0) <= bar * scale), (name, k)
    return done, dropped


@pytest.fixture(scope="module")
def qps():
    """The oracle's smoothing QP of every named polyline, per weight set (the B-spline pre-pass runs once)."""
    cache = {}

    def get(name, w):
        if (name, w) not in cache:
            x, y = sc.named()[name]
            o = S.smooth([float(v) for v in x], [float(v) for v in y], O.default_params(), weights=w)
            assert o["qp"] is not None, name
            cache[(name, w)] = o["qp"]
        return cache[(name, w)]
    return get


def _status_only(pl, qps, names, p, w=S.WEIGHTS):
    """Status and iterations of the device against the oracle's OSQP on the cached QPs; returns (compared, dropped,
    statuses seen)."""
    _, pts, off = sc.batch(names)
    got = _smooth(pl, pts, off, p, w)
    done = dropped = 0
    seen = set()
    for b, name in enumerate(names):
        _, _, info = S.osqp_solve(p, qps(name, w))
        if not info.margin >= NEAR:
            dropped += 1
            continue
        done += 1
        assert (got["status"][b], got["iters"][b]) == (info.status, info.iters), (name, w, p.max_iter)
        assert got["ok"][b] == (info.status == 1), name
        seen.add(int(info.status))
    return done, dropped, seen


# (names, settings, the oracle's status): pose17 at eps_dual_inf 0.01 is the solved control of the row above it
DUAL_INF_ROWS = [
    (["config1", "corner"], dict(eps_dual_inf=0.1, max_iter=1), DUAL_INFEASIBLE),
    (["config1"], dict(eps_dual_inf=1.0, check_termination=10), DUAL_INFEASIBLE),
    (["pose17"], dict(eps_dual_inf=0.03), DUAL_INFEASIBLE),
    (["pose17"], dict(eps_dual_inf=0.01), 1),
    (["config1"], dict(eps_dual_inf=0.01, max_iter=1), DUAL_INFEASIBLE_INACCURATE),
]


@pytest.mark.parametrize("row", range(len(DUAL_INF_ROWS)))
def test_dual_infeasibility_rows(pl, qps, row):
    """OSQP's dual-infeasibility verdicts through smooth_device, whose path is then refused (ok = 0).  The row at
    eps_dual_inf 1 is an exact tie in the oracle (the x0 pin row's A dx equals ||dx||) and is compared regardless."""
    names, over, status = DUAL_INF_ROWS[row]
    p = _params(**over)
    _, pts, off = sc.batch(names)
    got = _smooth(pl, pts, off, p)
    for b, name in enumerate(names):
        _, _, info = S.osqp_solve(p, qps(name, S.WEIGHTS))
        assert info.status == status, name
        assert (got["status"][b], got["iters"][b]) == (info.status, info.iters), name
        assert got["ok"][b] == (status == 1), name
        if status != 1:
            assert np.isnan(got["max_s"][b]), name


def test_large_deviation_weight_at_every_pose(pl):
    """Weights (10, 1e-6, 0) at every pose: 16 of the 24 took 100-400 iterations longer than OSQP while the width-4
    separator chain multiplied by explicit inverses of its Schur blocks."""
    names = [f"pose{k}" for k in range(24)]
    _, pts, off = sc.batch(names)
    w = (10.0, 1e-6, 0.0)
    got = _smooth(pl, pts, off, O.default_params(), w)
    want = S.smooth_batch(pts, off, O.default_params(), CAP, MAX_RAW, MAX_PTS, weights=w)
    done, dropped = _compare_smooth(got, want, names, pts, off)
    assert dropped <= 2 and done + dropped == 24


@pytest.mark.parametrize("wi", range(len(WEIGHTS)))
def test_weights(pl, wi):
    w = WEIGHTS[wi]
    names = ["config1", "corner", "u_turn", "straight_x", "pose0", "pose1", "pose17"]
    _, pts, off = sc.batch(names)
    got = _smooth(pl, pts, off, O.default_params(), w)
    want = S.smooth_batch(pts, off, O.default_params(), CAP, MAX_RAW, MAX_PTS, weights=w)
    # lopsided weights (deviation below 1e-4 of the largest curvature weight, 0 included) leave directions with little
    # curvature beyond sigma, along which two correct solvers differ by up to 1e-7 (tests/test_qp_stage_settings.py)
    bar = 1e-8 if w[0] >= 1e-4 * max(w[1], w[2]) else 1e-6
    done, dropped = _compare_smooth(got, want, names, pts, off, bar=bar)
    assert dropped <= 1, dropped


def test_settings_grid(pl, qps):
    """Every verdict schedule at max_iter 1, 7 and V.MAX_ITER; scaling 0; eps_dual_inf from 1e-4 to 1; the verdict
    suite's tolerance settings.  Together they reach every status the smoothing QP can end in."""
    done = dropped = 0
    seen = set()
    cases = []
    for check, interval, adaptive in V.SCHEDULES.values():
        for t in (1, 7, 60, V.MAX_ITER):
            cases.append(dict(check_termination=check, adaptive_rho_interval=interval, adaptive_rho=adaptive,
                              max_iter=t))
    cases += [dict(scaling=0, max_iter=t) for t in (1, 7, V.MAX_ITER)]
    cases += [dict(eps_dual_inf=e, max_iter=t) for e in (1e-4, 1e-2, 3e-2, 0.1, 1.0) for t in (1, 2, 60, V.MAX_ITER)]
    cases += [dict(max_iter=t, **over) for over in V.SETTINGS.values() for t in (7, 60, V.MAX_ITER)]
    for over in cases:
        d, r, s = _status_only(pl, qps, NAMES, _params(**over))
        done, dropped, seen = done + d, dropped + r, seen | s
    assert done >= 20 * dropped, (done, dropped)
    assert {1, 2, -2, DUAL_INFEASIBLE, DUAL_INFEASIBLE_INACCURATE} <= seen, sorted(seen)


def _accepts(pl, pts, off, max_points):
    import torch
    try:
        pl.smooth_device(_t(pts), _t(off), MAX_RAW, max_points, capacity=CAP)
        torch.cuda.synchronize()
        return True
    except planner.PqpError as e:
        assert f"rc={ERR_CAPACITY}" in str(e)
        return False


def test_max_points_cap(pl):
    """The largest max_points the entry accepts, found by asking it, solved at that cap on a gentle curve about cap - 2
    metres long; cap + 1 is ERR_CAPACITY."""
    _, pts, off = sc.batch(["config1"])
    lo, hi = MAX_PTS, 4096
    assert _accepts(pl, pts, off, lo) and not _accepts(pl, pts, off, hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if _accepts(pl, pts, off, mid):
            lo = mid
        else:
            hi = mid
    cap = lo
    assert not _accepts(pl, pts, off, cap + 1)
    # a clothoid-like arc near the origin, raw points every 5 m
    L = cap - 2.0
    s = np.linspace(0.0, L, int(L // 5) + 1)
    th = 0.3 * np.sin(s / L * math.pi)
    x = np.concatenate([[0.0], np.cumsum(np.cos(th[:-1]) * np.diff(s))])
    y = np.concatenate([[0.0], np.cumsum(np.sin(th[:-1]) * np.diff(s))])
    pts = np.zeros((len(x), 7))
    pts[:, 0], pts[:, 1] = x, y
    off = np.array([0, len(x)], dtype=np.int32)
    got = _smooth(pl, pts, off, O.default_params(), max_points=cap)
    want = S.smooth_batch(pts, off, O.default_params(), CAP, MAX_RAW, cap)
    assert want["ok"][0] == 1 and len(want["smoothed"][0]["s"]) >= cap - 8
    done, _ = _compare_smooth(got, want, ["arc"], pts, off)
    assert done == 1


POST_SETTINGS = [dict(), dict(max_iter=7), dict(max_iter=1), dict(check_termination=10, adaptive_rho_interval=7),
                 dict(scaling=0), dict(adaptive_rho=0), dict(eps_abs=0.5, eps_rel=0.5), dict(eps_dual_inf=1.0)]


@pytest.mark.parametrize("si", range(len(POST_SETTINGS)))
def test_post_smooth_settings(si):
    """post_smooth_device (the width-3 core) under solver settings through set_params, against the restatement."""
    import torch
    scene = cc.batch()
    p = _params(**POST_SETTINGS[si])
    pl = planner.PathPlanner(max_batch=256, max_total_points=4096)
    try:
        pl.set_maps(scene["maps"])
        pl.set_params(p)
        sp = scene["splines"]
        d = dict(knot_offsets=_t(sp["knot_offsets"]), knots=_t(sp["knots"]), x_coef=_t(sp["x_coef"]),
                 y_coef=_t(sp["y_coef"]))
        r = pl.post_smooth_device(d, _t(scene["max_s"]), _t(scene["start"]), 200, capacity=4096,
                                  map_index=_t(np.asarray(scene["map_index"], dtype=np.int32)))
        torch.cuda.synchronize()
        r = {k: (None if v is None else _np(v)) for k, v in r.items()}
    finally:
        pl.close()
    o = oc.post_smooth_batch(sp, scene["max_s"], scene["start"], scene["maps"], p, 4096,
                             map_index=scene["map_index"], max_layers=200)
    near = o["margin"] < NEAR
    assert near.sum() <= max(1, len(near) // 10)
    off, ooff = r["knot_offsets"], o["knot_offsets"]
    for b, name in enumerate(scene["names"]):
        if near[b]:
            continue
        assert (r["ok"][b], r["status"][b], r["iters"][b]) == (o["ok"][b], o["status"][b], o["iters"][b]), name
        if not o["ok"][b]:
            continue
        d_, h = slice(off[b], off[b + 1]), slice(ooff[b], ooff[b + 1])
        np.testing.assert_allclose(r["knots"][d_], o["knots"][h], rtol=0, atol=1e-8, err_msg=name)
        np.testing.assert_allclose(r["x_coef"][d_], o["x_coef"][h], rtol=0, atol=1e-8, err_msg=name)
        np.testing.assert_allclose(r["y_coef"][d_], o["y_coef"][h], rtol=0, atol=1e-8, err_msg=name)
