"""CPU restatement of TensionSmoother::smooth with smoothing_method TENSION and tension_solver OSQP (TEST
INFRASTRUCTURE, not product code): what pqp_smooth_reference_tension_device computes, path by path, in plain Python
floats.

The front (input check, bSpline, segmentRawReference), the OSQP call and the tail are those of the TENSION2
restatement in oracle/smooth.py, which this module reuses; what is new is TensionSmoother's QP
(tension_smoother.cpp:186-314), with the clearance of every station from oracle.map_distance, and the refusal of a path
whose map index lies outside the map set."""
import math

import numpy as np

from oracle import oracle as O
from oracle import smooth as S
from oracle.segment import reserve

SM_MAP = 11     # the path's map index lies outside the map set (pqp::SM_MAP)
WEIGHTS = (0.0, 1.0, 50.0)    # FLAGS_cartesian_deviation_weight, _curvature_weight, _curvature_rate_weight


def tension_qp(stations, clearance, weights=WEIGHTS):
    """TensionSmoother::setHessianMatrix / setConstraintMatrix (tension_smoother.cpp:239-314) as triplets in the
    reference's order -- unknowns x of every station, then y, then d; rows x_i, y_i, d_i -- with q = 0.  clearance[i]:
    Map::getObstacleDistance at station i, read for 0 < i < N - 1.  The dds and ddds blocks are added into a zero
    matrix block by block, each entry (v_a v_b) w rounded once; exact zeros are dropped as sparseView drops them."""
    w_dev, w_curv, w_rate = weights
    N = len(stations)
    X, Y, D = 0, N, 2 * N
    n = m = 3 * N
    dds, ddds = (1.0, -2.0, 1.0), (-1.0, 3.0, -3.0, 1.0)
    H = {}
    for i in range(N - 2):
        for base in (X, Y):
            for a in range(3):
                for b in range(3):
                    key = (base + i + a, base + i + b)
                    H[key] = H.get(key, 0.0) + dds[a] * dds[b] * w_curv
            if i != N - 3:
                for a in range(4):
                    for b in range(4):
                        key = (base + i + a, base + i + b)
                        H[key] = H.get(key, 0.0) + ddds[a] * ddds[b] * w_rate
    for i in range(N):
        H[(D + i, D + i)] = w_dev
    P = tuple(np.array(v) for v in zip(*[(i, j, v) for (i, j), v in sorted(H.items()) if i <= j and v != 0.0]))
    A = {}
    lo, up = np.zeros(m), np.zeros(m)
    for i, st in enumerate(stations):
        theta = st[2] + math.pi / 2
        A[(X + i, X + i)] = A[(Y + i, Y + i)] = A[(D + i, D + i)] = 1.0
        A[(X + i, D + i)] = -math.cos(theta)
        A[(Y + i, D + i)] = -math.sin(theta)
        lo[X + i] = up[X + i] = st[0]
        lo[Y + i] = up[Y + i] = st[1]
    lo[D + N - 1], up[D + N - 1] = -0.5, 0.5
    for i in range(1, N - 1):
        c = 2.0 if 2.0 < clearance[i] else clearance[i]      # std::min(clearance, default_clearance)
        lo[D + i], up[D + i] = -c, c
    At = tuple(np.array(v) for v in zip(*[(r, c, v) for (r, c), v in sorted(A.items()) if v != 0.0]))
    return dict(n=n, m=m, P=P, q=np.zeros(n), A=At, l=lo, u=up)


def clearances(dmap, stations):
    """Map::getObstacleDistance at every station (oracle.map_distance); 0 at the two ends, which the QP does not
    read."""
    c = [0.0] * len(stations)
    if len(stations) > 2:
        inner = O.map_distance(dmap, [(st[0], st[1]) for st in stations[1:-1]])
        c[1:-1] = [float(v) for v in inner]
    return c


def smooth(px, py, params, dmap, max_raw=1 << 30, max_points=1 << 30, weights=WEIGHTS):
    """One polyline through the whole stage on the distance map `dmap` (None: a map index outside the set):
    dict(reason, status, iters, raw, s_stations, stations, clearance, qp, qp_margin, x, y, s).  The refusals come in
    the kernels' order: the sample kernel's, then the map, then the rest of the front."""
    out = dict(reason=S.SM_OK, status=-100, iters=0, raw=None, stations=[], clearance=[], qp=None, qp_margin=math.inf,
               x=[], y=[], s=[])
    raw = S.b_spline(px, py, max_raw)
    out["raw"] = raw
    if raw["reason"] != S.SM_OK:
        out["reason"] = raw["reason"]
        return out
    if dmap is None:
        out["reason"] = SM_MAP
        return out
    if not S.increasing(raw["s"]):
        out["reason"] = S.SM_RAW_ORDER
        return out
    if not raw["s"][-1] <= max_points:
        out["reason"] = S.SM_MANY
        return out
    _, _, s, stations = S.segment_raw(raw)
    out["stations"], out["s_stations"] = stations, s
    if len(s) > max_points:
        out["reason"] = S.SM_MANY
        return out
    if len(s) < 3:
        out["reason"] = S.SM_SHORT
        return out
    out["clearance"] = clearances(dmap, stations)
    qp = tension_qp(stations, out["clearance"], weights)
    out["qp"] = qp
    sol, _, info = S.osqp_solve(params, qp)
    out.update(status=info.status, iters=info.iters, qp_margin=info.margin)
    if info.status != S.SOLVED:
        out["reason"] = S.SM_QP
        return out
    N = len(stations)
    acc = 0.0
    for i in range(N):
        out["x"].append(float(sol[i]))
        out["y"].append(float(sol[N + i]))
        if i != 0:
            dx, dy = out["x"][i] - out["x"][i - 1], out["y"][i] - out["y"][i - 1]
            acc += math.sqrt(dx * dx + dy * dy)
        out["s"].append(acc)
    if not S.increasing(out["s"]):
        out["reason"] = S.SM_S_ORDER
    return out


def smooth_batch(points, point_offsets, params, capacity, maps, map_index=None, max_raw=1 << 30, max_points=1 << 30,
                 weights=WEIGHTS):
    """A batch in the layout of pqp_smooth_reference_tension_device over the map set `maps` with the per-path
    `map_index` (None: map 0): points [P, >= 2] (x, y).  Returns dict(knot_offsets, knots, x_coef, y_coef, max_s, ok,
    status, iters, reason, qp_margin, smoothed)."""
    xy = np.asarray(points, dtype=np.float64)[:, :2]
    po = np.asarray(point_offsets)
    B = len(po) - 1

    def dmap(b):
        k = 0 if map_index is None else int(map_index[b])
        return maps[k] if 0 <= k < len(maps) else None
    res = [smooth([float(v) for v in xy[po[b]:po[b + 1], 0]], [float(v) for v in xy[po[b]:po[b + 1], 1]], params,
                  dmap(b), max_raw, max_points, weights) for b in range(B)]
    reason = np.array([r["reason"] for r in res], dtype=np.int32)
    counts = [len(r["s"]) if r["reason"] == S.SM_OK else 0 for r in res]
    kept = reserve(counts, capacity)
    n = np.array([c if k else 0 for c, k in zip(counts, kept)], dtype=np.int32)
    off = np.zeros(B + 1, dtype=np.int32)
    np.cumsum(n, out=off[1:])
    T = int(off[-1])
    knots, xco, yco = np.zeros(T), np.zeros((T, 4)), np.zeros((T, 4))
    ms = np.full(B, np.nan)
    for b, r in enumerate(res):
        if reason[b] == S.SM_OK and not kept[b]:
            reason[b] = S.SM_CAPACITY
        if not kept[b]:
            continue
        sl = slice(off[b], off[b + 1])
        knots[sl] = r["s"]
        xco[sl], yco[sl] = O.spline_fit(r["s"], r["x"]), O.spline_fit(r["s"], r["y"])
        ms[b] = r["s"][-1] + 3
    return dict(knot_offsets=off, knots=knots, x_coef=xco, y_coef=yco, max_s=ms, ok=np.array(kept, dtype=np.int32),
                status=np.array([r["status"] if r["qp"] is not None else -100 for r in res], dtype=np.int32),
                iters=np.array([r["iters"] for r in res], dtype=np.int32), reason=reason,
                qp_margin=np.array([r["qp_margin"] for r in res]), smoothed=res)
