"""CPU restatement of ReferencePathSmoother::graphSearchDp and ::postSmooth (TEST INFRASTRUCTURE, not product code):
what pqp_post_smooth_device computes, path by path, in plain Python floats.

Written from the reference's behaviour (src/reference_path_smoother/reference_path_smoother.cpp:110-143 calculateCostAt,
:145-301 graphSearchDp, :534-644 postSmooth and its matrices; findClosestPoint, getHeading, getCurvature and
global2Local of src/tools/tools.cpp:32-110).  Every operation is one IEEE double operation in the reference's order and
the transcendental functions are the C library's, so the search's per-thread device functions compiled with g++ give
the same bits.  The map lookups are the oracle's (pqp_oracle_env.c).  The post-smoothing QP is built as triplets in the
reference's variable order (x, then dx, then ddx of every layer) and solved by the oracle's OSQP restatement.

Every path also reports `margin`: how close the search's discrete decisions came to flipping -- a node's distance
against 1.45 m and its l against the turning radius, every cost comparison of the DP and of the last layer's argmin,
every probe of the bound march against 1.45 m, |vehicle_l| against the range and the truncation of the start's
lateral index.  `ties` counts the comparisons that met an exact tie, which the first index wins.  A device whose
atan2 / sin / cos / pow differ from the C library's in the last bits can only decide differently where that margin is
tiny.
"""
import ctypes as C
import math

import numpy as np

from oracle import oracle as O
from oracle.segment import Spline, constraint_angle, reserve, sample

(COR_OK, COR_BAD_SPLINE, COR_BAD_LENGTH, COR_BAD_START, COR_FAR, COR_TOO_MANY, COR_SHORT, COR_QP, COR_S_ORDER, COR_MAP,
 COR_CAPACITY, COR_WIDE) = range(12)
MAX_LATERAL = 64
MAX_LENGTH = 1048576.0      # 2^20 m
MAX_HEADING = 1048576.0     # 2^20 rad
THRESHOLD = 1.45
DBL_MAX = 1.7976931348623157e308
SOLVED = 1


def _div(a, b):
    with np.errstate(all="ignore"):
        return float(np.float64(a) / np.float64(b))


class MapLookup:
    """grid_map isInside / getObstacleDistance of one distance map, through the oracle."""

    def __init__(self, m):
        self.dm, self._keep = O._dm(m)
        self.L = O.lib()
        self.L.oracle_map_inside.restype = C.c_int

    def inside(self, x, y):
        return bool(self.L.oracle_map_inside(C.byref(self.dm), float(x), float(y)))

    def distance(self, x, y):
        return self.L.oracle_map_distance(C.byref(self.dm), float(x), float(y))


def lateral_lattice(range_, spacing):
    """cur_l += spacing from -range while cur_l <= range (:186-212), at most MAX_LATERAL + 1 nodes."""
    out, cur = [], -range_
    while cur <= range_ and len(out) <= MAX_LATERAL:
        out.append(cur)
        cur += spacing
    return out


def closest_s(xs, ys, max_s, x, y):
    """findClosestPoint(xs, ys, x, y, max_s).s (tools.cpp:66-110), start_s = 0."""
    tmp, min_dis, min_s = 0.0, DBL_MAX, 0.0
    while tmp <= max_s:
        dx, dy = xs(tmp) - x, ys(tmp) - y
        d = math.sqrt(dx * dx + dy * dy)
        if d < min_dis:
            min_dis, min_s = d, tmp
        tmp += 0.5
    cur = prev = min_s
    for _ in range(20):
        px, py = xs(cur) - x, ys(cur) - y
        dx, dy, ddx, ddy = xs(cur, 1), ys(cur, 1), xs(cur, 2), ys(cur, 2)
        j = px * dx + py * dy
        h = dx * dx + px * ddx + dy * dy + py * ddy
        cur -= _div(j, h)
        if abs(cur - prev) < 1e-5:
            break
        prev = cur
    return max_s if max_s < cur else cur


def march(ml, rx, ry, heading, rough_lo, rough_hi, margins):
    """The 0.2 m bound march of one chosen node (:256-287)."""
    ub, lb = 0.2 + rough_hi, -0.2 + rough_lo
    c, s = math.cos(heading + math.pi / 2), math.sin(heading + math.pi / 2)
    while ub < 6.0:
        x, y = rx + ub * c, ry + ub * s
        inside = ml.inside(x, y)
        d = ml.distance(x, y) if inside else 0.0
        if inside:
            margins.append(abs(d - THRESHOLD))
        if inside and d > THRESHOLD:
            ub += 0.2
        else:
            ub -= 0.2
            break
    while lb > -6.0:
        x, y = rx + lb * c, ry + lb * s
        inside = ml.inside(x, y)
        d = ml.distance(x, y) if inside else 0.0
        if inside:
            margins.append(abs(d - THRESHOLD))
        if inside and d > THRESHOLD:
            lb -= 0.2
        else:
            lb += 0.2
            break
    return lb, ub


def search(xs, ys, max_s, start, ml, range_=10.0, spacing=0.6, ds_long=1.5, max_layers=1 << 30):
    """graphSearchDp of one path.  start: (x, y, z) sequence.  Returns dict(reason, s [R], bounds [R][2], chain [R]
    node indices, vehicle_l, margin)."""
    sx, sy, sz = (float(v) for v in start[:3])
    out = dict(reason=COR_OK, s=[], bounds=[], chain=[], vehicle_l=math.nan, margin=math.inf, ties=0)
    margins = []

    def done(reason):
        out["reason"] = reason
        out["margin"] = min(margins) if margins else math.inf
        if reason != COR_OK:
            out["s"], out["bounds"], out["chain"] = [], [], []
        return out
    lat = lateral_lattice(range_, spacing)
    if len(lat) > MAX_LATERAL:
        return done(COR_WIDE)
    if ml is None:
        return done(COR_MAP)
    if len(xs.t) < 3:
        return done(COR_BAD_SPLINE)
    max_s = float(max_s)
    if not (max_s > 0.0 and max_s <= MAX_LENGTH):
        return done(COR_BAD_LENGTH)
    if not abs(sz) <= MAX_HEADING:
        return done(COR_BAD_START)
    s0 = closest_s(xs, ys, max_s, sx, sy)
    if not math.isfinite(s0):
        return done(COR_BAD_START)
    search_ds = ds_long if max_s > 6 else 0.5           # :154
    layers, tmp = [], s0
    while tmp < max_s and len(layers) <= max_layers:
        layers.append(tmp)
        tmp += search_ds
    layers.append(max_s)
    if len(layers) > max_layers:
        return done(COR_TOO_MANY)
    px, py, pz, _ = sample(xs, ys, s0)
    dx, dy = sx - px, sy - py
    vl = -dx * math.sin(pz) + dy * math.cos(pz)          # global2Local(proj_point, start).y
    out["vehicle_l"] = vl
    if not math.isfinite(vl):
        return done(COR_BAD_START)
    margins.append(abs(abs(vl) - range_))
    if abs(vl) > range_:
        return done(COR_FAR)
    v = (range_ + vl) / spacing
    margins.append(abs(v - round(v)))
    start_idx = int(v)
    n = len(lat)
    # sample every layer: node position, distance, feasibility, rough bounds (:178-229)
    nodes = []
    for i, s in enumerate(layers):
        rx, ry, heading, k = sample(xs, ys, s)
        r = _div(1, k)
        c, sn = math.cos(heading + math.pi / 2), math.sin(heading + math.pi / 2)
        row = []
        for j, l in enumerate(lat):
            x, y = rx + l * c, ry + l * sn
            inside = ml.inside(x, y)
            dis = ml.distance(x, y) if inside else -1.0
            feas = not ((k < 0 and l < r) or (k > 0 and l > r) or dis < THRESHOLD)
            if i > 0:
                if inside:
                    margins.append(abs(dis - THRESHOLD))
                if k != 0 and math.isfinite(r):
                    margins.append(abs(l - r))
            if i == 0:
                feas = j == start_idx
            row.append(dict(x=x, y=y, l=l, s=s, heading=heading, dis=dis, feas=feas, cost=DBL_MAX, dir=None,
                            parent=None))
        if i == 0 and 0 <= start_idx < n:
            row[start_idx]["dir"], row[start_idx]["cost"] = sz, 0.0
        for j in range(n):
            p = row[j]
            p["lo"] = p["l"] if (j == 0 or not row[j - 1]["feas"] or not p["feas"]) else row[j - 1]["lo"]
        for j in range(n - 1, -1, -1):
            p = row[j]
            p["hi"] = p["l"] if (j == n - 1 or not row[j + 1]["feas"] or not p["feas"]) else row[j + 1]["hi"]
        nodes.append((row, rx, ry, heading))
    # cost (:231-241)
    max_layer = 0
    for i in range(1, len(layers)):
        row, prow = nodes[i][0], nodes[i - 1][0]
        any_parent = False
        for p in row:
            if not p["feas"]:
                continue
            self_cost = 0.0
            if p["dis"] < 3.0:
                self_cost += (3.0 - p["dis"]) / 3.0 * 0.5
            self_cost += abs(p["l"]) / range_ * 1.0
            min_cost = DBL_MAX
            for k, q in enumerate(prow):
                if not q["feas"] or q["cost"] == DBL_MAX:     # unreached: self + edge + DBL_MAX never passes '<'
                    continue
                if abs(q["l"] - p["l"]) > p["s"] - q["s"]:
                    continue
                direction = math.atan2(p["y"] - q["y"], p["x"] - q["x"])
                edge = (abs(constraint_angle(direction - q["dir"])) / (math.pi / 2) * 16.0
                        + abs(constraint_angle(direction - p["heading"])) / (math.pi / 2) * 0.5)
                total = self_cost + edge + q["cost"]
                if min_cost < DBL_MAX:
                    margins.append(abs(total - min_cost))
                    out["ties"] += total == min_cost
                if total < min_cost:
                    min_cost, p["parent"], p["dir"] = total, k, direction
            if p["parent"] is not None:
                p["cost"] = min_cost
                any_parent = True
        if not any_parent:
            break
        max_layer = i
    # retrieve (:243-293)
    best, min_cost = None, DBL_MAX
    for j, p in enumerate(nodes[max_layer][0]):
        if min_cost < DBL_MAX and p["cost"] < DBL_MAX:
            margins.append(abs(p["cost"] - min_cost))
            out["ties"] += p["cost"] == min_cost
        if p["cost"] < min_cost:
            best, min_cost = j, p["cost"]
    chain, bounds = [], []
    i, j = max_layer, best
    while j is not None:
        row, rx, ry, heading = nodes[i]
        p = row[j]
        if i == 0:
            bounds.append((-10.0, 10.0))
        else:
            bounds.append(march(ml, rx, ry, heading, p["lo"], p["hi"], margins))
        chain.append(j)
        j = p["parent"]
        i -= 1
    chain.reverse()
    bounds.reverse()
    out["s"], out["bounds"], out["chain"] = layers[:len(bounds)], bounds, chain
    if len(bounds) < 4:
        return done(COR_SHORT)
    return done(COR_OK)


def post_smooth_qp(s, bounds, vehicle_l):
    """setPostHessianMatrix / setPostConstraintMatrix (:590-644) as triplets: dict(n, m, P (i, j, v) upper, A (i, j, v),
    l, u), variables x (0..R-1), dx (R..2R-1), ddx (2R..3R-1)."""
    R = len(s)
    P = ([], [], [])
    for i in range(R):
        for idx, w in ((i, 1.0), (R + i, 100.0), (2 * R + i, 1000.0)):
            P[0].append(idx); P[1].append(idx); P[2].append(w)
    A = ([], [], [])

    def put(r, c, v):
        A[0].append(r); A[1].append(c); A[2].append(v)
    for i in range(R):
        put(i, i, 1.0)
    for i in range(R - 1):
        put(R + i, i + 1, 1.0); put(R + i, i, -1.0); put(R + i, R + i, -(s[i + 1] - s[i]))
    for i in range(R - 1):
        put(2 * R - 1 + i, R + i + 1, 1.0); put(2 * R - 1 + i, R + i, -1.0)
        put(2 * R - 1 + i, 2 * R + i, -(s[i + 1] - s[i]))
    l, u = np.zeros(3 * R - 2), np.zeros(3 * R - 2)
    l[0] = u[0] = vehicle_l
    for i in range(1, R):
        l[i], u[i] = bounds[i]
    return dict(n=3 * R, m=3 * R - 2, P=tuple(np.array(a) for a in P), A=tuple(np.array(a) for a in A), l=l, u=u)


def osqp_solve(params, qp):
    """The oracle's OSQP restatement on a triplet QP: (x, y, info)."""
    n, m = qp["n"], qp["m"]
    i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)      # noqa: E731
    f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)    # noqa: E731
    pi, pj, pv = i32(qp["P"][0]), i32(qp["P"][1]), f64(qp["P"][2])
    ai, aj, av = i32(qp["A"][0]), i32(qp["A"][1]), f64(qp["A"][2])
    q, lo, up = np.zeros(n), f64(qp["l"]), f64(qp["u"])
    ip, dp = C.POINTER(C.c_int), C.POINTER(C.c_double)
    prob = O.OqpProblem(n, m, len(pv), len(av), pi.ctypes.data_as(ip), pj.ctypes.data_as(ip), pv.ctypes.data_as(dp),
                        ai.ctypes.data_as(ip), aj.ctypes.data_as(ip), av.ctypes.data_as(dp), q.ctypes.data_as(dp),
                        lo.ctypes.data_as(dp), up.ctypes.data_as(dp))
    x, y, info = np.zeros(n), np.zeros(m), O.OqpInfo()
    O.lib().oracle_osqp_solve(C.byref(params), C.byref(prob), x.ctypes.data, y.ctypes.data, C.byref(info), None, 0)
    return x, y, info


def post_smooth(xs, ys, found, params):
    """postSmooth (:534-588) on a search's result: dict(reason, status, iters, x, y, s lists, qp, qp_margin)."""
    s, bounds = found["s"], found["bounds"]
    R = len(s)
    qp = post_smooth_qp(s, bounds, found["vehicle_l"])
    sol, _, info = osqp_solve(params, qp)
    out = dict(reason=COR_OK, status=info.status, iters=info.iters, qp=qp, qp_margin=info.margin, x=[], y=[], s=[])
    if info.status != SOLVED:
        out["reason"] = COR_QP
        return out
    acc = 0.0
    for i in range(R):
        rx, ry, heading, _ = sample(xs, ys, s[i])
        out["x"].append(rx + sol[i] * math.cos(heading + math.pi / 2))
        out["y"].append(ry + sol[i] * math.sin(heading + math.pi / 2))
        if i > 0:
            dx, dy = out["x"][i] - out["x"][i - 1], out["y"][i] - out["y"][i - 1]
            acc += math.sqrt(dx * dx + dy * dy)
        out["s"].append(acc)
    if not all(out["s"][i] > out["s"][i - 1] for i in range(1, R)) or not math.isfinite(out["s"][-1]):
        out["reason"] = COR_S_ORDER
    return out


def post_smooth_batch(splines, max_s, start, maps, params, capacity, map_index=None, max_layers=1 << 30,
                      range_=10.0, spacing=0.6, ds_long=1.5):
    """A batch in the layout of pqp_post_smooth_device.  maps: the map set (dicts of synth's map format); start:
    STATE_DTYPE records or [B, >= 3] arrays.  Returns dict(knot_offsets, knots, x_coef, y_coef, max_s, ok, status,
    iters, layers [knots, 3], reason, margin, qp_margin, found, smoothed)."""
    ko = np.asarray(splines["knot_offsets"])
    kn, xc, yc = (np.asarray(splines[k], dtype=np.float64) for k in ("knots", "x_coef", "y_coef"))
    xc, yc = xc.reshape(-1, 4), yc.reshape(-1, 4)
    start = np.asarray(start)
    B = len(max_s)
    lookups = [MapLookup(m) for m in maps]
    found, smoothed = [], []
    for b in range(B):
        sl = slice(int(ko[b]), int(ko[b + 1]))
        xs, ys = Spline(kn[sl], xc[sl]), Spline(kn[sl], yc[sl])
        st = [start[b][f] for f in ("x", "y", "z")] if start.dtype.names else list(start[b][:3])
        mi = 0 if map_index is None else int(map_index[b])
        ml = lookups[mi] if 0 <= mi < len(lookups) else None
        f = search(xs, ys, max_s[b], st, ml, range_, spacing, ds_long, max_layers)
        found.append(f)
        smoothed.append(post_smooth(xs, ys, f, params) if f["reason"] == COR_OK else None)
    reason = np.array([f["reason"] if sm is None else sm["reason"] for f, sm in zip(found, smoothed)], dtype=np.int32)
    counts = [len(found[b]["s"]) if reason[b] == COR_OK else 0 for b in range(B)]
    kept = reserve(counts, capacity)
    n = np.array([c if k else 0 for c, k in zip(counts, kept)], dtype=np.int32)
    off = np.zeros(B + 1, dtype=np.int32)
    np.cumsum(n, out=off[1:])
    T = int(off[-1])
    knots, xco, yco, layers = np.zeros(T), np.zeros((T, 4)), np.zeros((T, 4)), np.zeros((T, 3))
    ms = np.full(B, np.nan)
    for b in range(B):
        if reason[b] == COR_OK and not kept[b]:
            reason[b] = COR_CAPACITY
        if not kept[b]:
            continue
        sm, f = smoothed[b], found[b]
        sl = slice(off[b], off[b + 1])
        knots[sl] = sm["s"]
        xco[sl], yco[sl] = O.spline_fit(sm["s"], sm["x"]), O.spline_fit(sm["s"], sm["y"])
        layers[sl, 0] = f["s"]
        layers[sl, 1:] = np.array(f["bounds"])
        ms[b] = sm["s"][-1]
    status = np.array([-100 if sm is None else sm["status"] for sm in smoothed], dtype=np.int32)
    iters = np.array([0 if sm is None else sm["iters"] for sm in smoothed], dtype=np.int32)
    return dict(knot_offsets=off, knots=knots, x_coef=xco, y_coef=yco, max_s=ms, ok=np.array(kept, dtype=np.int32),
                status=status, iters=iters, layers=layers, reason=reason,
                margin=np.array([f["margin"] for f in found]),
                qp_margin=np.array([math.inf if sm is None else sm["qp_margin"] for sm in smoothed]),
                found=found, smoothed=smoothed)
