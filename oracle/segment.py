"""CPU restatement of PathOptimizer::segmentSmoothedPath (TEST INFRASTRUCTURE, not product code): what
pqp_segment_reference_device computes, path by path, in plain Python floats.

Written from the reference's behaviour (src/path_optimizer/path_optimizer.cpp:119-178 and
ReferencePathImpl::buildReferenceFromSpline, src/data_struct/reference_path_impl.cpp:474-499) with tk::spline's
evaluation (src/tools/spline.cpp:250-318) and the helpers of src/tools/tools.cpp.  Every operation is one IEEE double
operation, in the reference's order, and the transcendental functions are the C library's (math.sin / cos / atan2 /
pow / sqrt), so the kernel's per-thread functions compiled with g++ give the same bits.  pow(v, 2) is the correctly
rounded square v * v.

Besides the result, every path reports `margin`: how close its discrete decisions came to flipping -- the sign of the
start's lateral offset, the heading error against 75 degrees, the end distance against 1e-6, every goal-search sample's
distance against 8 m and against the running minimum, the lattice against 0, and every walk sample's s against the cut
length.  A device whose atan2 / sin / pow differ from the C library's in the last bits can only decide differently
where that margin is tiny.
"""
import bisect
import math

import numpy as np

SEG_OK, SEG_BAD_SPLINE, SEG_HEADING, SEG_BAD_LENGTH, SEG_TOO_MANY, SEG_CAPACITY = range(6)
MAX_SEARCH = 4194304.0          # 2^22 goal-search samples
MAX_TURN = 1048576.0            # 2^20 rad: start.z minus the line's first heading, before constraintAngle
HEADING_LIMIT = 75 * math.pi / 180
DBL_MAX = 1.7976931348623157e308


def _div(a, b):
    with np.errstate(all="ignore"):
        return float(np.float64(a) / np.float64(b))


def _pow(a, e):
    try:
        return math.pow(a, e)
    except OverflowError:
        return math.inf


class Spline:
    """tk::spline with its default natural boundary, from the fitted rows: knots t[n], coef[n][4] = (a, b, c, y)."""

    def __init__(self, t, coef):
        self.t = [float(v) for v in t]
        self.c = [[float(v) for v in row] for row in np.asarray(coef).reshape(-1, 4)]

    def __call__(self, at, order=0):
        t, c = self.t, self.c
        n = len(t)
        idx = max(bisect.bisect_left(t, at) - 1, 0)
        h = at - t[idx]
        if at < t[0]:            # left: the first row's quadratic part (tk::spline's m_b0, m_c0)
            b0, c0 = c[0][1], c[0][2]
            if order == 0:
                return (b0 * h + c0) * h + c[0][3]
            return 2.0 * b0 * h + c0 if order == 1 else 2.0 * b0 * h
        if at > t[n - 1]:        # right: the last row, a quadratic
            e = c[n - 1]
            if order == 0:
                return (e[1] * h + e[2]) * h + e[3]
            return 2.0 * e[1] * h + e[2] if order == 1 else 2.0 * e[1]
        a, b, cc, y = c[idx]
        if order == 0:
            return ((a * h + b) * h + cc) * h + y
        if order == 1:
            return (3.0 * a * h + 2.0 * b) * h + cc
        return 6.0 * a * h + 2.0 * b


def sample(xs, ys, s):
    """(x, y, heading, curvature) at s: getHeading / getCurvature, tools.cpp:32-44."""
    x1, y1, x2, y2 = xs(s, 1), ys(s, 1), xs(s, 2), ys(s, 2)
    k = _div(x1 * y2 - y1 * x2, _pow(x1 * x1 + y1 * y1, 1.5))
    return xs(s), ys(s), math.atan2(y1, x1), k


def constraint_angle(a):
    """tools.hpp:24-35"""
    while a > math.pi:
        a -= 2 * math.pi
    while a < -math.pi:
        a += 2 * math.pi
    return a


def _step(s, k, ds_small, ds_large, dynamic):
    if not dynamic:
        return s + ds_large
    ak = abs(k)
    share = 1.0 if ak > 0.2 else 0.0 if ak < 0.08 else (ak - 0.08) / (0.2 - 0.08)
    return s + (ds_large - share * (ds_large - ds_small))


def segment_path(xs, ys, max_s, start, goal, ds_small=0.15, ds_large=0.3, dynamic=True, search_ds=0.5, max_n=1 << 30):
    """One path.  start / goal: (x, y, z, k) sequences.  Returns dict(reason, states [(x, y, z, k, s)], x0, cut_s,
    margin); states is empty unless reason == SEG_OK."""
    sx, sy, sz, sk = (float(v) for v in start[:4])
    gx, gy = float(goal[0]), float(goal[1])
    out = dict(reason=SEG_OK, states=[], x0=(0.0, 0.0, sk), cut_s=float(max_s), margin=math.inf)
    margins = []

    def done(reason):
        out["reason"] = reason
        out["states"] = [] if reason != SEG_OK else out["states"]
        out["margin"] = min(margins) if margins else math.inf
        return out
    if len(xs.t) < 3 or len(ys.t) < 3:
        return done(SEG_BAD_SPLINE)
    # initial error, path_optimizer.cpp:125-141
    fx, fy, fz, _ = sample(xs, ys, 0.0)
    dx, dy = fx - sx, fy - sy
    local_y = -dx * math.sin(sz) + dy * math.cos(sz) if math.isfinite(sz) else math.nan
    ex, ey = sx - fx, sy - fy
    min_distance = math.sqrt(ex * ex + ey * ey) if math.isfinite(ex * ex + ey * ey) else ex * ex + ey * ey
    offset = min_distance if local_y < 0 else -min_distance
    turn = sz - fz
    out["x0"] = (offset, turn, sk)
    margins.append(abs(local_y) if min_distance > 0 else math.inf)
    if not (abs(offset) <= DBL_MAX and abs(turn) <= MAX_TURN):
        return done(SEG_BAD_SPLINE)
    heading_error = constraint_angle(turn)
    out["x0"] = (offset, heading_error, sk)
    margins.append(abs(abs(heading_error) - HEADING_LIMIT))
    if abs(heading_error) > HEADING_LIMIT:
        return done(SEG_HEADING)
    max_s = float(max_s)
    if not (max_s > 0.0 and max_s <= search_ds * MAX_SEARCH):
        return done(SEG_BAD_LENGTH)
    # goal cut, :143-166
    length = max_s
    ux, uy = gx - xs(length), gy - ys(length)
    end_distance = math.sqrt(ux * ux + uy * uy)
    margins.append(abs(end_distance - 1e-6))
    if not abs(end_distance - 0.0) < 1e-6:
        tmp_s = length - search_ds
        min_d, min_s = end_distance, length
        while True:
            margins.append(abs(tmp_s))
            if not tmp_s > 0:
                break
            px, py = xs(tmp_s) - gx, ys(tmp_s) - gy
            d = math.sqrt(px * px + py * py)
            margins.append(abs(d - min_d))
            if d < min_d:
                min_d, min_s = d, tmp_s
            margins += [abs(d - 8), abs(min_d - 8)]
            if d > 8 and min_d < 8:
                break
            tmp_s -= search_ds
        length = min_s
    out["cut_s"] = length
    # buildReferenceFromSpline, reference_path_impl.cpp:474-499
    states = []
    s = 0.0
    while True:
        margins.append(abs(s - length))
        if not s <= length:
            break
        if len(states) == max_n:
            return done(SEG_TOO_MANY)
        x, y, z, k = sample(xs, ys, s)
        states.append((x, y, z, k, s))
        s = _step(s, k, ds_small, ds_large, dynamic)
    out["states"] = states
    return done(SEG_OK)


def reserve(counts, capacity):
    """Station reservation in index order: kept[b] when counts[b] > 0 and the stations of paths 0..b (refused ones
    counting 0) do not exceed capacity."""
    kept, before = [], 0
    for c in counts:
        kept.append(c > 0 and before + c <= capacity)
        before += c
    return kept


def segment_batch(splines, max_s, start, goal, capacity, **flags):
    """A batch in the layout of pqp_segment_reference_device.  splines: dict(knot_offsets [B+1], knots, x_coef,
    y_coef); start / goal: STATE_DTYPE records or [B, >= 4] arrays.  Returns dict(n_points, offsets, ref [offsets[B]]
    as (x, y, z, k, s, v, a) rows, x0 [B, 3], end_heading, ok, reason, cut_s, margin)."""
    ko = np.asarray(splines["knot_offsets"])
    kn, xc, yc = (np.asarray(splines[k], dtype=np.float64) for k in ("knots", "x_coef", "y_coef"))
    xc, yc = xc.reshape(-1, 4), yc.reshape(-1, 4)
    B = len(max_s)

    def row(a, b):
        if a.dtype.names:
            return [a[b][f] for f in ("x", "y", "z", "k")]
        return list(a[b][:4])
    res = []
    for b in range(B):
        sl = slice(int(ko[b]), int(ko[b + 1]))
        xs, ys = Spline(kn[sl], xc[sl]), Spline(kn[sl], yc[sl])
        res.append(segment_path(xs, ys, max_s[b], row(np.asarray(start), b), row(np.asarray(goal), b), **flags))
    counts = [len(r["states"]) for r in res]
    kept = reserve(counts, capacity)
    n = np.array([c if k else 0 for c, k in zip(counts, kept)], dtype=np.int32)
    off = np.zeros(B + 1, dtype=np.int32)
    np.cumsum(n, out=off[1:])
    ref = np.zeros((int(off[-1]), 7))
    for b in range(B):
        if kept[b]:
            ref[off[b]:off[b + 1], :5] = np.array(res[b]["states"])
    reason = np.array([r["reason"] if (r["reason"] != SEG_OK or kept[b]) else SEG_CAPACITY
                       for b, r in enumerate(res)], dtype=np.int32)
    goal = np.asarray(goal)
    end_heading = np.array([goal[b]["z"] if goal.dtype.names else goal[b][2] for b in range(B)], dtype=np.float64)
    return dict(n_points=n, offsets=off, ref=ref, x0=np.array([r["x0"] for r in res]).reshape(B, 3),
                end_heading=end_heading, ok=np.array(kept, dtype=np.int32), reason=reason,
                cut_s=np.array([r["cut_s"] for r in res]), margin=np.array([r["margin"] for r in res]))
