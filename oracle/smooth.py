"""CPU restatement of ReferencePathSmoother::bSpline and TensionSmoother2::smooth under the default flags (TEST
INFRASTRUCTURE, not product code): what pqp_smooth_reference_device computes, path by path, in plain Python floats.

Written from the reference's behaviour (src/reference_path_smoother/reference_path_smoother.cpp:36-39 input check,
:50-88 segmentRawReference, :498-532 bSpline; tension_smoother_2.cpp:163-301 osqpSmooth and its matrices;
tension_smoother.cpp:84-96 the smooth tail; distance of src/tools/tools.cpp:46-48).  tinyspline's clamped B-spline is
restated from its published definition: clamped uniform knots and de Boor's algorithm.  Every operation is one IEEE
double operation in the kernel's order and the transcendental functions are the C library's.  The smoothing QP is built
as triplets in the reference's own variable order (x, y, theta of every station, then k of all but the last) and row
order (x updates, y updates, theta updates, the x and y pins), exact zeros dropped as Eigen's sparseView drops them,
and solved by the oracle's OSQP restatement.
"""
import ctypes as C
import math

import numpy as np

from oracle import oracle as O
from oracle.segment import Spline, reserve, sample

(SM_OK, SM_FEW, SM_DEGREE, SM_LENGTH, SM_RAW_MANY, SM_RAW_ORDER, SM_MANY, SM_SHORT, SM_QP, SM_S_ORDER,
 SM_CAPACITY) = range(11)
DBL_MAX = 1.7976931348623157e308
SOLVED = 1
WEIGHTS = (0.005, 1.0, 10.0)


def degree(px, py):
    """bSpline's length and degree (:499-508)."""
    length = 0.0
    for i in range(len(px) - 1):
        dx, dy = px[i] - px[i + 1], py[i] - py[i + 1]
        length += math.sqrt(dx * dx + dy * dy)
    avg = length / (len(px) - 1)
    return (3 if avg > 10 else 4 if avg > 5 else 5), length


def knot(n, p, j):
    """Knot j of the clamped uniform knot vector of n control points, degree p."""
    if j <= p:
        return 0.0
    if j >= n:
        return 1.0
    return (j - p) / (n - p)


def bspline_eval(px, py, p, t):
    """de Boor's algorithm at t in [0, 1]."""
    n = len(px)
    k = p
    while k + 1 < n and knot(n, p, k + 1) <= t:
        k += 1
    dx = [px[j + k - p] for j in range(p + 1)]
    dy = [py[j + k - p] for j in range(p + 1)]
    for r in range(1, p + 1):
        for j in range(p, r - 1, -1):
            lo, hi = knot(n, p, j + k - p), knot(n, p, j + 1 + k - r)
            a = (t - lo) / (hi - lo)
            dx[j] = (1.0 - a) * dx[j - 1] + a * dx[j]
            dy[j] = (1.0 - a) * dy[j - 1] + a * dy[j]
    return dx[p], dy[p]


def sample_params(length, cap):
    """t = 0, delta_t, ... (accumulated) while t < 1, then 1; at most cap + 1 of them."""
    with np.errstate(all="ignore"):
        delta_t = float(np.float64(1.0) / np.float64(length))
    t, tmp = [], 0.0
    while tmp < 1 and len(t) <= cap:
        t.append(tmp)
        tmp += delta_t
    if len(t) <= cap:
        t.append(1.0)
    return t


def b_spline(px, py, max_raw=1 << 30):
    """bSpline on one polyline: dict(reason, degree, length, t, x, y, s)."""
    out = dict(reason=SM_OK, degree=None, length=None, t=[], x=[], y=[], s=[])
    if len(px) < 4:
        out["reason"] = SM_FEW
        return out
    p, length = degree(px, py)
    out["degree"], out["length"] = p, length
    if p >= len(px):
        out["reason"] = SM_DEGREE
        return out
    if not (0 < length <= DBL_MAX):
        out["reason"] = SM_LENGTH
        return out
    t = sample_params(length, max_raw)
    if len(t) > max_raw:
        out["reason"] = SM_RAW_MANY
        return out
    out["t"] = t
    s = 0.0
    for k, tk in enumerate(t):
        x, y = bspline_eval(px, py, p, tk)
        if k > 0:
            dx, dy = x - out["x"][-1], y - out["y"][-1]
            s += math.sqrt(dx * dx + dy * dy)
        out["x"].append(x)
        out["y"].append(y)
        out["s"].append(s)
    return out


def increasing(s):
    return len(s) >= 3 and all(s[i] > s[i - 1] for i in range(1, len(s))) and s[-1] <= DBL_MAX


def segment_raw(raw):
    """segmentRawReference (:50-88): the raw splines and the stations (x, y, heading, curvature) at s = 0, 1, 2, ..."""
    xs = Spline(raw["s"], O.spline_fit(raw["s"], raw["x"]))
    ys = Spline(raw["s"], O.spline_fit(raw["s"], raw["y"]))
    max_s = raw["s"][-1]
    s = [0.0]
    while s[-1] < max_s:
        s.append(s[-1] + 1.0)
    return xs, ys, s, [sample(xs, ys, v) for v in s]


def tension2_qp(stations, s, weights=WEIGHTS):
    """setHessianMatrix / setGradient / setConstraintMatrix (tension_smoother_2.cpp:221-301) as triplets in the
    reference's order: dict(n, m, P (i, j, v) upper, q, A (i, j, v), l, u)."""
    w_dev, w_curv, w_rate = weights
    N = len(stations)
    X, Y, T, K = 0, N, 2 * N, 3 * N
    n, m = 4 * N - 1, 3 * (N - 1) + 2
    H = {}
    for i in range(N):
        H[(X + i, X + i)] = H[(Y + i, Y + i)] = w_dev * 2
        if i != N - 1:
            H[(K + i, K + i)] = w_curv * 2
    for i in range(N - 2):
        for (a, b), c in (((0, 0), 1.0), ((0, 1), -1.0), ((1, 0), -1.0), ((1, 1), 1.0)):
            key = (K + i + a, K + i + b)
            H[key] = H.get(key, 0.0) + 2 * w_rate * c
    P = tuple(np.array(v) for v in zip(*[(i, j, v) for (i, j), v in sorted(H.items()) if i <= j and v != 0.0]))
    q = np.zeros(n)
    for i, st in enumerate(stations):
        q[X + i] = -2 * w_dev * st[0]
        q[Y + i] = -2 * w_dev * st[1]
    A = {}
    lo, up = np.zeros(m), np.zeros(m)
    cx, cy, ct = 0, N - 1, 2 * N - 2
    for i in range(N - 1):
        ds = s[i + 1] - s[i]
        ang, k = stations[i][2], stations[i][3]
        A[(cx + i, X + i + 1)] = A[(cy + i, Y + i + 1)] = A[(ct + i, T + i + 1)] = 1.0
        A[(cx + i, X + i)] = A[(cy + i, Y + i)] = A[(ct + i, T + i)] = -1.0
        A[(cx + i, T + i)] = ds * math.sin(ang)
        A[(cy + i, T + i)] = -ds * math.cos(ang)
        A[(ct + i, K + i)] = -ds
        lo[cx + i] = up[cx + i] = ds * math.cos(ang)
        lo[cy + i] = up[cy + i] = ds * math.sin(ang)
        lo[ct + i] = up[ct + i] = -ds * k
    A[(3 * N - 3, X)] = A[(3 * N - 2, Y)] = 1.0
    lo[3 * N - 3] = up[3 * N - 3] = stations[0][0]
    lo[3 * N - 2] = up[3 * N - 2] = stations[0][1]
    At = tuple(np.array(v) for v in zip(*[(r, c, v) for (r, c), v in sorted(A.items()) if v != 0.0]))
    return dict(n=n, m=m, P=P, q=q, A=At, l=lo, u=up)


def dense(qp):
    """(P full symmetric, q, A, l, u) as dense arrays."""
    P = np.zeros((qp["n"], qp["n"]))
    for i, j, v in zip(*qp["P"]):
        P[int(i), int(j)] = P[int(j), int(i)] = v
    A = np.zeros((qp["m"], qp["n"]))
    for r, c, v in zip(*qp["A"]):
        A[int(r), int(c)] = v
    return P, np.array(qp["q"]), A, np.array(qp["l"]), np.array(qp["u"])


def osqp_solve(params, qp):
    """The oracle's OSQP restatement on a triplet QP with its q: (x, y, info)."""
    n, m = qp["n"], qp["m"]
    i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)      # noqa: E731
    f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)    # noqa: E731
    pi, pj, pv = i32(qp["P"][0]), i32(qp["P"][1]), f64(qp["P"][2])
    ai, aj, av = i32(qp["A"][0]), i32(qp["A"][1]), f64(qp["A"][2])
    q, lo, up = f64(qp["q"]), f64(qp["l"]), f64(qp["u"])
    ip, dp = C.POINTER(C.c_int), C.POINTER(C.c_double)
    prob = O.OqpProblem(n, m, len(pv), len(av), pi.ctypes.data_as(ip), pj.ctypes.data_as(ip), pv.ctypes.data_as(dp),
                        ai.ctypes.data_as(ip), aj.ctypes.data_as(ip), av.ctypes.data_as(dp), q.ctypes.data_as(dp),
                        lo.ctypes.data_as(dp), up.ctypes.data_as(dp))
    x, y, info = np.zeros(n), np.zeros(m), O.OqpInfo()
    O.lib().oracle_osqp_solve(C.byref(params), C.byref(prob), x.ctypes.data, y.ctypes.data, C.byref(info), None, 0)
    return x, y, info


def smooth(px, py, params, max_raw=1 << 30, max_points=1 << 30, weights=WEIGHTS):
    """One polyline through the whole stage: dict(reason, status, iters, raw, s_raw, stations, qp, qp_margin, x, y, s)."""
    out = dict(reason=SM_OK, status=-100, iters=0, raw=None, stations=[], qp=None, qp_margin=math.inf, x=[], y=[], s=[])
    raw = b_spline(px, py, max_raw)
    out["raw"] = raw
    if raw["reason"] != SM_OK:
        out["reason"] = raw["reason"]
        return out
    if not increasing(raw["s"]):
        out["reason"] = SM_RAW_ORDER
        return out
    max_s = raw["s"][-1]
    if not max_s <= max_points:
        out["reason"] = SM_MANY
        return out
    _, _, s, stations = segment_raw(raw)
    out["stations"], out["s_stations"] = stations, s
    if len(s) > max_points:
        out["reason"] = SM_MANY
        return out
    if len(s) < 3:
        out["reason"] = SM_SHORT
        return out
    qp = tension2_qp(stations, s, weights)
    out["qp"] = qp
    sol, _, info = osqp_solve(params, qp)
    out.update(status=info.status, iters=info.iters, qp_margin=info.margin)
    if info.status != SOLVED:
        out["reason"] = SM_QP
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
    if not increasing(out["s"]):
        out["reason"] = SM_S_ORDER
    return out


def smooth_batch(points, point_offsets, params, capacity, max_raw=1 << 30, max_points=1 << 30, weights=WEIGHTS):
    """A batch in the layout of pqp_smooth_reference_device: points [P, >= 2] (x, y) or STATE_DTYPE records.  Returns
    dict(knot_offsets, knots, x_coef, y_coef, max_s, ok, status, iters, reason, qp_margin, smoothed)."""
    pts = np.asarray(points)
    xy = np.stack([pts["x"], pts["y"]], 1) if pts.dtype.names else np.asarray(pts, dtype=np.float64)[:, :2]
    po = np.asarray(point_offsets)
    B = len(po) - 1
    res = [smooth([float(v) for v in xy[po[b]:po[b + 1], 0]], [float(v) for v in xy[po[b]:po[b + 1], 1]], params,
                  max_raw, max_points, weights) for b in range(B)]
    reason = np.array([r["reason"] for r in res], dtype=np.int32)
    counts = [len(r["s"]) if r["reason"] == SM_OK else 0 for r in res]
    kept = reserve(counts, capacity)
    n = np.array([c if k else 0 for c, k in zip(counts, kept)], dtype=np.int32)
    off = np.zeros(B + 1, dtype=np.int32)
    np.cumsum(n, out=off[1:])
    T = int(off[-1])
    knots, xco, yco = np.zeros(T), np.zeros((T, 4)), np.zeros((T, 4))
    ms = np.full(B, np.nan)
    for b, r in enumerate(res):
        if reason[b] == SM_OK and not kept[b]:
            reason[b] = SM_CAPACITY
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
