"""CPU tests of the corridor search and post-smoothing restatement (oracle/corridor.py): an independent numpy twin of
graphSearchDp, vectorised per layer, gives the same reached layers, layer s, chosen nodes and bounds exactly; the
post-smoothing QP solved by the oracle's OSQP equals oracle/twin.py's osqp_twin in status and iterations with iterates
within 1e-9, and passes the KKT certificate; and the named scenes behave as they are built to."""
import math

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import corridor as oc
from oracle import oracle as O
from oracle import twin
from oracle.segment import Spline, sample
from tests import corridor_cases as cc
from tests.emu import corridor_emu

atan2_v = np.frompyfunc(math.atan2, 2, 1)


def _wrap(a):
    a = a.copy()
    while np.any(a > math.pi):
        a = np.where(a > math.pi, a - 2 * math.pi, a)
    while np.any(a < -math.pi):
        a = np.where(a < -math.pi, a + 2 * math.pi, a)
    return a


def _twin_closest(xs, ys, max_s, x, y):
    """findClosestPoint with the grid scan as one array: np.argmin takes the first index of the minimum."""
    grid = 0.5 * np.arange(int(math.floor(2 * max_s)) + 1)
    d = np.array([math.sqrt((xs(t) - x) ** 2 + (ys(t) - y) ** 2) for t in grid])
    cur = prev = float(grid[int(np.argmin(d))])
    for _ in range(20):
        px, py = xs(cur) - x, ys(cur) - y
        dx, dy, ddx, ddy = xs(cur, 1), ys(cur, 1), xs(cur, 2), ys(cur, 2)
        cur = cur - float(np.float64(px * dx + py * dy) / np.float64(dx * dx + px * ddx + dy * dy + py * ddy))
        if abs(cur - prev) < 1e-5:
            break
        prev = cur
    return min(cur, max_s)


def _twin_march(ml, rx, ry, h, lo, hi):
    """The bound march as two scans of a precomputed probe sequence: the first probe that fails stops each side."""
    c, s = math.cos(h + math.pi / 2), math.sin(h + math.pi / 2)
    out = []
    for start, step, limit in ((hi + 0.2, 0.2, 6.0), (-0.2 + lo, -0.2, -6.0)):
        probes = [start]
        while (probes[-1] < limit) if step > 0 else (probes[-1] > limit):
            probes.append(probes[-1] + step)
        ok = [ml.inside(rx + p * c, ry + p * s) and ml.distance(rx + p * c, ry + p * s) > 1.45 for p in probes[:-1]]
        k = ok.index(False) if False in ok else None
        out.append(probes[-1] if k is None else probes[k] - step)
    return out[1], out[0]


def twin_search(xs, ys, max_s, start, m, range_=10.0, spacing=0.6, ds_long=1.5):
    """graphSearchDp with the per-layer work on numpy arrays: (s list, chain, bounds) or None when refused."""
    ml = oc.MapLookup(m)
    lat = [-range_]
    while lat[-1] + spacing <= range_:
        lat.append(lat[-1] + spacing)
    lat = np.array(lat)
    n = len(lat)
    s0 = _twin_closest(xs, ys, max_s, start[0], start[1])
    ds = ds_long if max_s > 6 else 0.5
    layers = []
    t = s0
    while t < max_s:
        layers.append(t)
        t += ds
    layers.append(max_s)
    px, py, pz, _ = sample(xs, ys, s0)
    vl = -(start[0] - px) * math.sin(pz) + (start[1] - py) * math.cos(pz)
    if abs(vl) > range_:
        return None
    si = int((range_ + vl) / spacing)
    inside_v = np.frompyfunc(ml.inside, 2, 1)
    dist_v = np.frompyfunc(ml.distance, 2, 1)
    L = []
    for i, s in enumerate(layers):
        rx, ry, h, k = sample(xs, ys, s)
        x = rx + lat * math.cos(h + math.pi / 2)
        y = ry + lat * math.sin(h + math.pi / 2)
        inside = inside_v(x, y).astype(bool)
        dis = np.where(inside, dist_v(x, y).astype(float), -1.0)
        with np.errstate(all="ignore"):
            r = np.float64(1) / np.float64(k)
        feas = ~(((k < 0) & (lat < r)) | ((k > 0) & (lat > r)) | (dis < 1.45))
        if i == 0:
            feas = np.arange(n) == si
        L.append(dict(x=x, y=y, h=h, s=s, rx=rx, ry=ry, feas=feas, dis=dis))
    cost = np.where(L[0]["feas"], 0.0, np.inf)
    dirs = np.full(n, start[2])
    parents, top = [None], 0
    for i in range(1, len(layers)):
        p, q = L[i], L[i - 1]
        self_c = np.where(p["dis"] < 3.0, 0.0 + (3.0 - p["dis"]) / 3.0 * 0.5, 0.0) + np.abs(lat) / range_ * 1.0
        d = atan2_v(p["y"][None, :] - q["y"][:, None], p["x"][None, :] - q["x"][:, None]).astype(float)   # [pre, node]
        edge = (np.abs(_wrap(d - dirs[:, None])) / (math.pi / 2) * 16.0
                + np.abs(_wrap(d - p["h"])) / (math.pi / 2) * 0.5)
        tot = self_c[None, :] + edge + np.where(np.isfinite(cost), cost, 0.0)[:, None]
        ok = (np.isfinite(cost)[:, None] & q["feas"][:, None] & p["feas"][None, :]
              & ~(np.abs(lat[:, None] - lat[None, :]) > p["s"] - q["s"]))
        tot = np.where(ok, tot, np.inf)
        par = np.argmin(tot, axis=0)                     # first index of the minimum
        best = tot[par, np.arange(n)]
        reached = np.isfinite(best)
        if not reached.any():
            break
        cost = np.where(reached, best, np.inf)
        dirs = np.where(reached, d[par, np.arange(n)], 0.0)
        parents.append(np.where(reached, par, -1))
        top = i
    j = int(np.argmin(cost)) if np.isfinite(cost).any() else None
    chain = []
    for i in range(top, -1, -1):
        chain.append(j)
        if i > 0:
            j = int(parents[i][j])
    chain.reverse()
    bounds = [(-10.0, 10.0)]
    for i in range(1, top + 1):
        f, j = L[i]["feas"], chain[i]
        a, b = j, j
        while a > 0 and f[a - 1]:
            a -= 1
        while b + 1 < n and f[b + 1]:
            b += 1
        bounds.append(_twin_march(ml, L[i]["rx"], L[i]["ry"], L[i]["h"], lat[a], lat[b]))
    return layers[:top + 1], chain, bounds


def _scene(name):
    m, (kn, xco, yco), st = cc.scenes()[name]
    return m, Spline(kn, xco), Spline(kn, yco), float(kn[-1]), [float(st["x"]), float(st["y"]), float(st["z"])]


@pytest.mark.parametrize("name", list(cc.scenes()))
def test_restatement_equals_numpy_twin(name):
    m, xs, ys, max_s, st = _scene(name)
    f = oc.search(xs, ys, max_s, st, oc.MapLookup(m))
    t = twin_search(xs, ys, max_s, st, m)
    if f["reason"] == oc.COR_FAR:
        assert t is None
        return
    s, chain, bounds = t
    if f["reason"] == oc.COR_SHORT:
        assert len(s) < 4
        return
    assert f["reason"] == oc.COR_OK
    assert f["s"] == s
    assert f["chain"] == chain
    assert [tuple(b) for b in f["bounds"]] == [tuple(b) for b in bounds]


@pytest.mark.parametrize("name", [n for n in cc.scenes() if n not in ("far start", "near end")])
def test_qp_equals_osqp_twin(name):
    m, xs, ys, max_s, st = _scene(name)
    f = oc.search(xs, ys, max_s, st, oc.MapLookup(m))
    qp = oc.post_smooth_qp(f["s"], f["bounds"], f["vehicle_l"])
    prm = O.default_params()
    x, y, info = oc.osqp_solve(prm, qp)
    n, mm = qp["n"], qp["m"]
    P = sp.coo_matrix((qp["P"][2], (qp["P"][0], qp["P"][1])), shape=(n, n)).tocsc()
    A = sp.coo_matrix((qp["A"][2], (qp["A"][0], qp["A"][1])), shape=(mm, n)).tocsc()
    tw = twin.osqp_twin(prm, P, np.zeros(n), A, qp["l"], qp["u"])
    assert info.status == tw["status"] == oc.SOLVED
    assert info.iters == tw["iters"]
    np.testing.assert_allclose(x, tw["x"], rtol=0, atol=1e-9)
    np.testing.assert_allclose(y, tw["y"], rtol=0, atol=1e-9)
    # OSQP's own stopping rule on the unscaled problem, with the settings' eps
    cert = twin.kkt_certificate(P, np.zeros(n), A, qp["l"], qp["u"], x, y)
    Ax, Px, Aty = A @ x, P @ x, A.T @ y
    z = np.clip(Ax, qp["l"], qp["u"])
    assert cert["primal"] <= prm.eps_abs + prm.eps_rel * max(np.abs(Ax).max(), np.abs(z).max())
    assert cert["dual"] <= prm.eps_abs + prm.eps_rel * max(np.abs(Px).max(), np.abs(Aty).max())


def test_scenes_behave_as_built():
    b = cc.batch()
    r = oc.post_smooth_batch(b["splines"], b["max_s"], b["start"], b["maps"], O.default_params(), 100000,
                             map_index=b["map_index"], max_layers=200)
    got = dict(zip(b["names"], r["reason"]))
    assert got["far start"] == oc.COR_FAR
    assert got["near end"] == oc.COR_SHORT
    f = dict(zip(b["names"], r["found"]))
    assert all(c == f["clear"]["chain"][0] for c in f["clear"]["chain"])         # a clear road keeps its lane
    assert len(set(f["obstacle"]["chain"])) > 1                                 # an obstacle forces a detour
    assert len(f["wall"]["s"]) < len(f["clear"]["s"])                           # a wall cuts the layers reached
    assert np.allclose(np.diff(f["short"]["s"][:-1]), 0.5)                      # <= 6 m: 0.5 m layers
    assert f["moved q1"]["chain"] == f["moved q0"]["chain"] == f["moved q3"]["chain"]
    assert r["ok"].sum() == len(b["names"]) - 2


def _band(R):
    """Band position of the reference's variable order (x 0..R-1, dx R..2R-1, ddx 2R..3R-1)."""
    return np.concatenate([3 * np.arange(R), 3 * np.arange(R) + 1, 3 * np.arange(R) + 2])


@pytest.mark.parametrize("name", list(cc.scenes()) + ["tie"])
def test_emulator_equals_restatement(name):
    """pqp_corridor_core.cuh compiled with g++ equals the restatement bit for bit: reason, layer s, chain, bounds and
    vehicle_l, and its QP rows, columns and separators are the restatement's QP in band order."""
    if name == "tie":
        m, (kn, xco, yco), st = cc.tie_scene()
        kw = dict(spacing=cc.TIE_SPACING)
    else:
        m, (kn, xco, yco), st = cc.scenes()[name]
        kw = {}
    start = [float(st["x"]), float(st["y"]), float(st["z"])]
    f = oc.search(Spline(kn, xco), Spline(kn, yco), float(kn[-1]), start, oc.MapLookup(m), max_layers=400, **kw)
    e = corridor_emu.search(kn, xco, yco, float(kn[-1]), st, m, max_layers=400, **kw)
    assert e["reason"] == f["reason"]
    if f["reason"] != oc.COR_OK:
        return
    assert e["s"] == f["s"] and e["chain"] == f["chain"]
    assert [tuple(b) for b in e["bounds"]] == [tuple(b) for b in f["bounds"]]
    assert e["vehicle_l"] == f["vehicle_l"]
    R = len(f["s"])
    qp = oc.post_smooth_qp(f["s"], f["bounds"], f["vehicle_l"])
    band = _band(R)
    A = sp.coo_matrix((qp["A"][2], (qp["A"][0], band[qp["A"][1]])), shape=(qp["m"], 3 * R)).toarray()
    ell = np.zeros_like(A)
    for r in range(qp["m"]):
        for c, v in zip(e["A_col"][r], e["A_val"][r]):
            if c >= 0:
                ell[r, c] += v
    np.testing.assert_array_equal(ell, A)
    csc = sp.csc_matrix((e["csc_val"], e["csc_row"], e["csc_ptr"]), shape=(qp["m"], 3 * R))
    assert csc.has_sorted_indices
    np.testing.assert_array_equal(csc.toarray(), A)
    np.testing.assert_array_equal(e["l"], qp["l"])
    np.testing.assert_array_equal(e["u"], qp["u"])
    L = max(2, (R - 2) // 31 + 1)
    assert e["sep"] == [3 * k for k in range(0, R - 1, L)][:32]


def test_tie_goes_to_the_first_index():
    """On a lattice symmetric about the line and a mirror-symmetric map the DP meets exact ties; the restatement and
    the numpy twin agree on the chain, which the strict '<' in index order decides."""
    m, (kn, xco, yco), st = cc.tie_scene()
    start = [float(st["x"]), float(st["y"]), float(st["z"])]
    xs, ys = Spline(kn, xco), Spline(kn, yco)
    f = oc.search(xs, ys, float(kn[-1]), start, oc.MapLookup(m), spacing=cc.TIE_SPACING)
    assert f["reason"] == oc.COR_OK and f["ties"] > 0 and f["margin"] == 0
    s, chain, bounds = twin_search(xs, ys, float(kn[-1]), start, m, spacing=cc.TIE_SPACING)
    assert f["s"] == s and f["chain"] == chain
    assert [tuple(b) for b in f["bounds"]] == [tuple(b) for b in bounds]


def test_clear_road_keeps_the_line():
    """A start on the line of a clear road: the QP's offsets stay at 0 within OSQP's tolerance."""
    m, (kn, xco, yco), st = cc.scenes()["clear"]
    f = oc.search(Spline(kn, xco), Spline(kn, yco), float(kn[-1]), [st["x"], st["y"], st["z"]], oc.MapLookup(m))
    assert f["vehicle_l"] == 0.0
    x, _, info = oc.osqp_solve(O.default_params(), oc.post_smooth_qp(f["s"], f["bounds"], f["vehicle_l"]))
    assert info.status == oc.SOLVED
    assert np.abs(x[:len(f["s"])]).max() < 1e-3
