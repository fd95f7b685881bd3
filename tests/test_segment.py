"""CPU tests of the batched segmentation of smoothed reference lines (pqp_segment_reference_device).

* The CPU restatement (oracle/segment.py) against an independent numpy twin written here: vectorised spline evaluation,
  a vectorised goal search over the accumulated lattice, numpy's arctan2 / power / hypot and a modulo angle wrap.
* The kernel's per-thread functions compiled with g++ (tests/emu/segment_emu.cpp), in the order of its three launches,
  against the oracle bit for bit: refusals, counts, offsets, every state, x0 and the cut length.
* The count / reservation / write split: refusals by the station cap and by the capacity fall on the oracle's paths.
Lines, starts and goals: tests/segment_cases.py."""
import math

import numpy as np
import pytest

from oracle import segment as oseg
from tests import segment_cases as sc
from tests.emu import segment_emu

BIG = 10 ** 7
NEAR = 1e-9          # a decision this close to its threshold may go either way under another libm


# ---- the numpy twin --------------------------------------------------------------------------------------------------

def _ev(t, c, at, order):
    at = np.atleast_1d(np.asarray(at, dtype=np.float64))
    idx = np.maximum(np.searchsorted(t, at, side="left") - 1, 0)
    h = at - t[idx]
    a, b, cc, y = (c[idx, k] for k in range(4))
    v = [((a * h + b) * h + cc) * h + y, (3 * a * h + 2 * b) * h + cc, 6 * a * h + 2 * b][order]
    left, right = at < t[0], at > t[-1]
    e = c[-1]
    v = np.where(left, [(c[0, 1] * h + c[0, 2]) * h + c[0, 3], 2 * c[0, 1] * h + c[0, 2], 2 * c[0, 1] * h][order], v)
    return np.where(right, [(e[1] * h + e[2]) * h + e[3], 2 * e[1] * h + e[2], 2 * e[1] + 0 * h][order], v)


def twin_path(t, xc, yc, max_s, start, goal, ds_small, ds_large, dynamic, search_ds, max_n=BIG):
    """(ok, states [n, 5], x0) of one path, by another route than the oracle."""
    sx, sy, sz, sk = (float(start[f]) for f in "xyzk")
    gx, gy = float(goal["x"]), float(goal["y"])
    x1, y1 = _ev(t, xc, 0.0, 1)[0], _ev(t, yc, 0.0, 1)[0]
    fx, fy, fz = _ev(t, xc, 0.0, 0)[0], _ev(t, yc, 0.0, 0)[0], np.arctan2(y1, x1)
    cross = np.cos(sz) * (fy - sy) - np.sin(sz) * (fx - sx)
    off = np.hypot(sx - fx, sy - fy) * (1 if cross < 0 else -1)
    herr = (sz - fz + np.pi) % (2 * np.pi) - np.pi
    x0 = (off, herr, sk)
    if abs(herr) > math.radians(75) or not max_s > 0 or not np.isfinite(max_s):
        return False, np.zeros((0, 5)), x0
    L = max_s
    end = np.hypot(gx - _ev(t, xc, L, 0)[0], gy - _ev(t, yc, L, 0)[0])
    if end >= 1e-6:
        m = int(L / search_ds) + 2
        lat = np.subtract.accumulate(np.concatenate([[L], np.full(m, search_ds)]))[1:]
        lat = lat[lat > 0]
        d = np.hypot(_ev(t, xc, lat, 0) - gx, _ev(t, yc, lat, 0) - gy)
        run = np.minimum.accumulate(np.concatenate([[end], d]))[1:]
        stop = np.flatnonzero((d > 8) & (run < 8))
        last = stop[0] if len(stop) else len(d) - 1
        cand = np.concatenate([[end], d[:last + 1]])
        i = int(np.argmin(cand))
        L = max_s if i == 0 else float(lat[i - 1])
    rows, s = [], 0.0
    while s <= L:
        if len(rows) == max_n:
            return False, np.zeros((0, 5)), x0
        d1x, d1y, d2x, d2y = (_ev(t, c, s, o)[0] for c, o in ((xc, 1), (yc, 1), (xc, 2), (yc, 2)))
        k = (d1x * d2y - d1y * d2x) / np.power(d1x * d1x + d1y * d1y, 1.5)
        rows.append((_ev(t, xc, s, 0)[0], _ev(t, yc, s, 0)[0], np.arctan2(d1y, d1x), k, s))
        share = 0.0 if not dynamic else float(np.clip((abs(k) - 0.08) / 0.12, 0.0, 1.0))
        s = s + (ds_large - share * (ds_large - ds_small))
    return True, np.array(rows), x0


def _cases():
    return [("main", sc.main_batch()), ("lengths", sc.length_batch())]


@pytest.fixture(scope="module", params=list(sc.FLAGS))
def flags(request):
    return request.param


@pytest.mark.parametrize("which", ["main", "lengths"])
def test_oracle_against_numpy_twin(which, flags):
    b = dict(_cases())[which]
    kw = sc.flag_kw(flags)
    o = oseg.segment_batch(b["splines"], b["max_s"], b["start"], b["goal"], BIG, **kw)
    sp, ko = b["splines"], b["splines"]["knot_offsets"]
    checked = dropped = 0
    for i, name in enumerate(b["names"]):
        sl = slice(ko[i], ko[i + 1])
        if o["reason"][i] == oseg.SEG_BAD_SPLINE:
            continue       # the twin does not restate the guards against unusable splines and starts
        if o["margin"][i] < NEAR:
            dropped += 1
            continue
        if not b["max_s"][i] <= kw["search_ds"] * oseg.MAX_SEARCH:     # too long to search (or NaN): the guard
            assert o["reason"][i] == oseg.SEG_BAD_LENGTH, name
            continue
        ok, rows, x0 = twin_path(sp["knots"][sl], sp["x_coef"][sl], sp["y_coef"][sl], b["max_s"][i], b["start"][i],
                                 b["goal"][i], **kw)
        assert bool(o["ok"][i]) == ok, name
        assert np.allclose(o["x0"][i], x0, rtol=0, atol=1e-12), name
        assert o["n_points"][i] == len(rows), name
        if ok:
            got = o["ref"][o["offsets"][i]:o["offsets"][i + 1], :5]
            assert np.allclose(got, rows, rtol=0, atol=1e-9), (name, np.abs(got - rows).max())
            assert (o["ref"][o["offsets"][i]:o["offsets"][i + 1], 5:] == 0).all()
        checked += 1
    assert dropped <= len(b["names"]) // 10 and checked >= min(len(b["names"]) // 2, 6), (checked, dropped)


def test_cases_cover_the_issue(flags):
    """Curvature crossing 0.08 and 0.2, both signs of the initial offset, both sides of 75 degrees, goal cuts and full
    lengths all occur."""
    b = sc.main_batch()
    o = oseg.segment_batch(b["splines"], b["max_s"], b["start"], b["goal"], BIG, **sc.flag_kw(flags))
    k = np.abs(o["ref"][:, 3])
    assert (k < 0.08).any() and ((k > 0.08) & (k < 0.2)).any() and (k > 0.2).any()
    assert (o["x0"][o["ok"] == 1, 0] > 0.5).any() and (o["x0"][o["ok"] == 1, 0] < -0.5).any()
    assert (o["reason"] == oseg.SEG_HEADING).sum() >= 3 * 4
    kept = o["ok"] == 1
    assert (o["cut_s"][kept] < b["max_s"][kept]).any() and (o["cut_s"][kept] == b["max_s"][kept]).any()


# ---- the kernel source under g++ -------------------------------------------------------------------------------------

def _same_as_oracle(e, o):
    assert np.array_equal(e["reason"], o["reason"])
    assert np.array_equal(e["ok"], o["ok"]) and np.array_equal(e["n_points"], o["n_points"])
    assert np.array_equal(e["offsets"], o["offsets"])
    assert np.ascontiguousarray(e["ref"]).view(np.float64).tobytes() == np.ascontiguousarray(o["ref"]).tobytes()
    assert e["x0"].tobytes() == o["x0"].tobytes() and e["end_heading"].tobytes() == o["end_heading"].tobytes()
    assert e["cut_s"].tobytes() == o["cut_s"].tobytes()


@pytest.mark.parametrize("which", ["main", "lengths"])
def test_emulated_kernel_equals_oracle(which, flags):
    b = dict(_cases())[which]
    kw = sc.flag_kw(flags)
    o = oseg.segment_batch(b["splines"], b["max_s"], b["start"], b["goal"], BIG, **kw)
    e = segment_emu.segment(b["splines"], b["max_s"], b["start"], b["goal"], BIG, **kw)
    _same_as_oracle(e, o)


def test_config1_line():
    """The config-1 benchmark polyline, start and goal: kept, and the kernel source equals the oracle."""
    c = sc.config1()
    b = sc.batch_of([("config1", c["spl"], float(c["spl"][0][-1]), c["start"], c["goal"])])
    o = oseg.segment_batch(b["splines"], b["max_s"], b["start"], b["goal"], BIG)
    _same_as_oracle(segment_emu.segment(b["splines"], b["max_s"], b["start"], b["goal"], BIG), o)
    assert o["ok"][0] == 1 and o["n_points"][0] > 100


def test_cap_and_capacity_refusals():
    """The station cap refuses the long paths only; the capacity refuses the first path whose stations pass it and
    every later one with stations, and the kept paths' states equal those of the uncapped run."""
    b = sc.main_batch()
    free = oseg.segment_batch(b["splines"], b["max_s"], b["start"], b["goal"], BIG)
    n = free["n_points"]
    cap = int(np.median(n[n > 0]))
    for max_n, capacity in ((cap, BIG), (BIG, int(n.sum()) // 2), (cap, int(n.sum()) // 3), (BIG, 0)):
        o = oseg.segment_batch(b["splines"], b["max_s"], b["start"], b["goal"], capacity, max_n=max_n)
        e = segment_emu.segment(b["splines"], b["max_s"], b["start"], b["goal"], capacity, max_n=max_n)
        _same_as_oracle(e, o)
        counts = np.where(n <= max_n, n, 0)
        assert np.array_equal(o["reason"] == oseg.SEG_TOO_MANY, n > max_n)
        before = np.concatenate([[0], np.cumsum(counts)[:-1]])
        want_cap = (counts > 0) & (before + counts > capacity)
        assert np.array_equal(o["reason"] == oseg.SEG_CAPACITY, want_cap)
        assert o["offsets"][-1] <= capacity
        for i in np.flatnonzero(o["ok"]):
            got = o["ref"][o["offsets"][i]:o["offsets"][i + 1]]
            assert got.tobytes() == free["ref"][free["offsets"][i]:free["offsets"][i + 1]].tobytes()
        if capacity < n.sum():
            first = np.flatnonzero(want_cap)[0]
            assert not o["ok"][first:].any()


def test_refusals_leave_other_paths_alone():
    """Refused paths interleaved with kept ones: the kept paths' states, x0 and counts equal those of the batch without
    the refused ones."""
    b, lb = sc.main_batch(), sc.length_batch()
    o_l = oseg.segment_batch(lb["splines"], lb["max_s"], lb["start"], lb["goal"], BIG)
    bad = np.flatnonzero(o_l["ok"] == 0)
    good = list(range(0, len(b["names"]), 7))
    ko, lko = b["splines"]["knot_offsets"], lb["splines"]["knot_offsets"]

    def path(src, k, i):
        sp = src["splines"]
        sl = slice(k[i], k[i + 1])
        return (src["names"][i], (sp["knots"][sl], sp["x_coef"][sl], sp["y_coef"][sl]), src["max_s"][i],
                src["start"][i], src["goal"][i])
    mixed, is_bad = [], []
    for j in range(max(len(good), len(bad))):
        if j < len(good):
            mixed.append(path(b, ko, good[j])); is_bad.append(False)
        if j < len(bad):
            mixed.append(path(lb, lko, bad[j])); is_bad.append(True)
    mb = sc.batch_of(mixed)
    gb = sc.batch_of([path(b, ko, i) for i in good])
    e = segment_emu.segment(mb["splines"], mb["max_s"], mb["start"], mb["goal"], BIG)
    g = segment_emu.segment(gb["splines"], gb["max_s"], gb["start"], gb["goal"], BIG)
    is_bad = np.array(is_bad)
    assert not e["ok"][is_bad].any() and (e["n_points"][is_bad] == 0).all()
    keep = np.flatnonzero(~is_bad)
    assert np.array_equal(e["n_points"][keep], g["n_points"])
    assert e["ref"].tobytes() == g["ref"].tobytes()
    assert e["x0"][keep].tobytes() == g["x0"].tobytes()
