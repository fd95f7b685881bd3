"""CPU tests of the batched reference-spline fit (pqp_fit_splines_device) through its kernel source: the per-thread
functions of csrc/pqp_env_core.cuh compiled with g++ (tests/emu/fit_emu.cpp) in the kernel's order and scratch layout.

Every fitted path's knots and coefficient rows equal pqp_spline_fit's bit for bit, and its values and first and second
derivatives at the knots and interval midpoints agree with scipy's natural cubic spline; refused paths (fewer than 3
stations, an s that is not finite and strictly increasing) get ok = 0 and NaN rows and change no other path.  Lines:
tests/fit_lines.py."""
import numpy as np
import pytest
from scipy.interpolate import CubicSpline

from path_optimizer_b200 import planner
from path_optimizer_b200.solver import PqpError
from tests import fit_lines
from tests.emu import fit_emu

REL = 1e-9


def _u64(a):
    return np.ascontiguousarray(a).view(np.uint64)


def _host_rows(r):
    return planner.spline_fit(r["s"], r["x"]), planner.spline_fit(r["s"], r["y"])


@pytest.fixture(scope="module")
def good():
    lines = fit_lines.good_lines()
    b = fit_lines.batch_of(list(lines.values()))
    return list(lines), b, fit_emu.fit_splines(b["offsets"], b["ref"])


def test_rows_equal_host_fit_bit_for_bit(good):
    names, b, got = good
    assert got["ok"].all()
    o = b["offsets"]
    assert _u64(got["knots"]).tobytes() == _u64(b["ref"]["s"]).tobytes()
    for i, name in enumerate(names):
        r = b["ref"][o[i]:o[i + 1]]
        hx, hy = _host_rows(r)
        assert _u64(got["x_coef"][o[i]:o[i + 1]]).tobytes() == _u64(hx).tobytes(), name
        assert _u64(got["y_coef"][o[i]:o[i + 1]]).tobytes() == _u64(hy).tobytes(), name


def _eval(t, c, at, order):
    idx = np.clip(np.searchsorted(t, at, side="left") - 1, 0, len(t) - 1)
    h = at - t[idx]
    a, bb, cc, y = (c[idx, k] for k in range(4))
    if order == 0:
        return ((a * h + bb) * h + cc) * h + y
    if order == 1:
        return (3 * a * h + 2 * bb) * h + cc
    return 6 * a * h + 2 * bb


def test_values_and_derivatives_match_scipy(good):
    names, b, got = good
    o = b["offsets"]
    for i, name in enumerate(names):
        sl = slice(o[i], o[i + 1])
        t = got["knots"][sl]
        at = np.concatenate([t, 0.5 * (t[1:] + t[:-1])])
        for coord, coef in (("x", got["x_coef"][sl]), ("y", got["y_coef"][sl])):
            ref = CubicSpline(t, b["ref"][coord][sl], bc_type="natural")
            for order in range(3):
                want = ref(at, order)
                have = _eval(t, coef, at, order)
                scale = max(np.abs(want).max(), np.abs(ref(at, 0)).max() / max(t[-1] - t[0], 1e-300) ** order)
                err = np.abs(have - want).max()
                assert err <= REL * scale, (name, coord, order, err, scale)


@pytest.fixture(scope="module")
def refused():
    return fit_lines.refused_lines()


def test_refused_paths_get_nan_rows_and_change_nothing_else(good, refused):
    """Every refused line between good ones: ok = 0 and NaN knots and rows for it, and the good lines' rows equal those
    of the batch without it."""
    _, gb, gwant = good
    gref = [gb["ref"][gb["offsets"][i]:gb["offsets"][i + 1]] for i in range(len(gb["n_points"]))]
    bad = [r for r, _ in refused.values()]
    # good, bad, good, bad, ... then the rest of the good lines
    order, refs = [], []
    for k in range(max(len(gref), len(bad))):
        if k < len(gref):
            order.append(("good", k)); refs.append(gref[k])
        if k < len(bad):
            order.append(("bad", k)); refs.append(bad[k])
    b = fit_lines.batch_of(refs)
    got = fit_emu.fit_splines(b["offsets"], b["ref"])
    o, go = b["offsets"], gb["offsets"]
    names = list(refused)
    for j, (kind, k) in enumerate(order):
        sl = slice(o[j], o[j + 1])
        if kind == "bad":
            assert got["ok"][j] == 0, names[k]
            assert np.isnan(got["knots"][sl]).all() and np.isnan(got["x_coef"][sl]).all() and np.isnan(got["y_coef"][sl]).all()
        else:
            assert got["ok"][j] == 1
            gs = slice(go[k], go[k + 1])
            for f in ("knots", "x_coef", "y_coef"):
                assert _u64(got[f][sl]).tobytes() == _u64(gwant[f][gs]).tobytes(), (f, k)


def test_refusal_rule_against_host_fit(refused):
    """pqp_spline_fit refuses the same lines, except one whose first or last knot is infinite: it tests only that every
    interval is positive, so it accepts that line and returns non-finite rows."""
    for name, (r, host_accepts) in refused.items():
        b = fit_lines.batch_of([r])
        assert fit_emu.fit_splines(b["offsets"], b["ref"])["ok"][0] == 0, name
        if host_accepts:
            hx, hy = _host_rows(r)
            assert not (np.isfinite(hx).all() and np.isfinite(hy).all()), name
        else:
            with pytest.raises(PqpError):
                _host_rows(r)
    assert any(a for _, a in refused.values())
