"""GPU shape sweep (run with -m gpu on an H100): every path length of every kernel class, and the verdict paths of every
class, against the oracle.

The solver picks a kernel class per path from (formulation, N, keep_control_steps), and inside a class the partition
(separator spacing and count, length of the last interior, held-control count, where the long classes overlay their
end rows and held controls) changes with every N.  So the sweeps run one path per length, from 2 stations to the longest
path of the keep value, plus one station more (PQP_INVALID_PROBLEM for that path only).  Each path is held to the oracle
like the rest of the suite: identical status and iteration count, 1e-8 on the Frenet and Cartesian states (1e-6 for
runs past 1000 iterations, see shapes.TOL).  The class of every path is recorded, and each sweep asserts that it ran
both ends of every class the library selects at its keep values; test_classes.py asserts that the sweeps together
reach every class."""
import os

import numpy as np
import pytest

from oracle import oracle
from path_optimizer_b200 import _lib, synth
from path_optimizer_b200.abi import STATE_DTYPE
from tests import shapes
from tests.device_entries import device_classes as _device

pytestmark = pytest.mark.gpu
THREADS = max(1, min(16, os.cpu_count() or 1))
INVALID = -100


@pytest.fixture(scope="module")
def solver():
    from path_optimizer_b200.solver import BatchPathSolver
    s = BatchPathSolver(max_batch=512, max_total_points=100_000)
    yield s
    s.close()


def _concat(batches):
    out = {k: np.concatenate([b[k] for b in batches]) for k in ("n_points", "ref", "bounds", "x0", "end_heading")}
    out["offsets"] = np.zeros(len(out["n_points"]) + 1, dtype=np.int32)
    np.cumsum(out["n_points"], out=out["offsets"][1:])
    return out


def _respace(b, ds):
    """Stations every ds metres, accumulated in double as a resampler makes them."""
    o = b["offsets"]
    for i, n in enumerate(b["n_points"]):
        b["ref"]["s"][o[i]:o[i + 1]] = synth._accumulate_s(int(n), ds)
    return b


def _kpc_limits(b):
    """KPC limits from a speed profile with standstill stations (DBL_MAX limits: rows free on that side)."""
    total = int(b["offsets"][-1])
    b["ref"]["v"] = 4.0 + 3.0 * np.sin(np.arange(total) * 0.05)
    b["ref"]["a"] = 0.5 * np.cos(np.arange(total) * 0.05)
    b["ref"]["v"][::13] = 0.0
    return oracle.update_limits(oracle.default_params(), b["ref"])


def _keeps(form, b):
    o = b["offsets"]
    return np.array([shapes.keep_of(form, b["ref"][o[i]:o[i + 1]]) for i in range(len(b["n_points"]))], dtype=np.int32)


def _rows(b, idx):
    o = b["offsets"]
    return np.concatenate([np.arange(o[i], o[i + 1]) for i in idx])


def _assert_invalid(res, b, idx):
    for i in idx:
        sl = slice(b["offsets"][i], b["offsets"][i + 1])
        assert res["status"][i] == INVALID and res["iters"][i] == 0, (i, res["status"][i])
        assert np.isnan(res["frenet"][sl]).all()
        for f in "xyzk":     # (s: the oracle, like the reference, keeps s = 0 at station 0 of a refused corridor)
            assert np.isnan(res["states"][f][sl]).all()


def _bit_identical(a, b):
    assert np.array_equal(a["status"], b["status"]) and np.array_equal(a["iters"], b["iters"])
    assert a["frenet"].tobytes() == b["frenet"].tobytes()
    assert a["states"].tobytes() == b["states"].tobytes()


def _sweep(s, form, b, mk=None, mkp=None):
    """b holds one path per length 2..max + 1 (the formulation's longest path at the keep value of its stations, and one
    more).  Host-buffer entry against the oracle, coverage of every class at both ends, device-resident entries."""
    name = {shapes.KP: "KP", shapes.K: "K", shapes.KPC: "KPC"}[form]
    L = _lib.load()
    n = b["n_points"]
    keeps = _keeps(form, b)
    main = int(np.bincount(keeps).argmax())
    nmax = L.pqp_max_points_keep(s._h, form, main)
    assert nmax == shapes.max_points(form, main)            # (the device offers the H100's 227 KB per block)
    assert np.array_equal(n, np.arange(2, nmax + 2))
    cls = [shapes.class_of(form, ni, ki) for ni, ki in zip(n, keeps)]
    ok = np.array([c[1] for c in cls])
    assert ok[:-1].all() and not ok[-1]

    # every class the library selects at the keep values of the batch, at both of its ends
    seen = {}
    for ni, ki, (c, good) in zip(n, keeps, cls):
        if good:
            seen.setdefault((c, int(ki)), set()).add(int(ni))
    # (paths of 2..4 stations take keep 4 at 0.3 m and keep 8 at 0.15 m: at those spacings the main keep starts at 5
    # stations; test_gpu_parity.py::test_parameter_sweep runs the 2-station ends at keep 3)
    first = int(n[keeps == main].min())
    lines = []
    for ki in sorted(set(keeps.tolist())):
        for c, (lo, hi) in sorted(shapes.class_ranges(form, ki).items(), key=lambda kv: kv[1]):
            if ki != main and lo > int(n[keeps == ki].max()):
                continue
            got = seen.get((c, ki), set())
            if ki == main:
                assert max(lo, first) in got and hi in got, f"{name} keep {ki}: class {c} ({lo}..{hi}) not swept at both ends"
            lines.append(f"  {name} keep {ki:2d}  {c:40s} N = {lo:3d}..{hi:3d}  swept {len(got)}")
    print("\n" + "\n".join(lines))
    assert {c for (c, ki) in seen if ki == main} == {c for c in shapes.class_ranges(form, main)}

    res = s.solve(b, formulation=form, max_k=mk, max_kp=mkp)
    good = np.nonzero(ok)[0]
    sub = synth.take_paths(b, good)
    rows = _rows(b, good)
    ref = oracle.solve_batch(s.params, form, sub, threads=THREADS,
                             max_k=None if mk is None else mk[rows], max_kp=None if mk is None else mkp[rows])
    shapes.assert_matches(res, ref, good, rows, n[good], f"{name} sweep")
    _assert_invalid(res, b, np.nonzero(~ok)[0])

    # device-resident entries: per-class launches give the same bits; one class for every length up to the longest
    # path of the batch's keep values gives the same verdicts and the oracle's states
    _bit_identical(_device(s, form, b, keeps, mk=mk, mkp=mkp), res)
    dmax = min(L.pqp_max_points_keep(s._h, form, int(k)) for k in set(keeps.tolist()))
    idx = np.nonzero(n <= dmax)[0]
    db = synth.take_paths(b, idx)
    drows = _rows(b, idx)
    dres = _device(s, form, db, keeps[idx], nmax=dmax, mk=None if mk is None else mk[drows],
                   mkp=None if mk is None else mkp[drows])
    assert np.array_equal(dres["status"], res["status"][idx]) and np.array_equal(dres["iters"], res["iters"][idx])
    pos = np.searchsorted(good, idx)
    shapes.assert_matches(dres, dict(status=ref["status"][pos], iters=ref["iters"][pos],
                                     frenet=ref["frenet"][np.searchsorted(rows, drows)],
                                     states=ref["states"][np.searchsorted(rows, drows)]),
                          np.arange(len(idx)), np.arange(len(drows)), n[idx], f"{name} device entry, one class up to {dmax}")


def _kp_keep(ds):
    ref = np.zeros(20, dtype=STATE_DTYPE)
    ref["s"] = synth._accumulate_s(20, ds)
    return shapes.keep_of(shapes.KP, ref)


@pytest.mark.parametrize("ds", shapes.SPACINGS)
def test_kp_every_length_curved(solver, ds):
    """KP, curved corridors: N = 2 .. pqp_max_points_keep + 1 at 0.3 / 0.25 / 0.5 / 1.0 / 0.2 / 0.15 / 0.11 m stations
    (keep_control_steps 3 / 4 / 2 / 1 / 5 / 7 / 10)."""
    nmax = shapes.max_points(shapes.KP, _kp_keep(ds))
    b = _respace(synth.curvy_corridors(nmax, n_points=np.arange(2, nmax + 2)), ds)
    _sweep(solver, shapes.KP, b)


@pytest.mark.parametrize("ds", [0.3, 0.25])
def test_kp_every_length_straight(solver, ds):
    """KP, straight corridors (BASELINE configs 2 and 4): every length at keep 3 and 4."""
    nmax = shapes.max_points(shapes.KP, _kp_keep(ds))
    b = _concat([synth.straight_corridors(1, int(n), first_path=int(n)) for n in range(2, nmax + 2)])
    b["ref"]["x"] = b["ref"]["s"]
    _respace(b, ds)
    b["ref"]["x"] = b["ref"]["s"]
    _sweep(solver, shapes.KP, b)


def test_k_every_length(solver):
    nmax = shapes.max_points(shapes.K, 1)
    assert nmax == 416
    _sweep(solver, shapes.K, synth.curvy_corridors(nmax, n_points=np.arange(2, nmax + 2)))


def test_kpc_every_length(solver):
    nmax = shapes.max_points(shapes.KPC, 4)
    assert nmax == 256
    b = synth.curvy_corridors(nmax, n_points=np.arange(2, nmax + 2))
    mk, mkp = _kpc_limits(b)
    _sweep(solver, shapes.KPC, b, mk, mkp)


# ---- verdicts and bad inputs on every class ------------------------------------------------------------------------
VERDICT_SPACING = {3: 0.3, 4: 0.25, 5: 0.2, 1: 0.3}
KINDS = ("control", "infeasible", "lb>ub station 0", "lb>ub first separator", "lb>ub interior", "lb>ub last station",
         "collapsed row at a separator", "end heading > 70 deg", "x0 on a corridor bound")


def _separator(form, name, n, keep):
    """First separator after station 0 of the class's partition; the middle station for the classes without one."""
    if name.startswith("pqp_kp3_solve_kernel"):
        return shapes.kp3_partition(n, keep, int(name.split(",")[3].rstrip(">KPC")))[0]
    if name in ("pqp_kk_solve_kernel<4>", "pqp_kk_solve_kernel<8>"):
        return shapes.kk_partition(n, 26 if name.endswith("<4>") else 32)[0]
    return n // 2


def _verdict_batch(form, keeps):
    """For every (class, keep) the formulation selects at these keeps: one path of KINDS each, at the top of the class's
    length range."""
    parts, tags = [], []
    for keep in keeps:
        for c, (lo, hi) in sorted(shapes.class_ranges(form, keep).items(), key=lambda kv: kv[1]):
            n = hi
            pid = 1000 * keep + n
            seps = _separator(form, c, n, keep)
            inf = synth.infeasible_corridors(6, n, first_path=pid)
            for kind in KINDS:
                if kind == "infeasible":
                    # two kinds of infeasibility by turns; KPC's front circle row (c2) is soft: the first kind only
                    p = synth.take_paths(inf, [4 if len(tags) % 2 and form != shapes.KPC else 0])
                else:
                    p = synth.curvy_corridors(1, n, first_path=pid)
                bb = p["bounds"]
                pos = {"lb>ub station 0": 0, "lb>ub first separator": seps, "lb>ub interior": seps + 1,
                       "lb>ub last station": n - 1}.get(kind)
                if pos is not None:
                    bb["c0_lb"][pos] = bb["c0_ub"][pos] + 0.5
                elif kind == "collapsed row at a separator":
                    bb["c2_lb"][seps] = bb["c2_ub"][seps] = np.round(0.5 * (bb["c2_lb"][seps] + bb["c2_ub"][seps]), 1)
                elif kind == "end heading > 70 deg":
                    p["end_heading"][0] = p["ref"]["z"][n - 1] + 1.4
                elif kind == "x0 on a corridor bound":
                    p["x0"][0] = [bb["c0_ub"][0], 0.0, p["ref"]["k"][0]]
                parts.append(_respace(p, VERDICT_SPACING[keep]) if form == shapes.KP else p)
                tags.append((c, keep, n, kind))
    return _concat(parts), tags


@pytest.mark.parametrize("form", [shapes.KP, shapes.K, shapes.KPC], ids=["KP", "K", "KPC"])
def test_verdicts_on_every_class(solver, form):
    """Per class, at the top of its length range: primal infeasibility (status -3 at the oracle's iteration), an invalid
    corridor (lb > ub) at station 0 / the first separator / an interior station / the last station (-100, all-NaN output),
    a collapsed corridor row at a separator, a free end-heading row, a start on a corridor bound, and the same batch
    capped at 75 iterations.  Every path against the oracle; the well-posed paths come back bit-identical when solved
    without the invalid ones."""
    from path_optimizer_b200.solver import BatchPathSolver
    keeps = {shapes.KP: (3, 4, 5), shapes.K: (1,), shapes.KPC: (4,)}[form]
    b, tags = _verdict_batch(form, keeps)
    assert {(c, k) for c, k, _, _ in tags} == {(c, k) for k in keeps for c in shapes.class_ranges(form, k)}
    assert set(_keeps(form, b).tolist()) == set(keeps)
    mk = mkp = None
    if form == shapes.KPC:
        mk, mkp = _kpc_limits(b)
    kinds = np.array([t[3] for t in tags])
    bad = np.nonzero(np.char.startswith(kinds, "lb>ub"))[0]
    wellposed = np.nonzero(~np.char.startswith(kinds, "lb>ub"))[0]
    res = solver.solve(b, formulation=form, max_k=mk, max_kp=mkp)
    ref = oracle.solve_batch(solver.params, form, b, threads=THREADS, max_k=mk, max_kp=mkp)
    # (KPC's soft circle and curvature rows leave ADMM without a certificate within max_iter: status -2, as in the oracle)
    assert (ref["status"][kinds == "infeasible"] == (-2 if form == shapes.KPC else -3)).all()
    assert (ref["status"][bad] == INVALID).all()
    shapes.assert_matches(res, ref, np.arange(len(tags)), np.arange(int(b["offsets"][-1])), b["n_points"], "verdict batch")
    _assert_invalid(res, b, bad)
    # the well-posed paths alone: bit for bit what they gave beside the invalid ones
    rows = _rows(b, wellposed)
    alone = solver.solve(synth.take_paths(b, wellposed), formulation=form,
                         max_k=None if mk is None else mk[rows], max_kp=None if mk is None else mkp[rows])
    _bit_identical(alone, dict(status=res["status"][wellposed], iters=res["iters"][wellposed],
                               frenet=res["frenet"][rows], states=res["states"][rows]))
    # capped at 75, 2 and 1 iterations: same verdict and the same iterate as the oracle.  At max_iter 1 the verdict comes
    # from the residuals of OSQP's first iteration, which ends at x = 0 with z = clamp(0) and y = -rho clamp(0): the x0
    # rows (and any row whose bounds exclude 0) leave a primal residual, so no control path passes as solved.
    for cap in (75, 2, 1):
        p = oracle.default_params()
        p.max_iter = cap
        capped = BatchPathSolver(params=p, max_batch=len(tags), max_total_points=int(b["offsets"][-1]))
        try:
            rc = capped.solve(b, formulation=form, max_k=mk, max_kp=mkp)
        finally:
            capped.close()
        rr = oracle.solve_batch(p, form, b, threads=THREADS, max_k=mk, max_kp=mkp)
        assert (rr["iters"][wellposed] <= cap).all() and (rr["iters"][kinds == "control"] == cap).any()
        if cap <= 2:
            assert (rr["status"][kinds == "control"] == -2).all()
        shapes.assert_matches(rc, rr, np.arange(len(tags)), np.arange(int(b["offsets"][-1])), b["n_points"], f"max_iter {cap}")
