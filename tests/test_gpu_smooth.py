"""GPU tests (run with -m gpu on an H100) of the reference smoothing stage, pqp_smooth_reference_device
(PathPlanner.smooth_device): the device stage against the CPU restatement (oracle/smooth.py) on the named polylines of
tests/smooth_cases.py, isolated refusals, the capacity reservation across warp tiles, argument errors, and the whole of
PathOptimizer::solve from raw polylines -- smooth -> post-smooth -> segment -> fit -> plan -- in one CUDA graph."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import smooth as S
from path_optimizer_b200 import device, planner
from path_optimizer_b200.abi import ERR_ARG, ERR_CAPACITY
from tests import segment_cases, smooth_cases as sc

pytestmark = pytest.mark.gpu
NEAR = 1e-9
CAP = 16384
MAX_RAW, MAX_PTS = 400, 200
# Far from the origin the knots are not compared, only ok, status and iterations: the QP iterates on absolute coordinates
# and OSQP's stopping rule is relative to them (eps_rel |z|: 5e3 m at UTM northings, 1e4 m at 1e7 m), so the device and
# the restatement, equal in status and iterations, stop at points inside that tolerance that differ by far more than
# rounding (tests/test_smooth_emu.py meets the same between two CPU builds).
FAR = 1e5


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


@pytest.fixture(scope="module")
def pl():
    p = planner.PathPlanner(max_batch=256, max_total_points=CAP)
    p.set_maps([segment_cases.config1()["field"]])
    yield p
    p.close()


def _run(p, pts, off, capacity=CAP, **kw):
    import torch
    r = p.smooth_device(_t(pts), _t(off), MAX_RAW, MAX_PTS, capacity=capacity, **kw)
    torch.cuda.synchronize()
    return {k: _np(v) for k, v in r.items()}


def _compare(got, want, names, pts, off):
    """ok exact, status and iterations equal; within FAR of the origin, knots, max_s and every coefficient column within
    1e-8 of that column's magnitude.  Paths whose QP decisions came within NEAR of a threshold are dropped and
    counted."""
    dropped = 0
    ko_g, ko_w = got["knot_offsets"], want["knot_offsets"]
    for b, name in enumerate(names):
        if want["qp_margin"][b] < NEAR:
            dropped += 1
            continue
        assert got["ok"][b] == want["ok"][b], name
        assert (got["status"][b], got["iters"][b]) == (want["status"][b], want["iters"][b]), name
        if not want["ok"][b]:
            assert ko_g[b + 1] == ko_g[b] and np.isnan(got["max_s"][b]), name
            continue
        if np.nanmax(np.abs(pts[off[b]:off[b + 1], :2])) > FAR:
            continue
        g, w = slice(ko_g[b], ko_g[b + 1]), slice(ko_w[b], ko_w[b + 1])
        for k in ("knots", "x_coef", "y_coef"):
            a, e = got[k][g].reshape(len(got[k][g]), -1), want[k][w].reshape(len(want[k][w]), -1)
            scale = np.maximum(1.0, np.max(np.abs(e), axis=0))            # per column: a, b, c, y of the spline rows
            assert np.all(np.max(np.abs(a - e), axis=0) <= 1e-8 * scale), (name, k)
        assert abs(got["max_s"][b] - want["max_s"][b]) <= 1e-8 * max(1.0, abs(want["max_s"][b])), name
    return dropped


def test_device_equals_oracle(pl):
    names, pts, off = sc.batch()
    got = _run(pl, pts, off)
    want = S.smooth_batch(pts, off, O.default_params(), CAP, MAX_RAW, MAX_PTS)
    assert np.array_equal(got["knot_offsets"][:1], [0])
    dropped = _compare(got, want, names, pts, off)
    assert dropped <= 2
    ok = dict(zip(names, got["ok"]))
    assert ok["config1"] == ok["straight_x"] == ok["u_turn"] == ok["corner"] == ok["six_close"] == 1
    assert ok["four_close"] == ok["five_close"] == ok["three"] == ok["nan"] == ok["tiny"] == ok["short"] == 0
    assert all(ok[f"pose{k}"] == 1 for k in range(24))
    refused = [b for b, n in enumerate(names) if n in ("four_close", "five_close", "three", "nan", "tiny", "short")]
    assert all(got["status"][b] == -100 and got["iters"][b] == 0 for b in refused)


@pytest.mark.parametrize("caps", [dict(max_raw_samples=20), dict(max_points=20)])
def test_sample_and_station_caps(pl, caps):
    """More B-spline samples than max_raw_samples, or more stations than max_points: refused, as in the restatement."""
    import torch
    names, pts, off = sc.batch(["corner", "config1", "straight_x"])
    args = dict(max_raw_samples=MAX_RAW, max_points=MAX_PTS)
    args.update(caps)
    r = pl.smooth_device(_t(pts), _t(off), capacity=CAP, **args)
    torch.cuda.synchronize()
    want = S.smooth_batch(pts, off, O.default_params(), CAP, args["max_raw_samples"], args["max_points"])
    assert list(_np(r["ok"])) == list(want["ok"])
    assert want["ok"][1] == 0 and want["reason"][1] == (S.SM_RAW_MANY if "max_raw_samples" in caps else S.SM_MANY)
    assert _np(r["status"])[1] == -100 and _np(r["iters"])[1] == 0


def test_refusals_are_isolated(pl):
    names, pts, off = sc.batch(["config1", "corner", "u_turn"])
    alone = _run(pl, pts, off)
    names2, pts2, off2 = sc.batch(["nan", "config1", "four_close", "corner", "three", "u_turn", "five_close"])
    mixed = _run(pl, pts2, off2)
    assert list(mixed["ok"]) == [0, 1, 0, 1, 0, 1, 0]
    ka, km = alone["knot_offsets"], mixed["knot_offsets"]
    for a, m in ((0, 1), (1, 3), (2, 5)):
        for k in ("knots", "x_coef", "y_coef"):
            assert alone[k][ka[a]:ka[a + 1]].tobytes() == mixed[k][km[m]:km[m + 1]].tobytes()
        assert alone["iters"][a] == mixed["iters"][m]


def test_capacity_reservation(pl):
    base = ["config1", "corner", "u_turn", "four_close", "straight_x"]
    names = [base[i % len(base)] for i in range(70)]      # three warp tiles of the reservation
    _, pts, off = sc.batch(names)
    full = _run(pl, pts, off)
    counts = np.diff(full["knot_offsets"])
    total = np.concatenate([[0], np.cumsum(counts)])
    for end in (31, 32, 33, 64, 65):
        cap = int(total[end])
        got = _run(pl, pts, off, capacity=cap)
        want_ok = np.array([full["ok"][b] if total[b + 1] <= cap else 0 for b in range(70)])
        assert np.array_equal(got["ok"], want_ok), end
        k = int(got["knot_offsets"][-1])
        assert k <= cap and got["knots"][:k].tobytes() == full["knots"][:k].tobytes()
        assert np.all(np.isnan(got["max_s"][want_ok == 0]))


def test_bad_arguments(pl):
    import torch
    names, pts, off = sc.batch(["config1"])
    P, O_ = _t(pts), _t(off)
    for kw, rc in ((dict(max_raw_samples=2), ERR_ARG), (dict(max_points=2), ERR_ARG),
                   (dict(weights=(-1.0, 1.0, 10.0)), ERR_ARG), (dict(weights=(0.005, np.nan, 10.0)), ERR_ARG),
                   (dict(max_points=600), ERR_CAPACITY), (dict(capacity=CAP + 1), ERR_CAPACITY)):
        args = dict(max_raw_samples=MAX_RAW, max_points=MAX_PTS)
        args.update(kw)
        with pytest.raises(planner.PqpError, match=f"rc={rc}"):
            pl.smooth_device(P, O_, **args)
    # an empty batch writes offsets[0] = 0, and is fine without the array
    ko = torch.full((1,), 7, dtype=torch.int32, device=_dev())
    r = pl.smooth_device(P[:0], O_[:1], MAX_RAW, MAX_PTS, out=dict(knot_offsets=ko))
    torch.cuda.synchronize()
    assert int(r["knot_offsets"][0]) == 0
    rc = pl._L.pqp_smooth_reference_device(pl._h, 0, None, None, 0.005, 1.0, 10.0, MAX_RAW, MAX_PTS, CAP,
                                           *([None] * 8), None)
    assert rc == 0
    torch.cuda.synchronize()


def _chain_inputs(k):
    c = segment_cases.config1()
    names, pts, off = sc.batch(["config1"] * k)
    st = np.array([c["start"]] * k)
    gl = np.array([c["goal"]] * k)
    return pts, off, st, gl


def test_plan_on_smoothed_lines_equals_host_plan(pl):
    """smooth -> post-smooth -> segment -> plan_device equals pqp_plan_batch on host copies of the segmented states."""
    import torch
    pts, off, st, gl = _chain_inputs(4)
    sm = pl.smooth_device(_t(pts), _t(off), MAX_RAW, MAX_PTS)
    ps = pl.post_smooth_device(sm, sm["max_s"], _t(st), MAX_PTS)
    sg = pl.segment_device(ps, ps["max_s"], _t(st), _t(gl), 400)
    got = pl.plan_device(sg["n_points"], sg["offsets"], sg["ref"], sg["x0"], sg["end_heading"], max_n_points=400)
    torch.cuda.synchronize()
    assert _np(sm["ok"]).all() and _np(ps["ok"]).all() and _np(sg["ok"]).all()
    off_s = _np(sg["offsets"])
    hb = dict(n_points=_np(sg["n_points"]), offsets=off_s, ref=device.tensor_to_records(sg["ref"])[:off_s[-1]].copy(),
              x0=_np(sg["x0"]), end_heading=_np(sg["end_heading"]))
    want = pl.plan(hb)
    assert _bits(got, off_s) == _bits(want, off_s, host=True)
    assert (np.asarray(want["status"]) == 1).all()


def _bits(res, offsets, host=False):
    st = res["states"] if host else device.tensor_to_records(res["states"].reshape(-1, 7))
    g = (lambda k: res[k]) if host else (lambda k: _np(res[k]))   # noqa: E731
    return [(int(g("status")[i]), int(g("iters")[i]), int(g("n_out")[i]), int(g("ok")[i]),
             st[offsets[i]:offsets[i + 1]].tobytes()) for i in range(len(offsets) - 1)]


def test_graph_replay_equals_eager(pl):
    """smooth -> post-smooth -> segment -> fit -> plan_device, the whole of PathOptimizer::solve from raw polylines,
    captured in one CUDA graph; new points written into the captured tensor, a replay equals an eager run."""
    import torch
    pts, off, st0, gl0 = _chain_inputs(8)
    P, Of, st, gl = _t(pts), _t(off), _t(st0), _t(gl0)

    def cycle(o_sm=None, o_ps=None, o_sg=None, o_ft=None, o_pr=None):
        sm = pl.smooth_device(P, Of, MAX_RAW, MAX_PTS, out=o_sm)
        ps = pl.post_smooth_device(sm, sm["max_s"], st, MAX_PTS, out=o_ps)
        sg = pl.segment_device(ps, ps["max_s"], st, gl, 400, out=o_sg)
        ft = pl.fit_splines_device(sg["offsets"], sg["ref"], out=o_ft)
        idx = torch.where((sm["ok"] != 0) & (ps["ok"] != 0) & (sg["ok"] != 0) & (ft["ok"] != 0),
                          torch.zeros_like(sm["ok"]), torch.full_like(sm["ok"], -1))
        pr = pl.plan_device(sg["n_points"], sg["offsets"], sg["ref"], sg["x0"], sg["end_heading"], max_n_points=400,
                            bounds_mode=planner.BOUNDS_IMPROVED, splines=ft, map_index=idx, out=o_pr)
        return sm, ps, sg, ft, pr
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        outs = cycle()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cycle(*outs)
    rng = np.random.default_rng(11)
    p1 = pts.copy()
    p1[:, 1] += rng.uniform(-0.2, 0.2, len(p1))
    P.copy_(_t(p1))
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    got = [{k: _np(v).copy() for k, v in r.items() if v is not None} for r in outs]
    with torch.cuda.stream(stream):
        outs2 = cycle()
    torch.cuda.synchronize()
    want = [{k: _np(v) for k, v in r.items() if v is not None} for r in outs2]
    assert want[0]["ok"].all() and (want[4]["status"] == 1).sum() >= 4
    for gr, wr in zip(got, want):
        for k in gr:
            a, b = gr[k], wr[k]
            if k in ("knots", "x_coef", "y_coef") and "knot_offsets" in gr:
                a, b = a[:int(gr["knot_offsets"][-1])], b[:int(gr["knot_offsets"][-1])]
            elif k in ("knots", "x_coef", "y_coef", "ref") and "offsets" in gr:
                a, b = a[:int(gr["offsets"][-1])], b[:int(gr["offsets"][-1])]
            elif k in ("knots", "x_coef", "y_coef") and "offsets" not in gr:
                continue
            assert a.tobytes() == b.tobytes(), k
    del g
