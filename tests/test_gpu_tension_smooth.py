"""GPU tests (run with -m gpu on an H100) of the TENSION smoothing stage, pqp_smooth_reference_tension_device
(PathPlanner.smooth_device(method="TENSION")): the device stage against the CPU restatement
(tests/tension_restatement.py) on the named polylines of tests/smooth_cases.py, on the config-1 map and on that map
turned and shifted to the quarter-turn poses of tests/poses.py; per-path map indices on a two-map set against
single-map runs; isolated refusals; the station cap and the capacity reservation; argument errors and the empty batch;
and smooth(TENSION) -> post-smooth -> segment -> fit -> plan in one CUDA graph, and the plan on its output against
pqp_plan_batch."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import smooth as S
from path_optimizer_b200 import device, planner
from path_optimizer_b200.abi import ERR_ARG, ERR_CAPACITY
from tests import segment_cases, tension_cases as tc
from tests import tension_restatement as T
from tests.test_gpu_smooth import _bits, _compare, _dev, _np, _t

pytestmark = pytest.mark.gpu
CAP = 16384
MAX_RAW, MAX_PTS = 400, 200
MAX_STATIONS = 277          # the largest max_points whose TENSION QP fits one H100 SM (57 N + 13 248 doubles)
REFUSED = ("four_close", "five_close", "three", "nan", "tiny", "short")


@pytest.fixture(scope="module")
def pl():
    p = planner.PathPlanner(max_batch=256, max_total_points=CAP)
    yield p
    p.close()


def _run(p, pts, off, capacity=CAP, map_index=None, **kw):
    import torch
    mi = None if map_index is None else _t(np.asarray(map_index, dtype=np.int32))
    r = p.smooth_device(_t(pts), _t(off), kw.pop("max_raw_samples", MAX_RAW), kw.pop("max_points", MAX_PTS),
                        capacity=capacity, method="TENSION", map_index=mi, **kw)
    torch.cuda.synchronize()
    return {k: _np(v) for k, v in r.items()}


def _oracle(pts, off, maps, index, capacity=CAP, max_points=MAX_PTS, weights=None):
    return T.smooth_batch(pts, off, O.default_params(), capacity, maps, index, MAX_RAW, max_points,
                          T.WEIGHTS if weights is None else weights)


@pytest.mark.parametrize("moved", [False, True])
def test_device_equals_oracle(pl, moved):
    names, pts, off, maps, index = tc.batch(list(tc.named()), moved=moved)
    pl.set_maps(maps)
    got = _run(pl, pts, off, map_index=index)
    want = _oracle(pts, off, maps, index)
    assert got["knot_offsets"][0] == 0
    assert _compare(got, want, names, pts, off) <= 2
    ok = dict(zip(names, got["ok"]))
    assert all(ok[k] == 1 for k in ("config1", "straight_x", "u_turn", "corner", "six_close", "four_far", "down"))
    assert all(ok[k] == 0 for k in REFUSED) and all(ok[f"pose{k}"] == 1 for k in range(24))
    assert all(got["status"][b] == -100 and got["iters"][b] == 0 for b, n in enumerate(names) if n in REFUSED)


@pytest.mark.parametrize("w", tc.WEIGHTS[1:])
def test_weights(pl, w):
    names, pts, off, maps, index = tc.batch(["config1", "u_turn", "corner", "down", "pose3"])
    pl.set_maps(maps)
    got = _run(pl, pts, off, map_index=index, weights=w)
    want = _oracle(pts, off, maps, index, weights=w)
    assert _compare(got, want, names, pts, off) <= 1


def test_map_index_two_map_set(pl):
    """Per-path indices on a two-map set equal one run per map with that map alone (map_index None: map 0)."""
    names = ["config1", "pose3", "u_turn", "pose7", "corner", "pose3"]
    _, pts, off, _, _ = tc.batch(names)
    two = [tc.config1_map(), tc.pose_maps()["pose3"]]
    index = np.array([0, 1, 0, 1, 1, 0], dtype=np.int32)
    pl.set_maps(two)
    mixed = _run(pl, pts, off, map_index=index)
    assert mixed["ok"].sum() >= 4
    for k in (0, 1):
        pl.set_maps([two[k]])
        alone = _run(pl, pts, off)
        ka, km = alone["knot_offsets"], mixed["knot_offsets"]
        for b in np.flatnonzero(index == k):
            assert (alone["ok"][b], alone["status"][b], alone["iters"][b]) == \
                (mixed["ok"][b], mixed["status"][b], mixed["iters"][b])
            for f in ("knots", "x_coef", "y_coef"):
                assert alone[f][ka[b]:ka[b + 1]].tobytes() == mixed[f][km[b]:km[b + 1]].tobytes()
            assert alone["max_s"][b:b + 1].tobytes() == mixed["max_s"][b:b + 1].tobytes()


def test_refusals_are_isolated(pl):
    pl.set_maps([tc.config1_map()])
    names, pts, off, _, _ = tc.batch(["config1", "corner", "u_turn"])
    alone = _run(pl, pts, off)
    names2, pts2, off2, _, _ = tc.batch(["nan", "config1", "four_close", "corner", "config1", "u_turn", "three"])
    index = np.array([0, 0, 0, 0, 7, 0, -1], dtype=np.int32)          # path 4: a map index outside the set
    mixed = _run(pl, pts2, off2, map_index=index)
    assert list(mixed["ok"]) == [0, 1, 0, 1, 0, 1, 0]
    assert mixed["status"][4] == -100 and mixed["iters"][4] == 0 and np.isnan(mixed["max_s"][4])
    ka, km = alone["knot_offsets"], mixed["knot_offsets"]
    for a, m in ((0, 1), (1, 3), (2, 5)):
        for k in ("knots", "x_coef", "y_coef"):
            assert alone[k][ka[a]:ka[a + 1]].tobytes() == mixed[k][km[m]:km[m + 1]].tobytes()
        assert alone["iters"][a] == mixed["iters"][m]


def test_station_caps(pl):
    """More stations than max_points are refused as in the restatement; the largest max_points the entry accepts is
    277 and solves, one more is ERR_CAPACITY."""
    m = tc.config1_map()
    pl.set_maps([m])
    names, pts, off, maps, index = tc.batch(["corner", "config1", "straight_x"])
    got = _run(pl, pts, off, max_points=20)
    want = _oracle(pts, off, maps, index, max_points=20)
    assert list(got["ok"]) == list(want["ok"]) and want["reason"][1] == S.SM_MANY and got["status"][1] == -100
    x = np.arange(0.0, 262.0, 3.0)
    long = np.zeros((len(x), 7))
    long[:, 0], long[:, 1] = x, 4.0 * np.sin(x / 20.0)
    lo = np.array([0, len(x)], dtype=np.int32)
    got = _run(pl, long, lo, max_points=MAX_STATIONS)
    want = _oracle(long, lo, [m], None, max_points=MAX_STATIONS)
    assert want["ok"][0] == 1 and _compare(got, want, ["long"], long, lo) == 0
    with pytest.raises(planner.PqpError, match=f"rc={ERR_CAPACITY}"):
        _run(pl, long, lo, max_points=MAX_STATIONS + 1)


def test_capacity_reservation(pl):
    pl.set_maps([tc.config1_map()])
    base = ["config1", "corner", "u_turn", "four_close", "straight_x"]
    names = [base[i % len(base)] for i in range(70)]      # three warp tiles of the reservation
    _, pts, off, _, _ = tc.batch(names)
    full = _run(pl, pts, off)
    total = np.concatenate([[0], np.cumsum(np.diff(full["knot_offsets"]))])
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
    pl.set_maps([tc.config1_map()])
    names, pts, off, _, _ = tc.batch(["config1"])
    P, O_ = _t(pts), _t(off)
    for kw, rc in ((dict(max_raw_samples=2), ERR_ARG), (dict(max_points=2), ERR_ARG),
                   (dict(weights=(-1.0, 1.0, 50.0)), ERR_ARG), (dict(weights=(0.0, np.inf, 50.0)), ERR_ARG),
                   (dict(max_points=MAX_STATIONS + 1), ERR_CAPACITY), (dict(capacity=CAP + 1), ERR_CAPACITY)):
        args = dict(max_raw_samples=MAX_RAW, max_points=MAX_PTS)
        args.update(kw)
        with pytest.raises(planner.PqpError, match=f"rc={rc}"):
            pl.smooth_device(P, O_, method="TENSION", **args)
    with pytest.raises(ValueError):
        pl.smooth_device(P, O_, MAX_RAW, MAX_PTS, map_index=_t(np.zeros(1, dtype=np.int32)))      # TENSION2
    with pytest.raises(ValueError):
        pl.smooth_device(P, O_, MAX_RAW, MAX_PTS, method="ANGLE_DIFF")
    # an empty batch writes offsets[0] = 0, and is fine without the array
    ko = torch.full((1,), 7, dtype=torch.int32, device=_dev())
    r = pl.smooth_device(P[:0], O_[:1], MAX_RAW, MAX_PTS, method="TENSION", out=dict(knot_offsets=ko))
    torch.cuda.synchronize()
    assert int(r["knot_offsets"][0]) == 0
    rc = pl._L.pqp_smooth_reference_tension_device(pl._h, 0, None, None, 0.0, 1.0, 50.0, None, MAX_RAW, MAX_PTS, CAP,
                                                   *([None] * 8), None)
    assert rc == 0
    # no map set: ERR_ARG
    fresh = planner.PathPlanner(max_batch=4, max_total_points=1024)
    try:
        with pytest.raises(planner.PqpError, match=f"rc={ERR_ARG}"):
            fresh.smooth_device(P, O_, MAX_RAW, MAX_PTS, capacity=1024, method="TENSION")
    finally:
        fresh.close()
    torch.cuda.synchronize()


def _chain_inputs(k):
    c = segment_cases.config1()
    _, pts, off, _, _ = tc.batch(["config1"] * k)
    return pts, off, np.array([c["start"]] * k), np.array([c["goal"]] * k)


def test_plan_on_smoothed_lines_equals_host_plan(pl):
    """smooth(TENSION) -> post-smooth -> segment -> plan_device equals pqp_plan_batch on host copies."""
    import torch
    pl.set_maps([tc.config1_map()])
    pts, off, st, gl = _chain_inputs(4)
    sm = pl.smooth_device(_t(pts), _t(off), MAX_RAW, MAX_PTS, method="TENSION")
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


def test_graph_replay_equals_eager(pl):
    """smooth(TENSION) -> post-smooth -> segment -> fit -> plan_device captured in one CUDA graph; new points written
    into the captured tensor, a replay equals an eager run."""
    import torch
    pl.set_maps([tc.config1_map()])
    pts, off, st0, gl0 = _chain_inputs(8)
    P, Of, st, gl = _t(pts), _t(off), _t(st0), _t(gl0)
    mi = _t(np.zeros(8, dtype=np.int32))

    def cycle(o_sm=None, o_ps=None, o_sg=None, o_ft=None, o_pr=None):
        sm = pl.smooth_device(P, Of, MAX_RAW, MAX_PTS, method="TENSION", map_index=mi, out=o_sm)
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
    rng = np.random.default_rng(12)
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
