"""GPU tests (run with -m gpu on an H100) of the corridor search and post-smoothing, pqp_post_smooth_device
(PathPlanner.post_smooth_device): the device stage against the CPU restatement (oracle/corridor.py) on the scenes of
tests/corridor_cases.py and on a scene of exact cost ties, the plan chain on its outputs against pqp_plan_batch on host
copies, map indices, the capacity reservation, isolated refusals, argument errors, and post-smooth -> segment -> fit ->
plan in one CUDA graph."""
import numpy as np
import pytest

from oracle import corridor as oc
from oracle import oracle as O
from path_optimizer_b200 import device, planner
from path_optimizer_b200.abi import ERR_ARG, ERR_CAPACITY
from tests import corridor_cases as cc

pytestmark = pytest.mark.gpu
NEAR = 1e-9
CAP = 4096
MAXL = 200


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
def scene():
    return cc.batch()


@pytest.fixture(scope="module")
def pl(scene):
    p = planner.PathPlanner(max_batch=256, max_total_points=CAP)
    p.set_maps(scene["maps"])
    yield p
    p.close()


def _splines_dev(b):
    sp = b["splines"]
    return dict(knot_offsets=_t(sp["knot_offsets"]), knots=_t(sp["knots"]), x_coef=_t(sp["x_coef"]),
                y_coef=_t(sp["y_coef"]))


def _goals(b):
    """Every line's end point and heading, as the goal the segment stage cuts the post-smoothed line at."""
    ko, xc, yc = b["splines"]["knot_offsets"], b["splines"]["x_coef"], b["splines"]["y_coef"]
    g = np.array(b["start"]).copy()
    for i in range(len(g)):
        e = ko[i + 1] - 1
        g[i]["x"], g[i]["y"], g[i]["z"] = xc[e][3], yc[e][3], np.arctan2(yc[e][2], xc[e][2])
    return g


def _run(p, b, capacity=CAP, map_index="scene", **kw):
    import torch
    sp = b["splines"]
    d = dict(knot_offsets=_t(sp["knot_offsets"]), knots=_t(sp["knots"]), x_coef=_t(sp["x_coef"]), y_coef=_t(sp["y_coef"]))
    mi = b["map_index"] if isinstance(map_index, str) else map_index
    r = p.post_smooth_device(d, _t(b["max_s"]), _t(b["start"]), MAXL, capacity=capacity,
                             map_index=None if mi is None else _t(np.asarray(mi, dtype=np.int32)), want_layers=True, **kw)
    torch.cuda.synchronize()
    return {k: (None if v is None else _np(v)) for k, v in r.items()}


def _oracle(b, capacity=CAP, map_index="scene"):
    mi = b["map_index"] if isinstance(map_index, str) else map_index
    return oc.post_smooth_batch(b["splines"], b["max_s"], b["start"], b["maps"], O.default_params(), capacity,
                                map_index=mi, max_layers=MAXL)


def _tile(b, k):
    """The scene batch repeated k times."""
    B = len(b["names"])
    idx = np.tile(np.arange(B), k)
    sp = b["splines"]
    ko = sp["knot_offsets"]
    pieces = [slice(int(ko[i]), int(ko[i + 1])) for i in idx]
    nko = np.zeros(len(idx) + 1, dtype=np.int32)
    np.cumsum([s.stop - s.start for s in pieces], out=nko[1:])
    return dict(names=[b["names"][i] for i in idx], maps=b["maps"], map_index=b["map_index"][idx],
                splines=dict(knot_offsets=nko, knots=np.concatenate([sp["knots"][s] for s in pieces]),
                             x_coef=np.concatenate([sp["x_coef"][s] for s in pieces]),
                             y_coef=np.concatenate([sp["y_coef"][s] for s in pieces])),
                max_s=b["max_s"][idx], start=b["start"][idx])


def test_device_equals_oracle(pl, scene):
    """ok, knot offsets, layer s and bounds exact; QP status and iterations equal; knots, coefficients and max_s
    within 1e-8.  Paths whose discrete decisions lie within 1e-9 of a threshold are dropped and counted."""
    o, r = _oracle(scene), _run(pl, scene)
    near = o["margin"] < NEAR
    print(f"dropped {int(near.sum())} of {len(near)} paths near a threshold: "
          f"{[n for n, x in zip(scene['names'], near) if x]}")
    assert near.sum() <= max(1, len(near) // 10)
    off, ooff = r["knot_offsets"], o["knot_offsets"]
    for b, name in enumerate(scene["names"]):
        if near[b]:
            continue
        assert r["ok"][b] == o["ok"][b], name
        assert (off[b + 1] - off[b]) == (ooff[b + 1] - ooff[b]), name
        assert r["status"][b] == o["status"][b], name
        assert r["iters"][b] == o["iters"][b], name
        if not o["ok"][b]:
            assert np.isnan(r["max_s"][b]), name
            continue
        d, h = slice(off[b], off[b + 1]), slice(ooff[b], ooff[b + 1])
        np.testing.assert_array_equal(r["layers"][d], o["layers"][h], err_msg=name)
        np.testing.assert_allclose(r["knots"][d], o["knots"][h], rtol=0, atol=1e-8, err_msg=name)
        np.testing.assert_allclose(r["x_coef"][d], o["x_coef"][h], rtol=0, atol=1e-8, err_msg=name)
        np.testing.assert_allclose(r["y_coef"][d], o["y_coef"][h], rtol=0, atol=1e-8, err_msg=name)
        assert abs(r["max_s"][b] - o["max_s"][b]) <= 1e-8, name
    assert o["ok"].sum() >= 8


def test_map_index_refusals(pl, scene):
    """An index outside the map set refuses its path alone; every other path equals the run with valid indices."""
    base = _run(pl, scene)
    mi = scene["map_index"].copy()
    mi[1], mi[3] = -1, len(scene["maps"])
    r = _run(pl, scene, map_index=mi)
    assert r["ok"][1] == 0 and r["ok"][3] == 0
    assert np.isnan(r["max_s"][1]) and np.isnan(r["max_s"][3])
    for b in range(len(mi)):
        if b in (1, 3):
            assert r["knot_offsets"][b + 1] == r["knot_offsets"][b]
            continue
        assert r["ok"][b] == base["ok"][b]
        n0 = base["knot_offsets"][b + 1] - base["knot_offsets"][b]
        d0 = slice(base["knot_offsets"][b], base["knot_offsets"][b] + n0)
        d1 = slice(r["knot_offsets"][b], r["knot_offsets"][b] + n0)
        np.testing.assert_array_equal(r["x_coef"][d1], base["x_coef"][d0])
        np.testing.assert_array_equal(r["layers"][d1], base["layers"][d0])


def test_capacity_reservation(pl, scene):
    """Over 70 paths (three warp tiles), capacities ending on either side of a tile boundary: the refused paths are a
    suffix in index order, offsets match the restatement's reservation, kept paths equal the uncapped run bit for
    bit."""
    b = _tile(scene, 5)
    full = _run(pl, b)
    counts = np.diff(full["knot_offsets"])
    before = np.concatenate([[0], np.cumsum(counts)])
    for cut in (31, 32, 33, 64):
        capacity = int(before[cut])
        r = _run(pl, b, capacity=capacity)
        kept = oc.reserve(list(counts), capacity)
        np.testing.assert_array_equal(r["ok"], np.array(kept, dtype=np.int32))
        assert r["knot_offsets"][-1] <= capacity
        for k in range(len(counts)):
            if not kept[k]:
                continue
            d0 = slice(full["knot_offsets"][k], full["knot_offsets"][k + 1])
            d1 = slice(r["knot_offsets"][k], r["knot_offsets"][k + 1])
            for key in ("knots", "x_coef", "y_coef", "layers"):
                np.testing.assert_array_equal(r[key][d1], full[key][d0])
            assert r["max_s"][k] == full["max_s"][k]
            assert r["status"][k] == full["status"][k] and r["iters"][k] == full["iters"][k]


def test_bad_arguments(pl, scene):
    import torch
    sp = scene["splines"]
    d = dict(knot_offsets=_t(sp["knot_offsets"]), knots=_t(sp["knots"]), x_coef=_t(sp["x_coef"]), y_coef=_t(sp["y_coef"]))
    ms, st = _t(scene["max_s"]), _t(scene["start"])
    for kw, rc in ((dict(search_lateral_range=0.0), ERR_ARG), (dict(search_lateral_spacing=float("nan")), ERR_ARG),
                   (dict(search_longitudial_spacing=-1.0), ERR_ARG), (dict(capacity=CAP + 1), ERR_CAPACITY)):
        with pytest.raises(planner.PqpError, match=f"rc={rc}"):
            pl.post_smooth_device(d, ms, st, MAXL, **kw)
    with pytest.raises(planner.PqpError, match=f"rc={ERR_ARG}"):
        pl.post_smooth_device(d, ms, st, 3)
    with pytest.raises(planner.PqpError, match=f"rc={ERR_CAPACITY}"):
        pl.post_smooth_device(d, ms, st, 100000)
    empty = dict(knot_offsets=torch.zeros(1, dtype=torch.int32, device=_dev()), knots=d["knots"], x_coef=d["x_coef"],
                 y_coef=d["y_coef"])
    r = pl.post_smooth_device(empty, ms[:0], st[:0], MAXL, out=dict(knot_offsets=torch.full((1,), 7, dtype=torch.int32,
                                                                                           device=_dev())))
    torch.cuda.synchronize()
    assert int(r["knot_offsets"][0]) == 0


def test_tie_scene_equals_oracle(pl):
    """A lattice symmetric about the line (spacing 0.5) and a mirror-symmetric map: the DP meets exact ties, which the
    device resolves as the restatement does -- first index -- so chain, layers and bounds are equal bit for bit."""
    m, spl, st = cc.tie_scene()
    p = planner.PathPlanner(max_batch=4, max_total_points=512)
    try:
        p.set_maps([m])
        b = dict(names=["tie"], maps=[m], map_index=np.zeros(1, dtype=np.int32),
                 splines=dict(knot_offsets=np.array([0, len(spl[0])], dtype=np.int32), knots=spl[0],
                              x_coef=np.asarray(spl[1]), y_coef=np.asarray(spl[2])),
                 max_s=np.array([spl[0][-1]]), start=np.array([st]))
        o = oc.post_smooth_batch(b["splines"], b["max_s"], b["start"], [m], O.default_params(), 512, max_layers=MAXL,
                                 spacing=cc.TIE_SPACING)
        assert o["found"][0]["ties"] > 0 and o["ok"][0] == 1
        r = _run(p, b, capacity=512, search_lateral_spacing=cc.TIE_SPACING)
    finally:
        p.close()
    assert r["ok"][0] == 1 and r["knot_offsets"][1] == o["knot_offsets"][1]
    np.testing.assert_array_equal(r["layers"][:o["knot_offsets"][1]], o["layers"])
    assert r["status"][0] == o["status"][0] and r["iters"][0] == o["iters"][0]
    np.testing.assert_allclose(r["knots"][:o["knot_offsets"][1]], o["knots"], rtol=0, atol=1e-8)


def _bits(res, offsets, host=False):
    st = res["states"] if host else device.tensor_to_records(res["states"].reshape(-1, 7))
    g = (lambda k: res[k]) if host else (lambda k: _np(res[k]))   # noqa: E731
    return [(int(g("status")[i]), int(g("iters")[i]), int(g("n_out")[i]), int(g("ok")[i]),
             st[offsets[i]:offsets[i + 1]].tobytes()) for i in range(len(offsets) - 1)]


@pytest.mark.parametrize("form", ["KP", "K"])
def test_plan_on_post_smoothed_lines_equals_host_plan(pl, scene, form):
    """post-smooth -> segment -> plan_device (IMPROVED bounds on the post-smoothed splines) equals pqp_plan_batch on
    host copies of the segmented states and of the post-smoothed splines, bit for bit."""
    import torch
    d = _splines_dev(scene)
    st, mi = _t(scene["start"]), _t(scene["map_index"])
    gl = _t(_goals(scene))
    ps = pl.post_smooth_device(d, _t(scene["max_s"]), st, MAXL, map_index=mi)
    sg = pl.segment_device(ps, ps["max_s"], st, gl, 400)
    torch.cuda.synchronize()      # torch ops on the NULL stream are not ordered with the library's own stream
    idx = torch.where((ps["ok"] != 0) & (sg["ok"] != 0), mi, torch.full_like(mi, -1))
    torch.cuda.synchronize()
    got = pl.plan_device(sg["n_points"], sg["offsets"], sg["ref"], sg["x0"], sg["end_heading"], max_n_points=400,
                         formulation=form, bounds_mode=planner.BOUNDS_IMPROVED, splines=ps, map_index=idx)
    torch.cuda.synchronize()
    off = _np(sg["offsets"])
    assert int((_np(idx) >= 0).sum()) >= 8
    hb = dict(n_points=_np(sg["n_points"]), offsets=off, ref=device.tensor_to_records(sg["ref"])[:off[-1]].copy(),
              x0=_np(sg["x0"]), end_heading=_np(sg["end_heading"]))
    # host copies of the post-smoothed splines; a refused path (0 knots, map index -1) carries its input line instead,
    # since the host entry checks every path's splines before it reads the map index
    ko, sp = _np(ps["knot_offsets"]), scene["splines"]
    pk, px, py = _np(ps["knots"]), _np(ps["x_coef"]), _np(ps["y_coef"])
    parts = []
    for b in range(len(ko) - 1):
        if ko[b + 1] > ko[b]:
            sl = slice(ko[b], ko[b + 1])
            parts.append((pk[sl], px[sl], py[sl]))
        else:
            sl = slice(sp["knot_offsets"][b], sp["knot_offsets"][b + 1])
            parts.append((sp["knots"][sl], sp["x_coef"][sl], sp["y_coef"][sl]))
    hs = dict(n_knots=np.array([len(p[0]) for p in parts], dtype=np.int32), knots=np.concatenate([p[0] for p in parts]),
              x_coef=np.concatenate([p[1] for p in parts]), y_coef=np.concatenate([p[2] for p in parts]))
    want = pl.plan(hb, formulation=form, bounds_mode=planner.BOUNDS_IMPROVED, splines=hs, map_index=_np(idx))
    assert _bits(got, off) == _bits(want, off, host=True)
    assert sum(int(v) == 1 for v in want["status"]) >= 8


def test_graph_replay_equals_eager(pl, scene):
    """post-smooth -> segment -> fit -> plan_device captured in one CUDA graph (IMPROVED bounds on the splines the fit
    makes of the segmented states); new starts written into the captured tensor, a replay equals an eager run."""
    import torch
    d = _splines_dev(scene)
    ms, st, mi, gl = _t(scene["max_s"]), _t(scene["start"]), _t(scene["map_index"]), _t(_goals(scene))

    def cycle(out_ps=None, out_seg=None, out_fit=None, out_plan=None):
        ps = pl.post_smooth_device(d, ms, st, MAXL, map_index=mi, out=out_ps)
        sg = pl.segment_device(ps, ps["max_s"], st, gl, 400, out=out_seg)
        ft = pl.fit_splines_device(sg["offsets"], sg["ref"], out=out_fit)
        idx = torch.where((ps["ok"] != 0) & (sg["ok"] != 0) & (ft["ok"] != 0), mi, torch.full_like(mi, -1))
        pr = pl.plan_device(sg["n_points"], sg["offsets"], sg["ref"], sg["x0"], sg["end_heading"], max_n_points=400,
                            bounds_mode=planner.BOUNDS_IMPROVED, splines=ft, map_index=idx, out=out_plan)
        return ps, sg, ft, pr
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        ps, sg, ft, pr = cycle()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cycle(ps, sg, ft, pr)
    rng = np.random.default_rng(7)
    s0 = scene["start"].copy()
    s1 = s0.copy()
    s1["y"] += rng.uniform(-0.3, 0.3, len(s1))
    s1["z"] += rng.uniform(-0.05, 0.05, len(s1))
    st.copy_(_t(s1))
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    got = {k: _np(v).copy() for r in (ps, sg, pr) for k, v in r.items() if v is not None}
    with torch.cuda.stream(stream):
        ps2, sg2, ft2, pr2 = cycle()
    torch.cuda.synchronize()
    want = {k: _np(v) for r in (ps2, sg2, pr2) for k, v in r.items() if v is not None}
    assert int(_np(ps2["ok"]).sum()) >= 8 and int(_np(sg2["ok"]).sum()) >= 8
    assert int((_np(pr2["status"]) == 1).sum()) >= 8
    kt, tt = int(got["knot_offsets"][-1]), int(got["offsets"][-1])
    for k in got:
        a, b = got[k], want[k]
        if k in ("knots", "x_coef", "y_coef"):
            a, b = a[:kt], b[:kt]                     # rows past the offsets are not written
        if k == "ref":
            a, b = a[:tt], b[:tt]
        assert a.tobytes() == b.tobytes(), k
    del g
