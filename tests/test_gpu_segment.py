"""GPU tests (run with -m gpu on an H100) of the batched segmentation, pqp_segment_reference_device
(PathPlanner.segment_device): the device stage against the CPU restatement (oracle/segment.py), the plan chain on its
outputs against pqp_plan_batch on host copies of them, capacity as total_points, fit -> segment -> plan in one CUDA
graph, isolated refusals and argument errors.  Lines: tests/segment_cases.py."""
import numpy as np
import pytest

from oracle import segment as oseg
from path_optimizer_b200 import _lib, device, planner, synth
from path_optimizer_b200.abi import ERR_ARG, ERR_CAPACITY, STATE_DTYPE
from tests import segment_cases as sc

pytestmark = pytest.mark.gpu
NEAR = 1e-9
IMPROVED, SIMPLE, RAW, DENSIFY = planner.BOUNDS_IMPROVED, planner.BOUNDS_SIMPLE, planner.OUTPUT_RAW, planner.OUTPUT_DENSIFY
CAP = 64 * 400


def _dev():
    import torch
    return torch.device("cuda", 0)


def _np(t):
    return t.detach().cpu().numpy()


def _t(a, dtype=None):
    import torch
    a = np.ascontiguousarray(a)
    if a.dtype.names:
        a = a.view(np.float64).reshape(len(a), -1)
    return torch.from_numpy(a.copy()).to(_dev())


def _dev_inputs(b):
    sp = b["splines"]
    return dict(splines=dict(knot_offsets=_t(sp["knot_offsets"]), knots=_t(sp["knots"]), x_coef=_t(sp["x_coef"]),
                             y_coef=_t(sp["y_coef"])),
                max_s=_t(b["max_s"]), start=_t(b["start"]), goal=_t(b["goal"]))


def _segment(p, b, capacity=CAP, max_n=400, **kw):
    import torch
    d = _dev_inputs(b)
    r = p.segment_device(d["splines"], d["max_s"], d["start"], d["goal"], max_n, capacity=capacity, **kw)
    torch.cuda.synchronize()
    return d, r


def _flags_dev(name):
    ds_small, ds_large, dynamic, search_ds = sc.FLAGS[name]
    return dict(delta_s_smaller=ds_small, delta_s_larger=ds_large, dynamic_segmentation=dynamic,
                search_delta_s=search_ds)


@pytest.fixture(scope="module")
def pl():
    p = planner.PathPlanner(max_batch=256, max_total_points=CAP)
    c = sc.config1()
    p.set_maps([c["field"], synth.disc_field_map()])
    p.set_param_sets(synth.param_sets(3, seed=5))
    yield p
    p.close()


@pytest.mark.parametrize("which", ["main", "lengths"])
@pytest.mark.parametrize("flags", list(sc.FLAGS))
def test_device_equals_oracle(pl, which, flags):
    """ok, n_points and offsets exact; x, y, z, k, s and x0 within 1e-9; paths whose decisions lie within 1e-9 of a
    threshold are dropped and counted."""
    b = sc.main_batch() if which == "main" else sc.length_batch()
    o = oseg.segment_batch(b["splines"], b["max_s"], b["start"], b["goal"], CAP, max_n=400, **sc.flag_kw(flags))
    _, r = _segment(pl, b, **_flags_dev(flags))
    near = o["margin"] < NEAR
    if near.any():   # a flipped decision moves every later offset: compare path by path
        print(f"dropped {int(near.sum())} of {len(near)} paths near a threshold")
    ok, n, off = _np(r["ok"]), _np(r["n_points"]), _np(r["offsets"])
    ref, x0 = _np(r["ref"]), _np(r["x0"])
    keep = ~near
    assert np.array_equal(ok[keep], o["ok"][keep]) and np.array_equal(n[keep], o["n_points"][keep])
    if not near.any():
        assert np.array_equal(off, o["offsets"])
    assert np.allclose(x0[keep], o["x0"][keep], rtol=0, atol=1e-9, equal_nan=True)
    assert np.array_equal(_np(r["end_heading"]), b["goal"]["z"])
    for i in np.flatnonzero(keep & (o["ok"] == 1)):
        got = ref[off[i]:off[i + 1]]
        want = o["ref"][o["offsets"][i]:o["offsets"][i + 1]]
        assert np.allclose(got, want, rtol=0, atol=1e-9), (b["names"][i], np.abs(got - want).max())
    assert near.sum() <= len(near) // 10


# ---- the plan chain on segmented lines -------------------------------------------------------------------------------

def _plan_batch():
    """Config-1's line, start and goal (on map 0) and the main batch's lines moved onto the disc field (map 1)."""
    c = sc.config1()
    paths = [("config1", c["spl"], float(c["spl"][0][-1]), c["start"], c["goal"])] * 3
    m = sc.main_batch()
    ko = m["splines"]["knot_offsets"]
    for i in range(0, len(m["names"]), 4):
        sl = slice(ko[i], ko[i + 1])
        sp = m["splines"]
        shift = lambda c4, dx: np.concatenate([c4[:, :3], c4[:, 3:] + dx], axis=1)   # noqa: E731
        st, gl = m["start"][i].copy(), m["goal"][i].copy()
        st["x"] -= 60.0; gl["x"] -= 60.0
        paths.append((m["names"][i], (sp["knots"][sl], shift(sp["x_coef"][sl], -60.0), sp["y_coef"][sl]),
                      m["max_s"][i], st, gl))
    b = sc.batch_of(paths)
    B = len(paths)
    mi = np.where(np.arange(B) < 3, 0, 1).astype(np.int32)
    pi = (np.arange(B) % 3).astype(np.int32)
    return b, mi, pi


def _host_plan_inputs(r):
    n = _np(r["n_points"])
    off = _np(r["offsets"])
    ref = device.tensor_to_records(r["ref"])[:off[-1]].copy()
    return dict(n_points=n, offsets=off, ref=ref, x0=_np(r["x0"]), end_heading=_np(r["end_heading"]))


def _host_splines(b, ok):
    sp, ko = b["splines"], b["splines"]["knot_offsets"]
    return dict(n_knots=np.diff(ko).astype(np.int32), knots=sp["knots"], x_coef=sp["x_coef"], y_coef=sp["y_coef"])


def _bits(r, hb, output_mode, host=False):
    o = hb["offsets"]
    out = []
    st = r["states"] if host else (device.tensor_to_records(r["states"].reshape(-1, 7)) if output_mode == RAW else
                                   device.tensor_to_records(r["states"].reshape(-1, 7)).reshape(r["states"].shape[0], -1))
    g = (lambda k: r[k]) if host else (lambda k: _np(r[k]))   # noqa: E731
    for i in range(len(hb["n_points"])):
        s = st[o[i]:o[i + 1]] if output_mode == RAW else st[i, :int(g("n_out")[i])]
        out.append((int(g("status")[i]), int(g("iters")[i]), int(g("n_out")[i]), int(g("ok")[i]), s.tobytes()))
    return out


@pytest.mark.parametrize("output_mode", [RAW, DENSIFY], ids=["raw", "densify"])
@pytest.mark.parametrize("bounds_mode", [IMPROVED, SIMPLE], ids=["improved", "simple"])
@pytest.mark.parametrize("form", ["KP", "K"])
def test_plan_on_segmented_lines_equals_host_plan(pl, form, bounds_mode, output_mode):
    """plan_device on segment_device's outputs (total_points = the capacity) = pqp_plan_batch_sets on a host copy of
    those outputs, bit for bit, with map and parameter-set indices and IMPROVED bounds on the smoothed splines."""
    import torch
    b, mi, pi = _plan_batch()
    d, r = _segment(pl, b)
    ok = _np(r["ok"])
    assert ok[:3].all() and ok.sum() >= len(ok) // 2
    hb = _host_plan_inputs(r)
    mi_dev = torch.where(r["ok"] != 0, _t(mi), -1).to(torch.int32)
    pi_dev = _t(pi)
    torch.cuda.synchronize()      # torch ops on the NULL stream are not ordered with the library's own stream
    spl = d["splines"] if bounds_mode == IMPROVED else None
    got = pl.plan_device(r["n_points"], r["offsets"], r["ref"], r["x0"], r["end_heading"], max_n_points=400,
                         formulation=form, bounds_mode=bounds_mode, splines=spl, output_mode=output_mode, max_out=512,
                         map_index=mi_dev, param_index=pi_dev)
    exact = pl.plan_device(r["n_points"], r["offsets"][: len(ok) + 1], r["ref"][: int(hb["offsets"][-1])], r["x0"],
                           r["end_heading"], max_n_points=int(hb["n_points"].max()), formulation=form, bounds_mode=bounds_mode, splines=spl,
                           output_mode=output_mode, max_out=512, map_index=mi_dev, param_index=pi_dev)
    torch.cuda.synchronize()
    hmi = np.where(ok != 0, mi, -1).astype(np.int32)
    want = pl.plan(hb, formulation=form, bounds_mode=bounds_mode,
                   splines=_host_splines(b, ok) if bounds_mode == IMPROVED else None, output_mode=output_mode,
                   max_out=512, map_index=hmi, param_index=pi)
    w = _bits(want, hb, output_mode, host=True)
    assert _bits(got, hb, output_mode) == w
    assert _bits(exact, hb, output_mode) == w          # capacity as total_points: the same bits as the exact total
    assert int(want["ok"][0]) == 1 or int(want["status"][0]) == 1


def test_graph_fit_segment_plan(pl):
    """Fit -> segment -> plan captured in one graph; new starts and goals written into the captured tensors, then a
    replay equals an eager run of the same three calls."""
    import torch
    c = sc.config1()
    xs, ys = oseg.Spline(*c["spl"][:2]), oseg.Spline(c["spl"][0], c["spl"][2])
    t = c["spl"][0]
    B = 16
    poly = np.zeros(len(t) * B, dtype=STATE_DTYPE)
    for i in range(B):
        seg = poly[i * len(t):(i + 1) * len(t)]
        seg["s"] = t
        seg["x"] = [xs(v) for v in t]
        seg["y"] = [ys(v) for v in t]
        seg["y"] += 0.05 * i
    poff = np.arange(B + 1, dtype=np.int32) * len(t)
    rng = np.random.default_rng(3)

    def poses():
        st = np.array([c["start"]] * B)
        gl = np.array([c["goal"]] * B)
        st["x"] += rng.uniform(-0.5, 0.5, B); st["z"] += rng.uniform(-0.2, 0.2, B)
        gl["x"] += rng.uniform(-1, 1, B); gl["y"] += rng.uniform(-1, 1, B)
        return st, gl
    dev = _dev()
    d_off, d_poly = _t(poff), _t(poly)
    s0, g0 = poses()
    d_max_s = _t(np.full(B, t[-1]))
    d_start, d_goal = _t(s0), _t(g0)
    zero = torch.zeros(B, dtype=torch.int32, device=dev)

    def cycle(fit_out=None, seg_out=None, plan_out=None):
        spl = pl.fit_splines_device(d_off, d_poly, out=fit_out)
        seg = pl.segment_device(spl, d_max_s, d_start, d_goal, 400, out=seg_out)
        mi = torch.where((seg["ok"] != 0) & (spl["ok"] != 0), zero, -1)
        res = pl.plan_device(seg["n_points"], seg["offsets"], seg["ref"], seg["x0"], seg["end_heading"],
                             max_n_points=400, bounds_mode=IMPROVED, splines=spl, map_index=mi, out=plan_out)
        return spl, seg, res
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        spl, seg, res = cycle()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cycle(spl, seg, res)
    for _ in range(2):
        s1, g1 = poses()
        d_start.copy_(_t(s1)); d_goal.copy_(_t(g1))
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        got = {k: _np(v).copy() for k, v in list(seg.items()) + list(res.items()) if v is not None}
        with torch.cuda.stream(stream):
            spl2, seg2, res2 = cycle()
        torch.cuda.synchronize()
        want = {k: _np(v) for k, v in list(seg2.items()) + list(res2.items()) if v is not None}
        assert set(got) == set(want)
        total = int(got["offsets"][-1])
        got["ref"], want["ref"] = got["ref"][:total], want["ref"][:total]    # rows past offsets[B] are not written
        for k in got:
            assert got[k].tobytes() == want[k].tobytes(), k
        assert _np(seg2["ok"]).sum() >= B // 2
    del g


def test_refusals_are_isolated(pl):
    """Refused paths (lengths, NaN rows, heading) between kept ones: the kept paths' counts, states and x0 equal those
    of the batch without the refused ones."""
    m, lb = sc.main_batch(), sc.length_batch()
    o = oseg.segment_batch(lb["splines"], lb["max_s"], lb["start"], lb["goal"], CAP)
    bad = [i for i in range(len(lb["names"])) if not o["ok"][i]]
    good = list(range(0, len(m["names"]), 9))

    def path(src, i):
        sp, ko = src["splines"], src["splines"]["knot_offsets"]
        sl = slice(ko[i], ko[i + 1])
        return (src["names"][i], (sp["knots"][sl], sp["x_coef"][sl], sp["y_coef"][sl]), src["max_s"][i],
                src["start"][i], src["goal"][i])
    mixed, is_bad = [], []
    for j in range(max(len(good), len(bad))):
        if j < len(good):
            mixed.append(path(m, good[j])); is_bad.append(False)
        if j < len(bad):
            mixed.append(path(lb, bad[j])); is_bad.append(True)
    is_bad = np.array(is_bad)
    _, r = _segment(pl, sc.batch_of(mixed))
    _, g = _segment(pl, sc.batch_of([path(m, i) for i in good]))
    assert not _np(r["ok"])[is_bad].any() and (_np(r["n_points"])[is_bad] == 0).all()
    keep = np.flatnonzero(~is_bad)
    assert np.array_equal(_np(r["n_points"])[keep], _np(g["n_points"]))
    tot = int(_np(g["offsets"])[-1])
    assert _np(r["ref"])[:tot].tobytes() == _np(g["ref"])[:tot].tobytes()
    assert _np(r["x0"])[keep].tobytes() == _np(g["x0"]).tobytes()


def test_argument_errors():
    """NULL pointers, a negative batch or capacity, max_n_points < 1 and bad spacings: PQP_ERR_ARG; a batch or capacity
    beyond the handle: PQP_ERR_CAPACITY; nothing is written either way."""
    import torch
    L = _lib.load()
    p = planner.PathPlanner(max_batch=4, max_total_points=300)
    try:
        b = sc.batch_of([("p", sc.lines()["curved"], 10.0, sc.main_batch()["start"][0], sc.main_batch()["goal"][0])] * 4)
        d = _dev_inputs(b)
        dev = _dev()
        outs = [torch.full((4,), 5, dtype=torch.int32, device=dev), torch.full((5,), 5, dtype=torch.int32, device=dev),
                torch.full((300, 7), 7.0, dtype=torch.float64, device=dev),
                torch.full((4, 3), 7.0, dtype=torch.float64, device=dev),
                torch.full((4,), 7.0, dtype=torch.float64, device=dev), torch.full((4,), 5, dtype=torch.int32, device=dev)]
        ins = [d["splines"][k].data_ptr() for k in ("knot_offsets", "knots", "x_coef", "y_coef")] + \
              [d[k].data_ptr() for k in ("max_s", "start", "goal")]
        good = ins + [t.data_ptr() for t in outs]

        def seg(batch, ptrs, ds=(0.15, 0.3, 1, 0.5), max_n=100, cap=300, h=p._h):
            return L.pqp_segment_reference_device(h, batch, *ptrs[:7], ds[0], ds[1], ds[2], ds[3], max_n, cap,
                                                  *ptrs[7:], None)
        for i in range(len(good)):
            bad = list(good)
            bad[i] = None
            assert seg(4, bad) == ERR_ARG, i
        assert seg(-1, good) == ERR_ARG and seg(4, good, h=None) == ERR_ARG
        assert seg(4, good, cap=-1) == ERR_ARG and seg(4, good, max_n=0) == ERR_ARG
        for ds in ((0.0, 0.3, 1, 0.5), (0.3, 0.15, 1, 0.5), (0.15, float("inf"), 1, 0.5), (0.15, 0.3, 1, 0.0),
                   (float("nan"), 0.3, 1, 0.5), (0.15, 0.3, 1, float("nan"))):
            assert seg(4, good, ds=ds) == ERR_ARG, ds
        assert seg(5, good) == ERR_CAPACITY and seg(4, good, cap=301) == ERR_CAPACITY
        assert seg(0, [None] * len(good)) == 0
        torch.cuda.synchronize()
        assert all((_np(t) == (5 if t.dtype == torch.int32 else 7.0)).all() for t in outs)
        assert seg(4, good) == 0
        torch.cuda.synchronize()
        assert (_np(outs[5]) == 1).all() and int(_np(outs[1])[-1]) == 4 * int(_np(outs[0])[0])
        # an empty batch writes offsets[0] = 0 and nothing else
        outs[1].fill_(5)
        torch.cuda.synchronize()
        assert seg(0, good) == 0
        torch.cuda.synchronize()
        assert _np(outs[1]).tolist() == [0, 5, 5, 5, 5]
    finally:
        p.close()


# ---- the station cap and the capacity on the device -------------------------------------------------------------------

def _reserve(counts, capacity):
    kept = np.array(oseg.reserve([int(c) for c in counts], capacity), dtype=bool)
    n = np.where(kept, counts, 0).astype(np.int32)
    return kept.astype(np.int32), n, np.concatenate([[0], np.cumsum(n)]).astype(np.int32)


def test_cap_and_capacity_on_the_device(pl):
    """The device reservation (two warp scans per 32 paths, carried across tiles) on the main batch (120 paths, four
    tiles): with the station cap at the median count, capacities of about a half and a third of the total, and
    capacities that end exactly at, one before and one after the stations of paths 0..30, 0..31 and 0..32 (the first
    tile boundary).  ok, n_points and offsets equal the reservation rule applied to the device's own uncapped counts
    exactly, and the oracle's when no path lies near a threshold; every kept path's states and x0 equal the uncapped
    run's bit for bit; a refused path has 0 stations."""
    b = sc.main_batch()
    B = len(b["names"])
    assert B > 96
    _, free = _segment(pl, b, capacity=CAP, max_n=400)
    fn, foff = _np(free["n_points"]), _np(free["offsets"])
    fref, fx0 = _np(free["ref"]), _np(free["x0"])
    assert (fn > 0).sum() >= B // 2 and int(foff[-1]) < CAP
    o_free = oseg.segment_batch(b["splines"], b["max_s"], b["start"], b["goal"], CAP, max_n=400)
    near = o_free["margin"] < NEAR
    max_n = int(np.median(fn[fn > 0]))
    capped = np.where(fn <= max_n, fn, 0)
    pre = np.cumsum(capped)
    caps = {int(foff[-1]) // 2, int(foff[-1]) // 3}
    for j in (30, 31, 32):
        caps |= {int(pre[j]) - 1, int(pre[j]), int(pre[j]) + 1}
    checked = 0
    for max_n_i in (max_n, 400):
        counts = capped if max_n_i == max_n else fn
        for capacity in sorted(caps):
            _, r = _segment(pl, b, capacity=capacity, max_n=max_n_i)
            ok, n, off = _np(r["ok"]), _np(r["n_points"]), _np(r["offsets"])
            want_ok, want_n, want_off = _reserve(counts, capacity)
            assert np.array_equal(ok, want_ok), (max_n_i, capacity)
            assert np.array_equal(n, want_n) and np.array_equal(off, want_off), (max_n_i, capacity)
            assert off[-1] <= capacity and (n[ok == 0] == 0).all()
            assert ok.sum() < (counts > 0).sum() or max_n_i == max_n, (max_n_i, capacity)   # something is refused
            ref, x0 = _np(r["ref"]), _np(r["x0"])
            for i in np.flatnonzero(ok):
                assert ref[off[i]:off[i + 1]].tobytes() == fref[foff[i]:foff[i + 1]].tobytes(), (capacity, i)
            assert x0.tobytes() == fx0.tobytes()
            if not near.any():
                o = oseg.segment_batch(b["splines"], b["max_s"], b["start"], b["goal"], capacity, max_n=max_n_i)
                assert np.array_equal(ok, o["ok"]) and np.array_equal(n, o["n_points"])
                assert np.array_equal(off, o["offsets"])
                for i in np.flatnonzero(ok):
                    assert np.allclose(ref[off[i]:off[i + 1]], o["ref"][o["offsets"][i]:o["offsets"][i + 1]], rtol=0,
                                       atol=1e-9)
            checked += 1
    assert checked >= 10
