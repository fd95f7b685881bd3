"""GPU tests (run with -m gpu on an H100) of the batched reference-spline fit, pqp_fit_splines_device
(PathPlanner.fit_splines_device): its rows against pqp_spline_fit bit for bit, the IMPROVED plan chain on its splines
against pqp_plan_batch on host-fitted ones, fit and plan captured in one CUDA graph and replayed on a new batch, refused
paths routed out of the chain through the map index, and argument errors."""
import os

import numpy as np
import pytest

from path_optimizer_b200 import _lib, device, planner, synth, workloads
from path_optimizer_b200.abi import BOUNDS_DTYPE, ERR_ARG, ERR_CAPACITY
from tests import fit_lines
from tests.emu import fit_emu

pytestmark = pytest.mark.gpu
INVALID = -100
IMPROVED, RAW, DENSIFY = planner.BOUNDS_IMPROVED, planner.OUTPUT_RAW, planner.OUTPUT_DENSIFY
WILD = dict(y_range=(-3.0, 3.0), heading_range=0.05, curvature_amp=0.02)


def _dev():
    import torch
    return torch.device("cuda", 0)


def _np(t):
    return t.detach().cpu().numpy()


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64).tobytes()


@pytest.fixture(scope="module")
def big():
    p = planner.PathPlanner(max_batch=8192, max_total_points=8192 * 200)
    yield p
    p.close()


@pytest.fixture(scope="module")
def pl():
    p = planner.PathPlanner(max_batch=256, max_total_points=256 * 400)
    p.set_map(synth.disc_field_map())
    yield p
    p.close()


# torch's default stream is the NULL stream, which the library takes for the handle's own (non-blocking) stream: a
# torch op between two library calls is ordered with them only on another torch stream (or inside a capture).


def _fit(p, b, out=None):
    import torch
    d = device.batch_to_device(b, _dev())
    r = p.fit_splines_device(d["offsets"], d["ref"], out=out)
    torch.cuda.synchronize()
    return d, r


def _case(name):
    if name == "config3":
        return workloads.config3_candidates(8192)
    if name == "config5":
        return workloads.build(5)
    return fit_lines.batch_of(list(fit_lines.good_lines().values()))


@pytest.mark.parametrize("name", ["config3", "config5", "spacing"])
def test_rows_equal_host_fit(big, name):
    """Every path's knots and x / y rows equal pqp_spline_fit's (planner.reference_splines) bit for bit."""
    b = _case(name)
    _, r = _fit(big, b)
    want = planner.reference_splines(b)
    assert (_np(r["ok"]) == 1).all()
    assert _bits(_np(r["knots"])) == _bits(want["knots"])
    assert _bits(_np(r["x_coef"])) == _bits(want["x_coef"])
    assert _bits(_np(r["y_coef"])) == _bits(want["y_coef"])


def test_refused_rows_and_emulator(big):
    """Good and refused lines interleaved: ok and every finite row as the kernel source under g++ gives them, NaN rows
    for the refused paths."""
    good = list(fit_lines.good_lines().values())
    bad = [r for r, _ in fit_lines.refused_lines().values()]
    refs = [x for pair in zip(good, bad) for x in pair] + good[len(bad):] + bad[len(good):]
    b = fit_lines.batch_of(refs)
    _, r = _fit(big, b)
    want = fit_emu.fit_splines(b["offsets"], b["ref"])
    ok = _np(r["ok"])
    assert np.array_equal(ok, want["ok"]) and (ok == 0).sum() == len(bad)
    o = b["offsets"]
    for i in range(len(refs)):
        sl = slice(o[i], o[i + 1])
        for f in ("knots", "x_coef", "y_coef"):
            g = _np(r[f])[sl]
            if ok[i]:
                assert _bits(g) == _bits(want[f][sl]), (i, f)
            else:
                assert np.isnan(g).all(), (i, f)


# ---- the plan chain -------------------------------------------------------------------------------------------------

def _host(r, output_mode):
    import torch
    torch.cuda.synchronize()
    st = r["states"].reshape(-1, 7) if output_mode == RAW else r["states"]
    states = device.tensor_to_records(st)
    if output_mode == DENSIFY:
        states = states.reshape(r["states"].shape[0], -1)
    return dict(states=states, n_out=_np(r["n_out"]), ok=_np(r["ok"]), status=_np(r["status"]), iters=_np(r["iters"]),
                bounds=device.tensor_to_records(r["bounds"], BOUNDS_DTYPE))


def _path_bits(r, b, i, output_mode):
    o = b["offsets"]
    st = r["states"][o[i]:o[i + 1]] if output_mode == RAW else r["states"][i, :r["n_out"][i]]
    return (int(r["status"][i]), int(r["iters"][i]), int(r["n_out"][i]), int(r["ok"][i]), st.tobytes(),
            r["bounds"][o[i]:o[i + 1]].tobytes())


def _same(got, want, b, output_mode, idx=None, want_b=None, want_idx=None):
    """Path idx[k] of `got` (batch b) equals path want_idx[k] of `want` (batch want_b): status, iterations, out_n, ok,
    states and bounds, bit for bit."""
    idx = range(len(b["n_points"])) if idx is None else idx
    want_b = b if want_b is None else want_b
    want_idx = idx if want_idx is None else want_idx
    for i, j in zip(idx, want_idx):
        assert _path_bits(got, b, i, output_mode) == _path_bits(want, want_b, j, output_mode), (i, j)


def _plan_dev(p, d, b, spl, output_mode=RAW, **kw):
    return p.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"],
                         max_n_points=int(b["n_points"].max()), bounds_mode=IMPROVED, splines=spl,
                         output_mode=output_mode, max_out=256, want_bounds=True, **kw)


def _plan_batch(B=48, perm=None, first_path=0):
    n_points = synth.mixed_lengths(B, 20, 300)
    if perm is not None:
        n_points = n_points[perm]
    return synth.map_reference_paths(B, n_points=n_points, first_path=first_path, **WILD)


@pytest.mark.parametrize("output_mode", [RAW, DENSIFY], ids=["raw", "densify"])
@pytest.mark.parametrize("name", ["KP", "KPC", "K"])
def test_chain_equals_host_splines(pl, name, output_mode):
    """plan_device(IMPROVED) on device-fitted splines = pqp_plan_batch on host-fitted ones, bit for bit."""
    b = _plan_batch()
    want = pl.plan(b, formulation=name, bounds_mode=IMPROVED, splines=planner.reference_splines(b),
                   output_mode=output_mode, max_out=256, want_bounds=True)
    d, spl = _fit(pl, b)
    got = _host(_plan_dev(pl, d, b, spl, output_mode, formulation=name), output_mode)
    _same(got, want, b, output_mode)
    assert (want["status"] == 1).sum() >= 10 and (want["n_out"] < b["n_points"]).any()


def _config1():
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "config1_benchmark_map.npz"))
    field = dict(distance=g["map_distance"], rows=int(g["image_shape"][0]), cols=int(g["image_shape"][1]),
                 resolution=float(g["map_geo"][0]), center_x=float(g["map_geo"][1]), center_y=float(g["map_geo"][2]))
    b = dict(n_points=g["n_points"], ref=g["ref"], x0=g["x0"], end_heading=g["end_heading"])
    b["offsets"] = np.array([0, int(g["n_points"][0])], dtype=np.int32)
    return field, b


def test_chain_config1_golden():
    """BASELINE config 1 (the reference's benchmark map and path), both tails."""
    field, b = _config1()
    p = planner.PathPlanner(max_batch=1, max_total_points=256)
    try:
        p.set_map(field)
        for output_mode in (RAW, DENSIFY):
            want = p.plan(b, bounds_mode=IMPROVED, splines=planner.reference_splines(b), output_mode=output_mode,
                          max_out=256, want_bounds=True)
            d, spl = _fit(p, b)
            _same(_host(_plan_dev(p, d, b, spl, output_mode), output_mode), want, b, output_mode)
            assert int(want["ok"][0]) == 1
    finally:
        p.close()


def test_chain_maps_sets_forms():
    """A batch over three maps (the first the config-1 map), four parameter sets and per-path formulations."""
    import torch
    field, _ = _config1()
    maps, b, mi = synth.multi_map_batch(3, 12, n=120, first_maps=[field], order="interleaved",
                                        y_range=(-1.5, 1.5), heading_range=0.03, curvature_amp=0.01)
    total = int(b["offsets"][-1])
    b["ref"]["v"] = 4.0 + 3.0 * np.sin(np.arange(total) * 0.05)
    b["ref"]["a"] = 0.5 * np.cos(np.arange(total) * 0.05)
    B = len(mi)
    rng = np.random.default_rng(8)
    pi = rng.permutation(np.arange(B) % 4).astype(np.int32)
    forms = rng.permutation(np.arange(B) // 4 % 3).astype(np.int32)
    p = planner.PathPlanner(max_batch=64, max_total_points=64 * 200)
    try:
        p.set_maps(maps)
        p.set_param_sets(synth.param_sets(4, seed=11))
        dev = _dev()
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
        for output_mode in (RAW, DENSIFY):
            want = p.plan(b, formulation=forms, bounds_mode=IMPROVED, splines=planner.reference_splines(b),
                          output_mode=output_mode, max_out=256, want_bounds=True, map_index=mi, param_index=pi)
            d, spl = _fit(p, b)
            got = _host(_plan_dev(p, d, b, spl, output_mode, formulation=t(forms), map_index=t(mi), param_index=t(pi)),
                        output_mode)
            _same(got, want, b, output_mode)
            assert (want["status"] == 1).sum() >= 10
    finally:
        p.close()


def test_graph_fit_and_plan(pl):
    """Warm up, capture fit + the map-index route + plan in one graph, write a new batch (same path count and station
    total) into the captured inputs and replay, twice: pqp_plan_batch's results on host-fitted splines each time."""
    import torch
    B = 48
    first = _plan_batch(B)
    second = _plan_batch(B, perm=np.random.default_rng(5).permutation(B), first_path=777)
    assert int(first["offsets"][-1]) == int(second["offsets"][-1])
    max_n = int(max(first["n_points"].max(), second["n_points"].max()))
    dev = _dev()
    d = device.batch_to_device(first, dev)
    zero = torch.zeros(B, dtype=torch.int32, device=dev)

    def cycle(spl_out=None):
        spl = pl.fit_splines_device(d["offsets"], d["ref"], out=spl_out)
        mi = torch.where(spl["ok"] != 0, zero, -1)
        res = pl.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], max_n_points=max_n,
                             bounds_mode=IMPROVED, splines=spl, want_bounds=True, map_index=mi)
        return spl, res
    with torch.cuda.stream(torch.cuda.Stream()):   # library and torch.where on one stream (note above _fit)
        spl, _ = cycle()                  # warm-up
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _, res = cycle(spl)
    for b in (second, first):
        for k, v in device.batch_to_device(b, dev).items():
            if k in d:
                d[k].copy_(v)
        g.replay()
        torch.cuda.synchronize()          # (one call in flight per handle: the host chain below uses the same handle)
        want = pl.plan(b, bounds_mode=IMPROVED, splines=planner.reference_splines(b), want_bounds=True)
        _same(_host(res, RAW), want, b, RAW)
        assert (_np(spl["ok"]) == 1).all()
    del g


def test_refused_paths_through_the_map_index(pl):
    """Refused lines between planned ones: ok = 0, and with map_index = -1 from ok on the device, status -100, 0
    iterations, out_n = 0 and ok = 0; the planned paths equal those of the batch without the refused ones, bit for bit,
    and pqp_plan_batch on host-fitted splines."""
    import torch
    good_b = _plan_batch(24, first_path=300)
    o = good_b["offsets"]
    good = [good_b["ref"][o[i]:o[i + 1]] for i in range(24)]
    bad = [r for r, _ in fit_lines.refused_lines().values()]
    refs, is_bad = [], []
    for k in range(max(len(good), len(bad))):
        for lst, flag in ((good, False), (bad, True)):
            if k < len(lst):
                refs.append(lst[k]); is_bad.append(flag)
    is_bad = np.array(is_bad)
    b = fit_lines.batch_of(refs)
    gb = fit_lines.batch_of(good)

    def run(batch):
        with torch.cuda.stream(torch.cuda.Stream()):   # library and torch.where on one stream (note above _fit)
            d = device.batch_to_device(batch, _dev())
            spl = pl.fit_splines_device(d["offsets"], d["ref"])
            mi = torch.where(spl["ok"] != 0, 0, -1).to(torch.int32)
            res = _plan_dev(pl, d, batch, spl, map_index=mi)
        torch.cuda.synchronize()
        return _np(spl["ok"]), _host(res, RAW)
    ok, got = run(b)
    gok, gwant = run(gb)
    assert np.array_equal(ok == 0, is_bad) and (gok == 1).all()
    bi = np.flatnonzero(is_bad)
    assert (got["status"][bi] == INVALID).all() and (got["iters"][bi] == 0).all()
    assert (got["n_out"][bi] == 0).all() and (got["ok"][bi] == 0).all()
    _same(got, gwant, b, RAW, idx=np.flatnonzero(~is_bad), want_b=gb, want_idx=range(len(good)))
    host = pl.plan(gb, bounds_mode=IMPROVED, splines=planner.reference_splines(gb), want_bounds=True)
    _same(gwant, host, gb, RAW)


def test_argument_errors():
    """NULL pointers and a negative batch or total: PQP_ERR_ARG; a batch or total beyond the handle: PQP_ERR_CAPACITY;
    nothing is written either way.  IMPROVED without splines is still PQP_ERR_ARG."""
    import torch
    L = _lib.load()
    p = planner.PathPlanner(max_batch=4, max_total_points=240)
    try:
        b = synth.curvy_corridors(4, 60)
        dev = _dev()
        d = device.batch_to_device(b, dev)
        outs = [torch.full((240,), 7.0, dtype=torch.float64, device=dev),
                torch.full((240, 4), 7.0, dtype=torch.float64, device=dev),
                torch.full((240, 4), 7.0, dtype=torch.float64, device=dev), torch.full((4,), 5, dtype=torch.int32, device=dev)]
        good = [d["offsets"].data_ptr(), d["ref"].data_ptr()] + [t.data_ptr() for t in outs]

        def fit(batch, total, ptrs, h=p._h):
            return L.pqp_fit_splines_device(h, batch, total, *ptrs, None)
        for i in range(len(good)):
            bad = list(good)
            bad[i] = None
            assert fit(4, 240, bad) == ERR_ARG, i
        assert fit(-1, 240, good) == ERR_ARG
        assert fit(4, -1, good) == ERR_ARG
        assert fit(4, 240, good, h=None) == ERR_ARG
        assert fit(5, 240, good) == ERR_CAPACITY
        assert fit(4, 241, good) == ERR_CAPACITY
        assert fit(0, 0, [None] * 6) == 0
        torch.cuda.synchronize()
        assert all((_np(t) == (5 if t.dtype == torch.int32 else 7.0)).all() for t in outs)
        assert fit(4, 240, good) == 0
        torch.cuda.synchronize()
        assert (_np(outs[3]) == 1).all()
        # IMPROVED without splines: still refused by the plan entry
        p.set_map(synth.disc_field_map())
        with pytest.raises(planner.PqpError):
            p.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], max_n_points=60,
                          bounds_mode=IMPROVED)
    finally:
        p.close()
