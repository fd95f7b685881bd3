"""GPU tests (run with -m gpu on an H100) of the device-side class dispatch and the device-resident plan chain:
pqp_solve_batch_device_dispatch against pqp_solve_batch and pqp_plan_batch_device against pqp_plan_batch, bit for bit,
at the ends and partition edges of every class; stated bounds; CUDA graph capture and replay; argument errors."""
import ctypes as C
import os

import numpy as np
import pytest

from path_optimizer_b200 import _lib, device, planner, synth
from path_optimizer_b200.abi import ERR_ARG, ERR_CAPACITY, STATE_DTYPE
from tests import shapes

pytestmark = pytest.mark.gpu
INVALID = -100
WILD = dict(y_range=(-3.0, 3.0), heading_range=0.05, curvature_amp=0.02)


@pytest.fixture(scope="module")
def solver():
    from path_optimizer_b200.solver import BatchPathSolver
    s = BatchPathSolver(max_batch=1024, max_total_points=1024 * 400)
    yield s
    s.close()


@pytest.fixture(scope="module")
def field():
    return synth.disc_field_map()


@pytest.fixture(scope="module")
def pl(field):
    p = planner.PathPlanner(max_batch=256, max_total_points=256 * 400)
    p.set_map(field)
    yield p
    p.close()


def _u64(a):
    return np.ascontiguousarray(a).view(np.uint64).reshape(-1)


def _np(t):
    return t.detach().cpu().numpy()


def _respace(b, ds):
    o = b["offsets"]
    for i, n in enumerate(b["n_points"]):
        b["ref"]["s"][o[i]:o[i + 1]] = synth._accumulate_s(int(n), ds)
    return b


def _with_short(b):
    """Paths of 0 and 1 stations in front of the batch."""
    out = dict(n_points=np.r_[[0, 1], b["n_points"]].astype(np.int32), ref=np.r_[b["ref"][:1], b["ref"]],
               bounds=np.r_[b["bounds"][:1], b["bounds"]], x0=np.r_[np.zeros((1, 3)), b["x0"][:1], b["x0"]],
               end_heading=np.r_[[0.0], b["end_heading"][:1], b["end_heading"]])
    out["offsets"] = np.r_[0, np.cumsum(out["n_points"])].astype(np.int32)
    return out


def _kpc_limits(b):
    total = int(b["offsets"][-1])
    b["ref"]["v"] = 4.0 + 3.0 * np.sin(np.arange(total) * 0.05)
    b["ref"]["a"] = 0.5 * np.cos(np.arange(total) * 0.05)
    b["ref"]["v"][::13] = 0.0
    from oracle import oracle
    return oracle.update_limits(oracle.default_params(), b["ref"])


def _lengths(form, keep):
    """Both ends of every class at this keep, the partition edges of the thread-per-station classes, and 1 station past
    the longest path (paths of 0 and 1 stations come from _with_short)."""
    out = set()
    for name, (lo, hi) in shapes.class_ranges(form, keep).items():
        out.update((lo, hi))
        if name.startswith("pqp_kp3_solve_kernel"):
            mmax = int(name.split(",")[3].rstrip(">KPC"))
            out.update(shapes.partition_edges(lo, hi, lambda n: shapes.kp3_partition(n, keep, mmax)))
        elif name in ("pqp_kk_solve_kernel<4>", "pqp_kk_solve_kernel<8>"):
            ms = 26 if name.endswith("<4>") else 32
            out.update(shapes.partition_edges(lo, hi, lambda n: shapes.kk_partition(n, ms)))
    out.add(shapes.max_points(form, keep) + 1)
    return sorted(out)


def _batch(form, keep):
    lengths = _lengths(form, keep)
    b = synth.curvy_corridors(len(lengths), n_points=np.array(lengths, dtype=np.int32), first_path=100 * keep)
    if form == shapes.KP:
        _respace(b, 1.2 / (keep + 0.5))
    b = _with_short(b)
    mk = mkp = None
    if form == shapes.KPC:
        mk, mkp = _kpc_limits(b)
    return b, mk, mkp


def _dispatch(s, form, b, mk=None, mkp=None, **bounds):
    import torch
    dev = torch.device("cuda", 0)
    d = device.batch_to_device(b, dev)
    dmk = torch.from_numpy(mk).to(dev) if mk is not None else None
    dmkp = torch.from_numpy(mkp).to(dev) if mkp is not None else None
    r = s.solve_device(d["n_points"], d["offsets"], d["ref"], d["bounds"], d["x0"], d["end_heading"], formulation=form,
                       max_k=dmk, max_kp=dmkp, **bounds)
    torch.cuda.synchronize()
    return dict(states=device.tensor_to_records(r["states"]), frenet=_np(r["frenet"]), status=_np(r["status"]),
                iters=_np(r["iters"]))


def _same_bits(a, b, idx, rows):
    assert np.array_equal(a["status"][idx], b["status"][idx]), (a["status"][idx], b["status"][idx])
    assert np.array_equal(a["iters"][idx], b["iters"][idx])
    assert np.array_equal(_u64(a["frenet"][rows]), _u64(b["frenet"][rows]))
    assert np.array_equal(_u64(a["states"][rows]), _u64(b["states"][rows]))


def _rows(b, idx):
    o = b["offsets"]
    return np.concatenate([np.arange(o[i], o[i + 1]) for i in idx] + [np.zeros(0, dtype=np.int64)]).astype(np.int64)


def _check_rejected(res, b, idx):
    for i in idx:
        sl = slice(b["offsets"][i], b["offsets"][i + 1])
        assert res["status"][i] == INVALID and res["iters"][i] == 0, (i, res["status"][i])
        assert np.isnan(res["frenet"][sl]).all()
        for f in "xyzks":
            assert np.isnan(res["states"][f][sl]).all()


def _cases():
    return ([("KP", shapes.KP, k) for k in shapes.kp_keeps()] + [("K", shapes.K, 1), ("KPC", shapes.KPC, 4)])


@pytest.mark.parametrize("name,form,keep", _cases(), ids=[f"{n}-keep{k}" for n, _, k in _cases()])
def test_dispatch_equals_host_entry(solver, name, form, keep):
    """Every class at both ends and its partition edges, 0 / 1 / limit + 1 stations, in one mixed batch: the device
    dispatch gives the host entry's bits with unknown bounds and with bounds set exactly; tighter bounds turn the paths
    beyond them into INVALID_PROBLEM and leave every other path's bits alone; a repeat call gives the same bits."""
    b, mk, mkp = _batch(form, keep)
    n = b["n_points"]
    B = len(n)
    keeps = np.array([shapes.keep_of(form, b["ref"][b["offsets"][i]:b["offsets"][i + 1]]) for i in range(B)])
    assert (keeps[n >= 5] == keep).all()
    host = solver.solve(b, formulation=form, max_k=mk, max_kp=mkp)
    every, all_rows = np.arange(B), np.arange(int(b["offsets"][-1]))
    assert (host["status"][n == n.max()] == INVALID).all() and (host["status"][n < 2] == INVALID).all()
    got = _dispatch(solver, form, b, mk, mkp)
    _same_bits(got, host, every, all_rows)
    _same_bits(_dispatch(solver, form, b, mk, mkp), got, every, all_rows)
    k_lo, k_hi = int(keeps.min()), int(keeps.max())
    _same_bits(_dispatch(solver, form, b, mk, mkp, max_n_points=int(n.max()), min_keep=k_lo, max_keep=k_hi), host,
               every, all_rows)
    # tight bounds: the longest valid class ends one station short, and (KP) only the main keep
    top = int(n[host["status"] != INVALID].max())
    tight = dict(max_n_points=top - 1, min_keep=keep, max_keep=keep)
    out = (n > top - 1) | ((keeps != keep) if form == shapes.KP else False)
    assert (out & (host["status"] != INVALID)).any()
    res = _dispatch(solver, form, b, mk, mkp, **tight)
    inside = np.nonzero(~out)[0]
    _same_bits(res, host, inside, _rows(b, inside))
    _check_rejected(res, b, np.nonzero(out)[0])


def _plan_batch(form, B=48, perm=None, first_path=0):
    n_points = synth.mixed_lengths(B, 20, 400 if form == shapes.KP else 300)
    if perm is not None:
        n_points = n_points[perm]
    return synth.map_reference_paths(B, n_points=n_points, first_path=first_path, **WILD)


def _plan_device(p, form, b, bounds_mode, output_mode, max_out=256, out=None, max_n=None):
    import torch
    dev = torch.device("cuda", 0)
    d = device.batch_to_device(b, dev)
    spl = device.splines_to_device(planner.reference_splines(b), dev) if bounds_mode == planner.BOUNDS_IMPROVED else None
    return d, spl, p.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"],
                                 max_n_points=int(b["n_points"].max()) if max_n is None else max_n, formulation=form,
                                 bounds_mode=bounds_mode, splines=spl, output_mode=output_mode, max_out=max_out,
                                 want_bounds=True, out=out)


def _plan_same(got, want, b, output_mode):
    import torch
    torch.cuda.synchronize()
    for k in ("n_out", "ok", "status", "iters"):
        assert np.array_equal(_np(got[k]), want[k]), (k, _np(got[k]), want[k])
    assert np.array_equal(_u64(_np(got["bounds"])), _u64(want["bounds"]))
    gs = _np(got["states"])
    if output_mode == planner.OUTPUT_RAW:
        assert np.array_equal(_u64(gs), _u64(want["states"]))
    else:
        ws = want["states"].view(np.float64).reshape(len(b["n_points"]), -1, 7)
        for i, m in enumerate(want["n_out"]):
            assert np.array_equal(_u64(gs[i, :m]), _u64(ws[i, :m])), i


@pytest.mark.parametrize("output_mode", [planner.OUTPUT_RAW, planner.OUTPUT_DENSIFY], ids=["raw", "densify"])
@pytest.mark.parametrize("bounds_mode", [planner.BOUNDS_SIMPLE, planner.BOUNDS_IMPROVED], ids=["simple", "improved"])
@pytest.mark.parametrize("name", ["KP", "KPC", "K"])
def test_plan_device_equals_host_chain(pl, name, bounds_mode, output_mode):
    """Mixed lengths on the config-3 map (blocking shortens many paths, some onto another kernel class): the device chain
    gives pqp_plan_batch's states, out_n, out_ok, status, iterations and bounds bit for bit."""
    form = {"KP": shapes.KP, "K": shapes.K, "KPC": shapes.KPC}[name]
    b = _plan_batch(form)
    spl = planner.reference_splines(b) if bounds_mode == planner.BOUNDS_IMPROVED else None
    want = pl.plan(b, formulation=name, bounds_mode=bounds_mode, splines=spl, output_mode=output_mode, max_out=256,
                   want_bounds=True)
    _, _, got = _plan_device(pl, name, b, bounds_mode, output_mode)
    _plan_same(got, want, b, output_mode)
    # blocking moved at least one path onto another kernel class than its full length would take
    nv = pl.update_bounds(b, mode=bounds_mode, splines=spl)["n_valid"]
    o = b["offsets"]
    moved = 0
    for i, (n, m) in enumerate(zip(b["n_points"], nv)):
        k_full = shapes.keep_of(form, b["ref"][o[i]:o[i] + n])
        k_cut = shapes.keep_of(form, b["ref"][o[i]:o[i] + m])
        moved += shapes.class_of(form, n, k_full)[0] != shapes.class_of(form, m, k_cut)[0]
    assert (nv < b["n_points"]).any() and moved > 0


def test_plan_device_config1_golden():
    """BASELINE config 1 (the reference's benchmark map and path): device chain = host chain, both bounds variants."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "config1_benchmark_map.npz"))
    field = dict(distance=g["map_distance"], rows=int(g["image_shape"][0]), cols=int(g["image_shape"][1]),
                 resolution=float(g["map_geo"][0]), center_x=float(g["map_geo"][1]), center_y=float(g["map_geo"][2]))
    b = dict(n_points=g["n_points"], ref=g["ref"], x0=g["x0"], end_heading=g["end_heading"])
    b["offsets"] = np.array([0, int(g["n_points"][0])], dtype=np.int32)
    spl = dict(n_knots=np.array([len(g["knots"])], dtype=np.int32), knots=g["knots"], x_coef=g["x_coef"], y_coef=g["y_coef"])
    p = planner.PathPlanner(max_batch=1, max_total_points=256)
    p.set_map(field)
    import torch
    dev = torch.device("cuda", 0)
    try:
        for mode in (planner.BOUNDS_IMPROVED, planner.BOUNDS_SIMPLE):
            sp = spl if mode == planner.BOUNDS_IMPROVED else None
            want = p.plan(b, bounds_mode=mode, splines=sp, want_bounds=True)
            d = device.batch_to_device(b, dev)
            got = p.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"],
                                max_n_points=int(b["n_points"][0]), bounds_mode=mode,
                                splines=device.splines_to_device(sp, dev) if sp else None, want_bounds=True)
            _plan_same(got, want, b, planner.OUTPUT_RAW)
            assert int(_np(got["ok"])[0]) == 1
    finally:
        p.close()


def _copy_into(static, fresh):
    for k, t in fresh.items():
        if t is not None and static.get(k) is not None:
            static[k].copy_(t)


def test_plan_device_graph_replay(pl):
    """One warm-up call, capture plan_device in a CUDA graph, copy a new batch (same path count and station total, other
    lengths and paths) into the captured inputs, replay: pqp_plan_batch's results on the new batch."""
    import torch
    B = 48
    first = _plan_batch(shapes.KP, B)
    second = _plan_batch(shapes.KP, B, perm=np.random.default_rng(5).permutation(B), first_path=777)
    assert int(first["offsets"][-1]) == int(second["offsets"][-1])
    max_n = int(max(first["n_points"].max(), second["n_points"].max()))
    dev = torch.device("cuda", 0)
    for mode in (planner.BOUNDS_SIMPLE, planner.BOUNDS_IMPROVED):
        d, spl, _ = _plan_device(pl, "KP", first, mode, planner.OUTPUT_RAW, max_n=max_n)   # warm-up
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            res = pl.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], max_n_points=max_n,
                                 bounds_mode=mode, splines=spl, want_bounds=True)
        d2 = device.batch_to_device(second, dev)
        _copy_into(d, d2)
        if spl is not None:
            spl2 = device.splines_to_device(planner.reference_splines(second), dev)
            assert spl2["knots"].shape == spl["knots"].shape
            _copy_into(spl, spl2)
        g.replay()
        torch.cuda.synchronize()   # (one call in flight per handle: the host chain below uses the same handle)
        sp2 = planner.reference_splines(second) if mode == planner.BOUNDS_IMPROVED else None
        want = pl.plan(second, bounds_mode=mode, splines=sp2, want_bounds=True)
        _plan_same(res, want, second, planner.OUTPUT_RAW)
        del g


def test_solve_device_graph_replay(solver):
    """The same for solve_device on a mixed 50..400-station batch (BASELINE config 5 lengths)."""
    import torch
    B = 256
    n1 = synth.mixed_lengths(B, 50, 400)
    n2 = n1[np.random.default_rng(9).permutation(B)]
    first = synth.curvy_corridors(B, n_points=n1)
    second = synth.curvy_corridors(B, n_points=n2, first_path=5000)
    dev = torch.device("cuda", 0)
    d = device.batch_to_device(first, dev)
    args = (d["n_points"], d["offsets"], d["ref"], d["bounds"], d["x0"], d["end_heading"])
    solver.solve_device(*args, max_n_points=400)      # warm-up
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        res = solver.solve_device(*args, max_n_points=400)
    _copy_into(d, device.batch_to_device(second, dev))
    g.replay()
    torch.cuda.synchronize()
    want = solver.solve(second)
    got = dict(states=device.tensor_to_records(res["states"]), frenet=_np(res["frenet"]), status=_np(res["status"]),
               iters=_np(res["iters"]))
    _same_bits(got, want, np.arange(B), np.arange(int(second["offsets"][-1])))
    del g


def test_argument_errors(solver, pl):
    """Null pointers, an unknown formulation, batch or station total beyond the handle: the codes of
    pqp_solve_batch_device."""
    import torch
    L = _lib.load()
    dev = torch.device("cuda", 0)
    b = synth.curvy_corridors(4, 60)
    d = device.batch_to_device(b, dev)
    out = torch.empty((240, 7), dtype=torch.float64, device=dev)
    st = torch.empty(4, dtype=torch.int32, device=dev)
    p = [t.data_ptr() for t in (d["n_points"], d["offsets"], d["ref"], d["bounds"], d["x0"], d["end_heading"])]

    def both(form, batch, total, ptrs):
        args = (form, batch, total, 60, 3, 3, *ptrs[:6], None, None, ptrs[6], None, ptrs[7], None, None, None)
        return (L.pqp_solve_batch_device(solver._h, *args), L.pqp_solve_batch_device_dispatch(solver._h, *args))
    good = p + [out.data_ptr(), st.data_ptr()]
    assert both(0, 4, 240, good) == (0, 0)
    for i in range(8):
        bad = list(good)
        bad[i] = None
        assert both(0, 4, 240, bad) == (ERR_ARG, ERR_ARG), i
    assert both(7, 4, 240, good) == (ERR_ARG, ERR_ARG)
    assert both(2, 4, 240, good) == (ERR_ARG, ERR_ARG)          # KPC without limits
    assert both(0, 1025, 240, good) == (ERR_CAPACITY, ERR_CAPACITY)
    assert both(0, 4, 1024 * 400 + 1, good) == (ERR_CAPACITY, ERR_CAPACITY)
    torch.cuda.synchronize()

    # the plan chain: the same codes
    n_out = torch.empty(4, dtype=torch.int32, device=dev)
    ok = torch.empty(4, dtype=torch.int32, device=dev)

    def plan(form, batch, total, ptrs, bounds_mode=planner.BOUNDS_SIMPLE):
        return L.pqp_plan_batch_device(pl._h, form, bounds_mode, planner.OUTPUT_RAW, batch, total, 60, ptrs[0], ptrs[1],
                                       ptrs[2], None, None, None, None, ptrs[3], ptrs[4], 0.3, 1, 512, ptrs[5], ptrs[6],
                                       ptrs[7], ptrs[8], None, None, None, None)
    pp = [p[0], p[1], p[2], p[4], p[5], out.data_ptr(), n_out.data_ptr(), ok.data_ptr(), st.data_ptr()]
    assert plan(0, 4, 240, pp) == 0
    for i in range(len(pp)):
        bad = list(pp)
        bad[i] = None
        assert plan(0, 4, 240, bad) == ERR_ARG, i
    assert plan(0, 4, 240, pp, bounds_mode=planner.BOUNDS_IMPROVED) == ERR_ARG   # no splines
    assert plan(7, 4, 240, pp) == ERR_ARG
    assert plan(0, 257, 240, pp) == ERR_CAPACITY
    assert plan(0, 4, 256 * 400 + 1, pp) == ERR_CAPACITY
    torch.cuda.synchronize()
