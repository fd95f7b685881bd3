"""GPU tests (run with -m gpu on an H100) of planning one batch over several distance maps: pqp_set_maps with
pqp_plan_batch_maps / pqp_plan_batch_device_maps against pqp_plan_batch run per map after pqp_set_map (bit for bit) and
against the oracle with each path's own map; the device entry, CUDA graph replay across new inputs and a new map set;
a NULL index; indices outside the set; pqp_set_map after a set; argument errors; the C++ mirror.

Oracle tolerances are those of tests/test_gpu_env.py: identical status and iteration counts, 1e-8 on the states;
simple bounds bit for bit, improved bounds to 1e-9 (their offsets go through the device's sin/cos)."""
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle
from path_optimizer_b200 import _lib, device, planner, synth
from path_optimizer_b200.abi import BOUNDS_DTYPE, ERR_ARG, FORMULATIONS, OK, STATE_DTYPE, DistanceMap, ptr

pytestmark = pytest.mark.gpu
INVALID = -100
FRENET_TOL, FP_TOL = 1e-8, 1e-9
N_MAPS, N_CAND, N = 5, 12, 120
MIXED = dict(y_range=(-1.5, 1.5), heading_range=0.03, curvature_amp=0.01)


def _config1_map():
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "config1_benchmark_map.npz"))
    return dict(distance=g["map_distance"], rows=int(g["image_shape"][0]), cols=int(g["image_shape"][1]),
                resolution=float(g["map_geo"][0]), center_x=float(g["map_geo"][1]), center_y=float(g["map_geo"][2]))


def _with_speed(b):
    """v, a on the reference states (the KPC limits come from them)."""
    total = int(b["offsets"][-1])
    b["ref"]["v"] = 4.0 + 3.0 * np.sin(np.arange(total) * 0.05)
    b["ref"]["a"] = 0.5 * np.cos(np.arange(total) * 0.05)
    b["ref"]["v"][::13] = 0.0
    return b


@pytest.fixture(scope="module")
def scene():
    maps, b, mi = synth.multi_map_batch(N_MAPS, N_CAND, n=N, first_maps=[_config1_map()], order="interleaved", **MIXED)
    return maps, _with_speed(b), mi


@pytest.fixture(scope="module")
def multi(scene):
    p = planner.PathPlanner(max_batch=512, max_total_points=512 * N)
    p.set_maps(scene[0])
    yield p
    p.close()


@pytest.fixture(scope="module")
def single():
    p = planner.PathPlanner(max_batch=512, max_total_points=512 * N)
    yield p
    p.close()


def _np(t):
    return t.detach().cpu().numpy()


def _path_bits(r, b, i, output_mode):
    """RAW: the path's whole segment (stations past a cut read as zeros); DENSIFY: the samples it reports (the rest of
    its row is scratch)."""
    if output_mode == planner.OUTPUT_RAW:
        return r["states"][b["offsets"][i]:b["offsets"][i + 1]].tobytes()
    return r["states"][i, :r["n_out"][i]].tobytes()


def _same_path(got, gb, i, want, wb, k, output_mode, bounds=True):
    for f in ("n_out", "ok", "status", "iters"):
        assert got[f][i] == want[f][k], (f, i)
    assert _path_bits(got, gb, i, output_mode) == _path_bits(want, wb, k, output_mode), i
    if bounds:
        assert (got["bounds"][gb["offsets"][i]:gb["offsets"][i + 1]].tobytes()
                == want["bounds"][wb["offsets"][k]:wb["offsets"][k + 1]].tobytes()), i


def _spl(b, mode):
    return planner.reference_splines(b) if mode == planner.BOUNDS_IMPROVED else None


@pytest.mark.parametrize("output_mode", [planner.OUTPUT_RAW, planner.OUTPUT_DENSIFY])
@pytest.mark.parametrize("bounds_mode", [planner.BOUNDS_SIMPLE, planner.BOUNDS_IMPROVED])
@pytest.mark.parametrize("form", ["KP", "KPC", "K"])
def test_per_map_agreement(multi, single, scene, form, bounds_mode, output_mode):
    """pqp_plan_batch_maps over interleaved paths of five maps equals pqp_plan_batch run per map on that map's paths,
    bit for bit; for KP and K a sample of every map equals the oracle's plan on that map."""
    maps, b, mi = scene
    kw = dict(formulation=form, bounds_mode=bounds_mode, output_mode=output_mode, max_out=256, want_bounds=True)
    got = multi.plan(b, splines=_spl(b, bounds_mode), map_index=mi, **kw)
    assert (got["status"] == 1).sum() >= 10
    prm = oracle.default_params()
    for m in range(N_MAPS):
        idx = np.flatnonzero(mi == m)
        sub = synth.take_paths(b, idx)
        single.set_map(maps[m])
        want = single.plan(sub, splines=_spl(sub, bounds_mode), **kw)
        for k, i in enumerate(idx):
            _same_path(got, b, i, want, sub, k, output_mode)
        if form == "KPC":   # the chain's KPC limits are checked against pqp_plan_batch above, not the oracle's chain
            continue
        few = synth.take_paths(sub, [0, 1, 2])
        o = oracle.plan(prm, maps[m], few, formulation=FORMULATIONS[form], bounds_mode=bounds_mode,
                        splines=_spl(few, bounds_mode), output_mode=output_mode, max_out=256)
        nv = oracle.update_bounds(prm, maps[m], few, mode=bounds_mode, splines=_spl(few, bounds_mode))["n_valid"]
        for k in range(3):
            i = idx[k]
            assert got["status"][i] == o["status"][k] and got["iters"][i] == o["iters"][k]
            assert got["n_out"][i] == o["n_out"][k] and got["ok"][i] == o["ok"][k]
            c = o["n_out"][k]
            if output_mode == planner.OUTPUT_RAW:
                lo, lw = b["offsets"][i], few["offsets"][k]
                g, w = got["states"][lo:lo + c], o["states"][lw:lw + c]
            else:
                g, w = got["states"][i, :c], o["states"][k, :c]
            for f in ("x", "y", "z", "k", "s"):
                assert np.abs(g[f] - w[f]).max(initial=0.0) <= FRENET_TOL
            G = got["bounds"][b["offsets"][i]:b["offsets"][i] + nv[k]].view(np.float64)
            W = o["bounds"][few["offsets"][k]:few["offsets"][k] + nv[k]].view(np.float64)
            if bounds_mode == planner.BOUNDS_SIMPLE:
                assert G.tobytes() == W.tobytes()
            else:
                assert np.abs(G - W).max(initial=0.0) <= FP_TOL


def _plan_device(p, b, mi_t, mode, output_mode, d=None, spl=None, **kw):
    import torch
    dev = torch.device("cuda", 0)
    d = d or device.batch_to_device(b, dev)
    if spl is None and mode == planner.BOUNDS_IMPROVED:
        spl = device.splines_to_device(planner.reference_splines(b), dev)
    r = p.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], max_n_points=N, bounds_mode=mode,
                      splines=spl, output_mode=output_mode, max_out=256, want_bounds=True, map_index=mi_t, **kw)
    return d, spl, r


def _host(r, output_mode):
    import torch
    torch.cuda.synchronize()   # plan_device on torch's default stream is queued on the handle's own stream
    st = r["states"].reshape(-1, 7) if output_mode == planner.OUTPUT_RAW else r["states"]
    states = device.tensor_to_records(st)
    if output_mode == planner.OUTPUT_DENSIFY:
        states = states.reshape(r["states"].shape[0], -1)
    return dict(states=states, n_out=_np(r["n_out"]), ok=_np(r["ok"]), status=_np(r["status"]), iters=_np(r["iters"]),
                bounds=device.tensor_to_records(r["bounds"], BOUNDS_DTYPE))


@pytest.mark.parametrize("output_mode", [planner.OUTPUT_RAW, planner.OUTPUT_DENSIFY])
@pytest.mark.parametrize("bounds_mode", [planner.BOUNDS_SIMPLE, planner.BOUNDS_IMPROVED])
def test_device_entry_equals_host_entry(multi, scene, bounds_mode, output_mode):
    import torch
    maps, b, mi = scene
    want = multi.plan(b, bounds_mode=bounds_mode, splines=_spl(b, bounds_mode), output_mode=output_mode, max_out=256,
                      want_bounds=True, map_index=mi)
    _, _, r = _plan_device(multi, b, torch.from_numpy(mi).cuda(), bounds_mode, output_mode)
    got = _host(r, output_mode)
    for i in range(len(mi)):
        _same_path(got, b, i, want, b, i, output_mode)


def test_graph_replay_follows_new_inputs_and_a_new_map_set(scene):
    """Capture plan_device with a map index; write new candidates and indices into the captured buffers and replay;
    then upload a new set of maps of the same sizes and replay again: fresh host calls' results each time."""
    import torch
    maps, b, mi = scene
    p = planner.PathPlanner(max_batch=512, max_total_points=512 * N)
    try:
        p.set_maps(maps)
        dev = torch.device("cuda", 0)
        mi_t = torch.from_numpy(mi.copy()).to(dev)
        d, _, _ = _plan_device(p, b, mi_t, planner.BOUNDS_SIMPLE, planner.OUTPUT_RAW)   # warm-up
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            _, _, res = _plan_device(p, b, mi_t, planner.BOUNDS_SIMPLE, planner.OUTPUT_RAW, d=d)
        # new candidates (other lines, same station total) and a new assignment of paths to maps
        _, b2, _ = synth.multi_map_batch(N_MAPS, N_CAND, n=N, seed=synth.BASE_SEED + 77, first_maps=maps,
                                         order="interleaved", **MIXED)
        mi2 = np.random.default_rng(3).integers(0, N_MAPS, len(mi)).astype(np.int32)
        for k, t in device.batch_to_device(b2, dev).items():
            if k in d:
                d[k].copy_(t)
        mi_t.copy_(torch.from_numpy(mi2))
        g.replay()
        torch.cuda.synchronize()
        want = p.plan(b2, want_bounds=True, map_index=mi2)
        got = _host(res, planner.OUTPUT_RAW)
        for i in range(len(mi2)):
            _same_path(got, b2, i, want, b2, i, planner.OUTPUT_RAW)
        # a new map set of the same sizes (other obstacles): the table is rewritten in place
        new_maps = [dict(m, distance=np.ascontiguousarray(np.roll(m["distance"], 37 * (k + 1), axis=0)))
                    for k, m in enumerate(maps)]
        p.set_maps(new_maps)
        g.replay()
        torch.cuda.synchronize()
        want2 = p.plan(b2, want_bounds=True, map_index=mi2)
        got2 = _host(res, planner.OUTPUT_RAW)
        for i in range(len(mi2)):
            _same_path(got2, b2, i, want2, b2, i, planner.OUTPUT_RAW)
        assert (want2["n_out"] != want["n_out"]).any() or (want2["bounds"].tobytes() != want["bounds"].tobytes())
        del g
    finally:
        p.close()


@pytest.mark.parametrize("output_mode", [planner.OUTPUT_RAW, planner.OUTPUT_DENSIFY])
def test_null_index_is_map_zero(multi, single, scene, output_mode):
    maps, b, mi = scene
    single.set_map(maps[0])
    kw = dict(output_mode=output_mode, max_out=256, want_bounds=True)
    want = single.plan(b, **kw)
    for got in (multi.plan(b, **kw), multi.plan(b, map_index=np.zeros(len(mi), np.int32), **kw)):
        for i in range(len(mi)):
            _same_path(got, b, i, want, b, i, output_mode)
    _, _, r = _plan_device(multi, b, None, planner.BOUNDS_SIMPLE, output_mode)
    got = _host(r, output_mode)
    for i in range(len(mi)):
        _same_path(got, b, i, want, b, i, output_mode)


@pytest.mark.parametrize("output_mode", [planner.OUTPUT_RAW, planner.OUTPUT_DENSIFY])
@pytest.mark.parametrize("bad", [-1, N_MAPS])
def test_index_outside_the_set(multi, scene, bad, output_mode):
    """PQP_INVALID_PROBLEM, 0 iterations, ok = 0, n_out = 0 for those paths, on both entries; every other path keeps
    its bits."""
    import torch
    maps, b, mi = scene
    victims = [0, 7, len(mi) - 1]
    others = np.setdiff1d(np.arange(len(mi)), victims)
    bad_mi = mi.copy()
    bad_mi[victims] = bad
    kw = dict(output_mode=output_mode, max_out=256, want_bounds=True)
    good = multi.plan(b, map_index=mi, **kw)
    _, _, r = _plan_device(multi, b, torch.from_numpy(bad_mi).cuda(), planner.BOUNDS_SIMPLE, output_mode)
    for got in (multi.plan(b, map_index=bad_mi, **kw), _host(r, output_mode)):
        assert (got["status"][victims] == INVALID).all() and (got["iters"][victims] == 0).all()
        assert (got["ok"][victims] == 0).all() and (got["n_out"][victims] == 0).all()
        for i in others:
            _same_path(got, b, i, good, b, i, output_mode)


def test_set_map_after_set_maps(scene):
    """A pqp_set_map after a set leaves the single-map entries exactly as on a handle that only ever had that map."""
    maps, b, mi = scene
    field = maps[2]
    a = planner.PathPlanner(max_batch=512, max_total_points=512 * N)
    fresh = planner.PathPlanner(max_batch=512, max_total_points=512 * N)
    try:
        a.set_maps(maps)
        a.set_map(field)
        fresh.set_map(field)
        rng = np.random.default_rng(4)
        xy = np.stack([rng.uniform(-112, 112, 4000), rng.uniform(-26, 26, 4000)], 1)
        assert a.map_distance(xy).tobytes() == fresh.map_distance(xy).tobytes()
        assert a.check_states(b["ref"]).tobytes() == fresh.check_states(b["ref"]).tobytes()
        for mode in (planner.BOUNDS_SIMPLE, planner.BOUNDS_IMPROVED):
            u, v = a.update_bounds(b, mode=mode, splines=_spl(b, mode)), fresh.update_bounds(b, mode=mode, splines=_spl(b, mode))
            assert u["bounds"].tobytes() == v["bounds"].tobytes() and (u["n_valid"] == v["n_valid"]).all()
        n_points, paths = b["n_points"], b["ref"].copy()
        assert a.finish_raw(n_points, paths)["states"].tobytes() == fresh.finish_raw(n_points, paths)["states"].tobytes()
        u, v = a.densify(n_points, paths, max_out=256), fresh.densify(n_points, paths, max_out=256)
        assert u["states"].tobytes() == v["states"].tobytes() and (u["n_out"] == v["n_out"]).all()
        u, v = a.plan(b, want_bounds=True), fresh.plan(b, want_bounds=True)
        for i in range(len(mi)):
            _same_path(u, b, i, v, b, i, planner.OUTPUT_RAW)
        r = a.plan(b, map_index=np.ones(len(mi), np.int32))   # the set is gone: index 1 is outside a set of one
        assert (r["status"] == INVALID).all() and (r["n_out"] == 0).all()
    finally:
        a.close()
        fresh.close()


def test_argument_errors(scene):
    maps, b, mi = scene
    L = _lib.load()
    p = planner.PathPlanner(max_batch=512, max_total_points=512 * N)
    try:
        # no map set: both entries refuse
        B, T = len(mi), int(b["offsets"][-1])
        out = np.zeros(T, dtype=STATE_DTYPE)
        n_out, ok, st, it = (np.zeros(B, np.int32) for _ in range(4))
        ref, n_points = np.ascontiguousarray(b["ref"]), np.ascontiguousarray(b["n_points"])
        x0, eh = np.ascontiguousarray(b["x0"]), np.ascontiguousarray(b["end_heading"])
        assert L.pqp_plan_batch_maps(p._h, 0, planner.BOUNDS_SIMPLE, planner.OUTPUT_RAW, B, ptr(n_points), ptr(ref),
                                     ptr(mi), None, None, None, None, ptr(x0), ptr(eh), 0.3, 1, 256, ptr(out),
                                     ptr(n_out), ptr(ok), ptr(st), ptr(it), None, None) == ERR_ARG
        import torch
        d = device.batch_to_device(b, torch.device("cuda", 0))
        mi_t = torch.from_numpy(mi).cuda()
        o = torch.empty((T, 7), dtype=torch.float64, device="cuda")
        i32 = [torch.empty(B, dtype=torch.int32, device="cuda") for _ in range(3)]
        assert L.pqp_plan_batch_device_maps(p._h, 0, planner.BOUNDS_SIMPLE, planner.OUTPUT_RAW, B, T, N,
                                            d["n_points"].data_ptr(), d["offsets"].data_ptr(), d["ref"].data_ptr(),
                                            mi_t.data_ptr(), None, None, None, None, d["x0"].data_ptr(),
                                            d["end_heading"].data_ptr(), 0.3, 1, 256, o.data_ptr(), i32[0].data_ptr(),
                                            i32[1].data_ptr(), i32[2].data_ptr(), None, None, None, None) == ERR_ARG
        torch.cuda.synchronize()
        # bad sets: nothing changes
        p.set_maps(maps)
        before = p.plan(b, map_index=mi, want_bounds=True)
        keep = []

        def dms(ms):
            arr = (DistanceMap * len(ms))()
            for k, m in enumerate(ms):
                dist = np.ascontiguousarray(m["distance"], dtype=np.float32)
                keep.append(dist)
                arr[k] = DistanceMap(ptr(dist), dist.shape[0], dist.shape[1], float(m["resolution"]),
                                     float(m["center_x"]), float(m["center_y"]))
            return arr
        good = dms(maps[:2])
        assert L.pqp_set_maps(p._h, 0, good) == ERR_ARG
        assert L.pqp_set_maps(p._h, -1, good) == ERR_ARG
        assert L.pqp_set_maps(p._h, 2, None) == ERR_ARG
        assert L.pqp_set_maps(None, 2, good) == ERR_ARG
        for field, value in (("distance", None), ("rows", 0), ("cols", -3), ("resolution", 0.0), ("resolution", -0.2)):
            bad = dms(maps[:3])
            setattr(bad[2], field, value)
            assert L.pqp_set_maps(p._h, 3, bad) == ERR_ARG, field
        after = p.plan(b, map_index=mi, want_bounds=True)
        for i in range(len(mi)):
            _same_path(after, b, i, before, b, i, planner.OUTPUT_RAW)
        assert L.pqp_set_maps(p._h, 2, good) == OK
        with pytest.raises(Exception):
            p.plan(b, map_index=mi[:-1])                # wrong length
    finally:
        p.close()


def test_cpp_planner_maps_mirror(tmp_path):
    """include/pqp_planner.hpp: PathOptimizerGpu built from two maps and the batched solveWithoutSmoothing with a map
    index per reference, through tests/cpp/planner_maps_driver.cpp; results equal PathPlanner.plan(..., map_index)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.join(root, "path_optimizer_b200")
    exe = str(tmp_path / "planner_maps_driver")
    subprocess.run(["g++", "-O2", "-std=c++17", os.path.join(root, "tests", "cpp", "planner_maps_driver.cpp"), "-o", exe,
                    "-L" + libdir, "-lpqp", "-Wl,-rpath," + libdir], check=True)
    maps, b, mi = synth.multi_map_batch(2, 8, n=90, first_maps=[_config1_map()], order="interleaved",
                                        y_range=(-1.0, 1.0), heading_range=0.03, curvature_amp=0.008)
    B = len(mi)
    veh = np.column_stack([b["x0"], b["end_heading"]])
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(fin, "wb") as f:
        f.write(np.int32(len(maps)).tobytes())
        for m in maps:
            f.write(np.array([m["rows"], m["cols"]], dtype=np.int32).tobytes())
            f.write(np.array([m["resolution"], m["center_x"], m["center_y"]], dtype=np.float64).tobytes())
            f.write(np.ascontiguousarray(m["distance"], dtype=np.float32).tobytes())
        f.write(np.int32(B).tobytes()); f.write(b["n_points"].tobytes()); f.write(mi.tobytes())
        f.write(np.ascontiguousarray(b["ref"]).tobytes()); f.write(np.ascontiguousarray(veh).tobytes())
    subprocess.run([exe, str(fin), str(fout)], check=True)
    raw = open(fout, "rb").read()
    n_out = np.frombuffer(raw, dtype=np.int32, count=B)
    ok = np.frombuffer(raw, dtype=np.int32, count=B, offset=4 * B)
    status = np.frombuffer(raw, dtype=np.int32, count=B, offset=8 * B)
    p = planner.PathPlanner(max_batch=B, max_total_points=int(b["offsets"][-1]))
    try:
        p.set_maps(maps)
        want = p.plan(b, map_index=mi)
    finally:
        p.close()
    assert (n_out == want["n_out"]).all() and (ok == want["ok"]).all() and (status == want["status"]).all()
    assert (want["status"] == 1).any() and set(mi.tolist()) == {0, 1}
    o = 12 * B
    for i in range(B):
        got = raw[o:o + STATE_DTYPE.itemsize * int(n_out[i])]
        o += len(got)
        lo = b["offsets"][i]
        assert got == want["states"][lo:lo + n_out[i]].tobytes(), i
