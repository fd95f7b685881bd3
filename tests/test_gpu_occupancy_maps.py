"""GPU tests (run with -m gpu on an H100) of building distance maps on the device from occupancy grids:
pqp_set_maps_occupancy and pqp_set_maps_occupancy_device read back with pqp_get_map against the scipy recipe bit for bit;
the config-1 layer rebuilt from occupancy and planned on; many scenes planned from device-built maps against host layers;
CUDA graphs that capture the build with plan_device; argument errors; the C++ mirror."""
import os
import subprocess

import numpy as np
import pytest

from path_optimizer_b200 import _lib, device, planner, synth
from path_optimizer_b200.abi import ERR_ARG, OK, STATE_DTYPE, OccupancyMap
from path_optimizer_b200.solver import PqpError
from tests import test_occupancy_maps as cpu

pytestmark = pytest.mark.gpu
FRENET_TOL, FP_TOL = 1e-8, 1e-9
N_SCENES, N_CAND, N = 16, 16, 200


def _dev():
    import torch
    return torch.device("cuda", 0)


def _occ_map(occ, res, cx=0.0, cy=0.0):
    return dict(occupancy=occ, rows=occ.shape[0], cols=occ.shape[1], resolution=float(res), center_x=cx, center_y=cy)


def _on_device(maps):
    import torch
    return [dict(m, occupancy=torch.from_numpy(np.array(m["occupancy"], dtype=np.uint8, order="C")).to(_dev()))
            for m in maps]


def _check_layers(p, maps):
    import torch
    torch.cuda.synchronize()
    for k, m in enumerate(maps):
        cpu._same(p.get_map(k), cpu.expected(np.asarray(m["occupancy"]), m["resolution"]))


@pytest.fixture(scope="module")
def mixed_set():
    """Edge cases, random grids, two 1100 x 250 disc fields (0.2 m and 0.25 m) and the 495 x 497 config-1 grid."""
    maps = [_occ_map(occ, res) for _, occ, res in cpu.edge_grids()]
    maps += [_occ_map(occ, res, 3.0 * k, -1.0 * k) for k, (occ, res) in enumerate(cpu.random_grids(seed=7))]
    maps += [synth.disc_field_occupancy(), synth.disc_field_occupancy(resolution=0.25, seed=synth.BASE_SEED + 3,
                                                                      center=(40.0, -10.0))]
    occ, res, _ = cpu.config1_occupancy()
    maps.append(_occ_map(occ, res, 1.0, 2.0))
    return maps


def test_layers_bit_for_bit_host_and_device_entries(mixed_set):
    import torch
    p = planner.PathPlanner(max_batch=8, max_total_points=8 * 200)
    try:
        p.set_maps_occupancy(mixed_set)
        _check_layers(p, mixed_set)
        p.set_maps([dict(distance=np.zeros((3, 3), np.float32), rows=3, cols=3, resolution=0.2, center_x=0.0,
                         center_y=0.0)])
        dmaps = _on_device(mixed_set)
        p.set_maps_occupancy_device(dmaps)          # new layout
        _check_layers(p, mixed_set)
        rev = list(reversed(mixed_set))
        p.set_maps_occupancy(rev)                   # host entry, other layout
        _check_layers(p, rev)
        p.set_maps_occupancy_device(dmaps)          # the first layout again: laid out anew
        _check_layers(p, mixed_set)
        flipped = [dict(m, occupancy=np.asarray(m["occupancy"])[::-1].copy()) for m in mixed_set]
        for d, f in zip(dmaps, flipped):
            d["occupancy"].copy_(_on_device([f])[0]["occupancy"])
        torch.cuda.synchronize()                    # the NULL stream is the handle's stream to the library
        p.set_maps_occupancy_device(dmaps)          # same layout: launches only
        _check_layers(p, flipped)
    finally:
        p.close()


def test_large_grid_4096():
    rng = np.random.default_rng(11)
    occ = (rng.random((4096, 4096)) >= 0.0005).astype(np.uint8)
    m = _occ_map(occ, 0.1)
    p = planner.PathPlanner(max_batch=1, max_total_points=200)
    try:
        p.set_maps_occupancy([m])
        want = cpu.expected(occ, 0.1)
        cpu._same(p.get_map(0), want)
        # the same layout: the device entry only launches the transform, on other occupancy
        m2 = dict(m, occupancy=(rng.random((4096, 4096)) >= 0.002).astype(np.uint8))
        p.set_maps_occupancy_device(_on_device([m2]))
        _check_layers(p, [m2])
    finally:
        p.close()


def _config1():
    g = np.load(os.path.join(cpu.GOLDEN, "config1_benchmark_map.npz"))
    field = dict(distance=g["map_distance"], rows=int(g["image_shape"][0]), cols=int(g["image_shape"][1]),
                 resolution=float(g["map_geo"][0]), center_x=float(g["map_geo"][1]), center_y=float(g["map_geo"][2]))
    b = dict(n_points=g["n_points"], ref=g["ref"], x0=g["x0"], end_heading=g["end_heading"])
    b["offsets"] = np.array([0, int(g["n_points"][0])], dtype=np.int32)
    spl = dict(n_knots=np.array([len(g["knots"])], dtype=np.int32), knots=g["knots"], x_coef=g["x_coef"], y_coef=g["y_coef"])
    occ = dict(field, occupancy=(g["map_distance"] != 0).astype(np.uint8))
    del occ["distance"]
    return g, field, occ, b, spl


def test_config1_from_occupancy():
    """The rebuilt config-1 layer equals the fixture; plans on it equal plans on the fixture's layer bit for bit and meet
    the config-1 bar against the golden outputs."""
    g, field, occ, b, spl = _config1()
    p = planner.PathPlanner(max_batch=1, max_total_points=256)
    q = planner.PathPlanner(max_batch=1, max_total_points=256)
    try:
        p.set_maps_occupancy([occ])
        cpu._same(p.get_map(0), g["map_distance"])
        q.set_map(field)
        for mode, tag in ((planner.BOUNDS_IMPROVED, "improved"), (planner.BOUNDS_SIMPLE, "simple")):
            sp = spl if mode == planner.BOUNDS_IMPROVED else None
            r = p.plan(b, bounds_mode=mode, splines=sp, want_bounds=True)
            w = q.plan(b, bounds_mode=mode, splines=sp, want_bounds=True)
            for f in ("status", "iters", "n_out", "ok"):
                assert (r[f] == w[f]).all(), (tag, f)
            assert r["states"].tobytes() == w["states"].tobytes() and r["bounds"].tobytes() == w["bounds"].tobytes()
            assert r["status"][0] == g[f"plan_{tag}_status"][0] == 1 and r["iters"][0] == g[f"plan_{tag}_iters"][0]
            assert r["n_out"][0] == g[f"plan_{tag}_n_out"][0] and r["ok"][0] == 1
            assert np.abs(r["bounds"].view(np.float64) - g[f"bounds_{tag}"].view(np.float64)).max() <= FP_TOL
            for f in ("x", "y", "z", "k", "s"):
                assert np.abs(r["states"][f] - g[f"plan_{tag}_states"][f]).max() <= FRENET_TOL
    finally:
        p.close()
        q.close()


def _scene_occupancy(k, seed=synth.BASE_SEED):
    """Occupancy of synth.scene_map(k): the grids whose layers multi_map_batch plans on."""
    if k % 4 == 1:
        return synth.disc_field_occupancy(resolution=0.25, seed=seed + k, center=(35.0 + 10.0 * (k % 7), -20.0 + 3.0 * (k % 5)))
    return synth.disc_field_occupancy(seed=seed + k)


@pytest.fixture(scope="module")
def scenes():
    maps, b, mi = synth.multi_map_batch(N_SCENES, N_CAND, n=N, order="interleaved")
    occ = [_scene_occupancy(k) for k in range(N_SCENES)]
    for m, o in zip(maps, occ):
        assert synth.distance_layer(o["occupancy"], o["resolution"]).tobytes() == m["distance"].tobytes()
    total = int(b["offsets"][-1])
    b["ref"]["v"] = 4.0 + 3.0 * np.sin(np.arange(total) * 0.05)
    b["ref"]["a"] = 0.5 * np.cos(np.arange(total) * 0.05)
    pi = (np.arange(len(mi)) % 3).astype(np.int32)
    return maps, occ, b, mi, pi


def _host(r):
    import torch
    torch.cuda.synchronize()
    return dict(states=device.tensor_to_records(r["states"].reshape(-1, 7)), n_out=r["n_out"].cpu().numpy(),
                ok=r["ok"].cpu().numpy(), status=r["status"].cpu().numpy(), iters=r["iters"].cpu().numpy(),
                bounds=r["bounds"].cpu().numpy().tobytes())


def _same_plan(got, want):
    for f in ("n_out", "ok", "status", "iters"):
        assert (got[f] == want[f]).all(), f
    assert got["states"].tobytes() == want["states"].tobytes()
    assert got["bounds"] == want["bounds"]


@pytest.mark.parametrize("form", ["KP", "KPC", "K"])
def test_scenes_from_device_occupancy_equal_host_layers(scenes, form):
    """16 scenes x 16 candidates: set_maps_occupancy_device + plan_device(map_index) equals set_maps(host layers) + the
    same call bit for bit; once more with a parameter-set index."""
    import torch
    maps, occ, b, mi, pi = scenes
    dev = _dev()
    d = device.batch_to_device(b, dev)
    mi_t, pi_t = torch.from_numpy(mi).to(dev), torch.from_numpy(pi).to(dev)
    a = planner.PathPlanner(max_batch=len(mi), max_total_points=len(mi) * N)
    h = planner.PathPlanner(max_batch=len(mi), max_total_points=len(mi) * N)
    try:
        sets = synth.param_sets(3, seed=5)
        a.set_param_sets(sets)
        h.set_param_sets(sets)
        a.set_maps_occupancy_device(_on_device(occ))
        h.set_maps(maps)
        for kw in (dict(map_index=mi_t), dict(map_index=mi_t, param_index=pi_t)):
            run = [p.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], max_n_points=N,
                                 formulation=form, want_bounds=True, **kw) for p in (a, h)]
            got, want = _host(run[0]), _host(run[1])
            _same_plan(got, want)
            assert (got["status"] == 1).sum() >= len(mi) // 2
    finally:
        a.close()
        h.close()


def test_graphs_capture_the_build_with_the_plan(scenes):
    """set_maps_occupancy_device + plan_device captured in one graph: new occupancy written into the captured tensors
    replays like an uncaptured run; a layout change while capturing is refused and the capture completes; a replay after
    a host set_maps of another geometry leaves the new set unchanged and plans against it."""
    import torch
    maps, occ, b, mi, _ = scenes
    dev = _dev()
    d = device.batch_to_device(b, dev)
    mi_t = torch.from_numpy(mi).to(dev)
    p = planner.PathPlanner(max_batch=len(mi), max_total_points=len(mi) * N)
    ref = planner.PathPlanner(max_batch=len(mi), max_total_points=len(mi) * N)
    try:
        docc = _on_device(occ)

        def cycle():
            p.set_maps_occupancy_device(docc)
            return p.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], max_n_points=N,
                                 want_bounds=True, map_index=mi_t)
        cycle()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            res = cycle()
        # new occupancy: other seeds, same geometry
        occ2 = [_scene_occupancy(k, seed=synth.BASE_SEED + 101) for k in range(N_SCENES)]
        for t, o in zip(docc, occ2):
            t["occupancy"].copy_(torch.from_numpy(o["occupancy"]))
        g.replay()
        got = _host(res)
        _check_layers(p, occ2)
        ref.set_maps_occupancy(occ2)
        want = ref.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], max_n_points=N,
                               want_bounds=True, map_index=mi_t)
        _same_plan(got, _host(want))
        # a layout change while capturing: refused, the capture still completes
        g2 = torch.cuda.CUDAGraph()
        other = _on_device([_occ_map(np.ones((30, 40), np.uint8), 0.2)])
        with torch.cuda.graph(g2):
            with pytest.raises(PqpError):
                p.set_maps_occupancy_device(other)
            res2 = p.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], max_n_points=N,
                                 want_bounds=True, map_index=mi_t)
        g2.replay()
        _same_plan(_host(res2), _host(want))
        # a host set_maps with other geometry, then the old graph: the new set stays, the plan reads it
        new_maps = [synth.disc_field_map(rows=900, cols=300, seed=synth.BASE_SEED + 200 + k) for k in range(N_SCENES)]
        p.set_maps(new_maps)
        g.replay()
        got = _host(res)
        for k, m in enumerate(new_maps):
            assert p.get_map(k).tobytes() == m["distance"].tobytes(), k
        ref.set_maps(new_maps)
        want = ref.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], max_n_points=N,
                               want_bounds=True, map_index=mi_t)
        _same_plan(got, _host(want))
    finally:
        p.close()
        ref.close()


def test_argument_errors_leave_the_set(mixed_set):
    import torch
    L = _lib.load()
    p = planner.PathPlanner(max_batch=1, max_total_points=200)
    try:
        small = mixed_set[:3]
        p.set_maps_occupancy(small)
        cells = np.ones((4, 5), np.uint8)
        good = OccupancyMap(cells.ctypes.data, 4, 5, 0.2, 0.0, 0.0)
        tcells = torch.ones((4, 5), dtype=torch.uint8, device=_dev())
        dgood = OccupancyMap(tcells.data_ptr(), 4, 5, 0.2, 0.0, 0.0)
        for bad in (OccupancyMap(None, 4, 5, 0.2, 0.0, 0.0), OccupancyMap(cells.ctypes.data, 0, 5, 0.2, 0.0, 0.0),
                    OccupancyMap(cells.ctypes.data, 4, 0, 0.2, 0.0, 0.0), OccupancyMap(cells.ctypes.data, 4, 5, 0.0, 0.0, 0.0)):
            assert L.pqp_set_maps_occupancy(p._h, 2, cpu._occ_array([good, bad])) == ERR_ARG
            dbad = OccupancyMap(bad.cells and tcells.data_ptr(), bad.rows, bad.cols, bad.resolution, 0.0, 0.0)
            assert L.pqp_set_maps_occupancy_device(p._h, 2, cpu._occ_array([dgood, dbad]), None) == ERR_ARG
        for n in (0, -1):
            assert L.pqp_set_maps_occupancy(p._h, n, cpu._occ_array([good])) == ERR_ARG
            assert L.pqp_set_maps_occupancy_device(p._h, n, cpu._occ_array([dgood]), None) == ERR_ARG
        out = np.zeros(1 << 16, np.float32)
        for m in (-1, len(small), 1000):
            assert L.pqp_get_map(p._h, m, out.ctypes.data) == ERR_ARG
        assert L.pqp_get_map(p._h, 0, None) == ERR_ARG
        _check_layers(p, small)
        assert L.pqp_set_maps_occupancy(p._h, 1, cpu._occ_array([good])) == OK
        cpu._same(_raw(L, p, 0, (4, 5)), cpu.expected(cells, 0.2))
    finally:
        p.close()


def _raw(L, p, m, shape):
    out = np.empty(shape, np.float32)
    assert L.pqp_get_map(p._h, m, out.ctypes.data) == OK
    return out


def test_cpp_planner_occupancy_mirror(tmp_path, scenes):
    """include/pqp_planner.hpp: PathOptimizerGpu created from occupancy grids, getMap, the batched
    solveWithoutSmoothing with a map index per reference and setMaps, through tests/cpp/planner_occupancy_driver.cpp."""
    maps, occ, b, mi, _ = scenes
    n_maps = 4
    keep = np.flatnonzero(mi < n_maps)[:24]
    sub, smi = synth.take_paths(b, keep), mi[keep]
    occ, maps = occ[:n_maps], maps[:n_maps]
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.join(root, "path_optimizer_b200")
    exe = str(tmp_path / "planner_occupancy_driver")
    subprocess.run(["g++", "-O2", "-std=c++17", os.path.join(root, "tests", "cpp", "planner_occupancy_driver.cpp"), "-o",
                    exe, "-L" + libdir, "-lpqp", "-Wl,-rpath," + libdir], check=True)
    B = len(smi)
    veh = np.column_stack([sub["x0"], sub["end_heading"]])
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(fin, "wb") as f:
        f.write(np.int32(n_maps).tobytes())
        for m in occ:
            f.write(np.array([m["rows"], m["cols"]], dtype=np.int32).tobytes())
            f.write(np.array([m["resolution"], m["center_x"], m["center_y"]], dtype=np.float64).tobytes())
            f.write(np.ascontiguousarray(m["occupancy"], dtype=np.uint8).tobytes())
        f.write(np.int32(B).tobytes()); f.write(sub["n_points"].tobytes()); f.write(smi.tobytes())
        f.write(np.ascontiguousarray(sub["ref"]).tobytes()); f.write(np.ascontiguousarray(veh).tobytes())
    subprocess.run([exe, str(fin), str(fout)], check=True)
    raw = open(fout, "rb").read()
    o = 0
    for m in maps:
        n = m["rows"] * m["cols"] * 4
        assert raw[o:o + n] == m["distance"].tobytes()
        o += n
    n_out = np.frombuffer(raw, dtype=np.int32, count=B, offset=o)
    ok = np.frombuffer(raw, dtype=np.int32, count=B, offset=o + 4 * B)
    status = np.frombuffer(raw, dtype=np.int32, count=B, offset=o + 8 * B)
    o += 12 * B
    p = planner.PathPlanner(max_batch=B, max_total_points=int(sub["offsets"][-1]))
    try:
        p.set_maps(maps)
        want = p.plan(sub, map_index=smi)
    finally:
        p.close()
    assert (n_out == want["n_out"]).all() and (ok == want["ok"]).all() and (status == want["status"]).all()
    assert (want["status"] == 1).any()
    for i in range(B):
        lo = sub["offsets"][i]
        got = raw[o:o + STATE_DTYPE.itemsize * int(n_out[i])]
        o += len(got)
        assert got == want["states"][lo:lo + n_out[i]].tobytes(), i
    for m in reversed(maps):
        n = m["rows"] * m["cols"] * 4
        assert raw[o:o + n] == m["distance"].tobytes()
        o += n
    assert o == len(raw)
