"""GPU tests (run with -m gpu on an H100) of solving and planning one batch over several parameter sets: pqp_set_param_sets
with pqp_solve_batch_sets, pqp_solve_batch_device_dispatch_sets, pqp_plan_batch_sets and pqp_plan_batch_device_sets
against a handle whose only set is the path's own (bit for bit) and against the oracle with each path's own params; a
NULL index and a single set against the existing entries; indices outside the sets; CUDA graphs across new inputs, new
indices and new sets; argument errors; the C++ mirror.

The sets (synth.param_sets) differ in every group the stages read: vehicle geometry (radius, d1..d4), wheel base and
steering limit, a nonzero KP_deviation_weight and the K weights, expected_safety_margin, constraint_end_heading = 0, the
KPC limits (mu, curvature rate), and the OSQP settings (tight tolerances with adaptive_rho_interval = 100; a max_iter
that ends paths with PQP_MAX_ITER_REACHED).  Oracle tolerances are those of tests/test_gpu_env.py."""
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle
from path_optimizer_b200 import _lib, device, planner, solver, synth
from path_optimizer_b200.abi import BOUNDS_DTYPE, ERR_ARG, FORMULATIONS, OK, STATE_DTYPE, Params
from tests import shapes
from tests.device_entries import rows, u64

pytestmark = pytest.mark.gpu
INVALID, MAX_ITER = -100, -2
FRENET_TOL, FP_TOL = 1e-8, 1e-9
S = 6
N_MAPS, N_CAND, N = 3, 12, 120
MIXED = dict(y_range=(-1.5, 1.5), heading_range=0.03, curvature_amp=0.01)
# path lengths of the solve batches: short and long classes of every formulation; KP also a path at 0.2 m spacing
# (keep_control_steps 5..6, the one-warp kernel)
LENGTHS = {"KP": [20, 60, 100, 150, 230, 300, 400, 100], "KPC": [20, 60, 128, 129, 200, 256], "K": [20, 90, 200, 300, 416]}


@pytest.fixture(scope="module")
def sets():
    return synth.param_sets(S, seed=11)


def _solve_batch(form):
    lens = LENGTHS[form]
    b = synth.curvy_corridors(len(lens) * S, n_points=np.tile(lens, S).astype(np.int32), seed=synth.BASE_SEED + 5)
    if form == "KP":   # the last length of each round at 0.2 m spacing
        for i in range(len(lens) - 1, len(b["n_points"]), len(lens)):
            o, n = b["offsets"][i], b["n_points"][i]
            b["ref"]["s"][o:o + n] = np.arange(n) * 0.2
    return b


def _limits(b):
    total = int(b["offsets"][-1])
    ref = b["ref"].copy()
    ref["v"] = 4.0 + 3.0 * np.sin(np.arange(total) * 0.05)
    ref["a"] = 0.5 * np.cos(np.arange(total) * 0.05)
    return planner.update_limits(solver.default_params(), ref)


def _index(B, seed=1):
    pi = np.arange(B, dtype=np.int32) % S
    np.random.default_rng(seed).shuffle(pi)
    return pi


@pytest.fixture(scope="module")
def multi(sets):
    s = planner.PathPlanner(max_batch=512, max_total_points=512 * 420)
    s.set_param_sets(sets)
    yield s
    s.close()


@pytest.fixture(scope="module")
def single():
    s = planner.PathPlanner(max_batch=512, max_total_points=512 * 420)
    yield s
    s.close()


def _same_solve(got, want, i, k, gb, wb):
    assert got["status"][i] == want["status"][k] and got["iters"][i] == want["iters"][k], i
    g, w = slice(gb["offsets"][i], gb["offsets"][i + 1]), slice(wb["offsets"][k], wb["offsets"][k + 1])
    assert u64(got["states"][g]).tobytes() == u64(want["states"][w]).tobytes(), i
    assert u64(got["frenet"][g]).tobytes() == u64(want["frenet"][w]).tobytes(), i


@pytest.mark.parametrize("form", ["KP", "KPC", "K"])
def test_solve_sets_per_set_bits_and_oracle(multi, single, sets, form):
    """pqp_solve_batch_sets over six sets equals a one-set handle solving only that set's paths, bit for bit; a sample of
    every set equals the oracle with that set's params."""
    b = _solve_batch(form)
    B = len(b["n_points"])
    mk, mkp = _limits(b) if form == "KPC" else (None, None)
    pi = _index(B)
    got = multi.solve(b, form, max_k=mk, max_kp=mkp, param_index=pi)
    assert (got["status"] == MAX_ITER).any()
    assert len(set(got["iters"][got["status"] == 1].tolist())) > 3
    for k in range(S):
        idx = np.flatnonzero(pi == k)
        sub = synth.take_paths(b, idx)
        r = rows(b, idx)
        single.set_params(sets[k])
        want = single.solve(sub, form, max_k=None if mk is None else mk[r], max_kp=None if mkp is None else mkp[r])
        for j, i in enumerate(idx):
            _same_solve(got, want, i, j, b, sub)
        few = idx[:2]
        fb = synth.take_paths(b, few)
        fr = rows(b, few)
        o = oracle.solve_batch(sets[k], FORMULATIONS[form], fb, max_k=None if mk is None else mk[fr],
                               max_kp=None if mkp is None else mkp[fr])
        shapes.assert_matches(got, o, few, fr, fb["n_points"], (form, k))


@pytest.mark.parametrize("form", ["KP", "KPC", "K"])
def test_dispatch_sets_equals_host_entry(multi, form):
    import torch
    b = _solve_batch(form)
    B = len(b["n_points"])
    mk, mkp = _limits(b) if form == "KPC" else (None, None)
    pi = _index(B, seed=2)
    want = multi.solve(b, form, max_k=mk, max_kp=mkp, param_index=pi)
    dev = torch.device("cuda", 0)
    d = device.batch_to_device(b, dev)
    t = (lambda a: None if a is None else torch.from_numpy(a).to(dev))
    r = multi.solve_device(d["n_points"], d["offsets"], d["ref"], d["bounds"], d["x0"], d["end_heading"], formulation=form,
                           max_k=t(mk), max_kp=t(mkp), param_index=t(pi))
    torch.cuda.synchronize()
    got = dict(states=device.tensor_to_records(r["states"]), frenet=r["frenet"].cpu().numpy(),
               status=r["status"].cpu().numpy(), iters=r["iters"].cpu().numpy())
    for i in range(B):
        _same_solve(got, want, i, i, b, b)


def test_solve_null_index_and_single_set(multi, single, sets):
    """A NULL index is set 0; a one-set handle with an all-zero index equals pqp_solve_batch."""
    b = _solve_batch("KP")
    B = len(b["n_points"])
    single.set_params(sets[0])
    want = single.solve(b, "KP")
    for got in (multi.solve(b, "KP"), single.solve(b, "KP", param_index=np.zeros(B, np.int32))):
        for i in range(B):
            _same_solve(got, want, i, i, b, b)


def test_solve_invalid_indices_fail_only_their_path(multi, single, sets):
    import torch
    b = _solve_batch("KP")
    B = len(b["n_points"])
    pi = _index(B, seed=3)
    bad = {1: -1, 4: S, 9: 1000}
    for i, v in bad.items():
        pi[i] = v
    got = multi.solve(b, "KP", param_index=pi)
    # the device entry with n_param_sets = 3: indices 3..5 fail as well
    dev = torch.device("cuda", 0)
    d = device.batch_to_device(b, dev)
    r = multi.solve_device(d["n_points"], d["offsets"], d["ref"], d["bounds"], d["x0"], d["end_heading"],
                           param_index=torch.from_numpy(pi).to(dev), n_param_sets=3)
    torch.cuda.synchronize()
    dgot = dict(states=device.tensor_to_records(r["states"]), frenet=r["frenet"].cpu().numpy(),
                status=r["status"].cpu().numpy(), iters=r["iters"].cpu().numpy())
    for res, n_ok in ((got, S), (dgot, 3)):
        for i in range(B):
            if not (0 <= pi[i] < n_ok):
                assert res["status"][i] == INVALID and res["iters"][i] == 0, i
                o = slice(b["offsets"][i], b["offsets"][i + 1])
                assert np.isnan(res["states"]["x"][o]).all() and np.isnan(res["frenet"][o]).all()
                continue
            single.set_params(sets[pi[i]])
            want = single.solve(synth.take_paths(b, [i]), "KP")
            _same_solve(res, want, i, 0, b, synth.take_paths(b, [i]))


# ---- the plan chain -------------------------------------------------------------------------------------------------

def _config1_map():
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "config1_benchmark_map.npz"))
    return dict(distance=g["map_distance"], rows=int(g["image_shape"][0]), cols=int(g["image_shape"][1]),
                resolution=float(g["map_geo"][0]), center_x=float(g["map_geo"][1]), center_y=float(g["map_geo"][2]))


@pytest.fixture(scope="module")
def scene():
    maps, b, mi = synth.multi_map_batch(N_MAPS, N_CAND, n=N, first_maps=[_config1_map()], order="interleaved", **MIXED)
    total = int(b["offsets"][-1])
    b["ref"]["v"] = 4.0 + 3.0 * np.sin(np.arange(total) * 0.05)
    b["ref"]["a"] = 0.5 * np.cos(np.arange(total) * 0.05)
    b["ref"]["v"][::13] = 0.0
    return maps, b, mi, _index(len(mi), seed=4)


def _spl(b, mode):
    return planner.reference_splines(b) if mode == planner.BOUNDS_IMPROVED else None


def _path_bits(r, b, i, output_mode):
    if output_mode == planner.OUTPUT_RAW:
        return r["states"][b["offsets"][i]:b["offsets"][i + 1]].tobytes()
    return r["states"][i, :r["n_out"][i]].tobytes()


def _same_path(got, gb, i, want, wb, k, output_mode):
    for f in ("n_out", "ok", "status", "iters"):
        assert got[f][i] == want[f][k], (f, i)
    assert _path_bits(got, gb, i, output_mode) == _path_bits(want, wb, k, output_mode), i
    assert (got["bounds"][gb["offsets"][i]:gb["offsets"][i + 1]].tobytes()
            == want["bounds"][wb["offsets"][k]:wb["offsets"][k + 1]].tobytes()), i


@pytest.mark.parametrize("output_mode", [planner.OUTPUT_RAW, planner.OUTPUT_DENSIFY])
@pytest.mark.parametrize("bounds_mode", [planner.BOUNDS_SIMPLE, planner.BOUNDS_IMPROVED])
@pytest.mark.parametrize("form", ["KP", "KPC", "K"])
def test_plan_sets_per_set_bits(multi, single, sets, scene, form, bounds_mode, output_mode):
    """pqp_plan_batch_sets over three maps and six sets equals, per set, a one-set handle planning only that set's paths
    with pqp_plan_batch_maps; the device entry equals the host entry."""
    import torch
    maps, b, mi, pi = scene
    multi.set_maps(maps)
    single.set_maps(maps)
    kw = dict(formulation=form, bounds_mode=bounds_mode, output_mode=output_mode, max_out=256, want_bounds=True)
    got = multi.plan(b, splines=_spl(b, bounds_mode), map_index=mi, param_index=pi, **kw)
    assert (got["status"] == 1).sum() >= 10
    for k in range(S):
        idx = np.flatnonzero(pi == k)
        sub = synth.take_paths(b, idx)
        single.set_params(sets[k])
        want = single.plan(sub, splines=_spl(sub, bounds_mode), map_index=mi[idx], **kw)
        for j, i in enumerate(idx):
            _same_path(got, b, i, want, sub, j, output_mode)
    dev = torch.device("cuda", 0)
    d = device.batch_to_device(b, dev)
    spl = device.splines_to_device(_spl(b, bounds_mode), dev) if bounds_mode == planner.BOUNDS_IMPROVED else None
    r = multi.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], max_n_points=N,
                          formulation=form, bounds_mode=bounds_mode, splines=spl, output_mode=output_mode, max_out=256,
                          want_bounds=True, map_index=torch.from_numpy(mi).to(dev), param_index=torch.from_numpy(pi).to(dev))
    dgot = _host(r, output_mode)
    for i in range(len(pi)):
        _same_path(dgot, b, i, got, b, i, output_mode)


@pytest.mark.parametrize("form", ["KP", "K"])
def test_plan_sets_oracle_sample(multi, sets, scene, form):
    """Two paths of every set against oracle.plan with that set's params (the map of the path)."""
    maps, b, mi, pi = scene
    multi.set_maps(maps)
    got = multi.plan(b, formulation=form, map_index=mi, param_index=pi, max_out=256, want_bounds=True)
    for k in range(S):
        for i in np.flatnonzero(pi == k)[:2]:
            one = synth.take_paths(b, [i])
            o = oracle.plan(sets[k], maps[mi[i]], one, formulation=FORMULATIONS[form], max_out=256)
            nv = oracle.update_bounds(sets[k], maps[mi[i]], one)["n_valid"][0]
            assert got["status"][i] == o["status"][0] and got["iters"][i] == o["iters"][0], (k, i)
            assert got["n_out"][i] == o["n_out"][0] and got["ok"][i] == o["ok"][0], (k, i)
            c, lo = o["n_out"][0], b["offsets"][i]
            for f in ("x", "y", "z", "k", "s"):
                assert np.abs(got["states"][f][lo:lo + c] - o["states"][f][:c]).max(initial=0.0) <= FRENET_TOL
            G = got["bounds"][lo:lo + nv]
            assert G.tobytes() == o["bounds"][:nv].tobytes(), (k, i)


def _np(t):
    return t.detach().cpu().numpy()


def _host(r, output_mode):
    import torch
    torch.cuda.synchronize()
    st = r["states"].reshape(-1, 7) if output_mode == planner.OUTPUT_RAW else r["states"]
    states = device.tensor_to_records(st)
    if output_mode == planner.OUTPUT_DENSIFY:
        states = states.reshape(r["states"].shape[0], -1)
    return dict(states=states, n_out=_np(r["n_out"]), ok=_np(r["ok"]), status=_np(r["status"]), iters=_np(r["iters"]),
                bounds=device.tensor_to_records(r["bounds"], BOUNDS_DTYPE))


def test_plan_null_index_single_set_and_invalid(multi, single, sets, scene):
    """A NULL index is set 0; a one-set handle with an all-zero index equals pqp_plan_batch_maps; indices -1, n_sets and
    (device, n_param_sets = 2) >= 2 fail only their own path with status -100, 0 iterations, n_out = 0 and ok = 0."""
    import torch
    maps, b, mi, pi = scene
    multi.set_maps(maps)
    single.set_maps(maps)
    single.set_params(sets[0])
    kw = dict(formulation="KPC", max_out=256, want_bounds=True)
    want = single.plan(b, map_index=mi, **kw)
    for got in (multi.plan(b, map_index=mi, **kw), single.plan(b, map_index=mi, param_index=np.zeros_like(pi), **kw)):
        for i in range(len(pi)):
            _same_path(got, b, i, want, b, i, planner.OUTPUT_RAW)
    bad = pi.copy()
    bad[0], bad[5], bad[7] = -1, S, 2
    got = multi.plan(b, map_index=mi, param_index=bad, **kw)
    dev = torch.device("cuda", 0)
    d = device.batch_to_device(b, dev)
    r = multi.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], max_n_points=N,
                          formulation="KPC", max_out=256, want_bounds=True, map_index=torch.from_numpy(mi).to(dev),
                          param_index=torch.from_numpy(bad).to(dev), n_param_sets=2)
    dgot = _host(r, planner.OUTPUT_RAW)
    for res, n_ok in ((got, S), (dgot, 2)):
        for i in range(len(bad)):
            if not (0 <= bad[i] < n_ok):
                assert (res["status"][i], res["iters"][i], res["n_out"][i], res["ok"][i]) == (INVALID, 0, 0, 0), i
                continue
            single.set_params(sets[bad[i]])
            one = synth.take_paths(b, [i])
            w = single.plan(one, map_index=mi[[i]], **kw)
            _same_path(res, b, i, w, one, 0, planner.OUTPUT_RAW)


def test_graphs_follow_inputs_and_keep_their_sets(sets, scene):
    """A captured plan_device with a set index replays new inputs and indices; after pqp_set_param_sets a graph captured
    before keeps its old sets at every stage, and a graph captured again follows the new ones."""
    import torch
    maps, b, mi, pi = scene
    p = planner.PathPlanner(max_batch=512, max_total_points=512 * N)
    try:
        p.set_maps(maps)
        p.set_param_sets(sets)
        dev = torch.device("cuda", 0)
        d = device.batch_to_device(b, dev)
        mi_t, pi_t = torch.from_numpy(mi.copy()).to(dev), torch.from_numpy(pi.copy()).to(dev)

        def run(**kw):
            return p.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], max_n_points=N,
                                 formulation="KPC", max_out=256, want_bounds=True, map_index=mi_t, param_index=pi_t, **kw)
        run()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            res = run()
        _, b2, _ = synth.multi_map_batch(N_MAPS, N_CAND, n=N, seed=synth.BASE_SEED + 77, first_maps=maps,
                                         order="interleaved", **MIXED)
        b2["ref"]["v"], b2["ref"]["a"] = b["ref"]["v"], b["ref"]["a"]
        mi2 = np.random.default_rng(5).integers(0, N_MAPS, len(mi)).astype(np.int32)
        pi2 = np.random.default_rng(6).integers(0, S, len(pi)).astype(np.int32)
        for k, t in device.batch_to_device(b2, dev).items():
            if k in d:
                d[k].copy_(t)
        mi_t.copy_(torch.from_numpy(mi2))
        pi_t.copy_(torch.from_numpy(pi2))
        g.replay()
        torch.cuda.synchronize()
        want = p.plan(b2, formulation="KPC", max_out=256, want_bounds=True, map_index=mi2, param_index=pi2)
        got = _host(res, planner.OUTPUT_RAW)
        for i in range(len(pi2)):
            _same_path(got, b2, i, want, b2, i, planner.OUTPUT_RAW)
        # new sets: the old graph keeps the old ones at every stage
        new = list(reversed(synth.param_sets(S, seed=12)))
        p.set_param_sets(new)
        g.replay()
        torch.cuda.synchronize()
        got = _host(res, planner.OUTPUT_RAW)
        for i in range(len(pi2)):
            _same_path(got, b2, i, want, b2, i, planner.OUTPUT_RAW)
        # captured again: the new sets
        g2 = torch.cuda.CUDAGraph()
        run()
        torch.cuda.synchronize()
        with torch.cuda.graph(g2):
            res2 = run()
        g2.replay()
        torch.cuda.synchronize()
        want2 = p.plan(b2, formulation="KPC", max_out=256, want_bounds=True, map_index=mi2, param_index=pi2)
        got2 = _host(res2, planner.OUTPUT_RAW)
        for i in range(len(pi2)):
            _same_path(got2, b2, i, want2, b2, i, planner.OUTPUT_RAW)
        assert any(got2["iters"][i] != want["iters"][i] or got2["bounds"][b2["offsets"][i]:b2["offsets"][i + 1]].tobytes()
                   != want["bounds"][b2["offsets"][i]:b2["offsets"][i + 1]].tobytes() for i in range(len(pi2)))
    finally:
        p.close()


def test_argument_errors_leave_the_sets(multi, sets, scene):
    maps, b, mi, pi = scene
    multi.set_maps(maps)
    multi.set_param_sets(sets)
    before = multi.plan(b, map_index=mi, param_index=pi, max_out=256, want_bounds=True)
    L = _lib.load()
    arr = (Params * 65)(*([sets[1]] * 65))
    for n, a in ((0, arr), (65, arr), (-1, arr), (2, None)):
        assert L.pqp_set_param_sets(multi._h, n, a) == ERR_ARG
    assert L.pqp_set_param_sets(None, 1, arr) == ERR_ARG
    with pytest.raises(ValueError):
        multi.plan(b, map_index=mi, param_index=pi[:-1])
    after = multi.plan(b, map_index=mi, param_index=pi, max_out=256, want_bounds=True)
    for i in range(len(pi)):
        _same_path(after, b, i, before, b, i, planner.OUTPUT_RAW)
    assert L.pqp_set_param_sets(multi._h, 64, arr) == OK
    multi.set_param_sets(sets)


def test_cpp_planner_sets_mirror(tmp_path, sets, scene):
    """include/pqp_planner.hpp: PathOptimizerGpu built from three maps and six parameter sets, and the batched
    solveWithoutSmoothing with a map and a set index per reference, through tests/cpp/planner_sets_driver.cpp; results
    equal PathPlanner.plan(..., map_index, param_index)."""
    maps, b, mi, pi = scene
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.join(root, "path_optimizer_b200")
    exe = str(tmp_path / "planner_sets_driver")
    subprocess.run(["g++", "-O2", "-std=c++17", os.path.join(root, "tests", "cpp", "planner_sets_driver.cpp"), "-o", exe,
                    "-L" + libdir, "-lpqp", "-Wl,-rpath," + libdir], check=True)
    B = len(mi)
    veh = np.column_stack([b["x0"], b["end_heading"]])
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(fin, "wb") as f:
        f.write(np.int32(len(maps)).tobytes())
        for m in maps:
            f.write(np.array([m["rows"], m["cols"]], dtype=np.int32).tobytes())
            f.write(np.array([m["resolution"], m["center_x"], m["center_y"]], dtype=np.float64).tobytes())
            f.write(np.ascontiguousarray(m["distance"], dtype=np.float32).tobytes())
        f.write(np.int32(len(sets)).tobytes())
        for p_ in sets:
            f.write(bytes(p_))
        f.write(np.int32(B).tobytes()); f.write(b["n_points"].tobytes()); f.write(mi.tobytes()); f.write(pi.tobytes())
        f.write(np.ascontiguousarray(b["ref"]).tobytes()); f.write(np.ascontiguousarray(veh).tobytes())
    subprocess.run([exe, str(fin), str(fout)], check=True)
    raw = open(fout, "rb").read()
    n_out = np.frombuffer(raw, dtype=np.int32, count=B)
    ok = np.frombuffer(raw, dtype=np.int32, count=B, offset=4 * B)
    status = np.frombuffer(raw, dtype=np.int32, count=B, offset=8 * B)
    p = planner.PathPlanner(max_batch=B, max_total_points=int(b["offsets"][-1]))
    try:
        p.set_maps(maps)
        p.set_param_sets(sets)
        want = p.plan(b, map_index=mi, param_index=pi)
    finally:
        p.close()
    assert (n_out == want["n_out"]).all() and (ok == want["ok"]).all() and (status == want["status"]).all()
    assert (want["status"] == 1).any() and set(pi.tolist()) == set(range(S))
    o = 12 * B
    for i in range(B):
        got = raw[o:o + STATE_DTYPE.itemsize * int(n_out[i])]
        o += len(got)
        lo = b["offsets"][i]
        assert got == want["states"][lo:lo + n_out[i]].tobytes(), i
