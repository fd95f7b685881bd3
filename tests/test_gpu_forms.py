"""GPU tests (run with -m gpu on an H100) of solving and planning one batch over several formulations ("KP", "K" and
"KPC" per path): pqp_solve_batch_forms, pqp_solve_batch_device_dispatch_forms, pqp_plan_batch_forms and
pqp_plan_batch_device_forms against the _sets entry called with each path's own formulation (bit for bit), the host and
device entries against each other, a CUDA graph whose formulation tensor is rewritten between replays, paths whose
formulation is not one or lies outside form_mask, the str path, an oracle sample of every formulation, argument errors
and the C++ mirror.

The solve batch takes the lengths at the edges of every class of every formulation (tests/shapes.py) and one station
past each formulation's limit, with "KP" at station spacings that give keep_control_steps 3, 4 and 8, over four
parameter sets (synth.param_sets)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle
from path_optimizer_b200 import device, planner, solver, synth
from path_optimizer_b200.abi import ERR_ARG, STATE_DTYPE
from tests import shapes
from tests.device_entries import rows, same_bits, to_np

pytestmark = pytest.mark.gpu
INVALID = -100
S = 4
N_MAPS, N_CAND, N = 3, 12, 120
MIXED = dict(y_range=(-1.5, 1.5), heading_range=0.03, curvature_amp=0.01)
NAMES = ("KP", "K", "KPC")
KP_SPACINGS = {3: 0.3, 4: 0.25, 8: 0.149}   # keep_control_steps -> station spacing of the "KP" paths


def _edges(form, keep):
    out = set()
    for lo, hi in shapes.class_ranges(form, keep).values():
        out.update((lo, hi))
    out.add(shapes.max_points(form, keep) + 1)
    return sorted(out)


def _solve_case():
    """(batch, formulation [B], spacing [B] of every path)."""
    lens, forms, ds = [], [], []
    for keep, sp in KP_SPACINGS.items():
        e = _edges(shapes.KP, keep)
        lens += e; forms += [shapes.KP] * len(e); ds += [sp] * len(e)
    for f in (shapes.K, shapes.KPC):
        e = _edges(f, 1 if f == shapes.K else 4)
        lens += e; forms += [f] * len(e); ds += [0.3] * len(e)
    rng = np.random.default_rng(2)
    for f in (shapes.KP, shapes.K, shapes.KPC):   # 16 more of every formulation inside its limits (the oracle sample)
        lens += rng.integers(10, 250, 16).tolist(); forms += [f] * 16
        ds += rng.choice([0.3, 0.25, 0.149] if f == shapes.KP else [0.3], 16).tolist()
    order = np.random.default_rng(3).permutation(len(lens))
    lens, forms, ds = (np.asarray(a)[order] for a in (lens, forms, ds))
    b = synth.curvy_corridors(len(lens), n_points=lens.astype(np.int32), seed=synth.BASE_SEED + 9)
    for i in range(len(lens)):
        o, n = b["offsets"][i], b["n_points"][i]
        b["ref"]["s"][o:o + n] = synth._accumulate_s(n, float(ds[i]))
    total = int(b["offsets"][-1])
    b["ref"]["v"] = 4.0 + 3.0 * np.sin(np.arange(total) * 0.05)
    b["ref"]["a"] = 0.5 * np.cos(np.arange(total) * 0.05)
    return b, forms.astype(np.int32)


@pytest.fixture(scope="module")
def sets():
    return synth.param_sets(S, seed=11)


@pytest.fixture(scope="module")
def multi(sets):
    s = planner.PathPlanner(max_batch=512, max_total_points=512 * 420)
    s.set_param_sets(sets)
    yield s
    s.close()


@pytest.fixture(scope="module")
def case():
    b, forms = _solve_case()
    mk, mkp = planner.update_limits(solver.default_params(), b["ref"])
    pi = (np.arange(len(forms)) % S).astype(np.int32)
    np.random.default_rng(4).shuffle(pi)
    return b, forms, mk, mkp, pi


def _dev_solve(s, b, forms_t, mk, mkp, pi=None, **kw):
    import torch
    dev = torch.device("cuda", 0)
    d = device.batch_to_device(b, dev)
    t = (lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev))
    r = s.solve_device(d["n_points"], d["offsets"], d["ref"], d["bounds"], d["x0"], d["end_heading"], formulation=forms_t,
                       max_k=t(mk), max_kp=t(mkp), param_index=t(pi), **kw)
    torch.cuda.synchronize()
    return dict(states=device.tensor_to_records(r["states"]), frenet=to_np(r["frenet"]), status=to_np(r["status"]),
                iters=to_np(r["iters"]))


@pytest.mark.parametrize("indexed", [False, True])
def test_solve_forms_equal_sets_entry_per_formulation(multi, case, indexed):
    """Per path, pqp_solve_batch_forms equals the _sets entry called with that path's formulation, bit for bit; so does
    the device dispatch, with and without a set index."""
    import torch
    b, forms, mk, mkp, pi = case
    pi = pi if indexed else None
    got = multi.solve(b, forms, max_k=mk, max_kp=mkp, param_index=pi)
    dgot = _dev_solve(multi, b, torch.from_numpy(forms).cuda(), mk, mkp, pi)
    covered = set()
    for f in range(3):
        want = multi.solve(b, NAMES[f], max_k=mk if f == shapes.KPC else None, max_kp=mkp if f == shapes.KPC else None,
                           param_index=pi)
        idx = np.flatnonzero(forms == f)
        for res in (got, dgot):
            same_bits(res, want, idx, rows(b, idx))
        covered.update((f, int(s)) for s in (pi[idx] if indexed else [0]))
        solved = want["status"][idx] == 1
        assert solved.sum() >= 3 and (want["status"][idx] == INVALID).any(), NAMES[f]   # and a path past the limit
    assert len(covered) == (3 * S if indexed else 3)


def test_solve_forms_oracle_sample(multi, sets, case):
    """16 paths of every formulation (inside its limits) against the oracle with each path's set."""
    b, forms, mk, mkp, pi = case
    got = multi.solve(b, forms, max_k=mk, max_kp=mkp, param_index=pi)
    for f in range(3):
        idx = np.flatnonzero((forms == f) & (got["status"] != INVALID) & (b["n_points"] < 250))[:16]
        assert len(idx) == 16, NAMES[f]
        for k in range(S):
            few = idx[pi[idx] == k]
            if not len(few):
                continue
            fb, fr = synth.take_paths(b, few), rows(b, few)
            o = oracle.solve_batch(sets[k], f, fb, max_k=mk[fr] if f == shapes.KPC else None,
                                   max_kp=mkp[fr] if f == shapes.KPC else None)
            shapes.assert_matches(got, o, few, fr, fb["n_points"], (NAMES[f], k))


def test_solve_rejected_formulations_fail_only_their_path(multi, case):
    import torch
    b, forms, mk, mkp, pi = case
    want = multi.solve(b, forms, max_k=mk, max_kp=mkp, param_index=pi)
    bad = forms.copy()
    bad[1], bad[4] = -1, 3
    kpc = np.flatnonzero(forms == shapes.KPC)
    got = multi.solve(b, bad, max_k=mk, max_kp=mkp, param_index=pi)
    # the device entry with form_mask = KP | K: the "KPC" paths fail as well (the limits are then not needed)
    dgot = _dev_solve(multi, b, torch.from_numpy(bad).cuda(), None, None, pi, form_mask=["KP", "K"])
    for res, rejected in ((got, {1, 4}), (dgot, {1, 4} | set(kpc.tolist()))):
        for i in range(len(forms)):
            o = slice(b["offsets"][i], b["offsets"][i + 1])
            if i in rejected:
                assert res["status"][i] == INVALID and res["iters"][i] == 0, i
                assert np.isnan(res["states"]["x"][o]).all() and np.isnan(res["frenet"][o]).all()
            else:
                same_bits(res, want, [i], rows(b, [i]))


def test_solve_str_path_equals_an_array_of_one_formulation(multi, case):
    b, forms, mk, mkp, pi = case
    for f in range(3):
        lim = dict(max_k=mk, max_kp=mkp) if f == shapes.KPC else {}
        a = multi.solve(b, NAMES[f], param_index=pi, **lim)
        c = multi.solve(b, np.full(len(forms), f, np.int32), param_index=pi, **lim)
        d = multi.solve(b, [NAMES[f]] * len(forms), param_index=pi, **lim)
        idx = np.arange(len(forms))
        same_bits(a, c, idx, rows(b, idx))
        same_bits(a, d, idx, rows(b, idx))


def test_solve_argument_errors(multi, case):
    import torch
    b, forms, mk, mkp, pi = case
    with pytest.raises(solver.PqpError, match=f"rc={ERR_ARG}"):
        multi.solve(b, forms, param_index=pi)   # a "KPC" path and no limits
    with pytest.raises(ValueError):
        multi.solve(b, forms[:-1], max_k=mk, max_kp=mkp)
    kp_k = np.where(forms == shapes.KPC, shapes.KP, forms).astype(np.int32)
    multi.solve(b, kp_k)   # no "KPC" path: no limits needed
    t = torch.from_numpy(kp_k).cuda()
    with pytest.raises(solver.PqpError, match=f"rc={ERR_ARG}"):
        _dev_solve(multi, b, t, None, None)   # the mask (all three) holds "KPC"
    with pytest.raises(solver.PqpError, match=f"rc={ERR_ARG}"):
        _dev_solve(multi, b, t, None, None, form_mask=8)


def test_generic_switch_is_unsupported(tmp_path):
    """With PQP_GENERIC_K set, a batch with a "K" path returns PQP_ERR_UNSUPPORTED; one without is solved."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = (
        "import numpy as np\n"
        "from path_optimizer_b200 import solver, synth\n"
        "b = synth.curvy_corridors(4, 60)\n"
        "s = solver.BatchPathSolver(max_batch=4, max_total_points=240)\n"
        "r = s.solve(b, np.array([0, 0, 0, 0], np.int32))\n"
        "assert (r['status'] == 1).all()\n"
        "try:\n"
        "    s.solve(b, np.array([0, 1, 0, 0], np.int32))\n"
        "    raise SystemExit('no error')\n"
        "except solver.PqpError as e:\n"
        "    assert 'rc=4' in str(e), e\n"
        "s.close()\n")
    env = dict(os.environ, PQP_GENERIC_K="1", PYTHONPATH=root)
    subprocess.run([sys.executable, "-c", code], check=True, env=env, cwd=root)


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
    B = len(mi)
    rng = np.random.default_rng(8)
    pi = (np.arange(B) % S).astype(np.int32)
    rng.shuffle(pi)
    forms = (np.arange(B) // S % 3).astype(np.int32)   # every (set, formulation) pair
    rng.shuffle(forms)
    return maps, b, mi, pi, forms


def _spl(b, mode):
    return planner.reference_splines(b) if mode == planner.BOUNDS_IMPROVED else None


def _bits(r, b, i, output_mode):
    if output_mode == planner.OUTPUT_RAW:
        return r["states"][b["offsets"][i]:b["offsets"][i + 1]].tobytes()
    return r["states"][i, :r["n_out"][i]].tobytes()


def _same_path(got, want, b, i, output_mode):
    for f in ("n_out", "ok", "status", "iters"):
        assert got[f][i] == want[f][i], (f, i)
    assert _bits(got, b, i, output_mode) == _bits(want, b, i, output_mode), i
    o = slice(b["offsets"][i], b["offsets"][i + 1])
    assert got["bounds"][o].tobytes() == want["bounds"][o].tobytes(), i


def _host(r, output_mode):
    import torch
    from path_optimizer_b200.abi import BOUNDS_DTYPE
    torch.cuda.synchronize()
    st = r["states"].reshape(-1, 7) if output_mode == planner.OUTPUT_RAW else r["states"]
    states = device.tensor_to_records(st)
    if output_mode == planner.OUTPUT_DENSIFY:
        states = states.reshape(r["states"].shape[0], -1)
    return dict(states=states, n_out=to_np(r["n_out"]), ok=to_np(r["ok"]), status=to_np(r["status"]),
                iters=to_np(r["iters"]), bounds=device.tensor_to_records(r["bounds"], BOUNDS_DTYPE))


def _plan_device(p, b, dev, mi, pi, forms_t, bounds_mode=planner.BOUNDS_SIMPLE, output_mode=planner.OUTPUT_RAW, **kw):
    import torch
    d = device.batch_to_device(b, dev)
    spl = device.splines_to_device(_spl(b, bounds_mode), dev) if bounds_mode == planner.BOUNDS_IMPROVED else None
    t = (lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev))
    return p.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], formulation=forms_t,
                         bounds_mode=bounds_mode, splines=spl, output_mode=output_mode, max_out=256, want_bounds=True,
                         map_index=t(mi), param_index=t(pi), **kw)


@pytest.mark.parametrize("output_mode", [planner.OUTPUT_RAW, planner.OUTPUT_DENSIFY])
@pytest.mark.parametrize("bounds_mode", [planner.BOUNDS_SIMPLE, planner.BOUNDS_IMPROVED])
def test_plan_forms_equal_sets_entry_per_formulation(multi, scene, bounds_mode, output_mode):
    """Maps x sets x formulations: per path, pqp_plan_batch_forms and plan_device(formulation=) equal the _sets entry
    called with that path's formulation, bit for bit."""
    import torch
    maps, b, mi, pi, forms = scene
    multi.set_maps(maps)
    kw = dict(bounds_mode=bounds_mode, output_mode=output_mode, max_out=256, want_bounds=True, map_index=mi,
              param_index=pi)
    got = multi.plan(b, formulation=forms, splines=_spl(b, bounds_mode), **kw)
    dev = torch.device("cuda", 0)
    dgot = _host(_plan_device(multi, b, dev, mi, pi, torch.from_numpy(forms).to(dev), bounds_mode, output_mode), output_mode)
    for f in range(3):
        want = multi.plan(b, formulation=NAMES[f], splines=_spl(b, bounds_mode), **kw)
        idx = np.flatnonzero(forms == f)
        assert (want["status"][idx] == 1).sum() >= 5 and len(set(pi[idx].tolist())) == S, NAMES[f]
        for i in idx:
            _same_path(got, want, b, i, output_mode)
            _same_path(dgot, want, b, i, output_mode)


def test_plan_rejected_formulations_and_str_path(multi, scene):
    """Formulations -1 and 3, and (device) one outside form_mask, fail only their path: status -100, 0 iterations,
    out_n = 0, ok = 0.  The str path equals an array of one formulation."""
    import torch
    maps, b, mi, pi, forms = scene
    multi.set_maps(maps)
    kw = dict(max_out=256, want_bounds=True, map_index=mi, param_index=pi)
    want = multi.plan(b, formulation=forms, **kw)
    bad = forms.copy()
    bad[0], bad[3] = -1, 3
    got = multi.plan(b, formulation=bad, **kw)
    dev = torch.device("cuda", 0)
    mask = (1 << shapes.KP) | (1 << shapes.KPC)
    dgot = _host(_plan_device(multi, b, dev, mi, pi, torch.from_numpy(bad).to(dev), form_mask=mask), planner.OUTPUT_RAW)
    kk = set(np.flatnonzero(bad == shapes.K).tolist())
    for res, rejected in ((got, {0, 3}), (dgot, {0, 3} | kk)):
        for i in range(len(bad)):
            if i in rejected:
                assert (res["status"][i], res["iters"][i], res["n_out"][i], res["ok"][i]) == (INVALID, 0, 0, 0), i
            else:
                _same_path(res, want, b, i, planner.OUTPUT_RAW)
    for f in range(3):
        a = multi.plan(b, formulation=NAMES[f], **kw)
        c = multi.plan(b, formulation=np.full(len(forms), f, np.int32), **kw)
        for i in range(len(forms)):
            _same_path(c, a, b, i, planner.OUTPUT_RAW)


def test_plan_forms_oracle_sample(multi, sets, scene):
    """"KP" and "K" paths of every set against oracle.plan with that set's params on the path's map (the "KPC" QP is
    held to the oracle by the solve sample)."""
    maps, b, mi, pi, forms = scene
    multi.set_maps(maps)
    got = multi.plan(b, formulation=forms, map_index=mi, param_index=pi, max_out=256)
    for f in (shapes.KP, shapes.K):
        for k in range(S):
            for i in np.flatnonzero((forms == f) & (pi == k))[:2]:
                one = synth.take_paths(b, [i])
                o = oracle.plan(sets[k], maps[mi[i]], one, formulation=f, max_out=256)
                assert got["status"][i] == o["status"][0] and got["iters"][i] == o["iters"][0], (f, k, i)
                assert got["n_out"][i] == o["n_out"][0] and got["ok"][i] == o["ok"][0], (f, k, i)
                c, lo = o["n_out"][0], b["offsets"][i]
                for name in "xyzks":
                    assert np.abs(got["states"][name][lo:lo + c] - o["states"][name][:c]).max(initial=0.0) <= 1e-8


def test_graph_replays_rewritten_formulations(sets, scene):
    """A captured plan_device with a formulation tensor: rotate the formulations across the paths, replay, and the
    result equals a fresh call."""
    import torch
    maps, b, mi, pi, forms = scene
    p = planner.PathPlanner(max_batch=512, max_total_points=512 * N)
    try:
        p.set_maps(maps)
        p.set_param_sets(sets)
        dev = torch.device("cuda", 0)
        d = device.batch_to_device(b, dev)
        mi_t, pi_t = torch.from_numpy(mi.copy()).to(dev), torch.from_numpy(pi.copy()).to(dev)
        f_t = torch.from_numpy(forms.copy()).to(dev)

        def run():
            return p.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], formulation=f_t,
                                 max_out=256, want_bounds=True, map_index=mi_t, param_index=pi_t, n_param_sets=S)
        run()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            res = run()
        for shift in (1, 2):
            rot = np.roll(forms, shift).astype(np.int32)
            f_t.copy_(torch.from_numpy(rot))
            g.replay()
            got = _host(res, planner.OUTPUT_RAW)
            fresh = _host(run(), planner.OUTPUT_RAW)
            want = p.plan(b, formulation=rot, max_out=256, want_bounds=True, map_index=mi, param_index=pi)
            for i in range(len(rot)):
                _same_path(got, fresh, b, i, planner.OUTPUT_RAW)
                _same_path(got, want, b, i, planner.OUTPUT_RAW)
    finally:
        p.close()


def test_cpp_planner_forms_mirror(tmp_path, sets, scene):
    """include/pqp_planner.hpp: the batched solveWithoutSmoothing with a map index, a set index and a method string per
    reference, through tests/cpp/planner_forms_driver.cpp; results equal PathPlanner.plan(..., formulation=)."""
    maps, b, mi, pi, forms = scene
    forms = forms.copy()
    forms[2] = 7   # a method name the reference does not know
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.join(root, "path_optimizer_b200")
    exe = str(tmp_path / "planner_forms_driver")
    subprocess.run(["g++", "-O2", "-std=c++17", os.path.join(root, "tests", "cpp", "planner_forms_driver.cpp"), "-o", exe,
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
        f.write(forms.tobytes())
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
        want = p.plan(b, formulation=forms, map_index=mi, param_index=pi)
    finally:
        p.close()
    assert (n_out == want["n_out"]).all() and (ok == want["ok"]).all() and (status == want["status"]).all()
    assert status[2] == INVALID and (want["status"] == 1).any()
    o = 12 * B
    for i in range(B):
        got = raw[o:o + STATE_DTYPE.itemsize * int(n_out[i])]
        o += len(got)
        lo = b["offsets"][i]
        assert got == want["states"][lo:lo + n_out[i]].tobytes(), i
