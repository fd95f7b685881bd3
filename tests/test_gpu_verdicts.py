"""GPU: every named verdict branch of tests/verdicts.py on every kernel class of every formulation at both ends of its
length range, the cases batched as parameter sets (up to 64 per call, one set index per path), against the oracle
(shapes.assert_matches: same status and iteration count, 1e-8 on the output, 1e-6 past 1000 iterations); a subset again
through a single-set handle and through solve_device, bit for bit; and the refusal of every setting OSQP refuses."""
import ctypes as C
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from oracle import oracle
from path_optimizer_b200 import synth
from path_optimizer_b200.abi import ERR_ARG, OK, Params
from tests import device_entries, shapes, verdicts
from tests.test_gpu_parity import _class_ends_batch

pytestmark = pytest.mark.gpu
THREADS = max(1, min(16, os.cpu_count() or 1))
FORMS = {"KP": shapes.KP, "K": shapes.K, "KPC": shapes.KPC}


def _gather(batches, chunk):
    """One batch of the chunk's paths (a path may appear once per case) and its KPC limits."""
    kind = chunk[0]["kind"]
    b, mk, mkp = batches[kind]
    idx = [c["path"] for c in chunk]
    sub = synth.take_paths(b, idx)
    if mk is None:
        return sub, None, None
    rows = device_entries.rows(b, idx)
    return sub, np.ascontiguousarray(mk[rows]), np.ascontiguousarray(mkp[rows])


def _oracle(form, sub, mk, mkp, chunk):
    def one(i):
        c = chunk[i]
        p = synth.take_paths(sub, [i])
        rows = device_entries.rows(sub, [i])
        r = oracle.solve_batch(c["params"], form, p, max_k=None if mk is None else mk[rows],
                               max_kp=None if mk is None else mkp[rows])
        return r
    with ThreadPoolExecutor(max_workers=THREADS) as ex:
        rs = list(ex.map(one, range(len(chunk))))
    return dict(status=np.concatenate([r["status"] for r in rs]), iters=np.concatenate([r["iters"] for r in rs]),
                frenet=np.concatenate([r["frenet"] for r in rs]), states=np.concatenate([r["states"] for r in rs]))


def _report(res, ref, chunk, sub, what):
    """shapes.assert_matches' bar per case, naming the cases that miss it (length, schedule, setting, branch)."""
    o, bad = sub["offsets"], []
    for i, c in enumerate(chunk):
        r = slice(o[i], o[i + 1])
        tol = shapes.LONG_RUN_TOL if ref["iters"][i] > shapes.LONG_RUN_ITERS else shapes.TOL
        pairs = [(res["frenet"][r], ref["frenet"][r])] + [(res["states"][f][r], ref["states"][f][r]) for f in "xyzks"]
        err = max(float(np.max(np.where(np.isnan(a) & np.isnan(d), 0.0, np.abs(a - d)), initial=0.0)) for a, d in pairs)
        if res["status"][i] != ref["status"][i] or res["iters"][i] != ref["iters"][i] or not err <= tol:
            bad.append((int(sub["n_points"][i]), c["schedule"], c["label"], c["branch"], c["params"].max_iter,
                        int(ref["iters"][i]), int(res["iters"][i]), err))
    assert not bad, (what, bad)


@pytest.mark.parametrize("name", sorted(FORMS), ids=sorted(FORMS))
def test_every_branch_every_class(name):
    from path_optimizer_b200.solver import BatchPathSolver
    form = FORMS[name]
    b = _class_ends_batch(form)
    cases, dropped, batches = verdicts.batch_cases(form, b, threads=THREADS)
    assert {c["branch"] for c in cases} == set(verdicts.BRANCHES)
    s = BatchPathSolver(max_batch=64, max_total_points=64 * 416)
    single = BatchPathSolver(max_batch=64, max_total_points=64 * 416)
    gap, checked = 0.0, 0
    try:
        for kind in ("feasible", "infeasible"):
            mine = [c for c in cases if c["kind"] == kind]
            for k in range(0, len(mine), 64):
                chunk = mine[k:k + 64]
                sub, mk, mkp = _gather(batches, chunk)
                s.set_param_sets([c["params"] for c in chunk])
                pi = np.arange(len(chunk), dtype=np.int32)
                res = s.solve(sub, formulation=name, max_k=mk, max_kp=mkp, param_index=pi)
                ref = _oracle(form, sub, mk, mkp, chunk)
                assert np.array_equal(ref["status"], [c["status"] for c in chunk])
                _report(res, ref, chunk, sub, f"{name} {kind}")
                shapes.assert_matches(res, ref, pi, np.arange(int(sub["offsets"][-1])), sub["n_points"],
                                      f"{name} {kind} cases {k}..{k + len(chunk)}")
                if np.isfinite(ref["frenet"]).any():
                    gap = max(gap, float(np.nanmax(np.abs(res["frenet"] - ref["frenet"]))))
                checked += len(chunk)
                # the same paths through the device entry with the same sets, and every fourth case through a handle
                # holding its set alone: bit for bit
                import torch
                dpi = torch.from_numpy(pi).to("cuda")
                dev = device_entries.dispatch(s, name, sub, mk, mkp, param_index=dpi, n_param_sets=len(chunk))
                device_entries.same_bits(res, dev, pi, np.arange(int(sub["offsets"][-1])))
                for i in range(0, len(chunk), 4):
                    one = synth.take_paths(sub, [i])
                    rows = device_entries.rows(sub, [i])
                    single.set_params(chunk[i]["params"])
                    r1 = single.solve(one, formulation=name, max_k=None if mk is None else mk[rows],
                                      max_kp=None if mk is None else mkp[rows])
                    assert r1["status"][0] == res["status"][i] and r1["iters"][0] == res["iters"][i]
                    assert np.array_equal(device_entries.u64(r1["frenet"]), device_entries.u64(res["frenet"][rows]))
                    assert np.array_equal(device_entries.u64(r1["states"]), device_entries.u64(res["states"][rows]))
    finally:
        s.close()
        single.close()
    print(f"{name}: {checked} cases on {len(b['n_points'])} class-end paths x 2 kinds, {dropped} dropped for margin, "
          f"max |frenet - oracle| = {gap:.1e}")


def test_illegal_settings_are_refused():
    """pqp_create, pqp_set_params and pqp_set_param_sets refuse every setting OSQP refuses with PQP_ERR_ARG, and the
    handle keeps its previous sets: a solve afterwards matches the oracle under the defaults."""
    from path_optimizer_b200 import _lib
    from path_optimizer_b200.solver import BatchPathSolver
    L = _lib.load()
    b = synth.curvy_corridors(2, 40)
    s = BatchPathSolver(max_batch=4, max_total_points=400)
    try:
        good = oracle.default_params()
        for name, over in verdicts.ILLEGAL.items():
            p = oracle.default_params()
            for k, v in over.items():
                setattr(p, k, v)
            h = C.c_void_p()
            assert L.pqp_create(C.byref(h), C.byref(p), 0, 4, 400) == ERR_ARG and not h.value, name
            assert L.pqp_set_params(s._h, C.byref(p)) == ERR_ARG, name
            arr = (Params * 3)(good, p, good)
            assert L.pqp_set_param_sets(s._h, 3, arr) == ERR_ARG, name
        assert L.pqp_set_param_sets(s._h, 3, (Params * 3)(good, good, good)) == OK
        res = s.solve(b)
        ref = oracle.solve_batch(good, 0, b)
        shapes.assert_matches(res, ref, np.arange(2), np.arange(80), b["n_points"], "after refusals")
    finally:
        s.close()
