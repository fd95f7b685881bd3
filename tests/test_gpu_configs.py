"""GPU tests of BASELINE configs 3, 4, 5 AT THEIR NAMED PER-GPU SIZES (run with -m gpu on an H100): the whole
shard is solved through the C ABI, a >= 64-path sample of it is compared with the oracle (identical status, identical
ADMM iteration count, 1e-8 on the Frenet and Cartesian states), and the device-resident entry points are checked
against the host-buffer one bit for bit."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle
from path_optimizer_b200 import synth, workloads
from path_optimizer_b200.abi import BOUNDS_DTYPE, STATE_DTYPE, SOLVED

pytestmark = pytest.mark.gpu
TOL = 1e-8
SAMPLE = 64


def _solver(B, total):
    from path_optimizer_b200.planner import PathPlanner
    return PathPlanner(max_batch=B, max_total_points=total)


def _sample_vs_oracle(batch, res, oracle_params, idx):
    sub = synth.take_paths(batch, idx)
    ref = oracle.solve_batch(oracle_params, 0, sub, threads=8)
    o = batch["offsets"]
    sel = np.concatenate([np.arange(o[i], o[i + 1]) for i in idx])
    assert np.array_equal(res["status"][idx], ref["status"])
    assert np.array_equal(res["iters"][idx], ref["iters"])
    np.testing.assert_allclose(res["frenet"][sel], ref["frenet"], rtol=0, atol=TOL)
    for f in "xyzks":
        np.testing.assert_allclose(res["states"][f][sel], ref["states"][f], rtol=0, atol=TOL)
    return ref


def test_config4_full_shard_sampled(oracle_params):
    """8192 x 100 straight corridors (one GPU's shard of the 65 536-path config 4)."""
    batch = workloads.build(4)
    s = _solver(8192, 8192 * 100)
    res = s.solve(batch)
    assert (res["status"] == SOLVED).all()
    idx = np.arange(17, 8192, 8192 // SAMPLE)[:SAMPLE]
    _sample_vs_oracle(batch, res, oracle_params, idx)
    s.close()


def test_config3_full_shard_sampled(oracle_params):
    """8192 x 200 with clearance bounds from the random-obstacle distance map (bounds by the GPU clearance stage)."""
    field = synth.disc_field_map()
    s = _solver(8192 + 1024, (8192 + 1024) * 200)
    s.set_map(field)

    def fn(cand):
        r = s.update_bounds(cand)
        return r["bounds"], r["n_valid"]
    batch = workloads.build(3, bounds_fn=fn)
    assert len(batch["n_points"]) == 8192 and (batch["n_points"] == 200).all()
    res = s.solve(batch)
    idx = np.arange(5, 8192, 8192 // SAMPLE)[:SAMPLE]
    # the sample's bounds from the oracle's clearance stage: the two agree bit for bit
    sub = synth.take_paths(batch, idx)
    ob = oracle.update_bounds(oracle_params, field, sub, mode=1)
    assert (ob["n_valid"] == 200).all()
    for f in BOUNDS_DTYPE.names:
        assert np.array_equal(ob["bounds"][f], sub["bounds"][f])
    ref = _sample_vs_oracle(batch, res, oracle_params, idx)
    assert (ref["status"] == SOLVED).sum() >= SAMPLE // 2
    # whole planner iteration on the same reference lines: same QP statuses and iteration counts as QP-only
    pr = s.plan(batch)
    assert np.array_equal(pr["status"], res["status"]) and np.array_equal(pr["iters"], res["iters"])
    s.close()


def _device_call(s, batch, classes):
    """Device-resident entry points through raw device buffers (torch only moves the bytes)."""
    import torch
    from path_optimizer_b200 import _lib
    L = _lib.load()
    dev = torch.device("cuda", 0)
    B, total = len(batch["n_points"]), int(batch["offsets"][-1])

    def up(a):
        return torch.from_numpy(np.frombuffer(np.ascontiguousarray(a).tobytes(), dtype=np.uint8).copy()).to(dev)
    d_n, d_off, d_ref, d_bnd = up(batch["n_points"]), up(batch["offsets"]), up(batch["ref"]), up(batch["bounds"])
    d_x0, d_end = up(batch["x0"]), up(batch["end_heading"])
    d_out = torch.zeros(total * STATE_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    d_fr = torch.zeros(total * 3, dtype=torch.float64, device=dev)
    d_st = torch.zeros(B, dtype=torch.int32, device=dev)
    d_it = torch.zeros(B, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    off = batch["offsets"]
    keep = np.array([L.pqp_keep_control_steps(0, np.ascontiguousarray(batch["ref"][off[i]:off[i + 1]]).ctypes.data_as(C.c_void_p),
                                              int(batch["n_points"][i])) for i in range(B)], dtype=np.int32)
    if classes:
        hn = np.ascontiguousarray(batch["n_points"], dtype=np.int32)
        rc = L.pqp_solve_batch_device_classes(s._h, 0, B, total, hn.ctypes.data_as(C.c_void_p), keep.ctypes.data_as(C.c_void_p),
                                              d_n.data_ptr(), d_off.data_ptr(), d_ref.data_ptr(), d_bnd.data_ptr(),
                                              d_x0.data_ptr(), d_end.data_ptr(), None, None, d_out.data_ptr(), d_fr.data_ptr(),
                                              d_st.data_ptr(), d_it.data_ptr(), None, None)
    else:
        nmax, klo, khi = int(batch["n_points"].max()), int(keep.min()), int(keep.max())
        rc = L.pqp_solve_batch_device(s._h, 0, B, total, nmax, klo, khi, d_n.data_ptr(), d_off.data_ptr(), d_ref.data_ptr(),
                                      d_bnd.data_ptr(), d_x0.data_ptr(), d_end.data_ptr(), None, None, d_out.data_ptr(),
                                      d_fr.data_ptr(), d_st.data_ptr(), d_it.data_ptr(), None, None)
    assert rc == 0, _lib.last_error()
    torch.cuda.synchronize()
    return dict(status=d_st.cpu().numpy(), iters=d_it.cpu().numpy(), frenet=d_fr.cpu().numpy().reshape(-1, 3),
                states=np.frombuffer(d_out.cpu().numpy().tobytes(), dtype=STATE_DTYPE))


def test_config5_full_shard_sampled(oracle_params):
    """4096 paths of U{50..400} stations (one GPU's share of config 5): host-buffer call sampled against the oracle in
    every length bucket; the length-bucketed device entry point gives the same bits."""
    batch = workloads.build(5)
    B, total = len(batch["n_points"]), int(batch["offsets"][-1])
    assert B == 4096 and batch["n_points"].min() >= 50 and batch["n_points"].max() <= 400
    s = _solver(B, total)
    res = s.solve(batch)
    n = batch["n_points"]
    idx = []
    for lo, hi in [(50, 102), (103, 204), (205, 256), (257, 400)]:   # the four kernel classes of the range
        cand = np.nonzero((n >= lo) & (n <= hi))[0]
        idx += list(cand[:: max(1, len(cand) // (SAMPLE // 4))][: SAMPLE // 4])
    idx = np.array(sorted(idx))
    assert len(idx) >= SAMPLE - 4
    _sample_vs_oracle(batch, res, oracle_params, idx)
    dres = _device_call(s, batch, classes=True)
    assert np.array_equal(dres["status"], res["status"]) and np.array_equal(dres["iters"], res["iters"])
    assert np.array_equal(dres["frenet"], res["frenet"])
    for f in "xyzks":
        assert np.array_equal(dres["states"][f], res["states"][f])
    s.close()


@pytest.mark.parametrize("nmax,ds", [(128, 0.3), (150, 0.3), (150, 0.25), (256, 0.3), (400, 0.3)])
def test_device_entry_with_loose_hints(oracle_params, nmax, ds):
    """pqp_solve_batch_device picks ONE class from the caller's bounds: every path inside them must solve exactly as
    pqp_solve_batch solves it (round 1 rejected in-range paths because neither fits() nor the shared-memory need is
    monotone in the path length)."""
    rng = np.random.default_rng(nmax)
    n_points = rng.integers(2, nmax + 1, size=40)
    n_points[:3] = [2, nmax, nmax - 1]
    batch = synth.curvy_corridors(40, n_points=n_points)
    if ds != 0.3:
        o = batch["offsets"]
        for b in range(40):
            batch["ref"]["s"][o[b]:o[b + 1]] = np.arange(n_points[b]) * ds
    total = int(batch["offsets"][-1])
    s = _solver(40, total)
    res = s.solve(batch)
    dres = _device_call(s, batch, classes=False)
    assert (dres["status"] != -100).all()
    assert np.array_equal(dres["status"], res["status"]) and np.array_equal(dres["iters"], res["iters"])
    np.testing.assert_allclose(dres["frenet"], res["frenet"], rtol=0, atol=TOL)
    ref = oracle.solve_batch(oracle_params, 0, batch, threads=8)
    assert np.array_equal(dres["status"], ref["status"]) and np.array_equal(dres["iters"], ref["iters"])
    s.close()


def _kpc_limits(oracle_params, batch, still=True):
    total = int(batch["offsets"][-1])
    batch["ref"]["v"] = 4.0 + 3.0 * np.sin(np.arange(total) * 0.05)
    batch["ref"]["a"] = 0.5 * np.cos(np.arange(total) * 0.05)
    if still:
        batch["ref"]["v"][::13] = 0.0
    return oracle.update_limits(oracle_params, batch["ref"])


def test_kpc_thread_per_station_classes_and_fallback(oracle_params):
    """"KPC" runs on the thread-per-station kernel classes up to 256 stations (assembled in the kernel); a batch with a
    longer path takes the host-assembled generic kernel.  Both against the oracle; the device entry point gives the
    same bits as the host-buffer one."""
    import torch
    from path_optimizer_b200 import _lib
    L = _lib.load()
    v, t, sm = C.c_int(), C.c_int(), C.c_int64()
    assert L.pqp_class_info_kpc(100, 0, C.byref(v), C.byref(t), C.byref(sm)) == 0
    assert L.pqp_class_name(v.value).decode() == "pqp_kp3_solve_kernel<13,7,8,34,KPC>"
    assert L.pqp_class_info_kpc(200, 0, C.byref(v), C.byref(t), C.byref(sm)) == 0 and t.value == 256
    assert L.pqp_class_info_kpc(300, 0, C.byref(v), C.byref(t), C.byref(sm)) != 0
    rng = np.random.default_rng(4)
    n_points = rng.integers(2, 257, size=64)
    n_points[:4] = [2, 3, 128, 256]
    batch = synth.curvy_corridors(64, n_points=n_points)
    mk, mkp = _kpc_limits(oracle_params, batch)
    total = int(batch["offsets"][-1])
    s = _solver(64, total)
    res = s.solve(batch, formulation="KPC", max_k=mk, max_kp=mkp)
    assert res["stats"].kernel_launches >= 2            # thread-per-station classes (the generic path launches once)
    ref = oracle.solve_batch(oracle_params, 2, batch, threads=8, max_k=mk, max_kp=mkp)
    assert np.array_equal(res["status"], ref["status"]) and np.array_equal(res["iters"], ref["iters"])
    np.testing.assert_allclose(res["frenet"], ref["frenet"], rtol=0, atol=TOL)
    for f in "xyzks":
        np.testing.assert_allclose(res["states"][f], ref["states"][f], rtol=0, atol=TOL)
    # device-resident entry (limits computed on the device) == host-buffer entry
    dev = torch.device("cuda", 0)

    def up(a):
        return torch.from_numpy(np.frombuffer(np.ascontiguousarray(a).tobytes(), dtype=np.uint8).copy()).to(dev)
    d_n, d_off, d_ref, d_bnd = up(batch["n_points"]), up(batch["offsets"]), up(batch["ref"]), up(batch["bounds"])
    d_x0, d_end = up(batch["x0"]), up(batch["end_heading"])
    d_mk = torch.zeros(total, dtype=torch.float64, device=dev)
    d_mkp = torch.zeros(total, dtype=torch.float64, device=dev)
    d_out = torch.zeros(total * STATE_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    d_fr = torch.zeros(total * 3, dtype=torch.float64, device=dev)
    d_st = torch.zeros(64, dtype=torch.int32, device=dev)
    d_it = torch.zeros(64, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    assert L.pqp_update_limits_device(s._h, 0, total, d_ref.data_ptr(), d_mk.data_ptr(), d_mkp.data_ptr(), None) == 0
    hn = np.ascontiguousarray(batch["n_points"], dtype=np.int32)
    rc = L.pqp_solve_batch_device_classes(s._h, 2, 64, total, hn.ctypes.data_as(C.c_void_p), None, d_n.data_ptr(),
                                          d_off.data_ptr(), d_ref.data_ptr(), d_bnd.data_ptr(), d_x0.data_ptr(), d_end.data_ptr(),
                                          d_mk.data_ptr(), d_mkp.data_ptr(), d_out.data_ptr(), d_fr.data_ptr(), d_st.data_ptr(),
                                          d_it.data_ptr(), None, None)
    assert rc == 0, _lib.last_error()
    torch.cuda.synchronize()
    assert np.array_equal(d_st.cpu().numpy(), res["status"]) and np.array_equal(d_it.cpu().numpy(), res["iters"])
    assert np.array_equal(d_fr.cpu().numpy().reshape(-1, 3), res["frenet"], equal_nan=True)
    # a path beyond 256 stations has no class (nor would the generic kernel hold it in one SM): PQP_INVALID_PROBLEM for it,
    # the rest of the batch is untouched
    n2 = np.array([40, 300, 100], dtype=np.int32)
    b2 = synth.curvy_corridors(3, n_points=n2)
    mk2, mkp2 = _kpc_limits(oracle_params, b2, still=False)
    r2 = s.solve(b2, formulation="KPC", max_k=mk2, max_kp=mkp2)
    o2 = oracle.solve_batch(oracle_params, 2, b2, threads=4, max_k=mk2, max_kp=mkp2)
    assert r2["status"][1] == -100 and np.isnan(r2["frenet"][40:340]).all()
    assert L.pqp_max_points_keep(s._h, 2, 4) == 256 and s.max_points("KPC") == 256 and s.max_points("K") == 416
    keep = np.array([0, 2])
    assert np.array_equal(r2["status"][keep], o2["status"][keep]) and np.array_equal(r2["iters"][keep], o2["iters"][keep])
    np.testing.assert_allclose(r2["frenet"][:40], o2["frenet"][:40], rtol=0, atol=TOL)
    np.testing.assert_allclose(r2["frenet"][340:], o2["frenet"][340:], rtol=0, atol=TOL)
    # the generic kernel (diagnostics switch) still agrees on the paths it can hold
    s.close()


def test_kpc_plan_chain(oracle_params):
    """solveWithoutSmoothing with optimization_method "KPC": updateBounds -> updateLimits (from the v, a fields of the
    reference states) -> QP -> raw tail, chained on the device, against the oracle's chain."""
    field = synth.disc_field_map()
    b = synth.map_reference_paths(24, 150)
    total = int(b["offsets"][-1])
    b["ref"]["v"] = 5.0 + 2.0 * np.sin(np.arange(total) * 0.03)
    b["ref"]["a"] = 0.3 * np.cos(np.arange(total) * 0.04)
    s = _solver(24, total)
    s.set_map(field)
    r = s.plan(b, formulation="KPC")
    o = oracle.plan(oracle_params, field, b, formulation=2)
    assert np.array_equal(r["status"], o["status"]) and np.array_equal(r["iters"], o["iters"])
    assert np.array_equal(r["ok"], o["ok"]) and np.array_equal(r["n_out"], o["n_out"])
    assert (o["status"] == SOLVED).sum() >= 12
    for f in "xyzks":
        np.testing.assert_allclose(r["states"][f], o["states"][f], rtol=0, atol=TOL)
    s.close()


def test_k_thread_per_station_classes_and_plan(oracle_params):
    """"K" (SolverKAsInput) runs on its own thread-per-station classes (pqp_kk_core.cuh: 4 / 8 / 13 warps, up to 416
    stations; SPIKE form to 256 stations, block cyclic reduction beyond), assembled in the kernel: every length class and an infeasible corridor against the
    oracle; the device entry gives the same bits as the host-buffer one; a longer path is PQP_INVALID_PROBLEM for itself;
    the solveWithoutSmoothing chain takes "K" too."""
    import torch
    from path_optimizer_b200 import _lib
    L = _lib.load()
    v, t, sm = C.c_int(), C.c_int(), C.c_int64()
    assert L.pqp_class_info_form(1, 100, 0, 0, C.byref(v), C.byref(t), C.byref(sm)) == 0 and t.value == 128
    assert L.pqp_class_name(v.value).decode() == "pqp_kk_solve_kernel<4>"
    assert L.pqp_class_info_form(1, 200, 0, 0, C.byref(v), C.byref(t), C.byref(sm)) == 0 and t.value == 256
    assert L.pqp_class_info_form(1, 416, 0, 0, C.byref(v), C.byref(t), C.byref(sm)) == 0 and t.value == 416
    assert L.pqp_class_info_form(1, 417, 0, 0, C.byref(v), C.byref(t), C.byref(sm)) != 0
    rng = np.random.default_rng(9)
    n_points = rng.integers(2, 417, size=96)
    n_points[:8] = [2, 3, 4, 128, 129, 256, 257, 416]
    batch = synth.curvy_corridors(96, n_points=n_points)
    total = int(batch["offsets"][-1])
    s = _solver(96, total)
    assert s.max_points("K") == 416
    res = s.solve(batch, formulation="K")
    assert res["stats"].kernel_launches == 3
    ref = oracle.solve_batch(oracle_params, 1, batch, threads=8)
    assert np.array_equal(res["status"], ref["status"]) and np.array_equal(res["iters"], ref["iters"])
    assert (ref["status"] == SOLVED).sum() >= 90
    np.testing.assert_allclose(res["frenet"], ref["frenet"], rtol=0, atol=TOL)
    for f in "xyzks":
        np.testing.assert_allclose(res["states"][f], ref["states"][f], rtol=0, atol=TOL)
    # device-resident entry == host-buffer entry
    dev = torch.device("cuda", 0)

    def up(a):
        return torch.from_numpy(np.frombuffer(np.ascontiguousarray(a).tobytes(), dtype=np.uint8).copy()).to(dev)
    d_n, d_off, d_ref, d_bnd = up(batch["n_points"]), up(batch["offsets"]), up(batch["ref"]), up(batch["bounds"])
    d_x0, d_end = up(batch["x0"]), up(batch["end_heading"])
    d_out = torch.zeros(total * STATE_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    d_fr = torch.zeros(total * 3, dtype=torch.float64, device=dev)
    d_st = torch.zeros(96, dtype=torch.int32, device=dev)
    d_it = torch.zeros(96, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    hn = np.ascontiguousarray(batch["n_points"], dtype=np.int32)
    rc = L.pqp_solve_batch_device_classes(s._h, 1, 96, total, hn.ctypes.data_as(C.c_void_p), None, d_n.data_ptr(),
                                          d_off.data_ptr(), d_ref.data_ptr(), d_bnd.data_ptr(), d_x0.data_ptr(), d_end.data_ptr(),
                                          None, None, d_out.data_ptr(), d_fr.data_ptr(), d_st.data_ptr(), d_it.data_ptr(), None, None)
    assert rc == 0, _lib.last_error()
    torch.cuda.synchronize()
    assert np.array_equal(d_st.cpu().numpy(), res["status"]) and np.array_equal(d_it.cpu().numpy(), res["iters"])
    assert np.array_equal(d_fr.cpu().numpy().reshape(-1, 3), res["frenet"], equal_nan=True)
    # one class for a whole device batch from the caller's bound
    d_st.zero_()
    rc = L.pqp_solve_batch_device(s._h, 1, 96, total, 416, 0, 0, d_n.data_ptr(), d_off.data_ptr(), d_ref.data_ptr(), d_bnd.data_ptr(),
                                  d_x0.data_ptr(), d_end.data_ptr(), None, None, d_out.data_ptr(), d_fr.data_ptr(), d_st.data_ptr(),
                                  d_it.data_ptr(), None, None)
    assert rc == 0, _lib.last_error()
    torch.cuda.synchronize()
    assert np.array_equal(d_st.cpu().numpy(), res["status"]) and np.array_equal(d_it.cpu().numpy(), res["iters"])
    # infeasible corridors (default eps_prim_inf) and a path beyond the largest class
    b2 = synth.infeasible_corridors(8, 50)
    r2 = s.solve(b2, formulation="K")
    o2 = oracle.solve_batch(oracle_params, 1, b2, threads=8)
    assert np.array_equal(r2["status"], o2["status"]) and np.array_equal(r2["iters"], o2["iters"])
    assert (o2["status"][0::2] == -3).all() and np.isnan(r2["frenet"][:50]).all()
    s.close()
    n3 = np.array([40, 450, 100], dtype=np.int32)
    b3 = synth.curvy_corridors(3, n_points=n3)
    s3 = _solver(3, 590)
    r3 = s3.solve(b3, formulation="K")
    o3 = oracle.solve_batch(oracle_params, 1, b3, threads=4)
    assert r3["status"][1] == -100 and np.isnan(r3["frenet"][40:490]).all()
    keep = np.array([0, 2])
    assert np.array_equal(r3["status"][keep], o3["status"][keep]) and np.array_equal(r3["iters"][keep], o3["iters"][keep])
    np.testing.assert_allclose(r3["frenet"][:40], o3["frenet"][:40], rtol=0, atol=TOL)
    np.testing.assert_allclose(r3["frenet"][490:], o3["frenet"][490:], rtol=0, atol=TOL)
    s3.close()
    # the planner chain with optimization_method "K"
    field = synth.disc_field_map()
    b = synth.map_reference_paths(24, 150)
    sp = _solver(24, int(b["offsets"][-1]))
    sp.set_map(field)
    r = sp.plan(b, formulation="K")
    o = oracle.plan(oracle_params, field, b, formulation=1)
    assert np.array_equal(r["status"], o["status"]) and np.array_equal(r["iters"], o["iters"])
    assert np.array_equal(r["ok"], o["ok"]) and np.array_equal(r["n_out"], o["n_out"])
    assert (o["status"] == SOLVED).sum() >= 12
    for i in range(24):     # the kept part of every path (what solveWithoutSmoothing returns)
        lo_, k = int(b["offsets"][i]), int(o["n_out"][i])
        for f in "xyzks":
            np.testing.assert_allclose(r["states"][f][lo_:lo_ + k], o["states"][f][lo_:lo_ + k], rtol=0, atol=TOL)
    sp.close()


def test_order_hint_changes_the_launch_order_only(oracle_params):
    """pqp_set_order_hint: longest expected work first inside a class.  Results are bit-identical with and without it,
    through the per-class device entry and through pqp_solve_batch; a hint of another length is ignored."""
    import torch
    from path_optimizer_b200 import _lib
    L = _lib.load()
    rng = np.random.default_rng(3)
    n_points = rng.integers(20, 200, size=160)
    batch = synth.curvy_corridors(160, n_points=n_points)
    total = int(batch["offsets"][-1])
    s = _solver(160, total)
    r0 = s.solve(batch)
    it = np.ascontiguousarray(r0["iters"], dtype=np.int32)
    assert L.pqp_set_order_hint(s._h, 160, it.ctypes.data_as(C.c_void_p)) == 0
    r1 = s.solve(batch)
    assert np.array_equal(r0["status"], r1["status"]) and np.array_equal(r0["iters"], r1["iters"])
    assert np.array_equal(r0["frenet"], r1["frenet"], equal_nan=True)
    # a hint of another length is ignored; NULL clears it
    assert L.pqp_set_order_hint(s._h, 7, it.ctypes.data_as(C.c_void_p)) == 0
    r2 = s.solve(batch)
    assert np.array_equal(r0["frenet"], r2["frenet"], equal_nan=True)
    assert L.pqp_set_order_hint(s._h, 0, None) == 0 and L.pqp_set_order_hint(None, 0, None) != 0
    s.close()


def test_k_and_kpc_full_size_samples(oracle_params):
    """"K" and "KPC" at a BASELINE shard size (8192 paths x 100 stations, config-4 shape): every path reaches a verdict, and
    a 48-path sample of each agrees with the oracle (status, iteration count, states at 1e-8)."""
    from path_optimizer_b200 import planner
    b = synth.straight_corridors(8192, 100, config=4)
    total = 8192 * 100
    b["ref"]["v"] = 4.0 + 3.0 * np.sin(np.arange(total) * 0.05)
    b["ref"]["a"] = 0.5 * np.cos(np.arange(total) * 0.05)
    s = _solver(8192, total)
    mk, mkp = planner.update_limits(s.params, b["ref"])
    idx = np.sort(np.random.default_rng(5).choice(8192, size=48, replace=False))
    sub = synth.take_paths(b, idx)
    o = b["offsets"]
    sel = np.concatenate([np.arange(o[i], o[i + 1]) for i in idx])
    for form, fid, kw, okw in (("K", 1, {}, {}), ("KPC", 2, dict(max_k=mk, max_kp=mkp), dict(max_k=mk[sel], max_kp=mkp[sel]))):
        res = s.solve(b, formulation=form, **kw)
        assert (res["status"] != 0).all() and (res["status"] == SOLVED).mean() > 0.9
        ref = oracle.solve_batch(oracle_params, fid, sub, threads=8, **okw)
        assert np.array_equal(res["status"][idx], ref["status"]) and np.array_equal(res["iters"][idx], ref["iters"])
        np.testing.assert_allclose(res["frenet"][sel], ref["frenet"], rtol=0, atol=TOL)
        for f in "xyzks":
            np.testing.assert_allclose(res["states"][f][sel], ref["states"][f], rtol=0, atol=TOL)
    s.close()


def test_device_entry_input_derived_launch_order(oracle_params):
    """Batches of more paths than SMs and at most 2048 are launched by pqp_solve_batch_device in an order computed on the
    device from the inputs (pqp_order_kernel: stations x (1 + |e_y0| / w), largest first).  The order must be a
    permutation -- every path gets its verdict -- and the results must be those of the host-buffer entry, bit for bit,
    including with NaN / degenerate inputs in the key."""
    rng = np.random.default_rng(12)
    n_points = rng.integers(60, 103, size=700)
    batch = synth.curvy_corridors(700, n_points=n_points)
    batch["x0"][5, 0] = np.nan                      # NaN key (whatever the solve makes of a NaN start offset)
    o = batch["offsets"]
    batch["bounds"]["c0_ub"][o[9]] = batch["bounds"]["c0_lb"][o[9]]     # zero-width first station
    total = int(o[-1])
    s = _solver(700, total)
    res = s.solve(batch)
    dres = _device_call(s, batch, classes=False)
    assert (dres["status"] != 0).all()
    assert np.array_equal(dres["status"], res["status"]) and np.array_equal(dres["iters"], res["iters"])
    assert np.array_equal(dres["frenet"], res["frenet"], equal_nan=True)
    idx = np.arange(0, 700, 11)
    keep = idx[(idx != 5)]
    sub = synth.take_paths(batch, keep)
    ref = oracle.solve_batch(oracle_params, 0, sub, threads=8)
    assert np.array_equal(res["status"][keep], ref["status"]) and np.array_equal(res["iters"][keep], ref["iters"])
    s.close()
