"""GPU parity tests (run with -m gpu on an H100): the CUDA path, called through the C ABI
(libpqp.so), against the CPU oracle on the same seeded inputs, against the committed golden fixtures,
and -- at BASELINE.json's full sizes -- through size-independent properties.

Tolerances.  north_star asks for <= 1e-4 on lateral offset and heading states.  The kernels run the
same recurrence as the oracle in fp64, so the tests hold them to a much tighter bar:
  FRENET_TOL = 1e-8 on (e_y, e_phi, kappa) and on the Cartesian states, identical status and
  identical ADMM iteration count per path."""
import glob
import os

import numpy as np
import pytest

from oracle import oracle
from path_optimizer_b200 import synth
from path_optimizer_b200.abi import SOLVED

pytestmark = pytest.mark.gpu

FRENET_TOL = 1e-8
NORTH_STAR_TOL = 1e-4
GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "kp_*.npz")))


@pytest.fixture(scope="module")
def solver():
    from path_optimizer_b200.solver import BatchPathSolver
    s = BatchPathSolver(max_batch=8192, max_total_points=8192 * 200)
    yield s
    s.close()


def _compare(res, ref, tol=FRENET_TOL):
    assert np.array_equal(res["status"], ref["status"])
    assert np.array_equal(res["iters"], ref["iters"])
    np.testing.assert_allclose(res["frenet"], ref["frenet"], rtol=0, atol=tol)
    for f in "xyzks":
        np.testing.assert_allclose(res["states"][f], ref["states"][f], rtol=0, atol=tol)


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_golden_fixtures(solver, path):
    g = np.load(path)
    batch = dict(n_points=g["n_points"], ref=g["ref"], bounds=g["bounds"], x0=g["x0"], end_heading=g["end_heading"])
    res = solver.solve(batch)
    _compare(res, dict(status=g["status"], iters=g["iters"], frenet=g["frenet"], states=g["states"]))
    # and the north-star bound against the independent twin
    assert np.nanmax(np.abs(res["frenet"][:, :2] - g["twin_frenet"][:, :2])) <= NORTH_STAR_TOL


def test_config2_sample_vs_oracle(solver, oracle_params):
    """BASELINE config 2 (1024 x 100 straight corridors): a 64-path sample against the oracle."""
    batch = synth.straight_corridors(64, 100)
    _compare(solver.solve(batch), oracle.solve_batch(oracle_params, 0, batch, threads=8))


def test_curvy_and_mixed_lengths_vs_oracle(solver, oracle_params):
    rng = np.random.default_rng(7)
    n_points = rng.integers(2, 260, size=48)
    n_points[:4] = [2, 3, 4, 5]
    batch = synth.curvy_corridors(48, n_points=n_points)
    _compare(solver.solve(batch), oracle.solve_batch(oracle_params, 0, batch, threads=8))


@pytest.mark.parametrize("ds", [0.15, 0.25, 0.5, 1.0])
def test_other_keep_control_steps(solver, oracle_params, ds):
    b = synth.curvy_corridors(4, 80)
    for k in range(4):
        sl = slice(k * 80, (k + 1) * 80)
        b["ref"]["s"][sl] = np.arange(80) * ds
    _compare(solver.solve(b), oracle.solve_batch(oracle_params, 0, b, threads=4))


def test_edge_cases(solver, oracle_params):
    b = synth.straight_corridors(6, 40)
    b["bounds"]["c0_lb"][10] = 3.0                    # path 0: lb > ub -> invalid
    b["end_heading"][1] = 2.5                         # path 1: end heading unconstrained (> 70 deg)
    b["bounds"]["c3_ub"][2 * 40:3 * 40] = 4.0         # path 2: wide corridor (ill-conditioned regime)
    b["bounds"]["c3_lb"][2 * 40:3 * 40] = -4.0
    b["x0"][3] = [0.0, 0.0, 0.0]                      # path 3: already on the reference
    b["bounds"]["c2_lb"][4 * 40 + 7] = b["bounds"]["c2_ub"][4 * 40 + 7] = 0.1  # path 4: collapsed corridor row
    res = solver.solve(b)
    ref = oracle.solve_batch(oracle_params, 0, b)
    assert res["status"][0] == -100 and np.all(np.isnan(res["frenet"][:40]))
    assert np.array_equal(res["status"], ref["status"])
    assert np.array_equal(res["iters"], ref["iters"])
    np.testing.assert_allclose(res["frenet"][40:], ref["frenet"][40:], rtol=0, atol=FRENET_TOL)
    # empty batch is a no-op
    empty = dict(n_points=np.zeros(0, np.int32), ref=b["ref"][:0], bounds=b["bounds"][:0],
                 x0=np.zeros((0, 3)), end_heading=np.zeros(0))
    assert len(solver.solve(empty)["status"]) == 0


def test_max_iter_status(oracle_params):
    from path_optimizer_b200.solver import BatchPathSolver
    p = oracle_params.copy()
    p.max_iter = 75
    s = BatchPathSolver(params=p, max_batch=4, max_total_points=400)
    b = synth.curvy_corridors(4, 60)
    _compare(s.solve(b), oracle.solve_batch(p, 0, b))
    s.close()


def test_full_size_config2_properties(solver):
    """1024 x 100 at full size: every path solves; the solution satisfies the QP's own constraints to
    the solver tolerance; permuting the batch permutes the result bit for bit (paths are independent
    and the kernel is deterministic); a second run is bit-identical."""
    batch = synth.straight_corridors(1024, 100)
    res = solver.solve(batch)
    assert (res["status"] == SOLVED).all()
    fr = res["frenet"].reshape(1024, 100, 3)
    p = solver.params
    w = batch["bounds"]["c0_ub"].reshape(1024, 100)
    for d in (p.d1, p.d3):  # hard circles stay inside the corridor (to eps 1e-3 of OSQP + slack)
        off = fr[:, :, 0] + d * fr[:, :, 1]
        assert np.all(np.abs(off) <= w + 5e-3)
    assert np.all(np.abs(fr[:, :, 2]) <= np.tan(p.max_steering_angle) / p.wheel_base + 5e-3)
    np.testing.assert_allclose(fr[:, 0, 0], batch["x0"][:, 0], atol=5e-3)   # initial state row
    np.testing.assert_allclose(fr[:, 0, 1], batch["x0"][:, 1], atol=5e-3)
    again = solver.solve(batch)
    assert np.array_equal(again["frenet"], res["frenet"]) and np.array_equal(again["iters"], res["iters"])
    perm = np.random.default_rng(3).permutation(1024)
    pb = dict(n_points=batch["n_points"][perm], ref=batch["ref"].reshape(1024, 100)[perm].reshape(-1),
              bounds=batch["bounds"].reshape(1024, 100)[perm].reshape(-1), x0=batch["x0"][perm],
              end_heading=batch["end_heading"][perm])
    pres = solver.solve(pb)
    assert np.array_equal(pres["frenet"].reshape(1024, 100, 3), fr[perm])
    assert np.array_equal(pres["iters"], res["iters"][perm])


def test_osqp_solver_adaptor(solver, oracle_params):
    """Single-path adaptor with the reference's call shape (solver.hpp:31-36)."""
    from path_optimizer_b200.solver import OsqpSolver
    b = synth.curvy_corridors(1, 70)
    s = OsqpSolver.create("KP", b["ref"], b["bounds"], (b["x0"][0, 0], b["x0"][0, 1]), b["x0"][0, 2],
                          b["end_heading"][0], 70)
    path = []
    assert s.solve(path) is True
    assert len(path) == 70
    ref = oracle.solve_batch(oracle_params, 0, b)
    np.testing.assert_allclose([q["x"] for q in path], ref["states"]["x"], rtol=0, atol=FRENET_TOL)
    assert OsqpSolver.create("XYZ", b["ref"], b["bounds"], (0, 0), 0, 0, 70) is None


def test_cpp_host_mirror(oracle_params, tmp_path):
    """The C++ host side (include/pqp_solver.hpp: BatchPathSolver + GpuOsqpSolver with the reference's
    create()/solve() shape) through a small compiled driver."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "tests", "cpp", "host_driver")
    src = exe + ".cpp"
    if not os.path.exists(exe) or os.path.getmtime(src) > os.path.getmtime(exe):
        subprocess.run(["g++", "-O2", "-std=c++17", src, "-o", exe, "-L" + os.path.join(root, "path_optimizer_b200"),
                        "-lpqp", "-Wl,-rpath," + os.path.join(root, "path_optimizer_b200")], check=True)
    b = synth.curvy_corridors(5, n_points=[60, 33, 100, 7, 81])
    veh = np.column_stack([b["x0"], b["end_heading"]])
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(fin, "wb") as f:
        f.write(np.int32(5).tobytes()); f.write(b["n_points"].tobytes()); f.write(b["ref"].tobytes())
        f.write(b["bounds"].tobytes()); f.write(np.ascontiguousarray(veh).tobytes())
    subprocess.run([exe, str(fin), str(fout)], check=True)
    raw = open(fout, "rb").read()
    total = int(b["n_points"].sum())
    frenet = np.frombuffer(raw, dtype=np.float64, count=3 * total).reshape(total, 3)
    o = 24 * total
    status = np.frombuffer(raw, dtype=np.int32, count=5, offset=o)
    iters = np.frombuffer(raw, dtype=np.int32, count=5, offset=o + 20)
    ok = np.frombuffer(raw, dtype=np.int32, count=1, offset=o + 40)[0]
    from path_optimizer_b200.abi import STATE_DTYPE
    path0 = np.frombuffer(raw, dtype=STATE_DTYPE, count=60, offset=o + 44)
    ref = oracle.solve_batch(oracle_params, 0, b)
    assert np.array_equal(status, ref["status"]) and np.array_equal(iters, ref["iters"])
    np.testing.assert_allclose(frenet, ref["frenet"], rtol=0, atol=FRENET_TOL)
    assert ok == 1
    np.testing.assert_allclose(path0["x"], ref["states"]["x"][:60], rtol=0, atol=FRENET_TOL)
    np.testing.assert_allclose(path0["s"], ref["states"]["s"][:60], rtol=0, atol=FRENET_TOL)


@pytest.mark.parametrize("form,name", [(1, "K"), (2, "KPC")])
def test_k_and_kpc_formulations(solver, oracle_params, form, name):
    """The other two type strings of OsqpSolver::create (solver.cpp:34-39) behind the same ABI: host-side
    sparse assembly + the generic banded kernel, against the oracle's restatement of
    solver_k_as_input.cpp / solver_kp_as_input_constrained.cpp."""
    rng = np.random.default_rng(11)
    n_points = rng.integers(2, 180, size=24)
    n_points[:3] = [2, 3, 5]
    b = synth.curvy_corridors(24, n_points=n_points)
    total = int(n_points.sum())
    mk = mkp = None
    if form == 2:
        # KPC limits from a speed profile on the reference states, derived on the DEVICE by the library's restatement of
        # ReferencePathImpl::updateLimits (reference_path_impl.cpp:203-235) and checked against the oracle's bit for bit
        import ctypes as C
        import torch
        from path_optimizer_b200 import _lib
        from path_optimizer_b200.abi import STATE_DTYPE
        b["ref"]["v"] = 4.0 + 3.0 * np.sin(np.arange(total) * 0.05)
        b["ref"]["a"] = 0.5 * np.cos(np.arange(total) * 0.05)
        b["ref"]["v"][7] = 0.0     # standstill: DBL_MAX limits (rows free on that side)
        d_ref = torch.from_numpy(np.frombuffer(np.ascontiguousarray(b["ref"], dtype=STATE_DTYPE).tobytes(), dtype=np.uint8).copy()).cuda()
        d_mk = torch.zeros(total, dtype=torch.float64, device="cuda")
        d_mkp = torch.zeros(total, dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()
        rc = _lib.load().pqp_update_limits_device(solver._h, 0, total, d_ref.data_ptr(), d_mk.data_ptr(), d_mkp.data_ptr(), None)
        assert rc == 0, _lib.last_error()
        torch.cuda.synchronize()
        mk, mkp = d_mk.cpu().numpy(), d_mkp.cpu().numpy()
        omk, omkp = oracle.update_limits(oracle_params, b["ref"])
        assert np.array_equal(mk, omk) and np.array_equal(mkp, omkp)
        assert mk[7] == np.finfo(np.float64).max
    res = solver.solve(b, formulation=name, max_k=mk, max_kp=mkp)
    ref = oracle.solve_batch(oracle_params, form, b, threads=8, max_k=mk, max_kp=mkp)
    _compare(res, ref)


def test_primal_infeasible_corridors(solver):
    """No feasible path: status -3 at the oracle's check iteration, NaN output, on every kernel class
    (thread-per-station, chunked, generic fallback via a long keep), neighbours untouched."""
    prm = oracle.default_params()
    for n, ds in ((60, 0.3), (180, 0.3), (60, 0.2)):
        b = synth.infeasible_corridors(16, n)
        if ds != 0.3:
            b["ref"]["s"] = np.tile(np.arange(n) * ds, 16)
        res = solver.solve(b)
        ref = oracle.solve_batch(prm, 0, b, threads=8)
        assert np.array_equal(res["status"], ref["status"])
        assert np.array_equal(res["iters"], ref["iters"])
        assert (ref["status"][0::2] == -3).all() and (ref["iters"][0::2] < 4000).all()
        assert np.isnan(res["frenet"][:n]).all()
        ok = np.repeat(ref["status"] == SOLVED, n)
        np.testing.assert_allclose(res["frenet"][ok], ref["frenet"][ok], rtol=0, atol=FRENET_TOL)
    b = synth.infeasible_corridors(8, 50)
    res = solver.solve(b, "K")
    ref = oracle.solve_batch(prm, 1, b, threads=8)
    assert np.array_equal(res["status"], ref["status"]) and np.array_equal(res["iters"], ref["iters"])
    assert (ref["status"][0::2] == -3).all()


def test_pipelined_host_path_mixed_chunks(solver, oracle_params):
    """pqp_solve_batch cuts batches of >= 384 paths into up to four chunks pipelined over two streams.  A batch
    whose chunks differ in length mix, shape class (keep 3 and 4, N up to 250) and feasibility must come back
    exactly as the same paths solved alone: chunk boundaries, per-chunk launch order and the overlapped copies
    leave no trace.  Host buffers here are plain pageable numpy arrays."""
    rng = np.random.default_rng(23)
    B = 640
    n_points = rng.integers(20, 130, size=B)
    n_points[rng.integers(0, B, 24)] = rng.integers(130, 250, size=24)      # some long paths (other shape classes)
    b = synth.curvy_corridors(B, n_points=n_points)
    off = b["offsets"]
    for p in rng.integers(0, B, 60):                                          # keep = 4 paths (0.25 m stations)
        b["ref"]["s"][off[p]:off[p + 1]] = np.arange(n_points[p]) * 0.25
    bad = synth.infeasible_corridors(2, int(n_points[5]))
    b["bounds"][off[5]:off[6]] = bad["bounds"][:n_points[5]]                  # one infeasible path in chunk 0
    b["x0"][5] = bad["x0"][0]
    res = solver.solve(b)
    assert res["stats"].kernel_launches >= 4
    idx = np.r_[0:12, 155:170, 318:330, 470:482, B - 10:B]
    for lo, hi in ((0, 12), (155, 170), (318, 330), (470, 482), (B - 10, B)):
        sub = synth.slice_batch(b, lo, hi)
        ref = oracle.solve_batch(oracle_params, 0, sub, threads=8)
        assert np.array_equal(res["status"][lo:hi], ref["status"])
        assert np.array_equal(res["iters"][lo:hi], ref["iters"])
        np.testing.assert_allclose(res["frenet"][off[lo]:off[hi]], ref["frenet"], rtol=0, atol=FRENET_TOL)
        np.testing.assert_allclose(res["states"]["s"][off[lo]:off[hi]], ref["states"]["s"], rtol=0, atol=FRENET_TOL)
    assert res["status"][5] == -3
    # the same batch again, and as two half batches: bitwise identical
    res2 = solver.solve(b)
    assert res2["frenet"].tobytes() == res["frenet"].tobytes() and np.array_equal(res2["iters"], res["iters"])
    half = solver.solve(synth.slice_batch(b, 0, B // 2))
    assert half["frenet"].tobytes() == res["frenet"][:off[B // 2]].tobytes()
    assert len(idx) > 0


PARAM_CASES = {
    "adaptive_off": dict(adaptive_rho=0),
    "interval100": dict(adaptive_rho_interval=100),
    "eps1e-5": dict(eps_abs=1e-5, eps_rel=1e-5),
    "alpha1": dict(alpha=1.0),
    "check10": dict(check_termination=10),
    "check7_interval35": dict(check_termination=7, adaptive_rho_interval=35),
    "no_end_heading": dict(constraint_end_heading=0),
    "weights": dict(KP_curvature_weight=3.0, KP_curvature_rate_weight=50.0, KP_deviation_weight=0.7, KP_slack_weight=10.0),
    "rho1": dict(rho=1.0, sigma=1e-5),
    "scaling0": dict(scaling=0),
    "scaling3": dict(scaling=3),
    "margin": dict(expected_safety_margin=0.6),
    "maxiter60": dict(max_iter=60),
    "check0": dict(check_termination=0, max_iter=120),
    "vehicle": dict(car_length=4.2, car_width=1.8, rear_axle_to_center=1.2, wheel_base=2.6, max_steering_angle=0.45),
}


@pytest.mark.parametrize("case", sorted(PARAM_CASES))
def test_parameter_sweep(case):
    """Every field of pqp_params is honoured the way the oracle honours it, on every KP kernel class (thread-per-station,
    chunked, generic fallback) and on the generic K kernel: intervals, tolerances, relaxation, weights, scaling,
    end-heading switch, vehicle geometry (d1..d4 recomputed by pqp_params_update_config)."""
    import ctypes as C
    from path_optimizer_b200 import _lib
    from path_optimizer_b200.solver import BatchPathSolver
    p = oracle.default_params()
    for k, v in PARAM_CASES[case].items():
        setattr(p, k, v)
    _lib.load().pqp_params_update_config(C.byref(p))
    s = BatchPathSolver(params=p, max_batch=16, max_total_points=16 * 300)
    b = synth.curvy_corridors(6, n_points=[60, 100, 33, 150, 220, 48])
    off = b["offsets"]
    b["ref"]["s"][off[5]:off[6]] = np.arange(48) * 0.2          # keep = 6 -> generic fallback kernel
    res = s.solve(b)
    ref = oracle.solve_batch(p, 0, b, threads=6)
    assert np.array_equal(res["status"], ref["status"]), (res["status"], ref["status"])
    assert np.array_equal(res["iters"], ref["iters"]), (res["iters"], ref["iters"])
    np.testing.assert_allclose(res["frenet"], ref["frenet"], rtol=0, atol=FRENET_TOL)
    small = synth.slice_batch(b, 0, 3)
    rk = s.solve(small, "K")
    ok_ = oracle.solve_batch(p, 1, small, threads=3)
    assert np.array_equal(rk["status"], ok_["status"]) and np.array_equal(rk["iters"], ok_["iters"])
    np.testing.assert_allclose(rk["frenet"], ok_["frenet"], rtol=0, atol=FRENET_TOL)
    s.close()


def test_config5_mixed_lengths_up_to_400(solver, oracle_params):
    """BASELINE config 5 shape: path lengths drawn from 50..400 stations.  Every length has a kernel class (4-warp and
    8-warp thread-per-station classes up to 256, the one-warp kernel beyond -- with its scalings in the global
    workspace above ~340 stations); shards of equal total station count (parallel.shard_by_work) give the same results
    as the whole batch."""
    from path_optimizer_b200 import parallel
    rng = np.random.default_rng(31)
    n_points = rng.integers(50, 401, size=48)
    n_points[:4] = [400, 399, 344, 343]
    b = synth.curvy_corridors(48, n_points=n_points)
    res = solver.solve(b)
    ref = oracle.solve_batch(oracle_params, 0, b, threads=8)
    _compare(res, ref)
    assert (res["status"] == SOLVED).all()
    parts = parallel.shard_by_work(n_points, 2)                     # index sets of (nearly) equal station totals
    assert sorted(np.concatenate(parts).tolist()) == list(range(48))
    assert abs(int(n_points[parts[0]].sum()) - int(n_points[parts[1]].sum())) <= int(n_points.max())
    o = b["offsets"]
    for idx in parts:
        sub = dict(n_points=n_points[idx].astype(np.int32),
                   ref=np.concatenate([b["ref"][o[i]:o[i + 1]] for i in idx]),
                   bounds=np.concatenate([b["bounds"][o[i]:o[i + 1]] for i in idx]),
                   x0=b["x0"][idx], end_heading=b["end_heading"][idx])
        part = solver.solve(sub)
        assert np.array_equal(part["iters"], res["iters"][idx]) and np.array_equal(part["status"], res["status"][idx])
        want = np.concatenate([res["frenet"][o[i]:o[i + 1]] for i in idx])
        assert part["frenet"].tobytes() == want.tobytes()
