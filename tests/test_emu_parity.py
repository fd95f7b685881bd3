"""CPU tests of the KERNEL SOURCE: path_optimizer_b200/csrc/pqp_kp_core.cuh compiled with plain g++
under a 32-thread warp emulator (tests/emu) and compared with the oracle.  This checks the
matrix-free scaling, the partitioned banded KKT solve, the ADMM recurrence, termination and adaptive
rho without a GPU.  The emulator is a test harness only; the product has no CPU path."""
import re

import numpy as np
import pytest

from oracle import oracle
from path_optimizer_b200 import synth
from tests import shapes
from tests.emu import emu

TOL = 1e-9  # same recurrence in fp64: agreement is ~1e-13 in practice


def _variant_for(batch):
    """One emulator variant for the whole batch, from the library's own selection: the class pqp_solve_batch launches
    when every path maps onto the same one, else the one class pqp_solve_batch_device takes for all of them."""
    o = batch["offsets"]
    keeps = [shapes.keep_of(shapes.KP, batch["ref"][o[b]:o[b + 1]]) for b in range(len(batch["n_points"]))]
    names = {shapes.class_of(shapes.KP, n, k)[0] for n, k in zip(batch["n_points"], keeps)}
    if len(names) > 1:
        names = {shapes.device_class_of(int(batch["n_points"].max()), min(keeps), max(keeps))}
    return emu.VARIANTS[names.pop()]


def _check(batch, params, variant=None):
    e = emu.solve_batch(params, batch, variant=_variant_for(batch) if variant is None else variant)
    o = oracle.solve_batch(params, 0, batch)
    assert np.array_equal(e["status"], o["status"])
    assert np.array_equal(e["iters"], o["iters"])
    ok = o["status"] == 1
    assert ok.any()
    np.testing.assert_allclose(e["frenet"], o["frenet"], rtol=0, atol=TOL)
    for f in "xyzks":
        np.testing.assert_allclose(e["states"][f], o["states"][f], rtol=0, atol=TOL)


def test_emu_straight(oracle_params):
    _check(synth.straight_corridors(2, 100), oracle_params)


def test_emu_curvy_and_mixed_lengths(oracle_params):
    _check(synth.curvy_corridors(5, n_points=[2, 3, 9, 41, 130]), oracle_params)


@pytest.mark.parametrize("ds", [0.2, 0.4, 0.6, 1.3])
def test_emu_other_keep_values(oracle_params, ds):
    b = synth.curvy_corridors(1, 45)
    b["ref"]["s"] = np.arange(45) * ds
    b["ref"]["x"] = np.arange(45) * ds
    _check(b, oracle_params)


def test_emu_invalid_and_unconstrained_end(oracle_params):
    b = synth.straight_corridors(2, 20)
    b["bounds"]["c2_lb"][5] = 1.0
    b["bounds"]["c2_ub"][5] = -1.0      # path 0 invalid (l > u)
    b["end_heading"][1] = 2.0           # path 1: end_psi > 70 deg -> end heading row is free
    e = emu.solve_batch(oracle_params, b, variant=5)
    o = oracle.solve_batch(oracle_params, 0, b)
    assert e["status"][0] == o["status"][0] == -100
    assert np.all(np.isnan(e["frenet"][:20]))
    assert e["status"][1] == o["status"][1] and e["iters"][1] == o["iters"][1]
    np.testing.assert_allclose(e["frenet"][20:], o["frenet"][20:], rtol=0, atol=TOL)


def test_emu_max_iter_status(oracle_params):
    p = oracle_params.copy()
    p.max_iter = 50
    b = synth.straight_corridors(1, 30)
    e = emu.solve_batch(p, b, variant=5)
    o = oracle.solve_batch(p, 0, b)
    assert e["status"][0] == o["status"][0]
    assert e["iters"][0] == o["iters"][0] == 50
    np.testing.assert_allclose(e["frenet"], o["frenet"], rtol=0, atol=TOL)


def test_emu_generic_core_still_matches(oracle_params):
    """The generic fallback kernel source (pqp_kp_core.cuh, used for keep_control_steps > 4)."""
    _check(synth.curvy_corridors(2, n_points=[33, 70]), oracle_params, variant=0)


@pytest.mark.parametrize("variant,n,ds", [(8, 187, 0.3), (6, 125, 0.25), (5, 102, 0.3), (6, 128, 0.25), (6, 77, 0.5), (7, 128, 0.3), (7, 150, 0.3),
                                           (8, 200, 0.3), (8, 131, 0.3), (9, 200, 0.25),
                                           (10, 257, 0.3), (10, 408, 0.25), (11, 384, 0.3), (12, 300, 0.3),   # thirteen- / twelve- / ten-warp long-path classes
                                           (0, 400, 0.3)])   # one-warp kernel with its scalings in the global workspace
def test_emu_shape_classes(oracle_params, variant, n, ds):
    """One full-length solve on a given class (emu.VARIANTS) at a length it takes.  Mostly the class the library selects
    for the path; 7 (Kp3<27,7,8,34>, selected for 205..256 stations at keep 3) at 128 / 150 and the one-warp kernel at
    400 stations run a class's source at lengths the selection gives to another class.
    test_emu_selected_classes runs the selected class."""
    b = synth.curvy_corridors(1, n)
    if ds != 0.3:
        b["ref"]["s"] = np.arange(n) * ds
    _check(b, oracle_params, variant=variant)


@pytest.mark.parametrize("n", [205, 256, 414])
def test_emu_selected_classes(oracle_params, n):
    """One full-length solve on the class the library selects for the path (0.3 m accumulated: keep 3):
    Kp3<27,7,8,34> at both ends of its range, and the one-warp kernel at its longest path (414 stations), which needs
    the whole shared-memory allocation."""
    _check(synth.curvy_corridors(1, n), oracle_params)


# station spacing (accumulated) per keep value: int(1.2 / ds) == keep for every path length, 2 stations included
EDGE_SPACING = {1: 1.0, 2: 0.5, 3: 0.35, 4: 0.28}


def _edge_lengths(form, keep, name, lo, hi):
    m = re.fullmatch(r"pqp_kp3_solve_kernel<\d+,\d+,\d+,(\d+)(,KPC)?>", name)
    if m:
        return shapes.partition_edges(lo, hi, lambda n: shapes.kp3_partition(n, keep, int(m.group(1))))
    m = re.fullmatch(r"pqp_kk_solve_kernel<([48])>", name)      # SPIKE form (the 13-warp class has no partition)
    if m:
        return shapes.partition_edges(lo, hi, lambda n: shapes.kk_partition(n, 26 if m.group(1) == "4" else 32))
    return [lo, hi]


@pytest.mark.parametrize("form,keep", [(0, 1), (0, 2), (0, 3), (0, 4), (2, 4), (1, 1)], ids=["KP1", "KP2", "KP3", "KP4", "KPC", "K"])
def test_emu_partition_edges(oracle_params, form, keep):
    """Every class the library selects for (formulation, keep), at the path lengths where its partition changes
    (tests/shapes.py: partition_edges -- ends of the class, both sides of every change of the separator spacing, first
    and last new separator at each spacing, odd and even separator counts), run on that class under the emulator and
    compared with the oracle.  max_iter = 50: both sides stop there, after the rho updates and termination checks on
    the way; the full-length runs are the GPU shape sweep (test_gpu_shapes.py)."""
    p = oracle_params.copy()
    p.max_iter = 50
    n_points, names = [], []
    for name, (lo, hi) in sorted(shapes.class_ranges(form, keep).items(), key=lambda kv: kv[1]):
        edges = _edge_lengths(form, keep, name, lo, hi)
        n_points += edges
        names += [name] * len(edges)
    b = synth.curvy_corridors(len(n_points), n_points=n_points)
    o = b["offsets"]
    ds = EDGE_SPACING.get(keep, 0.3)
    for i, n in enumerate(n_points):
        b["ref"]["s"][o[i]:o[i + 1]] = synth._accumulate_s(n, ds)
        assert shapes.keep_of(form, b["ref"][o[i]:o[i + 1]]) == keep
        assert shapes.class_of(form, n, keep) == (names[i], True)
    mk = mkp = None
    if form == shapes.KPC:
        b["ref"]["v"] = 4.0 + 3.0 * np.sin(np.arange(o[-1]) * 0.05)
        b["ref"]["a"] = 0.5 * np.cos(np.arange(o[-1]) * 0.05)
        b["ref"]["v"][::11] = 0.0
        mk, mkp = oracle.update_limits(oracle_params, b["ref"])
    ref = oracle.solve_batch(p, form, b, threads=8, max_k=mk, max_kp=mkp)
    names = np.array(names)
    for name in dict.fromkeys(names):
        idx = np.nonzero(names == name)[0]
        sub = synth.take_paths(b, idx)
        sel = np.concatenate([np.arange(o[i], o[i + 1]) for i in idx])
        e = emu.solve_batch(p, sub, variant=name, max_k=None if mk is None else mk[sel], max_kp=None if mk is None else mkp[sel])
        bad = (e["status"] != ref["status"][idx]) | (e["iters"] != ref["iters"][idx])
        assert not bad.any(), (name, "N =", np.asarray(n_points)[idx][bad].tolist())
        for f in range(3):
            np.testing.assert_allclose(e["frenet"][:, f], ref["frenet"][sel, f], rtol=0, atol=TOL, err_msg=name)
        for f in "xyzks":
            np.testing.assert_allclose(e["states"][f], ref["states"][f][sel], rtol=0, atol=TOL, err_msg=name)


def _limits(batch):
    """KPC limits as ReferencePathImpl::updateLimits derives them (reference_path_impl.cpp:203-235) for a
    synthetic speed profile: friction circle and curvature-rate limit."""
    total = int(batch["offsets"][-1])
    v = 4.0 + 3.0 * np.sin(np.arange(total) * 0.05)
    a = 0.5 * np.cos(np.arange(total) * 0.05)
    max_k = np.sqrt((0.4 * 9.8) ** 2 - a ** 2) / v ** 2
    max_kp = 0.1 / v
    return max_k, max_kp


@pytest.mark.parametrize("form", [1, 2])
def test_emu_generic_kernel_k_and_kpc(oracle_params, form):
    """"K" (SolverKAsInput) and "KPC" (SolverKpAsInputConstrained) on the generic banded kernel source +
    host assembly (pqp_gen_core.cuh, pqp_forms.h) against the oracle's own restatement of those files."""
    b = synth.curvy_corridors(4, n_points=[2, 9, 47, 120])
    mk, mkp = _limits(b) if form == 2 else (None, None)
    e = emu.solve_batch_generic(oracle_params, form, b, max_k=mk, max_kp=mkp)
    o = oracle.solve_batch(oracle_params, form, b, max_k=mk, max_kp=mkp)
    assert np.array_equal(e["status"], o["status"]) and np.array_equal(e["iters"], o["iters"])
    assert (o["status"] == 1).any()
    np.testing.assert_allclose(e["frenet"], o["frenet"], rtol=0, atol=TOL)
    for f in "xyzks":
        np.testing.assert_allclose(e["states"][f], o["states"][f], rtol=0, atol=TOL)


@pytest.mark.parametrize("variant", [0, 5, 7])
def test_emu_primal_infeasible(oracle_params, variant):
    """Corridors with no feasible path: OSQP's primal-infeasibility certificate fires (status -3) at the
    same check iteration as in the oracle, the output is NaN, feasible neighbours are untouched.  Kp3<17,6,4,17> (5)
    and Kp3<27,7,8,34> (7) at lengths the library selects them for; the one-warp kernel (0) forced at 60 stations."""
    n = 220 if variant == 7 else 60
    b = synth.infeasible_corridors(6 if variant == 0 else 2, n)
    if variant != 0:
        assert emu.VARIANTS[shapes.class_of(shapes.KP, n, 3)[0]] == variant
    e = emu.solve_batch(oracle_params, b, variant=variant)
    o = oracle.solve_batch(oracle_params, 0, b)
    assert np.array_equal(e["status"], o["status"]) and np.array_equal(e["iters"], o["iters"])
    assert (o["status"][0::2] == -3).all() and (o["status"][1::2] == 1).all()
    assert (o["iters"][0::2] < 4000).all()
    assert np.isnan(e["frenet"][:n]).all()
    ok = np.repeat(o["status"] == 1, n)
    np.testing.assert_allclose(e["frenet"][ok], o["frenet"][ok], rtol=0, atol=TOL)


def test_emu_generic_kernel_primal_infeasible(oracle_params):
    b = synth.infeasible_corridors(4, 40)
    e = emu.solve_batch_generic(oracle_params, 1, b)
    o = oracle.solve_batch(oracle_params, 1, b)
    assert np.array_equal(e["status"], o["status"]) and np.array_equal(e["iters"], o["iters"])
    assert (o["status"][0::2] == -3).all()


PARAM_CASES = {
    "adaptive_off_maxiter": dict(adaptive_rho=0, max_iter=300),
    "interval100": dict(adaptive_rho_interval=100),
    "check7_interval35": dict(check_termination=7, adaptive_rho_interval=35),
    "no_end_heading_weights": dict(constraint_end_heading=0, KP_curvature_weight=3.0, KP_curvature_rate_weight=50.0,
                                   KP_deviation_weight=0.7, KP_slack_weight=10.0),
    "scaling0_rho1": dict(scaling=0, rho=1.0, sigma=1e-5),
    "check0": dict(check_termination=0, max_iter=120),
}


@pytest.mark.parametrize("case", sorted(PARAM_CASES))
def test_emu_parameter_sweep(oracle_params, case):
    """Every setting in pqp_params is honoured the way the oracle (= OSQP's rules) honours it: check and adaptation
    intervals, adaptive rho off, no end-heading row, other weights, no scaling, no termination checks at all."""
    p = oracle_params.copy()
    for k, v in PARAM_CASES[case].items():
        setattr(p, k, v)
    b = synth.curvy_corridors(2, n_points=[60, 100])
    e = emu.solve_batch(p, b, variant=5)
    o = oracle.solve_batch(p, 0, b)
    assert np.array_equal(e["status"], o["status"]) and np.array_equal(e["iters"], o["iters"])
    np.testing.assert_allclose(e["frenet"], o["frenet"], rtol=0, atol=TOL)


@pytest.mark.parametrize("variant,n_points", [(20, [2, 3, 9, 60, 128]), (21, [200, 256]), (22, [5, 100, 136])])
def test_emu_kpc_thread_per_station(oracle_params, variant, n_points):
    """"KPC" (SolverKpAsInputConstrained) on the thread-per-station skeleton, assembled in the kernel: same status,
    iteration count and iterates as the oracle's restatement of solver_kp_as_input_constrained.cpp, including limits
    from a speed profile with standstill stations (DBL_MAX limits: rows free on that side)."""
    b = synth.curvy_corridors(len(n_points), n_points=n_points)
    total = int(b["offsets"][-1])
    ref = b["ref"].copy()
    ref["v"] = 4.0 + 3.0 * np.sin(np.arange(total) * 0.05)
    ref["a"] = 0.5 * np.cos(np.arange(total) * 0.05)
    ref["v"][::11] = 0.0
    mk, mkp = oracle.update_limits(oracle_params, ref)
    e = emu.solve_batch(oracle_params, b, variant=variant, max_k=mk, max_kp=mkp)
    o = oracle.solve_batch(oracle_params, 2, b, threads=4, max_k=mk, max_kp=mkp)
    assert np.array_equal(e["status"], o["status"]) and np.array_equal(e["iters"], o["iters"])
    assert (o["status"] == 1).any()
    np.testing.assert_allclose(e["frenet"], o["frenet"], rtol=0, atol=TOL)
    for f in "xyzks":
        np.testing.assert_allclose(e["states"][f], o["states"][f], rtol=0, atol=TOL)


def test_emu_kpc_infeasible_and_parameters(oracle_params):
    # (the emulator runs one pthread per lane: a 4000-iteration path costs ~20 s, so cap the iteration count here; the
    # full-length run is the GPU test test_gpu_parity.py::test_k_and_kpc_formulations / test_primal_infeasible_corridors)
    p = oracle_params.copy()
    p.max_iter = 600
    b = synth.infeasible_corridors(2, 60)
    mk, mkp = _limits(b)
    e = emu.solve_batch(p, b, variant=20, max_k=mk, max_kp=mkp)
    o = oracle.solve_batch(p, 2, b, threads=4, max_k=mk, max_kp=mkp)
    assert np.array_equal(e["status"], o["status"]) and np.array_equal(e["iters"], o["iters"])
    assert (o["status"] != 1).any()
    p = oracle_params.copy()
    p.constraint_end_heading = 0; p.KP_deviation_weight = 0.7; p.KP_slack_weight = 10.0
    p.check_termination = 7; p.adaptive_rho_interval = 35
    b = synth.curvy_corridors(2, n_points=[60, 100])
    mk, mkp = _limits(b)
    e = emu.solve_batch(p, b, variant=20, max_k=mk, max_kp=mkp)
    o = oracle.solve_batch(p, 2, b, threads=4, max_k=mk, max_kp=mkp)
    assert np.array_equal(e["status"], o["status"]) and np.array_equal(e["iters"], o["iters"])
    np.testing.assert_allclose(e["frenet"], o["frenet"], rtol=0, atol=TOL)


def _check_k(batch, params, variant):
    e = emu.solve_batch(params, batch, variant=variant)
    o = oracle.solve_batch(params, 1, batch, threads=4)
    assert np.array_equal(e["status"], o["status"]) and np.array_equal(e["iters"], o["iters"])
    np.testing.assert_allclose(e["frenet"], o["frenet"], rtol=0, atol=TOL)
    for f in "xyzks":
        np.testing.assert_allclose(e["states"][f], o["states"][f], rtol=0, atol=TOL)
    return o


@pytest.mark.parametrize("variant,n_points", [(30, [2, 3, 5, 26, 27, 53, 100, 105, 128]), (31, [129]), (32, [416])])
def test_emu_k_thread_per_station(oracle_params, variant, n_points):
    """"K" (SolverKAsInput) on its thread-per-station kernels (pqp_kk_core.cuh: stencils in registers; reduced KKT in SPIKE
    form with dense inverses in the four- and eight-warp classes -- lengths either side of every change of the chunk length
    of the former --, by block cyclic reduction with warp-local shuffle levels in the thirteen-warp class): same status, iteration count
    and iterates as the oracle's restatement of solver_k_as_input.cpp, for both corridor kinds."""
    p = oracle_params.copy()
    if variant != 30:
        p.max_iter = 150     # (256 / 416 host threads per barrier and shuffle: keep the emulated run short; both sides stop at max_iter)
    o = _check_k(synth.curvy_corridors(len(n_points), n_points=n_points), p, variant)
    assert (o["status"] == 1).all() if variant == 30 else (o["iters"] == 150).all()
    if variant == 30:
        _check_k(synth.straight_corridors(1, 64), oracle_params, variant)


def test_emu_k_infeasible_and_parameters(oracle_params):
    # (eps_prim_inf 1e-2 lets the certificate fire after 325 iterations instead of 1875: same code path, a fifth of the
    # emulated barriers; the default tolerance runs on the GPU, test_gpu_parity.py::test_k_thread_per_station_classes)
    p = oracle_params.copy()
    p.eps_prim_inf = 1e-2
    b = synth.infeasible_corridors(2, 40)
    o = _check_k(b, p, 30)
    assert o["status"][0] == -3 and o["status"][1] == 1 and o["iters"][0] < 1000
    for case in ("adaptive_off_maxiter", "check7_interval35", "scaling0_rho1", "check0"):
        p = oracle_params.copy()
        for k, v in PARAM_CASES[case].items():
            setattr(p, k, v)
        _check_k(synth.curvy_corridors(1, n_points=[24]), p, 30)
    p = oracle_params.copy()
    p.constraint_end_heading = 0; p.K_curvature_weight = 7.0; p.K_curvature_rate_weight = 60.0
    p.K_deviation_weight = 0.4; p.KP_slack_weight = 10.0; p.max_steering_angle = 0.2
    _check_k(synth.curvy_corridors(1, n_points=[40]), p, 30)
    # an invalid corridor (lower bound above the upper bound): OSQP's setup refuses it
    b = synth.curvy_corridors(2, n_points=[30, 30])
    b["bounds"]["c0_lb"][10] = b["bounds"]["c0_ub"][10] + 1.0
    e = emu.solve_batch(oracle_params, b, variant=30)
    o = oracle.solve_batch(oracle_params, 1, b)
    assert np.array_equal(e["status"], o["status"]) and e["status"][0] == -100 and e["status"][1] == 1
