"""CPU tests of the kernel source across the parameter envelope (tests/envelope.py): the emulator build of every kernel
family (tests/emu) against the oracle on every named case, max_iter 1 on every kernel class, the spacing ends of the
keep rule, and KPC limits that come out NaN.  The GPU side is test_gpu_envelope.py."""
import numpy as np
import pytest

from oracle import oracle
from path_optimizer_b200 import synth
from tests import envelope, shapes
from tests.emu import emu
from tests.envelope import kpc_limits

TOL = 1e-9
CAP = 150       # iterations per emulated solve (the emulator runs one host thread per lane); full runs are on the GPU

# one class per family, at a length it takes: (name, formulation, emulator variant, N)
FAMILIES = [("KP thread per station", shapes.KP, 5, 60), ("KP one warp", shapes.KP, 0, 40),
            ("K", shapes.K, 30, 40), ("KPC", shapes.KPC, 20, 40)]


def _run(p, form, variant, b, mk=None, mkp=None):
    e = emu.solve_batch(p, b, variant=variant, max_k=mk, max_kp=mkp)
    o = oracle.solve_batch(p, form, b, threads=4, max_k=mk, max_kp=mkp)
    return e, o


def _assert_same(e, o, what):
    assert np.array_equal(e["status"], o["status"]), (what, e["status"], o["status"])
    assert np.array_equal(e["iters"], o["iters"]), (what, e["iters"], o["iters"])
    np.testing.assert_allclose(e["frenet"], o["frenet"], rtol=0, atol=TOL, err_msg=what)
    for f in "xyzk":
        np.testing.assert_allclose(e["states"][f], o["states"][f], rtol=0, atol=TOL, err_msg=what)


@pytest.mark.parametrize("case", sorted(envelope.CASES))
def test_emu_envelope(case):
    """Each case on one class per kernel family: same status and iteration count as the oracle, 1e-9 on the iterate."""
    p = envelope.params(case)
    p.max_iter = min(p.max_iter, CAP)
    for name, form, variant, n in FAMILIES:
        b = envelope.apply(case, synth.curvy_corridors(2, n_points=[n, n - 7]))
        mk = mkp = None
        if form == shapes.KPC:
            mk, mkp = kpc_limits(b, p)
        e, o = _run(p, form, variant, b, mk, mkp)
        _assert_same(e, o, f"{case}: {name}")


def test_envelope_cases_do_what_they_say():
    """The geometry and weight cases reach the magnitudes their names promise."""
    rb, tr, d2 = envelope.params("robot"), envelope.params("truck"), envelope.params("d2_zero")
    assert d2.d2 == 0.0
    assert np.tan(rb.max_steering_angle) / rb.wheel_base > 1.6
    assert tr.d4 - tr.d1 == pytest.approx(9.0)
    assert envelope.params("no_steering").max_steering_angle == 0.0
    b = envelope.apply("open_bounds", synth.curvy_corridors(1, 30))
    assert (b["bounds"]["c0_ub"] == 1e30).any() and (b["bounds"]["c2_lb"] == -1e30).any()
    b = envelope.apply("narrow_rows", synth.curvy_corridors(1, 30))
    w = b["bounds"]["c0_ub"] - b["bounds"]["c0_lb"]
    assert w.min() < 1e-3 < w.max() < 1e-2


@pytest.mark.parametrize("max_iter", [1, 2])
def test_emu_first_iterations_every_class(max_iter):
    """max_iter 1 and 2 on every kernel class the emulator builds, at the top of its length range.  OSQP's first
    iteration from zero ends at x = 0, z = clamp(0), y = -rho clamp(0); the x0 rows then leave a primal residual, so the
    verdict is MAX_ITER_REACHED (-2), as in the oracle."""
    p = oracle.default_params()
    p.max_iter = max_iter
    runs = {}      # class name -> (formulation, N at the top of its range, station spacing)
    for form, keep, ds in [(shapes.KP, 3, 0.35), (shapes.KP, 4, 0.25), (shapes.KP, 5, 0.2), (shapes.K, 1, 0.3),
                           (shapes.KPC, 4, 0.3)]:
        for name, (lo, hi) in shapes.class_ranges(form, keep).items():
            runs.setdefault(name, (form, hi, ds))
    runs.setdefault("pqp_kp3_solve_kernel<23,7,4,17,KPC>", (shapes.KPC, 128, 0.3))   # (the device entries' KPC class)
    assert set(runs) == set(emu.VARIANTS)
    for name, (form, n, ds) in runs.items():
        variant = emu.VARIANTS[name]
        b = synth.curvy_corridors(2, n_points=[n, n])
        b["ref"]["s"] = np.concatenate([synth._accumulate_s(n, ds)] * 2)
        mk = mkp = None
        if form == shapes.KPC:
            mk, mkp = kpc_limits(b, p)
        e, o = _run(p, form, variant, b, mk, mkp)
        assert (o["status"] == -2).all() and (o["iters"] == max_iter).all(), (name, o["status"])
        _assert_same(e, o, f"max_iter {max_iter}: {name}")
    for form in (shapes.K, shapes.KPC):       # the generic banded source + host assembly
        b = synth.curvy_corridors(2, n_points=[9, 40])
        mk = mkp = None
        if form == shapes.KPC:
            mk, mkp = kpc_limits(b, p)
        e = emu.solve_batch_generic(p, form, b, max_k=mk, max_kp=mkp)
        o = oracle.solve_batch(p, form, b, max_k=mk, max_kp=mkp)
        _assert_same(e, o, f"max_iter {max_iter}: generic form {form}")


@pytest.mark.parametrize("form,ds,variant", [(shapes.KP, 0.11, 0), (shapes.KP, 1.1, 5), (shapes.K, 0.02, 30),
                                              (shapes.KPC, 0.02, 20)], ids=["KP0.11", "KP1.1", "K0.02", "KPC0.02"])
def test_emu_spacing_ends(form, ds, variant):
    """KP at 0.11 m (keep 10, the largest KP accepts) and 1.1 m (keep 1: the ds couplings of stations a metre apart);
    K and KPC, whose keep does not follow the spacing, at 0.02 m."""
    p = oracle.default_params()
    p.max_iter = CAP
    b = synth.curvy_corridors(2, n_points=[40, 33])
    o_ = b["offsets"]
    for i in range(2):
        b["ref"]["s"][o_[i]:o_[i + 1]] = synth._accumulate_s(int(b["n_points"][i]), ds)
    if form == shapes.KP:
        assert shapes.keep_of(form, b["ref"][:40]) == (10 if ds < 0.5 else 1)
    mk = mkp = None
    if form == shapes.KPC:
        mk, mkp = kpc_limits(b, p)
    e, o = _run(p, form, variant, b, mk, mkp)
    _assert_same(e, o, f"ds {ds}")


def test_emu_kpc_nan_limits():
    """KPC limits at standstill and at |a| > mu g.  updateLimits gives DBL_MAX at a speed below 1e-4 (the curvature rows
    are free on that side: path 1 is solved) and NaN where |a| > mu g; the oracle refuses that path (-100, OSQP's
    l <= u check fails on NaN) and so does the kernel."""
    p = oracle.default_params()
    p.max_iter = CAP
    b = synth.curvy_corridors(3, n_points=[40, 40, 40])
    total = int(b["offsets"][-1])
    b["ref"]["v"] = 5.0
    b["ref"]["a"] = 0.0
    b["ref"]["v"][45] = 0.0                                  # standstill inside path 1
    b["ref"]["a"][100] = 1.5 * p.mu * 9.8                    # |a| > mu g inside path 2
    mk, mkp = oracle.update_limits(p, b["ref"])
    assert np.isfinite(mk[:40]).all() and not np.isfinite(mk[100]), (mk[40:50], mk[100])
    e, o = _run(p, shapes.KPC, 20, b, mk, mkp)
    assert mk[45] == np.finfo(np.float64).max
    assert o["status"][2] == -100 and o["status"][0] == 1 and o["status"][1] == 1
    assert np.array_equal(e["status"], o["status"]) and np.array_equal(e["iters"], o["iters"])
    ok = np.repeat(o["status"] != -100, 40)
    assert np.isnan(e["frenet"][~ok]).all()
    np.testing.assert_allclose(e["frenet"][ok], o["frenet"][ok], rtol=0, atol=TOL)
    assert total == 120


# (formulation, emulator variant, the bound fields that open one row of a slack pair)
PAIR_FIELDS = [(shapes.KP, 5, ("c1_lb", "c1_ub", "c3_lb", "c3_ub")), (shapes.KP, 0, ("c1_lb", "c3_ub")),
               (shapes.K, 30, ("c1_lb", "c1_ub")), (shapes.KPC, 20, ("c2_lb", "c2_ub"))]


@pytest.mark.parametrize("form,variant,fields", PAIR_FIELDS, ids=["KP", "KP-one-warp", "K", "KPC"])
def test_emu_one_open_side_of_a_slack_pair(form, variant, fields):
    """A caller bound of +-1e30 on the open side of one row of a slack pair (KP: c1, c3; K: c1; KPC: c2) makes that row
    free on both sides: OSQP gives it RHO_MIN (constr_type -1) while its partner keeps the inequality rho.  The kernels
    eliminate the slack on the premise that both rows weigh the same, so they refuse such a path: PQP_INVALID_PROBLEM,
    0 iterations, NaN output; the path beside it is solved as the oracle solves it.  The generic banded kernel (per-row
    weights) solves the refused layout as the oracle does.  A bound opened on a box row (K: c3) is not refused."""
    p = oracle.default_params()
    p.max_iter = CAP
    for field in fields + (("c3_lb",) if form == shapes.K else ()):
        b = synth.curvy_corridors(2, n_points=[40, 33])
        idx = np.arange(40)
        b["bounds"][field][:40][idx % 5 == 2] = -1e30 if field.endswith("lb") else 1e30
        mk = mkp = None
        if form == shapes.KPC:
            mk, mkp = kpc_limits(b, p)
        e, o = _run(p, form, variant, b, mk, mkp)
        if field == "c3_lb" and form == shapes.K:
            _assert_same(e, o, field)
            continue
        assert o["status"][0] != -100, field          # (OSQP solves it)
        assert e["status"][0] == -100 and e["iters"][0] == 0, (field, e["status"], e["iters"])
        assert np.isnan(e["frenet"][:40]).all()
        assert e["status"][1] == o["status"][1] and e["iters"][1] == o["iters"][1], field
        np.testing.assert_allclose(e["frenet"][40:], o["frenet"][40:], rtol=0, atol=TOL, err_msg=field)
        if form != shapes.KP:
            g = emu.solve_batch_generic(p, form, b, max_k=mk, max_kp=mkp)
            _assert_same(g, o, f"generic kernel, {field}")
