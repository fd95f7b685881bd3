"""CPU tests of how a run ends (tests/verdicts.py): every named verdict branch is reached in every formulation, the
independent twin (oracle/twin.py) takes the oracle's branch on every case, the kernel source under the emulator
(tests/emu) takes it on one class per kernel family, adaptive rho lands on its lower clamp, and the oracle refuses the
settings OSQP refuses.  The GPU side is test_gpu_verdicts.py."""
import collections

import numpy as np
import pytest

from oracle import oracle, twin
from path_optimizer_b200 import synth
from path_optimizer_b200.abi import INVALID_PROBLEM
from tests import envelope, verdicts
from tests.emu import emu

TOL = 1e-9
LONG_RUN = 1500
FORMS = {"KP": 0, "K": 1, "KPC": 2}
ASSEMBLE = {0: twin.assemble_kp, 1: twin.assemble_k, 2: twin.assemble_kpc}
# one class per kernel family: (formulation, emulator variant; "generic": the banded kernel with host assembly)
FAMILIES = {"kp3 KP": (0, 5), "kp3 KPC": (2, 20), "K": (1, 30), "generic K": (1, "generic"), "one-warp KP": (0, 0)}

_cache = {}


def _cases(form, n_points=(40, 33)):
    key = (form, tuple(n_points))
    if key not in _cache:
        _cache[key] = verdicts.batch_cases(form, synth.curvy_corridors(len(n_points), n_points=list(n_points)), threads=8)
    return _cache[key]


def _path(batches, c):
    b, mk, mkp = batches[c["kind"]]
    sub = synth.take_paths(b, [c["path"]])
    rows = slice(b["offsets"][c["path"]], b["offsets"][c["path"] + 1])
    return sub, (None, None) if mk is None else (np.ascontiguousarray(mk[rows]), np.ascontiguousarray(mkp[rows]))


@pytest.mark.parametrize("form", sorted(FORMS), ids=sorted(FORMS))
def test_witness_every_branch(form):
    """Every named branch is reached in this formulation, with and without termination checks, and max_iter lands on
    an adaptation iteration that is not a check iteration; no case lies within MIN_MARGIN of its threshold."""
    cases, dropped, _ = _cases(FORMS[form])
    got = collections.Counter(c["branch"] for c in cases)
    assert set(got) == set(verdicts.BRANCHES), sorted(set(verdicts.BRANCHES) - set(got))
    check0 = {c["branch"] for c in cases if c["params"].check_termination == 0}
    assert check0 == {b for b in verdicts.BRANCHES if b.endswith("_final")}, check0
    assert any(c["adapt_not_check"] for c in cases)
    assert {c["schedule"] for c in cases} == set(verdicts.SCHEDULES)
    assert {c["label"] for c in cases} == {""} | set(verdicts.SETTINGS)
    assert all(c["margin"] >= verdicts.MIN_MARGIN for c in cases)
    print(f"{form}: {len(cases)} cases, {dropped} dropped for margin, {dict(sorted(got.items()))}")


@pytest.mark.parametrize("form", sorted(FORMS), ids=sorted(FORMS))
def test_twin_takes_the_oracles_branch(form):
    """The twin against the oracle on every case of a short path up to LONG_RUN iterations: same status, iteration
    count and rho updates, and the iterate to 1e-9 (NaN where the status carries no solution).  (Past that the two
    linear algebras' rounding can tip an adaptive-rho decision: on "K", one update more after 4000 iterations.)"""
    f = FORMS[form]
    cases, _, batches = _cases(f, (24,))
    short = [c for c in cases if c["iters"] <= LONG_RUN]
    assert {c["branch"] for c in short} == {c["branch"] for c in cases} and len(short) > 0.75 * len(cases)
    cases = short
    for c in cases:
        sub, (mk, mkp) = _path(batches, c)
        args = (sub["ref"], sub["bounds"], sub["x0"][0], float(sub["end_heading"][0]))
        r = oracle.solve_qp(c["params"], f, *args, max_k=mk, max_kp=mkp)
        qp = ASSEMBLE[f](c["params"], *args, *((mk, mkp) if f == 2 else ()))
        t = twin.osqp_twin(c["params"], *qp)
        what = (form, c["kind"], c["schedule"], c["label"], c["branch"], c["params"].max_iter)
        assert (t["status"], t["iters"]) == (r["info"].status, r["info"].iters) == (c["status"], c["iters"]), (what, t["status"], t["iters"])
        assert t["rho_updates"] == r["info"].rho_updates and t["rho"] == pytest.approx(r["info"].rho_final, rel=1e-9), what
        np.testing.assert_allclose(t["x"], r["x"], rtol=0, atol=TOL, err_msg=str(what))


def _emu(p, form, variant, b, mk, mkp):
    if variant == "generic":
        return emu.solve_batch_generic(p, form, b, max_k=mk, max_kp=mkp)
    return emu.solve_batch(p, b, variant=variant, max_k=mk, max_kp=mkp)


def _assert_same(e, o, what):
    assert np.array_equal(e["status"], o["status"]) and np.array_equal(e["iters"], o["iters"]), \
        (what, e["status"], o["status"], e["iters"], o["iters"])
    np.testing.assert_allclose(e["frenet"], o["frenet"], rtol=0, atol=TOL, err_msg=str(what))
    for f in "xyzk":
        np.testing.assert_allclose(e["states"][f], o["states"][f], rtol=0, atol=TOL, err_msg=str(what))


@pytest.mark.parametrize("family", sorted(FAMILIES), ids=sorted(FAMILIES))
def test_emu_every_branch(family):
    """The kernel source of one class per family against the oracle on every branch (the shortest case of each, and
    of each without termination checks, with fixed rho and with max_iter on an adaptation iteration off the check
    grid): same status and iteration count, 1e-9 on the output."""
    form, variant = FAMILIES[family]
    cases, _, batches = _cases(form)
    picked = verdicts.one_per_branch(cases)
    assert {c["branch"] for c in picked} == set(verdicts.BRANCHES)
    for c in picked:
        sub, (mk, mkp) = _path(batches, c)
        o = oracle.solve_batch(c["params"], form, sub, max_k=mk, max_kp=mkp)
        assert o["status"][0] == c["status"] and o["iters"][0] == c["iters"]
        _assert_same(_emu(c["params"], form, variant, sub, mk, mkp), o,
                     (family, c["kind"], c["schedule"], c["label"], c["branch"], c["params"].max_iter))


@pytest.mark.parametrize("family", sorted(FAMILIES), ids=sorted(FAMILIES))
def test_rho_lands_on_its_lower_clamp(family):
    """Adaptation every iteration from rho = 1e-5 and 1e5 on a QP that x = 0 solves: the first estimate is 0 and the
    update lands exactly on RHO_MIN (the oracle's rho_final, one update; the twin agrees); the kernels end as the
    oracle does, at a check iteration and at an off-grid max_iter."""
    form, variant = FAMILIES[family]
    b = verdicts.rho_clamp_path(synth.straight_corridors(1, 40))
    base = oracle.default_params()
    mk, mkp = verdicts.kpc_limits(base, b) if form == 2 else (None, None)
    path = dict(ref=b["ref"], bounds=b["bounds"], x0=b["x0"][0], end_heading=float(b["end_heading"][0]))
    for rho in (1e-5, 1e5):
        cases, dropped = verdicts.pick(base, form, path, mk, mkp, schedules=("c25_a25", "c25_a7"),
                                       over=dict(rho=rho, adaptive_rho_interval=1))
        assert dropped == 0 and {c["branch"] for c in cases} >= {"solved_check", "solved_final"}, cases
        for c in cases:
            assert c["rho_final"] == verdicts.RHO_MIN and c["rho_updates"] >= 1, c
            if c["iters"] > 100:
                continue
            t = twin.osqp_twin(c["params"], *ASSEMBLE[form](c["params"], path["ref"], path["bounds"], path["x0"],
                                                           path["end_heading"], *((mk, mkp) if form == 2 else ())))
            assert t["rho"] == verdicts.RHO_MIN and (t["status"], t["iters"]) == (c["status"], c["iters"])
            o = oracle.solve_batch(c["params"], form, b, max_k=mk, max_kp=mkp)
            _assert_same(_emu(c["params"], form, variant, b, mk, mkp), o, (family, rho, c["branch"]))


@pytest.mark.parametrize("name", sorted(verdicts.ILLEGAL))
def test_oracle_refuses_illegal_settings(name):
    """OSQP's osqp_setup refuses these settings (validate_settings), so the reference's solve() fails: the oracle
    reports PQP_INVALID_PROBLEM with 0 iterations and NaN output on every path, in every formulation."""
    p = oracle.default_params()
    for k, v in verdicts.ILLEGAL[name].items():
        setattr(p, k, v)
    assert not verdicts.legal(p)
    b = synth.infeasible_corridors(2, 20)
    mk, mkp = verdicts.kpc_limits(p, b)
    for form in (0, 1, 2):
        r = oracle.solve_batch(p, form, b, max_k=mk if form == 2 else None, max_kp=mkp if form == 2 else None)
        assert (r["status"] == INVALID_PROBLEM).all() and (r["iters"] == 0).all(), (name, form, r["status"])
        assert np.isnan(r["frenet"]).all()


def test_every_named_case_is_legal():
    """The defaults, every envelope case (tests/envelope.py) and every verdict schedule and setting are inside OSQP's
    legal settings, and the oracle solves them."""
    ps = [oracle.default_params()] + [envelope.params(c) for c in envelope.CASES]
    ps += [verdicts.params(oracle.default_params(), s, 50, **o) for s in verdicts.SCHEDULES
           for o in [{}] + list(verdicts.SETTINGS.values())]
    b = synth.curvy_corridors(1, 20)
    for p in ps:
        assert verdicts.legal(p)
        q = p.copy()
        q.max_iter = min(q.max_iter, 30)
        assert oracle.solve_batch(q, 0, b)["status"][0] != INVALID_PROBLEM
