"""GPU: every named case of tests/envelope.py on every kernel class of every formulation at both ends of its length
range, against the oracle (same status and iteration count; 1e-8 on the iterate, 1e-6 past 1000 iterations), and the
refusal of a slack pair opened on one side on every class."""
import os

import numpy as np
import pytest

from oracle import oracle
from path_optimizer_b200 import synth
from tests import envelope, shapes
from tests.envelope import kpc_limits
from tests.test_gpu_parity import _class_ends_batch

pytestmark = pytest.mark.gpu
THREADS = max(1, min(16, os.cpu_count() or 1))

# rho 1e-9 is clamped to RHO_MIN = 1e-6 = sigma: the KKT system's constraint block is then as small as its primal block
# and the long paths' iterates carry the rounding of the factorisation (on an H100: the same status and iteration count
# on every class, up to 2.0e-7 on the 273-station class <37,7,12,34>).  The bar there is 1e-6.
LOOSE = {"rho_1e-9": 1e-6}


def _clip_limits(mk, mkp):
    """updateLimits' DBL_MAX at standstill, as the kernels read it: any bound at or beyond OSQP_INFTY is infinite.  The
    oracle scales a DBL_MAX bound by E > 1 to inf, and inf * 0 makes its infeasibility certificate NaN for the whole
    path; with 1e30 it certifies where the kernels do."""
    return np.minimum(mk, 1e30), np.minimum(mkp, 1e30)


@pytest.mark.parametrize("case", sorted(envelope.CASES))
def test_envelope_every_class(case):
    from path_optimizer_b200.solver import BatchPathSolver
    p = envelope.params(case)
    s = BatchPathSolver(params=p, max_batch=64, max_total_points=16384)
    try:
        for form in (shapes.KP, shapes.K, shapes.KPC):
            b = envelope.apply(case, _class_ends_batch(form))
            mk = mkp = None
            if form == shapes.KPC:
                mk, mkp = kpc_limits(b, p)
            res = s.solve(b, formulation=form, max_k=mk, max_kp=mkp)
            if form == shapes.KPC:
                # the oracle on the limits as the kernels read them; where DBL_MAX changes its verdict, it is only the
                # NaN certificate (status -2 at max_iter instead of -3)
                ref = oracle.solve_batch(p, form, b, threads=THREADS, max_k=_clip_limits(mk, mkp)[0],
                                         max_kp=_clip_limits(mk, mkp)[1])
                raw = oracle.solve_batch(p, form, b, threads=THREADS, max_k=mk, max_kp=mkp)
                differ = raw["status"] != ref["status"]
                assert ((raw["status"][differ] == -2) & (ref["status"][differ] == -3)).all()
                if case != "narrow_rows":
                    assert not differ.any()
            else:
                ref = oracle.solve_batch(p, form, b, threads=THREADS)
            n = len(b["n_points"])
            rows = np.arange(int(b["offsets"][-1]))
            if case in LOOSE:
                assert np.array_equal(res["status"], ref["status"]) and np.array_equal(res["iters"], ref["iters"])
                ok = np.isfinite(ref["frenet"])
                assert np.array_equal(ok, np.isfinite(res["frenet"]))
                np.testing.assert_allclose(res["frenet"][ok], ref["frenet"][ok], rtol=0, atol=LOOSE[case])
            else:
                shapes.assert_matches(res, ref, np.arange(n), rows, b["n_points"], f"{case} formulation {form}")
            gap = np.nanmax(np.abs(res["frenet"] - ref["frenet"])) if np.isfinite(ref["frenet"]).any() else 0.0
            print(f"{case:16s} form {form}: max |frenet - oracle| = {gap:.1e}, iters {ref['iters'].min()}..{ref['iters'].max()}")
    finally:
        s.close()


@pytest.mark.parametrize("form,fields", [(shapes.KP, ("c1_lb", "c3_ub")), (shapes.K, ("c1_ub",)), (shapes.KPC, ("c2_lb",))],
                         ids=["KP", "K", "KPC"])
def test_one_open_side_of_a_slack_pair_every_class(form, fields):
    """A +-1e30 bound on the open side of one row of a slack pair: every thread-per-station class refuses the path
    (PQP_INVALID_PROBLEM, 0 iterations, NaN), the paths without it are solved as the oracle solves them."""
    from path_optimizer_b200.solver import BatchPathSolver
    p = oracle.default_params()
    s = BatchPathSolver(params=p, max_batch=64, max_total_points=16384)
    try:
        for field in fields:
            b = _class_ends_batch(form)
            n = len(b["n_points"])
            o = b["offsets"]
            opened = np.arange(0, n, 2)
            for i in opened:
                b["bounds"][field][o[i] + (o[i + 1] - o[i]) // 2] = -1e30 if field.endswith("lb") else 1e30
            mk = mkp = None
            if form == shapes.KPC:
                mk, mkp = _clip_limits(*kpc_limits(b, p))
            res = s.solve(b, formulation=form, max_k=mk, max_kp=mkp)
            assert (res["status"][opened] == -100).all() and (res["iters"][opened] == 0).all(), (field, res["status"])
            rest = np.arange(1, n, 2)
            sub = synth.take_paths(b, rest)
            rows = np.concatenate([np.arange(o[i], o[i + 1]) for i in rest])
            assert np.isnan(np.delete(res["frenet"], rows, axis=0)).all()
            ref = oracle.solve_batch(p, form, sub, threads=THREADS, max_k=None if mk is None else mk[rows],
                                     max_kp=None if mk is None else mkp[rows])
            shapes.assert_matches(res, ref, rest, rows, b["n_points"][rest], f"{field} formulation {form}")
    finally:
        s.close()
