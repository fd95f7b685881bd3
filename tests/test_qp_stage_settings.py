"""CPU tests of the width-4 generic core (csrc/pqp_gen_core.cuh, gen_solve_qp<4, true>, compiled with g++ through
tests/emu/smooth_emu.cpp) on the TENSION2 smoothing QP away from the defaults, against the oracle's OSQP
(oracle/smooth.py): every schedule of tests/verdicts.py, scaling 0 and 10, max_iter from 1 to past the first verdict,
eps_dual_inf from 1e-4 to 1, the verdict suite's tolerance settings, and the cost weights at 0, tiny and large.

Status and iterations must be equal; near the origin the stations' x and y (what the stage keeps) must agree within 1e-9
of their scale (test_weights documents a looser bar for lopsided weights).  The headings are not compared: with a tiny curvature weight the last heading is fixed only by a cost
of order 1e-6 and moves by 1e-6 rad between two correct solvers.  A case whose
deciding comparison in the oracle lies within 1e-9 (relative) of its threshold is a rounding coin flip and is dropped
and counted.  The named cases reproduce two defects of the core: it never tested OSQP's dual infeasibility, and far
from the origin with a large deviation weight its explicit inverses of the separator Schur blocks lost the x-step."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import smooth as S
from path_optimizer_b200 import abi
from tests import smooth_cases as sc
from tests import verdicts as V
from tests.emu import smooth_emu as E

CASES = sc.named()
NEAR = 1e-9
FAR = 1e5
NAMES = ["config1", "corner", "u_turn", "straight_x", "pose0", "pose1", "pose17"]
WEIGHTS = [S.WEIGHTS, (0.0, 1.0, 10.0), (0.005, 0.0, 10.0), (0.005, 1.0, 0.0), (1e-6, 1.0, 10.0),
           (0.005, 1e-6, 10.0), (10.0, 1.0, 10.0), (1000.0, 1.0, 10.0), (0.005, 1000.0, 1000.0), (10.0, 1e-6, 0.0)]
HAS_SOL = (abi.SOLVED, abi.SOLVED_INACCURATE, abi.MAX_ITER_REACHED)
_STAGES = {}


def _params(**over):
    p = O.default_params()
    for k, v in over.items():
        setattr(p, k, v)
    return p


def _stage(name, w):
    key = (name, w)
    if key not in _STAGES:
        x, y = CASES[name]
        g = E.stage(x, y, weights=w)
        o = S.smooth([float(v) for v in x], [float(v) for v in y], O.default_params(), weights=w)
        assert g["reason"] == S.SM_OK and o["qp"] is not None, name
        _STAGES[key] = (g, o["qp"])
    return _STAGES[key]


def _check(name, w, p, must=False, bar=1e-9):
    """Run both; returns 1 when compared, 0 when dropped for its margin."""
    g, qp = _stage(name, w)
    sol, _, info = S.osqp_solve(p, qp)
    if not must and not info.margin >= NEAR:
        return 0
    e = E.solve(p, g)
    assert (e["status"], e["iters"]) == (info.status, info.iters), (name, w, info.margin)
    N = g["N"]
    if info.status in HAS_SOL and np.max(np.abs(CASES[name][0])) < FAR and np.max(np.abs(CASES[name][1])) < FAR:
        want = np.stack([sol[:N], sol[N:2 * N]], 1)
        scale = max(1.0, np.max(np.abs(want)))
        assert np.max(np.abs(e["frenet"][:, :2] - want)) <= bar * scale, (name, w, p.max_iter)
    elif info.status not in HAS_SOL:
        assert np.all(np.isnan(e["frenet"])), name
    return 1


def _k1(name, w, **over):
    """The first iteration with an exact verdict (check at every iteration)."""
    g, qp = _stage(name, w)
    _, _, info = S.osqp_solve(_params(**dict(over, check_termination=1, max_iter=V.MAX_ITER)), qp)
    return int(info.iters)


# The rows of the defect report: (name, weights, settings) -- the oracle's status first.
DUAL_INF_ROWS = [
    ("config1", S.WEIGHTS, dict(eps_dual_inf=0.1, max_iter=1)),
    ("corner", S.WEIGHTS, dict(eps_dual_inf=0.1, max_iter=1)),
    ("config1", S.WEIGHTS, dict(eps_dual_inf=1.0, check_termination=10)),
    ("pose17", S.WEIGHTS, dict(eps_dual_inf=0.03)),
    ("pose17", S.WEIGHTS, dict(eps_dual_inf=0.01)),
]


@pytest.mark.parametrize("row", range(len(DUAL_INF_ROWS)))
def test_dual_infeasibility_rows(row):
    """OSQP's dual-infeasibility verdict.  Row 2 is an exact tie in both (the x0 pin row's A dx equals ||dx|| and the
    test is strict), so it is compared whatever its margin."""
    name, w, over = DUAL_INF_ROWS[row]
    assert _check(name, w, _params(**over), must=True)


def test_large_deviation_weight_at_every_pose():
    """Weights (10, 1e-6, 0): 16 of the 24 poses ran 100-400 iterations longer than OSQP before the separator chain
    solved with LDL' factors instead of explicit inverses.  At most one pose may be dropped for its margin."""
    done = sum(_check(f"pose{k}", (10.0, 1e-6, 0.0), _params()) for k in range(len(sc.poses.POSES)))
    assert done >= len(sc.poses.POSES) - 1, done


def test_dual_infeasible_inaccurate():
    """The x10 re-check at max_iter: eps_dual_inf 0.01 fails the exact test at iteration 1, 0.1 passes it."""
    g, qp = _stage("config1", S.WEIGHTS)
    p = _params(eps_dual_inf=0.01, max_iter=1)
    _, _, info = S.osqp_solve(p, qp)
    assert info.status == abi.DUAL_INFEASIBLE_INACCURATE
    assert _check("config1", S.WEIGHTS, p)


@pytest.mark.parametrize("name", NAMES)
def test_settings_grid(name):
    done = dropped = 0
    w = S.WEIGHTS
    for s, (check, interval, adaptive) in V.SCHEDULES.items():
        k1 = _k1(name, w, adaptive_rho_interval=interval, adaptive_rho=adaptive)
        for t in sorted({1, 7, max(k1 - 1, 1), k1, V.MAX_ITER}):
            r = _check(name, w, _params(check_termination=check, adaptive_rho_interval=interval,
                                        adaptive_rho=adaptive, max_iter=t))
            done += r
            dropped += 1 - r
    for scaling in (0, 10):
        for t in (1, 7, V.MAX_ITER):
            r = _check(name, w, _params(scaling=scaling, max_iter=t))
            done += r
            dropped += 1 - r
    for eps in (1e-4, 1e-3, 1e-2, 3e-2, 0.1, 1.0):
        k1 = _k1(name, w, eps_dual_inf=eps)
        for t in sorted({1, 2, 7, max(k1 - 1, 1), k1, V.MAX_ITER}):
            r = _check(name, w, _params(eps_dual_inf=eps, max_iter=t))
            done += r
            dropped += 1 - r
    for over in V.SETTINGS.values():
        k1 = _k1(name, w, **over)
        for t in sorted({max(k1 - 1, 1), k1, V.MAX_ITER}):
            r = _check(name, w, _params(max_iter=t, **over))
            done += r
            dropped += 1 - r
    assert done >= 3 * dropped, (name, done, dropped)


@pytest.mark.parametrize("name", ["config1", "u_turn", "pose1", "pose17"])
@pytest.mark.parametrize("wi", range(len(WEIGHTS)))
def test_weights(name, wi):
    """Status and iterations at every weight set, and the iterates near the origin: within 1e-9 of their scale, or 1e-6
    where the deviation weight is below 1e-4 of the largest curvature weight (0 included).  Such weights leave x and
    y with little cost curvature beyond sigma (1e-6); along those directions two correct solvers differ by up to 1e-7
    of the scale after the same iterations (4e-8 on config1 at deviation weight 0, 1e-7 on u_turn at (0.005, 1000,
    1000) one iteration after a rho update)."""
    w = WEIGHTS[wi]
    bar = 1e-9 if w[0] >= 1e-4 * max(w[1], w[2]) else 1e-6
    for t in sorted({7, V.MAX_ITER, _k1(name, w)}):
        _check(name, w, _params(max_iter=t), bar=bar)


def test_every_branch_reached():
    """Every status the smoothing QP can end in, each found from the oracle on config1 and compared."""
    want = {abi.SOLVED, abi.SOLVED_INACCURATE, abi.MAX_ITER_REACHED, abi.DUAL_INFEASIBLE, abi.DUAL_INFEASIBLE_INACCURATE}
    g, qp = _stage("config1", S.WEIGHTS)
    seen = set()
    candidates = [_params(eps_dual_inf=0.1, max_iter=1), _params(eps_dual_inf=0.01, max_iter=1)]
    candidates += [_params(max_iter=t) for t in range(_k1("config1", S.WEIGHTS), 0, -1)]
    for p in candidates:
        _, _, info = S.osqp_solve(p, qp)
        if info.status in want - seen and _check("config1", S.WEIGHTS, p):
            seen.add(int(info.status))
        if seen == want:
            break
    assert seen == want, sorted(seen)
