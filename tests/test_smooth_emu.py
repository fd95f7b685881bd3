"""CPU tests of the smoothing stage's device source (csrc/pqp_smooth_core.cuh and the width-4 generic core of
csrc/pqp_gen_core.cuh) compiled with g++ (tests/emu/smooth_emu.cpp) against the CPU restatement (oracle/smooth.py): the
B-spline samples, the raw fit and the stations bit for bit, the band-order QP equal to the reference-order one entry
for entry, and the width-4 core's status, iterations and solution against the oracle's OSQP."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import smooth as S
from tests import smooth_cases as sc
from tests.emu import smooth_emu as E

CASES = sc.named()
# Far from the origin the solutions are not compared, only status and iterations: the QP iterates on absolute
# coordinates and OSQP's stopping rule is relative to them (eps_rel |z|: 5e3 m at UTM northings, 1e4 m at 1e7 m), so two
# restatements of the same recurrence, equal in status and iterations, stop at points inside that tolerance that differ
# by far more than rounding (5e-4 m at UTM northings, metres at 1e7 m).
FAR = 1e5
ACCEPTED = ["config1", "straight_x", "u_turn", "corner", "six_close", "four_far"] + [f"pose{k}" for k in range(24)]


def _lists(name):
    x, y = CASES[name]
    return [float(v) for v in x], [float(v) for v in y]


def _ref_col(N, g):
    """Band position g = 4i + t of the generic core -> the reference's column (x, y, theta blocks, then k)."""
    i, t = divmod(int(g), 4)
    return t * N + i


@pytest.mark.parametrize("name", ACCEPTED)
def test_stage_bits_equal_restatement(name):
    x, y = _lists(name)
    g = E.stage(x, y)
    r = S.smooth(x, y, O.default_params())
    assert g["reason"] == S.SM_OK and r["qp"] is not None
    raw = r["raw"]
    for k in ("t", "x", "y", "s"):
        assert g[k].tobytes() == np.array(raw[k]).tobytes(), k
    assert g["xc"].tobytes() == O.spline_fit(raw["s"], raw["x"]).tobytes()
    assert g["yc"].tobytes() == O.spline_fit(raw["s"], raw["y"]).tobytes()
    st = np.stack([g["stations"][f] for f in ("x", "y", "z", "k")], 1)
    assert st.tobytes() == np.array([list(v) for v in r["stations"]]).tobytes()
    # the band-order QP, mapped to the reference's columns, equals the reference-order triplets entry for entry
    N = g["N"]
    n, m = 4 * N - 1, 3 * N - 1
    P, q, A, lo, up = S.dense(r["qp"])
    Ab = np.zeros((m, n))
    for row in range(m):
        for c, v in zip(g["A_col"][row], g["A_val"][row]):
            if c >= 0:
                Ab[row, _ref_col(N, c)] += v
    assert Ab.tobytes() == A.tobytes()
    assert g["l"].tobytes() == lo.tobytes() and g["u"].tobytes() == up.tobytes()
    Pb, qb = np.zeros((n, n)), np.zeros(n)
    for j in range(n):
        cj = _ref_col(N, j)
        Pb[cj, cj] = g["Pd"][j]
        qb[cj] = g["q"][j]
        for k, v in zip(g["Po_idx"][j], g["Po_val"][j]):
            if k >= 0:
                Pb[cj, _ref_col(N, k)] = v
    assert Pb.tobytes() == P.tobytes() and qb.tobytes() == q.tobytes()
    # the CSC columns are the rows' transpose, rows ascending; ptr[n] = 9N - 7
    cp, cr, cv = g["csc_ptr"], g["csc_row"], g["csc_val"]
    assert cp[0] == 0 and cp[n] == 9 * N - 7 and np.all(np.diff(cp) >= 0)
    Ac = np.zeros((m, n))
    for j in range(n):
        rows = cr[cp[j]:cp[j + 1]]
        assert np.all(np.diff(rows) > 0)
        Ac[rows, _ref_col(N, j)] = cv[cp[j]:cp[j + 1]]
    assert Ac.tobytes() == A.tobytes() or np.array_equal(Ac, A)
    # separators: station e's four unknowns every L stations, never the last station
    L = max(2, (N - 2) // 31 + 1)
    assert list(g["sep"]) == [4 * e for e in range(0, N - 1, L)][:32]


@pytest.mark.parametrize("name", ACCEPTED)
def test_width4_core_equals_oracle(name):
    prm = O.default_params()
    x, y = _lists(name)
    g = E.stage(x, y)
    r = S.smooth(x, y, prm)
    sol = E.solve(prm, g)
    if r["qp_margin"] < 1e-9:
        pytest.skip("a termination decision within 1e-9 of its threshold")
    assert (sol["status"], sol["iters"]) == (r["status"], r["iters"])
    if max(abs(v) for v in x + y) > FAR:
        return    # status and iterations only: see FAR
    want, _, _ = S.osqp_solve(prm, r["qp"])
    N = g["N"]
    got = np.concatenate([sol["frenet"][:, 0], sol["frenet"][:, 1], sol["frenet"][:, 2]])
    scale = max(1.0, float(np.max(np.abs(want[:3 * N]))))
    assert np.max(np.abs(got - want[:3 * N])) <= 1e-9 * scale


def test_refusals_equal_restatement():
    prm = O.default_params()
    want = {"three": S.SM_FEW, "four_close": S.SM_DEGREE, "five_close": S.SM_DEGREE, "nan": S.SM_LENGTH,
            "tiny": S.SM_RAW_ORDER, "short": S.SM_SHORT}
    for name, reason in want.items():
        x, y = _lists(name)
        assert E.stage(x, y)["reason"] == S.smooth(x, y, prm)["reason"] == reason, name
    x, y = _lists("config1")
    assert E.stage(x, y, max_raw=20)["reason"] == S.smooth(x, y, prm, max_raw=20)["reason"] == S.SM_RAW_MANY
    assert E.stage(x, y, max_points=20)["reason"] == S.smooth(x, y, prm, max_points=20)["reason"] == S.SM_MANY
