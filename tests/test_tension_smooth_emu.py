"""CPU tests of the TENSION smoothing stage's device source (the TENSION assembly of csrc/pqp_smooth_core.cuh and the
width-9 generic core of csrc/pqp_gen_core.cuh) compiled with g++ (tests/emu/tension_emu.cpp) against the CPU
restatement (tests/tension_restatement.py): the clearances equal to oracle.map_distance bit for bit, the
band-order rows, P, bounds and CSC columns equal to the reference-order QP bit for bit, the separators, and the core's
status and iterations equal to the oracle's OSQP, with its solution within the bar of tests/test_tension_smooth.py."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import smooth as S
from tests import tension_cases as tc
from tests import tension_restatement as T
from tests.emu import tension_emu as E
from tests.test_tension_smooth import bar

CASES = tc.named()
FAR = 1e5      # farther out only status and iterations are compared (tests/test_smooth_emu.py)
NAMES = ["config1", "u_turn", "corner", "four_far", "six_close", "straight_x", "down"] + [f"pose{k}" for k in range(24)]


def _lists(name):
    return tuple([float(v) for v in a] for a in CASES[name])


def _map(name):
    return tc.pose_maps().get(name, tc.config1_map())


def _ref_col(N, g):
    """Band position g = 3i + t -> the reference's column (x block, y block, d block)."""
    i, t = divmod(int(g), 3)
    return t * N + i


def _stage_equals(name, w):
    x, y = _lists(name)
    dmap = _map(name)
    g = E.stage(x, y, dmap, weights=w)
    r = T.smooth(x, y, O.default_params(), dmap, weights=w)
    assert g["reason"] == r["reason"] == S.SM_OK, name
    N = g["N"]
    st = np.stack([g["stations"][f] for f in ("x", "y", "z", "k")], 1)
    assert st.tobytes() == np.array([list(v) for v in r["stations"]]).tobytes()
    # the clearances, bit for bit, and oracle.map_distance at every interior station
    assert g["clearance"].tobytes() == np.array(r["clearance"]).tobytes()
    xy = np.array([[v[0], v[1]] for v in r["stations"][1:-1]])
    assert g["clearance"][1:-1].tobytes() == O.map_distance(dmap, xy).tobytes()
    n = m = 3 * N
    P, _, A, lo, up = S.dense(r["qp"])
    # rows: the band-order row r is the reference's row r
    Ab = np.zeros((m, n))
    for row in range(m):
        for c, v in zip(g["A_col"][row], g["A_val"][row]):
            if c >= 0:
                assert v != 0.0
                Ab[row, _ref_col(N, c)] = v
    assert Ab.tobytes() == A.tobytes()
    assert g["l"].tobytes() == lo.tobytes() and g["u"].tobytes() == up.tobytes()
    Pb = np.zeros((n, n))
    for j in range(n):
        cj = _ref_col(N, j)
        Pb[cj, cj] = g["Pd"][j]
        ks = [k for k in g["Po_idx"][j] if k >= 0]
        assert ks == sorted(ks) and all(abs(k - j) <= 9 for k in ks)
        for k, v in zip(g["Po_idx"][j], g["Po_val"][j]):
            if k >= 0:
                assert v != 0.0
                Pb[cj, _ref_col(N, k)] = v
    assert Pb.tobytes() == P.tobytes()
    # CSC: the rows' transpose, rows ascending, exactly the reference's non-zeros
    cp, cr, cv = g["csc_ptr"], g["csc_row"], g["csc_val"]
    assert cp[0] == 0 and cp[n] == len(r["qp"]["A"][2]) and np.all(np.diff(cp) >= 0)
    Ac = np.zeros((m, n))
    for j in range(n):
        rows = cr[cp[j]:cp[j + 1]]
        assert np.all(np.diff(rows) > 0)
        Ac[rows, _ref_col(N, j)] = cv[cp[j]:cp[j + 1]]
    assert Ac.tobytes() == A.tobytes()
    # separators: three stations every L >= 6 stations from station 0, never reaching the last station
    L = max(6, (N - 4) // 31 + 1)
    assert list(g["sep"]) == [3 * e for e in range(0, N, L) if e == 0 or e + 3 <= N - 1][:32]
    return g, r


@pytest.mark.parametrize("name", NAMES)
def test_stage_bits_equal_restatement(name):
    _stage_equals(name, T.WEIGHTS)


@pytest.mark.parametrize("w", tc.WEIGHTS[1:])
def test_stage_bits_under_weights(w):
    for name in ("config1", "corner", "down"):
        _stage_equals(name, w)


def _core_equals(name, w):
    prm = O.default_params()
    g, r = _stage_equals(name, w)
    sol = E.solve(prm, g)
    if r["qp_margin"] < 1e-9:
        return False
    assert (sol["status"], sol["iters"]) == (r["status"], r["iters"]), name
    x, y = _lists(name)
    if max(abs(v) for v in x + y) > FAR:
        return True
    want, _, _ = S.osqp_solve(prm, r["qp"])
    N = g["N"]
    got = np.concatenate([sol["frenet"][:, 0], sol["frenet"][:, 1], sol["frenet"][:, 2]])
    scale = max(1.0, float(np.max(np.abs(want))))
    assert np.max(np.abs(got - want)) <= bar(w) * scale, name
    return True


@pytest.mark.parametrize("name", NAMES)
def test_width9_core_equals_oracle(name):
    if not _core_equals(name, T.WEIGHTS):
        pytest.skip("a termination decision within 1e-9 of its threshold")


@pytest.mark.parametrize("w", tc.WEIGHTS[1:])
def test_width9_core_under_weights(w):
    assert sum(_core_equals(name, w) for name in ("config1", "u_turn", "corner")) >= 2


def test_long_line_separators():
    """Close to 277 stations, the most one SM holds: about 30 separators, the core equal to the oracle."""
    x = np.arange(0.0, 262.0, 3.0)
    y = 4.0 * np.sin(x / 20.0)
    CASES["long"] = (x, y)
    g = E.stage(list(x), list(y), tc.config1_map(), max_points=277)
    assert g["reason"] == S.SM_OK and g["N"] <= 277 and len(g["sep"]) >= 28
    _core_equals("long", T.WEIGHTS)
    assert E.stage(list(x), list(y), tc.config1_map(), max_points=g["N"] - 1)["reason"] == S.SM_MANY


def test_refusals_equal_restatement():
    prm = O.default_params()
    m = tc.config1_map()
    want = {"three": S.SM_FEW, "four_close": S.SM_DEGREE, "five_close": S.SM_DEGREE, "nan": S.SM_LENGTH,
            "tiny": S.SM_RAW_ORDER, "short": S.SM_SHORT}
    for name, reason in want.items():
        x, y = _lists(name)
        assert E.stage(x, y, m)["reason"] == T.smooth(x, y, prm, m)["reason"] == reason, name
    x, y = _lists("config1")
    assert E.stage(x, y, None)["reason"] == T.smooth(x, y, prm, None)["reason"] == T.SM_MAP
    x, y = _lists("tiny")
    assert E.stage(x, y, None)["reason"] == T.SM_MAP      # the map check comes before the raw-order one
    x, y = _lists("three")
    assert E.stage(x, y, None)["reason"] == S.SM_FEW
