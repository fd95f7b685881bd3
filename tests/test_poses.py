"""CPU tests of scenes under rigid motions (tests/poses.py): every heading, and coordinates of UTM size.

First the relation itself, on the oracle and the twin: a translated batch assembles to the same QP entry for entry and
solves to the same Frenet bits; a rotated one to the same status and iteration count and the same Frenet solution
within 1e-9 (only the end-heading row may move, by rounding); the Cartesian outputs are the moved outputs.  Then the
product's kernel source under g++ (tests/emu) against the oracle under those motions: one length per solver class family
on poses and on lines whose goal heading is reached through a wrap; the map, clearance, collision, tail and spline-fit
stages bit for bit (both sides call glibc here, so a differing bit is a logic difference)."""
import os

import numpy as np
import pytest
from scipy.interpolate import CubicSpline

from oracle import oracle, twin
from path_optimizer_b200 import planner, synth
from path_optimizer_b200.abi import BOUNDS_DTYPE, STATE_DTYPE
from tests import poses, shapes, spacing
from tests.emu import emu, fit_emu

KP, K, KPC = shapes.KP, shapes.K, shapes.KPC
FORMS = [KP, K, KPC]
REL_TOL = 1e-9           # Frenet solutions of a rotated batch against the unmoved one
UTM, FAR = poses.TRANSLATIONS[1], poses.TRANSLATIONS[2]
# a pure translation, then headings on both sides of +-pi, an axis, a diagonal and a seeded angle, far from the origin
SIX = [(0.0,) + UTM, (np.pi,) + UTM, (-np.pi,) + FAR, (poses.THETAS[5], 0.0, 0.0), (-3 * np.pi / 4,) + UTM,
       (np.pi / 2,) + FAR, (poses.THETAS[8],) + UTM]


def _u64(a):
    return np.ascontiguousarray(a).view(np.uint64).reshape(-1)


def _limits(params, b):
    ref = b["ref"].copy()
    ref["v"] = 4.0 + 3.0 * np.sin(np.arange(len(ref)) * 0.05)
    ref["a"] = 0.5 * np.cos(np.arange(len(ref)) * 0.05)
    ref["v"][::13] = 0.0
    return oracle.update_limits(params, ref)


def _base_batch():
    """Uneven curved corridors of several lengths, the U-turn and the S-bend, and the lines with wrapped goals."""
    b = spacing.corridors([spacing.dynamic_s(n, spacing.sine_kappa(0.15, 20.0)) for n in (9, 37, 80, 130)], first_path=5)
    t = poses.turning_lines(120)
    return poses.concat([b, t["u-turn"], t["s-bend"], poses.wrap_goal_lines()])


# ---- the convention of a turned map --------------------------------------------------------------------------------
def test_turned_map_convention():
    """A map moved by move_map reads, at its cell centres, what the original reads at the centres they came from: pins np.rot90 to the
    grid_map index convention, on a map with rows != cols, for the four quarter turns and the three translations."""
    m = synth.disc_field_map(rows=46, cols=30, n_discs=12, keep_clear_halfwidth=0.5, center=(3.0, -2.0))
    xs, ys = poses.cell_centers(m)
    X, Y = np.meshgrid(xs, ys, indexing="ij")
    want = oracle.map_distance(m, np.stack([X.ravel(), Y.ravel()], 1))
    assert (want == m["distance"].ravel()).all() and len(np.unique(want)) > 20
    for q, theta in enumerate([0.0, np.pi / 2, np.pi, -np.pi / 2]):
        for tx, ty in poses.TRANSLATIONS:
            mm = poses.move_map(m, tx, ty, q)
            assert (mm["rows"], mm["cols"]) == ((46, 30) if q % 2 == 0 else (30, 46))
            # where the original cell centres land, and the moved map's own cell there (its centre, by the lookup's
            # arithmetic: a point a rounding error off a centre already blends 1e-9 of a neighbour in)
            mx, my = (v.astype(np.float64) for v in poses.move_xy(X.ravel(), Y.ravel(), theta, tx, ty))
            cx, cy = poses.cell_centers(mm)
            a, c = np.abs(mx[:, None] - cx[None, :]).argmin(1), np.abs(my[:, None] - cy[None, :]).argmin(1)
            assert np.abs(cx[a] - mx).max() < 1e-6 and np.abs(cy[c] - my).max() < 1e-6
            assert len(set(zip(a.tolist(), c.tolist()))) == len(a)
            pts = np.stack([cx[a], cy[c]], 1)
            assert (oracle.map_distance(mm, pts) == want).all(), (q, tx)
            assert (emu.map_distance(mm, pts) == want).all(), (q, tx)
    assert poses.quarter_turns(-np.pi) == 2 and poses.quarter_turns(poses.THETAS[5]) is None


# ---- the relation, on the oracle and the twin -----------------------------------------------------------------------
@pytest.mark.parametrize("form", FORMS, ids=["KP", "K", "KPC"])
def test_translation_changes_no_entry_and_no_frenet_bit(oracle_params, form):
    """The assemblies read no x or y: a translated batch gives the same triplets and bounds and, solved, the same Frenet
    bits, status and iterations.  The Cartesian outputs are the translated outputs."""
    b = _base_batch()
    mk, mkp = _limits(oracle_params, b) if form == KPC else (None, None)
    base = oracle.solve_batch(oracle_params, form, b, max_k=mk, max_kp=mkp)
    assert (base["status"] == 1).mean() > 0.5
    o = b["offsets"]
    for tx, ty in poses.TRANSLATIONS[1:]:
        mb = poses.move(b, 0.0, tx, ty)
        assert np.array_equal(_u64(mb["ref"]["z"]), _u64(b["ref"]["z"]))
        for i in range(len(b["n_points"])):
            sl = slice(o[i], o[i + 1])
            kw = dict(max_k=np.ascontiguousarray(mk[sl]), max_kp=np.ascontiguousarray(mkp[sl])) if form == KPC else {}
            q0 = oracle.assemble(oracle_params, form, b["ref"][sl], b["bounds"][sl], b["x0"][i], b["end_heading"][i], **kw)
            q1 = oracle.assemble(oracle_params, form, mb["ref"][sl], mb["bounds"][sl], mb["x0"][i], mb["end_heading"][i], **kw)
            for k in ("P", "A"):
                assert all(np.array_equal(a, c) for a, c in zip(q0[k], q1[k])), (i, k)
            for k in ("q", "l", "u"):
                assert np.array_equal(q0[k], q1[k]), (i, k)
        r = oracle.solve_batch(oracle_params, form, mb, max_k=mk, max_kp=mkp)
        assert np.array_equal(r["status"], base["status"]) and np.array_equal(r["iters"], base["iters"])
        assert np.array_equal(_u64(r["frenet"]), _u64(base["frenet"]))
        _assert_moved_outputs(r, base, np.repeat(0.0, len(o) - 1), tx, ty, o)
    if form == KP:                                             # the dense-block twin reads no x or y either
        sl = slice(o[2], o[3])
        t0 = twin.assemble_kp(oracle_params, b["ref"][sl], b["bounds"][sl], b["x0"][2], b["end_heading"][2])
        t1 = twin.assemble_kp(oracle_params, mb["ref"][sl], mb["bounds"][sl], mb["x0"][2], mb["end_heading"][2])
        assert all(np.array_equal(a, c) for a, c in zip(t0, t1))


def _assert_moved_outputs(got, base, thetas, tx, ty, o, tol=1e-8):
    """got's Cartesian outputs are base's under the motion (per path thetas[i]; one translation)."""
    for i, theta in enumerate(thetas):
        sl = slice(o[i], o[i + 1])
        if base["status"][i] != 1:
            continue
        want = poses.move_states(base["states"][sl], theta, tx, ty)
        g = got["states"][sl]
        bar = poses.xy_tol(want["x"], want["y"], tol)
        assert (np.abs(g["x"] - want["x"]) <= bar).all() and (np.abs(g["y"] - want["y"]) <= bar).all(), i
        # the output heading is reference heading + e_phi, not wrapped (as getOptimizedPath leaves it): modulo 2 pi
        assert np.abs(poses.angle_diff(g["z"], base["states"]["z"][sl] + theta)).max() <= tol, i
        assert np.abs(g["k"] - base["states"]["k"][sl]).max() <= tol and np.abs(g["s"] - base["states"]["s"][sl]).max() <= bar.max(), i


@pytest.mark.parametrize("form", FORMS, ids=["KP", "K", "KPC"])
def test_rotation_moves_only_the_end_heading_row(oracle_params, form):
    """Every pose heading at the far translation: same status and iterations as the unmoved batch, Frenet within 1e-9,
    Cartesian outputs the moved outputs.  Of the assembly only the end-heading bounds may differ, by rounding."""
    b = _base_batch()
    mk, mkp = _limits(oracle_params, b) if form == KPC else (None, None)
    base = oracle.solve_batch(oracle_params, form, b, max_k=mk, max_kp=mkp)
    o = b["offsets"]
    worst = 0.0
    for theta in poses.THETAS:
        mb = poses.move(b, theta, *FAR)
        r = oracle.solve_batch(oracle_params, form, mb, max_k=mk, max_kp=mkp)
        assert np.array_equal(r["status"], base["status"]) and np.array_equal(r["iters"], base["iters"]), theta
        ok = np.repeat(base["status"] == 1, b["n_points"])
        worst = max(worst, np.abs(r["frenet"][ok] - base["frenet"][ok]).max())
        _assert_moved_outputs(r, base, np.repeat(theta, len(o) - 1), *FAR, o)
        sl = slice(o[1], o[2])
        kw = dict(max_k=np.ascontiguousarray(mk[sl]), max_kp=np.ascontiguousarray(mkp[sl])) if form == KPC else {}
        q0 = oracle.assemble(oracle_params, form, b["ref"][sl], b["bounds"][sl], b["x0"][1], b["end_heading"][1], **kw)
        q1 = oracle.assemble(oracle_params, form, mb["ref"][sl], mb["bounds"][sl], mb["x0"][1], mb["end_heading"][1], **kw)
        assert all(np.array_equal(a, c) for k in ("P", "A") for a, c in zip(q0[k], q1[k]))
        moved = np.nonzero((q0["l"] != q1["l"]) | (q0["u"] != q1["u"]))[0]
        assert len(moved) <= 1 and np.abs(q0["l"][moved] - q1["l"][moved]).max(initial=0.0) < 1e-14
    assert worst <= REL_TOL, worst


def test_wrap_goal_lines_cover_the_end_heading_switch(oracle_params):
    """From the oracle's own assembly: the lines of poses.WRAP_GOALS have an end-heading row constrained through a wrap
    (from both sides of +-pi), one unconstrained past 70 degrees, and one constrained below -70 degrees (the reference
    takes no absolute value)."""
    b = poses.wrap_goal_lines()
    o = b["offsets"]
    psi = poses.end_psi(b)
    raw = b["end_heading"] - b["ref"]["z"][o[1:] - 1]
    seen = set()
    for i, (_, _, what) in enumerate(poses.WRAP_GOALS):
        sl = slice(o[i], o[i + 1])
        qp = oracle.assemble(oracle_params, KP, b["ref"][sl], b["bounds"][sl], b["x0"][i], b["end_heading"][i])
        lo, hi = qp["l"], qp["u"]
        window = np.nonzero(np.isclose(hi - lo, 10 * np.pi / 180, atol=1e-12) & np.isclose(0.5 * (lo + hi), psi[i], atol=1e-12))[0]
        if what == "unconstrained":
            assert len(window) == 0 and psi[i] > 70 * np.pi / 180 and abs(raw[i]) > np.pi
        else:
            assert len(window) == 1, (i, what)
            if what == "constrained through a wrap":
                assert abs(raw[i]) > np.pi and abs(psi[i]) < 70 * np.pi / 180
            else:
                assert psi[i] < -70 * np.pi / 180
        seen.add(what)
    assert seen == {"constrained through a wrap", "unconstrained", "negative below -70 deg"}
    assert (raw[[0, 4]] * [1, -1] < -np.pi).all()          # through the wrap from either side


# ---- the kernel source under the emulator against the oracle, under motion -------------------------------------------
# (formulation, stations, keep of a KP step profile or None, max_iter): one length per class family
FAMILIES = {
    "thread per station, dense": (KP, 60, 3, 100),
    "thread per station, banded": (KP, 150, 3, 50),
    "one warp": (KP, 40, 5, 100),
    "KPC": (KPC, 100, None, 100),
    "K four warps": (K, 60, None, 100),
    "K eight warps": (K, 140, None, 50),
    "K thirteen warps": (K, 270, None, 50),
}
FAMILY_CLASS = {"thread per station, dense": r"pqp_kp3_solve_kernel<\d+,\d+,4,17>", "thread per station, banded":
                r"pqp_kp3_solve_kernel<\d+,\d+,8,34>", "one warp": "pqp_kp_solve_kernel", "KPC": r"pqp_kp3_solve_kernel<.*KPC>",
                "K four warps": r"pqp_kk_solve_kernel<4>", "K eight warps": r"pqp_kk_solve_kernel<8>",
                "K thirteen warps": r"pqp_kk_solve_kernel<13>"}


def _family_batch(form, n, keep, count):
    if keep is not None:
        s_list = [spacing.step_profile(n, keep, (2 * k) % 9, seed=n + k) for k in range(count)]
    else:
        s_list = [spacing.dynamic_s(n, spacing.sine_kappa(0.15, 20.0 + k)) for k in range(count)]
    return spacing.corridors(s_list, first_path=3 * n)


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_emu_under_motion(oracle_params, family):
    """One line per pose of SIX plus the same lines unmoved, on the class the library selects: the oracle's status,
    iterations and iterates on the moved inputs (the bar of the other emulator tests); the unmoved and the purely
    translated line give the same Frenet bits, so no row of the kernel's assembly reads x or y."""
    import re
    form, n, keep, max_iter = FAMILIES[family]
    p = oracle_params.copy()
    p.max_iter = max_iter
    few = family == "K thirteen warps"                    # 416 host threads per barrier: three poses
    chosen = SIX[:3] if few else SIX
    b = _family_batch(form, n, keep, 1)
    b = synth.take_paths(b, np.zeros(1 + len(chosen), dtype=np.int64))
    names = {shapes.class_of(form, n, shapes.keep_of(form, b["ref"][:n]))[0]}
    name = names.pop()
    assert re.fullmatch(FAMILY_CLASS[family], name), name
    mb = poses.move_each(b, [(0.0, 0.0, 0.0)] + chosen)
    mk = mkp = None
    if form == KPC:                                       # the same limits for every copy of the line
        mk, mkp = (np.tile(a[:n], 1 + len(chosen)) for a in _limits(p, mb))
    e = emu.solve_batch(p, mb, variant=name, max_k=mk, max_kp=mkp)
    r = oracle.solve_batch(p, form, mb, threads=4, max_k=mk, max_kp=mkp)
    every, rows = np.arange(len(mb["n_points"])), np.arange(int(mb["offsets"][-1]))
    shapes.assert_matches(e, r, every, rows, mb["n_points"], family)
    assert np.isfinite(e["frenet"]).all()
    assert np.array_equal(_u64(e["frenet"][:n]), _u64(e["frenet"][n:2 * n])), "translation changed a Frenet bit"
    for i in range(1, len(chosen) + 1):
        assert e["iters"][i] == e["iters"][0] and e["status"][i] == e["status"][0]
        assert np.abs(e["frenet"][i * n:(i + 1) * n] - e["frenet"][:n]).max() <= REL_TOL, i


@pytest.mark.parametrize("name", ["pqp_kp3_solve_kernel<17,6,8,34>", "pqp_kp_solve_kernel", "pqp_kk_solve_kernel<4>",
                                  "pqp_kp3_solve_kernel<13,7,8,34,KPC>"])
def test_emu_wrapped_goals_and_tight_turns(oracle_params, name):
    """The lines whose goal heading is reached through a wrap, the U-turn and the S-bend near the steering limit, and the
    same with headings a caller integrated (4 and -4 turns off): against the oracle, and the unwrapped ones against the
    wrapped ones."""
    form = KPC if name.endswith("KPC>") else K if name.startswith("pqp_kk") else KP
    p = oracle_params.copy()
    p.max_iter = 100
    t = poses.turning_lines(100)
    # far from the origin; the goal lines keep their last headings beside +-pi, the turns cross +-pi in their middle
    b = poses.concat([poses.move(poses.wrap_goal_lines(), 0.0, *UTM),
                      poses.move(poses.concat([t["u-turn"], t["s-bend"]]), np.pi / 2 + 0.3, *UTM)])
    raw = b["end_heading"] - b["ref"]["z"][b["offsets"][1:] - 1]
    assert (raw > np.pi).any() and (raw < -np.pi).any()
    z = b["ref"]["z"][b["offsets"][-3]:b["offsets"][-2]]
    assert np.abs(np.diff(z)).max() > 6.0                          # the wrapped heading jumps by 2 pi inside the path
    mk, mkp = _limits(p, b) if form == KPC else (None, None)
    r = oracle.solve_batch(p, form, b, threads=4, max_k=mk, max_kp=mkp)
    every, rows = np.arange(len(b["n_points"])), np.arange(int(b["offsets"][-1]))
    assert np.isfinite(r["frenet"]).all()
    e = emu.solve_batch(p, b, variant=name, max_k=mk, max_kp=mkp)
    shapes.assert_matches(e, r, every, rows, b["n_points"], name)
    for turns in (4, -4):
        ub = poses.move(b, 0.0, 0.0, 0.0, unwrap_turns=turns)
        assert np.abs(ub["ref"]["z"]).min() > 3 * np.pi
        u = emu.solve_batch(p, ub, variant=name, max_k=mk, max_kp=mkp)
        shapes.assert_matches(u, oracle.solve_batch(p, form, ub, threads=4, max_k=mk, max_kp=mkp), every, rows,
                              b["n_points"], (name, turns))
        assert np.array_equal(u["status"], e["status"]) and np.array_equal(u["iters"], e["iters"]), turns
        assert np.abs(u["frenet"] - e["frenet"]).max() <= REL_TOL
        bar = poses.xy_tol(e["states"]["x"], e["states"]["y"])
        assert (np.abs(u["states"]["x"] - e["states"]["x"]) <= bar).all()
        assert (np.abs(u["states"]["y"] - e["states"]["y"]) <= bar).all()
        assert np.abs(poses.angle_diff(u["states"]["z"], e["states"]["z"])).max() <= 1e-8


# ---- the stages either side of the QP, bit for bit --------------------------------------------------------------------
def _config1_map():
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "config1_benchmark_map.npz"))
    field = dict(distance=g["map_distance"], rows=int(g["image_shape"][0]), cols=int(g["image_shape"][1]),
                 resolution=float(g["map_geo"][0]), center_x=float(g["map_geo"][1]), center_y=float(g["map_geo"][2]))
    b = dict(n_points=g["n_points"], ref=g["ref"], x0=g["x0"], end_heading=g["end_heading"])
    b["offsets"] = np.array([0, int(g["n_points"][0])], dtype=np.int32)
    return field, b


@pytest.fixture(scope="module")
def scenes():
    """name -> (map, lines): the disc field with lines along its corridor and leaving through its ends, the config-1
    map with its own line and copies shifted sideways, and a square disc field with lines in every direction."""
    disc = synth.disc_field_map()
    lines = synth.map_reference_paths(24, 110, x_range=(-109.0, 100.0), y_range=(-6.0, 6.0), heading_range=0.08, curvature_amp=0.02)
    c1, c1b = _config1_map()
    shifted = synth.take_paths(dict(c1b, bounds=np.zeros(len(c1b["ref"]), dtype=BOUNDS_DTYPE)), np.zeros(4, dtype=np.int64))
    n = int(c1b["n_points"][0])
    for i in range(4):
        shifted["ref"]["y"][i * n:(i + 1) * n] += (0.0, 1.5, -2.5, 30.0)[i]
    square = synth.disc_field_map(rows=1100, cols=1100, n_discs=1300)
    return dict(disc=(disc, lines), config1=(c1, shifted), square=(square, lines))


def _bits_equal(a, b):
    return np.ascontiguousarray(a).tobytes() == np.ascontiguousarray(b).tobytes()


def _env_stages_equal(p, m, b, what, want_leaving=False):
    """Every stage of pqp_env_core.cuh on one scene, emulator against oracle, every bit.  Returns what the scene
    covered: (blocked paths, free paths, paths with a station off the map)."""
    n_points = b["n_points"]
    for mode in (planner.BOUNDS_SIMPLE, planner.BOUNDS_IMPROVED):
        spl = planner.reference_splines(b) if mode == planner.BOUNDS_IMPROVED else None
        want = oracle.update_bounds(p, m, b, mode=mode, splines=spl)
        got = emu.update_bounds(p, m, b, mode=mode, splines=spl)
        assert np.array_equal(got["n_valid"], want["n_valid"]), (what, mode, got["n_valid"], want["n_valid"])
        for i in range(len(n_points)):
            sl = slice(b["offsets"][i], b["offsets"][i] + want["n_valid"][i])
            assert _bits_equal(got["bounds"][sl], want["bounds"][sl]), (what, mode, i)
        if mode == planner.BOUNDS_SIMPLE:
            n_valid = want["n_valid"]
    ok = oracle.check_states(p, m, b["ref"])
    assert np.array_equal(emu.check_states(p, m, b["ref"]), ok), what
    paths = b["ref"].copy()
    paths["s"] = 0.0
    for cc in (True, False):
        want = oracle.finish_raw(p, m, n_points, paths, collision_check=cc)
        got = emu.finish_raw(p, m, n_points, paths, collision_check=cc)
        assert np.array_equal(got["n_kept"], want["n_kept"]) and np.array_equal(got["ok"], want["ok"]), (what, cc)
        for i in range(len(n_points)):
            sl = slice(b["offsets"][i], b["offsets"][i] + want["n_kept"][i])
            assert _bits_equal(got["states"][sl], want["states"][sl]), (what, cc, i)
    src = want["states"]                                   # s re-accumulated, nothing cut
    for cc in (True, False):
        want = oracle.densify(p, m, n_points, src, 0.3, cc, 160)
        got = emu.densify(p, m, n_points, src, 0.3, cc, 160)
        assert np.array_equal(got["n_out"], want["n_out"]) and np.array_equal(got["ok"], want["ok"]), (what, cc)
        for i, k in enumerate(want["n_out"]):
            assert _bits_equal(got["states"][i, :k], want["states"][i, :k]), (what, "densify", cc, i)
    xy = np.concatenate([poses.border_points(m), np.stack([b["ref"]["x"], b["ref"]["y"]], 1)[::7]])
    d = oracle.map_distance(m, xy)
    assert np.array_equal(emu.map_distance(m, xy), d), what
    off_map = np.array([not _inside(m, b["ref"][b["offsets"][i]:b["offsets"][i + 1]]).all() for i in range(len(n_points))])
    return n_valid < n_points, n_valid == n_points, off_map


def _inside(m, st):
    lx, ly = m["rows"] * m["resolution"], m["cols"] * m["resolution"]
    return (np.abs(st["x"] - m["center_x"]) < lx / 2) & (np.abs(st["y"] - m["center_y"]) < ly / 2)


def _exit_edges(m, b):
    """The map edges ('+x', '-x', '+y', '-y') through which the lines of a batch leave the map."""
    lx, ly = m["rows"] * m["resolution"], m["cols"] * m["resolution"]
    dx, dy = b["ref"]["x"] - m["center_x"], b["ref"]["y"] - m["center_y"]
    return {e for e, hit in (("+x", dx > lx / 2), ("-x", dx < -lx / 2), ("+y", dy > ly / 2), ("-y", dy < -ly / 2)) if hit.any()}


@pytest.mark.parametrize("scene", ["disc", "config1"])
def test_env_stages_on_turned_and_shifted_maps(scenes, scene):
    """The map turned by each quarter turn (both signs of pi) and shifted by each translation, with its lines: bounds of
    both modes, collision flags, both tails and the lookups, the borders included, equal the oracle's in every bit."""
    p = oracle.default_params()
    m, b = scenes[scene]
    edges = set()
    covered = np.zeros(3, dtype=bool)
    for theta, tx, ty in poses.QUARTER_POSES:
        q = poses.quarter_turns(theta)
        mm, mb = poses.move_map(m, tx, ty, q), poses.move(b, theta, tx, ty)
        blocked, free, off = _env_stages_equal(p, mm, mb, (scene, theta, tx))
        covered |= [blocked.any(), free.any(), off.any()]
        if (tx, ty) == FAR:
            edges |= _exit_edges(mm, mb)
    assert covered.all(), covered
    if scene == "disc":
        assert edges == {"+x", "-x", "+y", "-y"}, edges


@pytest.mark.parametrize("k", range(len(poses.THETAS)))
def test_env_stages_at_every_heading(scenes, k):
    """The lines turned by pose heading k at each translation, on a 220 m square disc field centred at the translation:
    rays in every direction, across the rows and columns of the map and against them, equal the oracle's in every bit."""
    p = oracle.default_params()
    m, b = scenes["square"]
    theta = poses.THETAS[k]
    for tx, ty in poses.TRANSLATIONS:
        blocked, free, _ = _env_stages_equal(p, poses.move_map(m, tx, ty), poses.move(b, theta, tx, ty), (theta, tx))
        assert blocked.any() and free.any()


def test_densify_heading_follows_every_quadrant():
    """The resampled heading of a circle driven once around (atan2 of the spline derivatives) follows the path through
    all four quadrants and over the branch cut: within 1e-3 of the line's own heading modulo 2 pi, in the oracle and,
    bit for bit, in the kernel source."""
    p = oracle.default_params()
    b = poses.move(poses.turning_lines(300)["circle"], 2.0, *UTM)
    m = poses.move_map(dict(distance=np.full((800, 800), 50.0, dtype=np.float32), rows=800, cols=800, resolution=0.2,
                            center_x=0.0, center_y=0.0), float(b["ref"]["x"].mean()), float(b["ref"]["y"].mean()))
    want = oracle.densify(p, m, b["n_points"], b["ref"], 0.3, False, 320)
    got = emu.densify(p, m, b["n_points"], b["ref"], 0.3, False, 320)
    k = int(want["n_out"][0])
    assert k >= 299 and got["n_out"][0] == k and _bits_equal(got["states"][0, :k], want["states"][0, :k])
    z = want["states"]["z"][0, :k]
    assert np.abs(poses.angle_diff(z[3:k - 3], b["ref"]["z"][3:k - 3])).max() < 1e-3
    assert (np.histogram(z, bins=4, range=(-np.pi, np.pi))[0] > 50).all()


# ---- the spline fit at UTM-sized values --------------------------------------------------------------------------------
def test_fit_on_moved_lines():
    """Lines of several spacings under every pose: the kernel source's rows equal pqp_spline_fit's bit for bit, and agree
    with scipy's natural cubic spline to 1e-9 of the values (1e-9 max(1, |x|)) and 1e-9 relative on the derivatives."""
    s_list = [0.3 * np.arange(50), spacing.dynamic_s(120, spacing.sine_kappa(0.15, 20.0)),
              spacing.jitter(spacing.dynamic_s(200, spacing.sine_kappa(0.1, 25.0)), 0.3, 3), 0.15 * np.arange(3)]
    base = spacing.corridors(s_list, first_path=21)
    o = base["offsets"]
    worst = 0.0
    for theta, tx, ty in poses.POSES:
        b = poses.move(base, theta, tx, ty)
        got = fit_emu.fit_splines(o, b["ref"])
        assert got["ok"].all()
        for i in range(len(s_list)):
            r = b["ref"][o[i]:o[i + 1]]
            for coord, rows in (("x", got["x_coef"]), ("y", got["y_coef"])):
                assert _bits_equal(rows[o[i]:o[i + 1]], planner.spline_fit(r["s"], r[coord])), (theta, tx, i, coord)
                if (tx, ty) == poses.TRANSLATIONS[0] or len(r) < 4:
                    continue
                t = r["s"]
                cs = CubicSpline(t, r[coord], bc_type="natural")
                c = rows[o[i]:o[i + 1]]
                mid = 0.5 * (t[1:] - t[:-1])
                val = ((c[:-1, 0] * mid + c[:-1, 1]) * mid + c[:-1, 2]) * mid + c[:-1, 3]
                d1 = (3 * c[:-1, 0] * mid + 2 * c[:-1, 1]) * mid + c[:-1, 2]
                at = t[:-1] + mid
                scale = max(1.0, np.abs(r[coord]).max())
                assert np.abs(val - cs(at)).max() <= 1e-9 * scale
                # a derivative carries the cancellation of the value differences it is made of: ulp(value) / interval
                assert np.abs(d1 - cs(at, 1)).max() <= 1e-9 + 8 * np.spacing(scale) / np.diff(t).min()
                worst = max(worst, np.abs(val - cs(at)).max() / scale)
    assert worst < 1e-12


def test_moved_batches_keep_their_frenet_fields():
    """move() leaves s, kappa, bounds and x0 alone, stores headings in (-pi, pi] or k turns off, and is exact for a
    quarter turn."""
    b = _base_batch()
    for theta, tx, ty in poses.POSES:
        mb = poses.move(b, theta, tx, ty)
        for f in ("s", "k", "v", "a"):
            assert _bits_equal(mb["ref"][f], b["ref"][f])
        assert _bits_equal(mb["bounds"], b["bounds"]) and _bits_equal(mb["x0"], b["x0"])
        assert (np.abs(mb["ref"]["z"]) <= np.pi).all() and (np.abs(mb["end_heading"]) <= np.pi).all()
        back = poses.move_xy(*poses.move_xy(b["ref"]["x"], b["ref"]["y"], theta, 0.0, 0.0), -theta, 0.0, 0.0)
        assert np.abs(back[0] - b["ref"]["x"]).max() < 1e-12
    q = poses.move(b, np.pi / 2, 0.0, 0.0)
    assert np.array_equal(q["ref"]["x"], -b["ref"]["y"]) and np.array_equal(q["ref"]["y"], b["ref"]["x"])
    u = poses.move(b, 1.0, 0.0, 0.0, unwrap_turns=4)
    assert np.abs(u["ref"]["z"] - (b["ref"]["z"] + 1.0 + 8 * np.pi)).max() < 1e-13
    assert np.asarray(mb["ref"]).dtype == STATE_DTYPE
