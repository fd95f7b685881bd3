"""GPU tests (run with -m gpu on an H100) of scenes under rigid motions (tests/poses.py): every solver kernel class at
every pose of the grid (16 headings x the origin, a UTM position and 1e7) against the oracle and against the same paths
unmoved; lines that turn through +-pi and goals reached through a wrap; the map, clearance, collision and tail stages on
turned and shifted maps and at every heading; the plan chain over twelve scenes, each under its own pose, and the
config-1 fixture moved to UTM coordinates; the device spline fit on moved lines.

Measured differences are printed (run with -rP) for DESIGN.md section 3."""
import os

import numpy as np
import pytest

from oracle import oracle
from path_optimizer_b200 import device, planner, synth
from path_optimizer_b200.abi import BOUNDS_DTYPE
from tests import poses, shapes, spacing
from tests.device_entries import device_classes, dispatch, same_bits, to_np, u64
from tests.device_entries import rows as poses_rows

pytestmark = pytest.mark.gpu
THREADS = max(1, min(16, os.cpu_count() or 1))
KP, K, KPC = shapes.KP, shapes.K, shapes.KPC
REL_TOL = 1e-9          # Frenet solution of a rotated path against the unmoved one
FP_TOL, FRENET_TOL, FLIP_BUDGET = 1e-9, 1e-8, 0          # the bars of test_gpu_env.py
UTM, FAR = poses.TRANSLATIONS[1], poses.TRANSLATIONS[2]
SIMPLE, IMPROVED, RAW, DENSIFY = planner.BOUNDS_SIMPLE, planner.BOUNDS_IMPROVED, planner.OUTPUT_RAW, planner.OUTPUT_DENSIFY


@pytest.fixture(scope="module")
def solver():
    from path_optimizer_b200.solver import BatchPathSolver
    s = BatchPathSolver(max_batch=1024, max_total_points=1024 * 420)
    yield s
    s.close()


def _kpc_limits(b):
    ref = b["ref"].copy()
    ref["v"] = 4.0 + 3.0 * np.sin(np.arange(len(ref)) * 0.05)
    ref["a"] = 0.5 * np.cos(np.arange(len(ref)) * 0.05)
    ref["v"][::13] = 0.0
    return oracle.update_limits(oracle.default_params(), ref)


def _keeps(form, b):
    o = b["offsets"]
    return np.array([shapes.keep_of(form, b["ref"][o[i]:o[i + 1]]) for i in range(len(b["n_points"]))], dtype=np.int32)


def _assert_against_oracle(res, ref, b, what):
    """Status and iterations equal; Frenet, curvature and heading to shapes.TOL (1e-6 past 1000 iterations); x and y to
    that plus 4 ulp of the coordinate; s, a running sum of chords of x and y, to that plus 2 ulp per chord.  Returns the
    worst Frenet difference and the worst x / y difference in ulp of the coordinate (over coordinates past 1e5)."""
    assert np.array_equal(res["status"], ref["status"]) and np.array_equal(res["iters"], ref["iters"]), (
        what, np.nonzero((res["status"] != ref["status"]) | (res["iters"] != ref["iters"]))[0].tolist())
    tol = np.repeat(np.where(ref["iters"] > shapes.LONG_RUN_ITERS, shapes.LONG_RUN_TOL, shapes.TOL), b["n_points"])
    live = np.isfinite(ref["frenet"]).all(axis=1)
    assert np.array_equal(live, np.isfinite(res["frenet"]).all(axis=1)), what
    g, w = res["states"][live], ref["states"][live]
    tol = tol[live]
    d_fr = np.abs(res["frenet"][live] - ref["frenet"][live])
    assert (d_fr <= tol[:, None]).all(), (what, "frenet", d_fr.max())
    for f in "zk":
        assert (np.abs(g[f] - w[f]) <= tol).all(), (what, f)
    ulp = np.spacing(np.maximum(np.abs(w["x"]), np.abs(w["y"])))
    d_xy = np.maximum(np.abs(g["x"] - w["x"]), np.abs(g["y"] - w["y"]))
    assert (d_xy <= tol + 4 * ulp).all(), (what, "xy", (d_xy / ulp).max())
    station = np.concatenate([np.arange(n) for n in b["n_points"]])[live]
    assert (np.abs(g["s"] - w["s"]) <= tol + 2 * ulp * (station + 1)).all(), (what, "s", np.abs(g["s"] - w["s"]).max())
    far = np.maximum(np.abs(w["x"]), np.abs(w["y"])) > 1e5
    return d_fr.max(initial=0.0), (d_xy[far] / ulp[far]).max(initial=0.0)


# ---- every kernel class at every pose ---------------------------------------------------------------------------------
def _class_lines(form):
    """Per class the library selects (KP at keep 1, 3, 4 and keep 5 of the one-warp kernel), a line of its shortest and
    one of its longest length.  Returns (batch of the lines, their class names)."""
    keeps = (1, 3, 4, 5) if form == KP else ((4,) if form == KPC else (1,))
    s_list, names = [], []
    for keep in keeps:
        for name, (lo, hi) in sorted(shapes.class_ranges(form, keep).items(), key=lambda kv: kv[1]):
            if keep == 5 and name != shapes.GENERIC:
                continue
            for n in (max(lo, 3), hi):
                if form == KP:
                    s_list.append(spacing.step_profile(n, keep, len(s_list) % 9, seed=100 * keep + n))
                else:
                    s_list.append(spacing.dynamic_s(n, spacing.sine_kappa(0.15, 20.0 + len(s_list) % 7)))
                names.append(name)
    b = spacing.corridors(s_list, first_path=60 * form + 7)
    assert all(shapes.class_of(form, n, k)[0] == c for n, k, c in zip(b["n_points"], _keeps(form, b), names))
    return b, names


@pytest.mark.parametrize("form", [KP, K, KPC], ids=["KP", "K", "KPC"])
def test_every_class_at_every_pose(solver, form):
    """Every (class, pose) pair once in one solve call, the class's shortest and longest line alternating over the poses.
    Against the oracle on the same moved inputs; against the same lines unmoved: a translation changes no Frenet bit, no
    status and no iteration count, a rotation no status and no iteration count and the Frenet solution by at most 1e-9;
    pqp_solve_batch_device_classes and the device dispatch give pqp_solve_batch's bits."""
    lines, names = _class_lines(form)
    assert set(names) == set(shapes.CLASSES[form])
    pick, pose_of = [], []
    for c in range(0, len(names), 2):
        for j, pose in enumerate(poses.POSES):
            pick.append(c + j % 2)
            pose_of.append(pose)
    pick = np.array(pick)
    b = poses.move_each(synth.take_paths(lines, pick), pose_of)
    mk = mkp = lmk = lmkp = None
    if form == KPC:                                    # limits per line, the same for every copy of it
        lmk, lmkp = _kpc_limits(lines)
        lo = lines["offsets"]
        mk, mkp = (np.concatenate([a[lo[i]:lo[i + 1]] for i in pick]) for a in (lmk, lmkp))
    res = solver.solve(b, formulation=form, max_k=mk, max_kp=mkp)
    ref = oracle.solve_batch(solver.params, form, b, threads=THREADS, max_k=mk, max_kp=mkp)
    assert (ref["status"] == 1).mean() > 0.7
    worst_fr, worst_ulp = _assert_against_oracle(res, ref, b, f"form {form}")
    base = solver.solve(lines, formulation=form, max_k=lmk, max_kp=lmkp)
    o, lo = b["offsets"], lines["offsets"]
    worst_rot = 0.0
    for i, (src, (theta, tx, ty)) in enumerate(zip(pick, pose_of)):
        what = (names[src], int(b["n_points"][i]), theta, tx)
        assert res["status"][i] == base["status"][src] and res["iters"][i] == base["iters"][src], what
        g, w = res["frenet"][o[i]:o[i + 1]], base["frenet"][lo[src]:lo[src + 1]]
        if theta == 0.0:
            assert np.array_equal(u64(g), u64(w)), ("a translation changed a Frenet bit", what)
        elif np.isfinite(w).all():
            worst_rot = max(worst_rot, np.abs(g - w).max())
            assert np.abs(g - w).max() <= REL_TOL, what
    every, rows = np.arange(len(pick)), np.arange(int(o[-1]))
    same_bits(device_classes(solver, form, b, _keeps(form, b), mk=mk, mkp=mkp), res, every, rows)
    same_bits(dispatch(solver, form, b, mk, mkp), res, every, rows)
    print(f"form {form}: {len(pick)} paths, {int(o[-1])} stations; against the oracle Frenet {worst_fr:.2e}, x/y "
          f"{worst_ulp:.2f} ulp; rotated against unmoved Frenet {worst_rot:.2e}")


@pytest.mark.parametrize("form", [KP, K, KPC], ids=["KP", "K", "KPC"])
def test_turning_lines_and_wrapped_goals(solver, form):
    """The U-turn, the full circle, the figure of eight and the S-bend (400 stations; 250 for KPC) and the lines whose
    goal heading is reached through a wrap, at the origin and turned far from it, against the oracle; then with headings
    4, 1 and -4 turns off (a caller that integrates its heading): the wrapped lines' status and iterations, their Frenet
    solution within 1e-9 and their Cartesian outputs."""
    t = poses.turning_lines(250 if form == KPC else 400)
    one = poses.concat(list(t.values()) + [poses.wrap_goal_lines()])
    b = poses.concat([one, poses.move(one, np.pi / 2 + 0.3, *UTM), poses.move(one, -2.5, *FAR)])
    psi = poses.end_psi(b)
    raw = b["end_heading"] - b["ref"]["z"][b["offsets"][1:] - 1]
    lim = 70 * np.pi / 180
    assert ((np.abs(raw) > np.pi) & (np.abs(psi) < lim)).any() and (psi > lim).any() and (psi < -lim).any()
    z = b["ref"]["z"]
    assert (np.abs(np.diff(z)) > 6.0).sum() >= 6 and (np.abs(z) <= np.pi).all()       # jumps of 2 pi inside paths
    mk, mkp = _kpc_limits(b) if form == KPC else (None, None)
    ref = oracle.solve_batch(solver.params, form, b, threads=THREADS, max_k=mk, max_kp=mkp)
    # A path the oracle leaves unconverged at max_iter is left out: whether its last iterate counts as solved
    # inaccurately is a threshold on iterates that 4000 iterations of rounding have moved apart.  (KP finishes all.)
    done = np.nonzero(ref["iters"] < solver.params.max_iter)[0]
    assert len(done) >= 18 and (form != KP or len(done) == len(psi))
    if form == KPC:
        mk, mkp = mk[poses_rows(b, done)], mkp[poses_rows(b, done)]
    b, psi, raw = synth.take_paths(b, done), psi[done], raw[done]
    assert ((np.abs(raw) > np.pi) & (np.abs(psi) < lim)).any() and (psi > lim).any()
    res = solver.solve(b, formulation=form, max_k=mk, max_kp=mkp)
    ref = oracle.solve_batch(solver.params, form, b, threads=THREADS, max_k=mk, max_kp=mkp)
    assert (ref["status"] == 1).mean() >= 0.5, ref["status"]
    _assert_against_oracle(res, ref, b, f"turning lines, form {form}")
    live = np.isfinite(res["frenet"]).all(axis=1)
    for turns in (4, 1, -4):
        ub = poses.move(b, 0.0, 0.0, 0.0, unwrap_turns=turns)
        u = solver.solve(ub, formulation=form, max_k=mk, max_kp=mkp)
        assert np.array_equal(u["status"], res["status"]) and np.array_equal(u["iters"], res["iters"]), turns
        assert np.abs(u["frenet"][live] - res["frenet"][live]).max() <= REL_TOL, turns
        bar = poses.xy_tol(res["states"]["x"][live], res["states"]["y"][live])
        for f in "xy":
            assert (np.abs(u["states"][f][live] - res["states"][f][live]) <= bar).all(), (turns, f)
        # the output heading is the reference heading plus e_phi, as getOptimizedPath leaves it: off by the same turns
        assert np.abs(poses.angle_diff(u["states"]["z"][live], res["states"]["z"][live])).max() <= 1e-8
        assert np.abs(u["states"]["z"][live] - res["states"]["z"][live] - 2 * np.pi * turns).max() <= 1e-8


# ---- the stages either side of the QP ---------------------------------------------------------------------------------
def _lines():
    return synth.map_reference_paths(24, 110, x_range=(-109.0, 100.0), y_range=(-6.0, 6.0), heading_range=0.08,
                                     curvature_amp=0.02)


def _inside(m, st):
    lx, ly = m["rows"] * m["resolution"], m["cols"] * m["resolution"]
    return (np.abs(st["x"] - m["center_x"]) < lx / 2) & (np.abs(st["y"] - m["center_y"]) < ly / 2)


def _exit_edges(m, b):
    lx, ly = m["rows"] * m["resolution"], m["cols"] * m["resolution"]
    dx, dy = b["ref"]["x"] - m["center_x"], b["ref"]["y"] - m["center_y"]
    return {e for e, hit in (("+x", dx > lx / 2), ("-x", dx < -lx / 2), ("+y", dy > ly / 2), ("-y", dy < -ly / 2)) if hit.any()}


def _env_stages(pl, prm, m, b, what, tally):
    """Every map-based stage on one scene against the oracle, with the bars of test_gpu_env.py.  tally: counts of
    compared stations / states and of differing bits, for the report."""
    pl.set_map(m)
    n_points = b["n_points"]
    for mode in (SIMPLE, IMPROVED):
        spl = planner.reference_splines(b) if mode == IMPROVED else None
        want = oracle.update_bounds(prm, m, b, mode=mode, splines=spl)
        got = pl.update_bounds(b, mode=mode, splines=spl)
        assert np.array_equal(got["n_valid"], want["n_valid"]), (what, mode)
        W, G = want["bounds"].view(np.float64).reshape(-1, 8), got["bounds"].view(np.float64).reshape(-1, 8)
        flips = 0
        for i in range(len(n_points)):
            sl = slice(b["offsets"][i], b["offsets"][i] + want["n_valid"][i])
            flips += int((np.abs(G[sl] - W[sl]) > FP_TOL).any(axis=1).sum())
            tally["bound values"] += G[sl].size
            tally["bound values differing in a bit"] += int((u64(G[sl]) != u64(W[sl])).sum())
        assert flips <= FLIP_BUDGET, (what, mode, flips)
        if mode == SIMPLE:
            n_valid = want["n_valid"]
    ok = oracle.check_states(prm, m, b["ref"])
    assert np.array_equal(pl.check_states(b["ref"]), ok), what
    paths = b["ref"].copy()
    paths["s"] = 0.0
    for cc in (True, False):
        want = oracle.finish_raw(prm, m, n_points, paths, collision_check=cc)
        got = pl.finish_raw(n_points, paths, collision_check=cc)
        assert np.array_equal(got["n_kept"], want["n_kept"]) and np.array_equal(got["ok"], want["ok"]), (what, cc)
    src = want["states"]
    ulp = np.spacing(max(abs(m["center_x"]), abs(m["center_y"]), 1.0))
    for cc in (True, False):
        want = oracle.densify(prm, m, n_points, src, 0.3, cc, 160)
        got = pl.densify(n_points, src, 0.3, cc, 160)
        assert np.array_equal(got["n_out"], want["n_out"]) and np.array_equal(got["ok"], want["ok"]), (what, cc)
        for i, k in enumerate(want["n_out"]):
            for f in "xyzks":
                d = np.abs(got["states"][f][i, :k] - want["states"][f][i, :k]).max(initial=0.0)
                assert d <= FP_TOL + (4 * ulp if f in "xy" else 0.0), (what, "densify", cc, i, f, d)
            tally["resampled values"] += 5 * int(k)
            tally["resampled values differing in a bit"] += sum(
                int((u64(got["states"][f][i, :k]) != u64(want["states"][f][i, :k])).sum()) for f in "xyzks")
    xy = np.concatenate([poses.border_points(m), np.stack([b["ref"]["x"], b["ref"]["y"]], 1)[::3]])
    assert np.array_equal(pl.map_distance(xy), oracle.map_distance(m, xy)), what
    tally["scenes"] += 1
    off_map = np.array([not _inside(m, b["ref"][b["offsets"][i]:b["offsets"][i + 1]]).all() for i in range(len(n_points))])
    return (n_valid < n_points).any(), (n_valid == n_points).any(), off_map.any()


@pytest.fixture(scope="module")
def env_planner():
    p = planner.PathPlanner(max_batch=64, max_total_points=64 * 200)
    yield p
    p.close()


def _tally():
    from collections import Counter
    return Counter()


def test_env_stages_on_turned_and_shifted_maps(env_planner):
    """The disc field under the four quarter turns (both signs of pi) x the three translations, with its lines: blocked
    paths, free paths and paths that leave the map in every scene, through each of its four edges over the turns."""
    prm = oracle.default_params()
    m, b = synth.disc_field_map(), _lines()
    tally, edges = _tally(), set()
    for theta, tx, ty in poses.QUARTER_POSES:
        mm, mb = poses.move_map(m, tx, ty, poses.quarter_turns(theta)), poses.move(b, theta, tx, ty)
        covered = _env_stages(env_planner, prm, mm, mb, (theta, tx), tally)
        assert all(covered), (theta, tx, covered)
        edges |= _exit_edges(mm, mb)
    assert edges == {"+x", "-x", "+y", "-y"}
    print("turned and shifted maps:", dict(tally))


def test_env_stages_at_every_heading(env_planner):
    """The lines under every pose of the grid on a 220 m square disc field (1100 x 1100 cells) centred at the pose's
    translation: rays in every direction."""
    prm = oracle.default_params()
    m, b = synth.disc_field_map(rows=1100, cols=1100, n_discs=1300), _lines()
    tally = _tally()
    for theta, tx, ty in poses.POSES:
        blocked, free, _ = _env_stages(env_planner, prm, poses.move_map(m, tx, ty), poses.move(b, theta, tx, ty),
                                       (theta, tx), tally)
        assert blocked and free, (theta, tx)
    print("every heading:", dict(tally))


# ---- the plan chain -----------------------------------------------------------------------------------------------------
def _host(r, output_mode):
    import torch
    torch.cuda.synchronize()
    st = r["states"].reshape(-1, 7) if output_mode == RAW else r["states"]
    states = device.tensor_to_records(st)
    if output_mode == DENSIFY:
        states = states.reshape(r["states"].shape[0], -1)
    return dict(states=states, n_out=to_np(r["n_out"]), ok=to_np(r["ok"]), status=to_np(r["status"]),
                iters=to_np(r["iters"]), bounds=device.tensor_to_records(r["bounds"], BOUNDS_DTYPE))


def _path(r, b, i, output_mode):
    o = b["offsets"]
    return r["states"][o[i]:o[i] + r["n_out"][i]] if output_mode == RAW else r["states"][i, :r["n_out"][i]]


def _plan_states_match(g, w, tol, what, densified=False):
    """x and y to tol + 4 ulp of the coordinate, s to tol + 2 ulp per chord.  Heading and curvature to tol in the raw
    output.  In the resampled output they are first and second derivatives of splines through x and y over 0.3 m
    intervals, so a coordinate that differs by one ulp moves them by ulp / 0.3 and ulp / 0.09: bars tol + 8 ulp / 0.3
    and tol + 32 ulp / 0.09 (3.3e-7 at 5.2e6, against 4.3e-8 measured on an H100)."""
    bar = poses.xy_tol(w["x"], w["y"], tol)
    ulp = (bar - tol) / 4
    for f in "xy":
        assert (np.abs(g[f] - w[f]) <= bar).all(), (what, f, np.abs(g[f] - w[f]).max(initial=0.0))
    for f, amp in (("z", 8 / 0.3), ("k", 32 / 0.09)):
        assert (np.abs(g[f] - w[f]) <= tol + (amp * ulp if densified else 0.0)).all(), (what, f, np.abs(g[f] - w[f]).max(initial=0.0))
    station = np.arange(len(w))
    assert (np.abs(g["s"] - w["s"]) <= tol + 2 * ulp * (station + 1)).all(), (what, "s")


SCENE_POSES = [poses.QUARTER_POSES[k] for k in (1, 2, 4, 5, 7, 8, 10, 11, 13, 14, 3, 0)]      # twelve, the origin last


@pytest.mark.parametrize("output_mode", [RAW, DENSIFY], ids=["raw", "densify"])
@pytest.mark.parametrize("bounds_mode", [SIMPLE, IMPROVED], ids=["simple", "improved"])
def test_plan_chain_twelve_scenes(bounds_mode, output_mode):
    """Twelve disc fields in one batch, each turned and shifted by its own pose, five lines per scene, KP / K / KPC per
    path: plan (host buffers, a map index per path) against oracle.plan scene by scene; plan_device, on splines fitted
    on the device for IMPROVED, gives plan's results bit for bit."""
    import torch
    prm = oracle.default_params()
    per = 5
    maps, parts = [], []
    for k, (theta, tx, ty) in enumerate(SCENE_POSES):
        maps.append(poses.move_map(synth.disc_field_map(seed=synth.BASE_SEED + k), tx, ty, poses.quarter_turns(theta)))
        lines = synth.map_reference_paths(per, 120, first_path=per * k, y_range=(-1.5, 1.5), heading_range=0.03,
                                          curvature_amp=0.01)
        parts.append(poses.move(lines, theta, tx, ty))
    b = poses.concat(parts)
    total = int(b["offsets"][-1])
    b["ref"]["v"] = 4.0 + 3.0 * np.sin(np.arange(total) * 0.05)
    b["ref"]["a"] = 0.5 * np.cos(np.arange(total) * 0.05)
    mi = np.repeat(np.arange(len(maps), dtype=np.int32), per)
    forms = (np.arange(len(mi)) % 3).astype(np.int32)
    spl = planner.reference_splines(b) if bounds_mode == IMPROVED else None
    p = planner.PathPlanner(max_batch=64, max_total_points=64 * 128)
    try:
        p.set_maps(maps)
        got = p.plan(b, formulation=forms, bounds_mode=bounds_mode, splines=spl, output_mode=output_mode, max_out=160,
                     want_bounds=True, map_index=mi)
        ko = np.concatenate([[0], np.cumsum(b["n_points"])])
        for i in range(len(mi)):
            one = synth.take_paths(b, [i])
            sp = None if spl is None else dict(n_knots=one["n_points"], knots=spl["knots"][ko[i]:ko[i + 1]],
                                               x_coef=spl["x_coef"][ko[i]:ko[i + 1]], y_coef=spl["y_coef"][ko[i]:ko[i + 1]])
            want = oracle.plan(prm, maps[mi[i]], one, formulation=int(forms[i]), bounds_mode=bounds_mode, splines=sp,
                               output_mode=output_mode, max_out=160)
            for f in ("status", "iters", "n_out", "ok"):
                assert got[f][i] == want[f][0], (i, f, got[f][i], want[f][0])
            tol = shapes.LONG_RUN_TOL if want["iters"][0] > shapes.LONG_RUN_ITERS else FRENET_TOL
            _plan_states_match(_path(got, b, i, output_mode), _path(want, one, 0, output_mode), tol, (i, SCENE_POSES[mi[i]]),
                               densified=output_mode == DENSIFY)
        assert (got["status"] == 1).sum() >= 20 and (got["n_out"] < b["n_points"]).any()
        dev = torch.device("cuda", 0)
        d = device.batch_to_device(b, dev)
        dspl = None
        if bounds_mode == IMPROVED:
            dspl = p.fit_splines_device(d["offsets"], d["ref"])
            torch.cuda.synchronize()
            assert (to_np(dspl["ok"]) == 1).all()
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
        r = p.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], max_n_points=120,
                          formulation=t(forms), bounds_mode=bounds_mode, splines=dspl, output_mode=output_mode,
                          max_out=160, want_bounds=True, map_index=t(mi))
        dv = _host(r, output_mode)
        for f in ("status", "iters", "n_out", "ok"):
            assert np.array_equal(dv[f], got[f]), f
        assert np.array_equal(u64(dv["bounds"]), u64(got["bounds"]))
        for i in range(len(mi)):
            assert _path(dv, b, i, output_mode).tobytes() == _path(got, b, i, output_mode).tobytes(), i
    finally:
        p.close()


def test_config1_fixture_at_utm_coordinates():
    """The reference's benchmark map and path moved to (4.5e5, 5.2e6) and turned a quarter turn: the fixture's stored
    oracle outputs under the same motion are the expected values (no new fixture); same status and iteration count."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "config1_benchmark_map.npz"))
    field = dict(distance=g["map_distance"], rows=int(g["image_shape"][0]), cols=int(g["image_shape"][1]),
                 resolution=float(g["map_geo"][0]), center_x=float(g["map_geo"][1]), center_y=float(g["map_geo"][2]))
    b = dict(n_points=g["n_points"], ref=g["ref"], x0=g["x0"], end_heading=g["end_heading"],
             bounds=np.zeros(len(g["ref"]), dtype=BOUNDS_DTYPE))
    b["offsets"] = np.array([0, int(g["n_points"][0])], dtype=np.int32)
    theta = np.pi / 2
    mb, mm = poses.move(b, theta, *UTM), poses.move_map(field, *UTM, 1)
    # the fixture's reference splines under the same motion: (x, y) -> (-y + tx, x + ty), the shift on the value column
    xc, yc = -g["y_coef"], g["x_coef"].copy()
    xc[:, 3], yc[:, 3] = (v.astype(np.float64) for v in poses.move_xy(g["x_coef"][:, 3], g["y_coef"][:, 3], theta, *UTM))
    spl = dict(n_knots=np.array([len(g["knots"])], dtype=np.int32), knots=g["knots"], x_coef=xc, y_coef=yc)
    p = planner.PathPlanner(max_batch=1, max_total_points=256)
    try:
        p.set_map(mm)
        for mode, tag in ((IMPROVED, "improved"), (SIMPLE, "simple")):
            r = p.plan(mb, bounds_mode=mode, splines=spl if mode == IMPROVED else None, want_bounds=True)
            assert r["status"][0] == g[f"plan_{tag}_status"][0] == 1 and r["iters"][0] == g[f"plan_{tag}_iters"][0]
            assert r["n_out"][0] == g[f"plan_{tag}_n_out"][0] and r["ok"][0] == 1
            # (IMPROVED adds an offset computed from coordinates of 5e6: a few ulp of them)
            assert np.abs(r["bounds"].view(np.float64) - g[f"bounds_{tag}"].view(np.float64)).max() <= (
                FP_TOL if mode == SIMPLE else 1e-7)
            k = int(r["n_out"][0])
            want = poses.move_states(g[f"plan_{tag}_states"][:k], theta, *UTM)
            got = r["states"][:k]
            want["z"] = got["z"]                      # compared modulo 2 pi below
            _plan_states_match(got, want, FRENET_TOL, tag)
            assert np.abs(poses.angle_diff(got["z"], g[f"plan_{tag}_states"]["z"][:k] + theta)).max() <= FRENET_TOL
    finally:
        p.close()


def test_fit_splines_device_on_moved_lines():
    """pqp_fit_splines_device on lines under every pose: knots and rows equal pqp_spline_fit's bit for bit."""
    import torch
    s_list = [0.3 * np.arange(50), spacing.dynamic_s(120, spacing.sine_kappa(0.15, 20.0)),
              spacing.jitter(spacing.dynamic_s(200, spacing.sine_kappa(0.1, 25.0)), 0.3, 3), 0.15 * np.arange(3),
              synth._accumulate_s(416)]
    base = spacing.corridors(s_list, first_path=21)
    b = poses.concat([poses.move(base, *pose) for pose in poses.POSES])
    p = planner.PathPlanner(max_batch=256, max_total_points=256 * 200)
    try:
        d = device.batch_to_device(b, torch.device("cuda", 0))
        r = p.fit_splines_device(d["offsets"], d["ref"])
        torch.cuda.synchronize()
        want = planner.reference_splines(b)
        assert (to_np(r["ok"]) == 1).all()
        for f in ("knots", "x_coef", "y_coef"):
            assert np.array_equal(u64(to_np(r[f])), u64(want[f])), f
        print(f"fit: {len(b['n_points'])} lines, {int(b['offsets'][-1])} stations, no differing bit")
    finally:
        p.close()
