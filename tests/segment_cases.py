"""Smoothed reference lines, starts and goals for the segmentation tests, shared by the CPU and GPU modules: straight,
curved (curvature ramping through 0.08 and 0.2), S-shaped and U-turn lines, fitted with pqp_spline_fit on their
chord-length s as a smoother's output would be; starts on, left of and right of the line and with heading errors
either side of 75 degrees; goals at the end, inside the line, beyond it, off to the side and far from it; the four
spacing settings of segmentSmoothedPath's flags; and the config-1 benchmark polyline, start and goal."""
import math
import os

import numpy as np

from oracle import segment as oseg
from path_optimizer_b200 import planner
from path_optimizer_b200.abi import STATE_DTYPE

# (ds_small, ds_large, dynamic, search_ds): FLAGS_enable_raw_output on / off x dynamic segmentation on / off, with
# both goal-search steps (FLAGS_enable_exact_position) between them
FLAGS = {"raw dynamic": (0.15, 0.3, True, 0.5), "raw fixed": (0.15, 0.3, False, 0.1),
         "dense dynamic": (0.5, 1.0, True, 0.1), "dense fixed": (0.5, 1.0, False, 0.5)}


def flag_kw(name):
    ds_small, ds_large, dynamic, search_ds = FLAGS[name]
    return dict(ds_small=ds_small, ds_large=ds_large, dynamic=dynamic, search_ds=search_ds)


def _polyline(kappa, length, ds=0.7071067811865476, x0=0.0, y0=0.0, th0=0.0):
    s = np.arange(0.0, length + 1e-9, ds)
    k = kappa(s)
    th = th0 + np.concatenate([[0.0], np.cumsum(0.5 * (k[1:] + k[:-1]) * np.diff(s))])
    x = x0 + np.concatenate([[0.0], np.cumsum(np.cos(0.5 * (th[1:] + th[:-1])) * np.diff(s))])
    y = y0 + np.concatenate([[0.0], np.cumsum(np.sin(0.5 * (th[1:] + th[:-1])) * np.diff(s))])
    return x, y


def fit(x, y):
    """(knots, x_coef, y_coef) of a polyline: pqp_spline_fit on the chord-length s, as the reference's smoothers hand
    x_s and y_s over."""
    t = np.concatenate([[0.0], np.cumsum(np.hypot(np.diff(x), np.diff(y)))])
    return t, planner.spline_fit(t, x), planner.spline_fit(t, y)


def lines():
    """name -> (knots, x_coef, y_coef)"""
    ramp = lambda s: np.minimum(0.3, 0.3 * s / 30.0)                                  # noqa: E731
    return {
        "straight": fit(*_polyline(lambda s: 0.0 * s, 45.0, x0=3.0, y0=-2.0, th0=0.4)),
        "curved": fit(*_polyline(ramp, 42.0, x0=-5.0, y0=1.0, th0=-0.3)),
        "s-curve": fit(*_polyline(lambda s: 0.17 * np.sin(2 * np.pi * s / 25.0), 50.0, th0=1.2)),
        "u-turn": fit(*_polyline(lambda s: np.where((s > 10.0) & (s < 10.0 + math.pi * 4.5), 1 / 4.5, 0.0), 40.0,
                                 x0=10.0, y0=5.0, th0=2.5)),
    }


def _pose(x, y, z, k=0.0):
    r = np.zeros(1, dtype=STATE_DTYPE)[0]
    r["x"], r["y"], r["z"], r["k"] = x, y, z, k
    return r


def poses(t, xc, yc):
    """[(name, start, goal)] on one line: 5 starts x 5 goals, plus starts with heading errors either side of 75 deg."""
    xs, ys = oseg.Spline(t, xc), oseg.Spline(t, yc)
    L = float(t[-1])

    def at(s, lateral=0.0, ahead=0.0):
        h = math.atan2(ys(s, 1), xs(s, 1))
        return (xs(s) - lateral * math.sin(h) + ahead * math.cos(h), ys(s) + lateral * math.cos(h) + ahead * math.sin(h),
                h)
    x0, y0, h0 = at(0.0)
    starts = {"on": _pose(x0, y0, h0, 0.02), "left": _pose(*at(0.0, 1.3), 0.0), "right": _pose(*at(0.0, -0.9), -0.01),
              "behind": _pose(*at(0.0, 0.3, -2.0)), "yawed": _pose(x0 + 0.2, y0 - 0.4, h0 + 0.6)}
    gx, gy, gh = at(L)
    goals = {"end": _pose(gx, gy, gh), "inside": _pose(*at(0.6 * L)), "beyond": _pose(*at(L, 0.0, 5.37)),
             "side": _pose(*at(0.7 * L, 3.0)), "far": _pose(*at(0.5 * L, 12.0))}
    out = [(f"{a}/{b}", sa, gb) for a, sa in starts.items() for b, gb in goals.items()]
    for deg in (74.0, -74.5, 76.0, -75.5, 179.0):
        out.append((f"heading {deg:+.1f}/inside", _pose(x0, y0, h0 + math.radians(deg)), goals["inside"]))
    return out


def batch_of(paths):
    """paths: [(name, (knots, x_coef, y_coef), max_s, start, goal)] -> dict(names, splines, max_s, start, goal) in the
    layout of pqp_segment_reference_device."""
    ko = np.zeros(len(paths) + 1, dtype=np.int32)
    np.cumsum([len(p[1][0]) for p in paths], out=ko[1:])
    cat = lambda i, w: np.concatenate([np.asarray(p[1][i], dtype=np.float64).reshape(-1, w) for p in paths]  # noqa: E731
                                      + [np.zeros((0, w))])
    return dict(names=[p[0] for p in paths],
                splines=dict(knot_offsets=ko, knots=cat(0, 1).reshape(-1), x_coef=cat(1, 4), y_coef=cat(2, 4)),
                max_s=np.array([p[2] for p in paths], dtype=np.float64),
                start=np.array([p[3] for p in paths], dtype=STATE_DTYPE),
                goal=np.array([p[4] for p in paths], dtype=STATE_DTYPE))


def main_batch():
    """Every line with every start and goal, at its full length."""
    paths = []
    for name, spl in lines().items():
        for pname, st, gl in poses(*spl):
            paths.append((f"{name} {pname}", spl, float(spl[0][-1]), st, gl))
    return batch_of(paths)


def length_batch():
    """Lengths that are refused (0, negative, NaN, infinite, too long to search) and kept (shorter than the knots, and
    past the last knot, where tk::spline extrapolates), between good paths."""
    spl = lines()["curved"]
    t = spl[0]
    _, st, gl = poses(*spl)[0]
    far = poses(*spl)[4][2]
    paths = []
    for v in (t[-1], 0.0, -1.0, float("nan"), float("inf"), 0.5 * t[-1], t[-1] + 3.0, 1e7, 1e-3):
        paths.append((f"max_s {v}", spl, float(v), st, far if v == 1e7 else gl))
    nan_spl = (spl[0], np.full_like(spl[1], np.nan), spl[2])
    paths.append(("nan rows", nan_spl, float(t[-1]), st, gl))
    paths.append(("two knots", (t[:2], spl[1][:2], spl[2][:2]), float(t[1]), st, gl))
    paths.append(("nan start", spl, float(t[-1]), _pose(np.nan, 0.0, 0.0), gl))
    paths.append(("inf heading", spl, float(t[-1]), _pose(st["x"], st["y"], np.inf), gl))
    paths.append(("huge heading", spl, float(t[-1]), _pose(st["x"], st["y"], 3e6), gl))
    return batch_of(paths)


def config1():
    """The config-1 benchmark polyline (path_optimizer_benchmark.cpp:47-82), fitted with pqp_spline_fit, its start
    and goal, and the map: dict(spl, start, goal, field)."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "config1_benchmark_map.npz"))
    field = dict(distance=g["map_distance"], rows=int(g["image_shape"][0]), cols=int(g["image_shape"][1]),
                 resolution=float(g["map_geo"][0]), center_x=float(g["map_geo"][1]), center_y=float(g["map_geo"][2]))
    spl = fit(g["poly_x"], g["poly_y"])
    return dict(spl=spl, start=_pose(*g["start"]), goal=_pose(*g["goal"]), field=field)
