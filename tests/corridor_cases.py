"""Scenes for the corridor search and post-smoothing tests (pqp_post_smooth_device, oracle/corridor.py), shared by the
CPU and GPU modules: lines fitted with pqp_spline_fit on their chord-length s, as a smoother hands them over, on small
distance maps built from discs and walls.  Named cases: a clear road, an obstacle on the line, symmetric obstacles, a
wall across the road, a start more than 10 m off the line, a start near the end, a line of 6 m or less, tight curves
either way, a line running off the map, the config-1 benchmark map with its polyline shifted sideways, and moved
copies of the obstacle scene at every quarter turn and far from the origin."""
import math

import numpy as np

from path_optimizer_b200 import synth
from path_optimizer_b200.abi import STATE_DTYPE
from tests import poses as P
from tests import segment_cases as sc

RES = 0.2


def grid_map(discs=(), walls=(), rows=400, cols=250, center=(20.0, 0.0)):
    """A distance map of rows x cols cells at 0.2 m centred on `center`, obstacles: discs (x, y, r) and walls
    (x0, y0, x1, y1) boxes."""
    cx, cy = center
    xs = cx + 0.5 * rows * RES - (np.arange(rows) + 0.5) * RES
    ys = cy + 0.5 * cols * RES - (np.arange(cols) + 0.5) * RES
    X, Y = np.meshgrid(xs, ys, indexing="ij")
    occ = np.ones((rows, cols), dtype=np.uint8)
    for x, y, r in discs:
        occ[(X - x) ** 2 + (Y - y) ** 2 <= r * r] = 0
    for x0, y0, x1, y1 in walls:
        occ[(X >= x0) & (X <= x1) & (Y >= y0) & (Y <= y1)] = 0
    return dict(distance=synth.distance_layer(occ, RES), rows=rows, cols=cols, resolution=RES, center_x=float(cx),
                center_y=float(cy))


def _line(length, kappa=lambda s: 0.0 * s, x0=0.0, y0=0.0, th0=0.0):
    return sc.fit(*sc._polyline(kappa, length, x0=x0, y0=y0, th0=th0))


def _start(x, y, z):
    r = np.zeros(1, dtype=STATE_DTYPE)[0]
    r["x"], r["y"], r["z"] = x, y, z
    return r


def scenes():
    """name -> (map, (knots, x_coef, y_coef), start)"""
    clear = grid_map()
    one = grid_map(discs=[(20.0, 0.0, 1.5)])
    sym = grid_map(discs=[(20.0, 3.0, 1.2), (20.0, -3.0, 1.2)])
    wall = grid_map(walls=[(30.0, -15.0, 31.0, 15.0)])
    road = _line(45.0)
    wave = lambda s: np.where(s < 12.0, 1 / 7.0, np.where(s < 24.0, -1 / 7.0, 0.0))   # noqa: E731
    out = {
        "clear": (clear, road, _start(0.3, 0.0, 0.05)),
        "obstacle": (one, road, _start(0.0, 0.0, 0.0)),
        "symmetric": (sym, road, _start(0.0, 0.0, 0.0)),
        "wall": (wall, road, _start(0.0, 0.0, 0.0)),
        "far start": (clear, road, _start(2.0, 10.5, 0.0)),
        "near end": (clear, road, _start(42.0, 0.5, 0.0)),
        "short": (clear, _line(5.5, x0=2.0), _start(2.0, 0.25, 0.0)),
        "tight curves": (clear, _line(36.0, wave, x0=2.0, y0=0.0), _start(2.0, 0.0, 0.0)),
        "off map": (clear, _line(60.0, x0=10.0, th0=0.1), _start(10.0, 0.0, 0.1)),
    }
    c = sc.config1()
    kn, xco, yco = c["spl"]
    # shifted sideways by 1.2 m along the normal of the first knot's heading
    th = math.atan2(yco[0][2], xco[0][2])
    xs = np.array([r[3] for r in xco]) - 1.2 * math.sin(th)
    ys = np.array([r[3] for r in yco]) + 1.2 * math.cos(th)
    out["config-1 shifted"] = (c["field"], sc.fit(xs, ys), c["start"])
    # the obstacle scene moved: every quarter turn, and far from the origin
    for q, (tx, ty) in enumerate([(0.0, 0.0), (1e4, -2e4), (-3e5, 4e5), (7e5, 7e5)]):
        th = q * math.pi / 2
        m = P.move_map(one, tx, ty, quarter_turns=q)
        x, y = sc._polyline(lambda s: 0.0 * s, 45.0)
        mx, my = P.move_xy(x, y, th, tx, ty)
        sx, sy = P.move_xy(np.array([0.0]), np.array([0.3]), th, tx, ty)
        out[f"moved q{q}"] = (m, sc.fit(mx.astype(np.float64), my.astype(np.float64)),
                                _start(float(sx[0]), float(sy[0]), th))
    return out


TIE_SPACING = 0.5


def tie_scene():
    """(map, line, start) for a lateral spacing of TIE_SPACING, where the lattice -10, -9.5, ..., 10 is symmetric about
    the line: a straight line along the x axis (heading exactly 0, so every node lies at (x, l) exactly once x >= 8),
    a mirror-symmetric map with a block across the middle of the road, and the start at x = 10.  Mirrored detours cost
    the same to the last bit (atan2 is odd), so the DP meets exact ties and the first index must win them."""
    m = grid_map(walls=[(25.0, -1.5, 27.0, 1.5)])
    occ = (m["distance"] > 0).astype(np.uint8)
    occ &= occ[:, ::-1]
    m = dict(m, distance=synth.distance_layer(occ, RES))
    return m, _line(45.0), _start(10.0, 0.1, 0.0)


def batch(names=None):
    """dict(names, maps, map_index, splines, max_s, start) of the named scenes (all by default), one map per scene."""
    sc_ = scenes()
    names = list(sc_) if names is None else names
    paths = [(n, sc_[n][1], float(sc_[n][1][0][-1]), sc_[n][2], sc_[n][2]) for n in names]
    b = sc.batch_of(paths)
    return dict(names=names, maps=[sc_[n][0] for n in names], map_index=np.arange(len(names), dtype=np.int32),
                splines=b["splines"], max_s=b["max_s"], start=b["start"])
