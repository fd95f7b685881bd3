"""Named raw polylines for the smoothing stage (pqp_smooth_reference_device) and its CPU restatement
(oracle/smooth.py): the config-1 benchmark polyline, a straight line along x (exact-zero ds sin entries), a U-turn, a
sharp corner, the config-1 polyline at every pose of tests/poses.py (every heading, UTM-sized coordinates), 4, 5 and 6
points (the degree refusal), a repeated point (a repeated control point, which the B-spline smooths over), a NaN, and
polylines too short for the raw or the smoothed spline."""
import math
import os

import numpy as np

from tests import poses

_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "config1_benchmark_map.npz")


def config1():
    d = np.load(_GOLDEN)
    return np.asarray(d["poly_x"], dtype=np.float64), np.asarray(d["poly_y"], dtype=np.float64)


def named():
    """dict name -> (x, y) float64 arrays."""
    cx, cy = config1()
    c = {"config1": (cx, cy)}
    c["straight_x"] = (np.arange(30, dtype=np.float64) * 2.0, np.zeros(30))
    a = np.linspace(-math.pi / 2, math.pi / 2, 40)
    c["u_turn"] = (np.concatenate([np.arange(-20.0, 0.0, 2.0), 8 * np.cos(a), np.arange(0.0, -20.0, -2.0)]),
                   np.concatenate([np.full(10, -8.0), 8 * np.sin(a), np.full(10, 8.0)]))
    c["corner"] = (np.concatenate([np.arange(0.0, 20.0, 1.0), np.full(20, 20.0)]),
                   np.concatenate([np.zeros(20), np.arange(0.0, 20.0, 1.0)]))
    for k, (th, tx, ty) in enumerate(poses.POSES):
        ct, st = math.cos(th), math.sin(th)
        c[f"pose{k}"] = (tx + ct * cx - st * cy, ty + st * cx + ct * cy)
    c["four_close"] = (np.array([0.0, 1.0, 2.0, 3.0]), np.array([0.0, 0.5, 0.0, 0.5]))
    c["five_close"] = (np.array([0.0, 1.0, 2.0, 3.0, 4.0]), np.array([0.0, 0.5, 0.0, 0.5, 0.0]))
    c["six_close"] = (np.array([0.0, 1.0, 2.0, 3.0, 4.0, 5.0]), np.array([0.0, 0.5, 0.0, 0.5, 0.0, 0.5]))
    c["four_far"] = (np.array([0.0, 12.0, 24.0, 36.0]), np.array([0.0, 3.0, 0.0, 3.0]))
    x, y = cx.copy(), cy.copy()
    x[40], y[40] = x[39], y[39]
    c["repeated"] = (x, y)
    x = cx.copy()
    x[10] = np.nan
    c["nan"] = (x, cy.copy())
    c["three"] = (np.array([0.0, 5.0, 10.0]), np.zeros(3))
    # under 1 m long: two B-spline samples (t = 0 and 1), which tk::spline refuses
    c["tiny"] = (np.array([0.0, 0.2, 0.4, 0.6, 0.8, 0.9]), np.array([0.0, 0.05, 0.0, 0.05, 0.0, 0.05]))
    # a zigzag over 2 m whose B-spline is under 1 m: enough samples, but only 2 stations
    c["short"] = (np.array([0.0, 0.16, 0.32, 0.48, 0.64, 0.8]), np.array([0.0, 0.4, 0.0, 0.4, 0.0, 0.4]))
    return c


def batch(names=None):
    """(names, points [P, 7] float64 with x, y set, point_offsets int32 [B + 1])."""
    c = named()
    names = list(c) if names is None else names
    xs = [c[k][0] for k in names]
    ys = [c[k][1] for k in names]
    off = np.zeros(len(names) + 1, dtype=np.int32)
    off[1:] = np.cumsum([len(x) for x in xs])
    pts = np.zeros((int(off[-1]), 7))
    pts[:, 0] = np.concatenate(xs)
    pts[:, 1] = np.concatenate(ys)
    return names, pts, off
