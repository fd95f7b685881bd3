"""Polylines, maps and weights for the TENSION smoothing tests (pqp_smooth_reference_tension_device and its CPU
restatement, tests/tension_restatement.py): the named polylines of tests/smooth_cases.py, a line heading
straight down -y (theta = heading + pi/2 is exactly 0 there, so the -sin(theta) entries of A are exact zeros that
sparseView drops), the config-1 map, and that map turned and shifted to every quarter-turn pose of tests/poses.py
together with the config-1 polyline moved to the same pose."""
import numpy as np

from tests import poses as P
from tests import segment_cases
from tests import smooth_cases as sc

WEIGHTS = [(0.0, 1.0, 50.0), (0.5, 1.0, 50.0), (0.0, 0.0, 50.0), (1e-3, 2.0, 0.0), (0.1, 0.3, 7.7)]
# the config-1 polyline at pose 3 (a quarter turn at the origin) keeps a station's offset on a clearance of 0.23 m
BINDING = "pose3"


def config1_map():
    return segment_cases.config1()["field"]


def named():
    """dict name -> (x, y): smooth_cases.named() plus "down"."""
    c = sc.named()
    c["down"] = (np.full(25, 12.0), -2.0 * np.arange(25, dtype=np.float64))
    return c


def pose_maps():
    """dict "pose{k}" -> the config-1 map moved to pose k, for the quarter-turn poses of tests/poses.py."""
    m = config1_map()
    out = {}
    for k, (th, tx, ty) in enumerate(P.POSES):
        if (th, tx, ty) in P.QUARTER_POSES:
            out[f"pose{k}"] = P.move_map(m, tx, ty, P.quarter_turns(th))
    return out


def batch(names, moved=False):
    """(names, points [P, 7], point_offsets [B + 1], maps, map_index): the config-1 map is map 0; with `moved`, a path
    "pose{k}" at a quarter-turn pose runs on the config-1 map moved to that pose (maps 1, 2, ...)."""
    c = named()
    xs, ys = [c[k][0] for k in names], [c[k][1] for k in names]
    off = np.zeros(len(names) + 1, dtype=np.int32)
    off[1:] = np.cumsum([len(x) for x in xs])
    pts = np.zeros((int(off[-1]), 7))
    if len(names):
        pts[:, 0], pts[:, 1] = np.concatenate(xs), np.concatenate(ys)
    maps, index = [config1_map()], np.zeros(len(names), dtype=np.int32)
    pm = pose_maps() if moved else {}
    for b, k in enumerate(names):
        if k in pm:
            index[b] = len(maps)
            maps.append(pm[k])
    return names, pts, off, maps, index
