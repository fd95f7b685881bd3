"""Scenes moved by a rigid motion, and lines that turn through every heading, shared by the CPU and GPU pose tests
(like tests/spacing.py).

Every generator of the suite starts near the origin at heading ~0 and runs along +x, so the wraps of constraintAngle,
the branch cut of atan2, rays with a negative x component and map lookups at UTM-sized coordinates run on one branch
only.  A vehicle drives in every direction, in map-frame coordinates that are often UTM (x ~ 5e5, y ~ 5e6).

A rigid motion changes x, y and heading and nothing else: s, kappa, the corridor bounds and x0 are Frenet quantities.
So a moved batch must solve to the same Frenet solution, and its Cartesian outputs are the moved outputs.  The motion is
computed in numpy.longdouble and rounded once, so that expected values do not carry the rounding pattern of a second
float64 implementation; quarter turns use exact cosines and sines, so that a map turned with np.rot90 stays aligned
with the lines turned by the same pose."""
import numpy as np

from path_optimizer_b200 import synth
from tests import spacing

LD = np.longdouble
PI = 2 * np.arctan2(LD(1), LD(0))            # pi in long double
TWO_PI = 2 * PI

_QUARTER = {0.0: 0, float(np.pi / 2): 1, float(np.pi): 2, float(-np.pi): 2, float(-np.pi / 2): 3}

# headings: the axes, pi from both sides, the last double below pi, the diagonals of the left half plane, 8 seeded
THETAS = [0.0, np.pi / 2, -np.pi / 2, np.pi, -np.pi, np.nextafter(np.pi, 0.0), 3 * np.pi / 4, -3 * np.pi / 4]
THETAS += np.random.default_rng(synth.BASE_SEED).uniform(-np.pi, np.pi, 8).tolist()
TRANSLATIONS = [(0.0, 0.0), (4.5e5, 5.2e6), (-1.0e7, 1.0e7)]          # the origin, a UTM easting / northing, 1e7
POSES = [(float(th), tx, ty) for th in THETAS for tx, ty in TRANSLATIONS]
QUARTER_POSES = [p for p in POSES if p[0] in _QUARTER]


def quarter_turns(theta):
    """0..3 for a pose heading that is a multiple of 90 degrees (as a double), else None."""
    return _QUARTER.get(float(theta))


def _cos_sin(theta):
    q = quarter_turns(theta)
    if q is not None:
        return [(LD(1), LD(0)), (LD(0), LD(1)), (LD(-1), LD(0)), (LD(0), LD(-1))][q]
    return np.cos(LD(theta)), np.sin(LD(theta))


def move_xy(x, y, theta, tx, ty):
    """(x, y) turned by theta about the origin, then shifted by (tx, ty): long double arrays."""
    c, s = _cos_sin(theta)
    x, y = np.asarray(x, dtype=LD), np.asarray(y, dtype=LD)
    return x * c - y * s + LD(tx), x * s + y * c + LD(ty)


def move_heading(z, theta, unwrap_turns=None):
    """Headings turned by theta, as long double.  unwrap_turns None: atan2(sin, cos) of the sum, in (-pi, pi] as the
    reference's getHeading gives them; k: the sum plus 2 pi k, for a caller that integrates its heading."""
    a = np.asarray(z, dtype=LD) + LD(theta)
    if unwrap_turns is None:
        return np.arctan2(np.sin(a), np.cos(a))
    return a + TWO_PI * unwrap_turns


def move_states(states, theta, tx, ty, unwrap_turns=None):
    """A copy of a state array with x, y and heading moved; every other field as it was."""
    out = np.array(states)
    x, y = move_xy(states["x"], states["y"], theta, tx, ty)
    out["x"], out["y"] = x.astype(np.float64), y.astype(np.float64)
    out["z"] = move_heading(states["z"], theta, unwrap_turns).astype(np.float64)
    return out


def move(batch, theta, tx, ty, unwrap_turns=None):
    """A copy of a batch under a rigid motion: ref x, y, z and end_heading move, nothing else does."""
    out = {k: np.array(v) for k, v in batch.items()}
    out["ref"] = move_states(batch["ref"], theta, tx, ty, unwrap_turns)
    out["end_heading"] = move_heading(batch["end_heading"], theta, unwrap_turns).astype(np.float64)
    return out


def move_each(batch, poses, unwrap_turns=None):
    """Path i of the batch under poses[i]."""
    out = {k: np.array(v) for k, v in batch.items()}
    o = batch["offsets"]
    for i, (theta, tx, ty) in enumerate(poses):
        out["ref"][o[i]:o[i + 1]] = move_states(batch["ref"][o[i]:o[i + 1]], theta, tx, ty, unwrap_turns)
        out["end_heading"][i] = float(move_heading(batch["end_heading"][i], theta, unwrap_turns))
    return out


def move_map(m, tx, ty, quarter_turns=0):
    """A distance (or occupancy) map turned by quarter_turns * 90 degrees about the origin, then shifted.  grid_map
    index convention (include/pqp_env.h): cell (0, 0) is the +x / +y corner and indices grow towards -x / -y, so a
    counter-clockwise quarter turn of the scene is np.rot90 of the layer, with rows and cols swapped."""
    q = quarter_turns % 4
    out = dict(m)
    for layer in ("distance", "occupancy"):
        if layer in m:
            out[layer] = np.ascontiguousarray(np.rot90(m[layer], q))
            out["rows"], out["cols"] = out[layer].shape
    cx, cy = move_xy(m["center_x"], m["center_y"], [0.0, np.pi / 2, np.pi, -np.pi / 2][q], tx, ty)
    out["center_x"], out["center_y"] = float(cx), float(cy)
    return out


def cell_centers(m):
    """x [rows] and y [cols] of the cell centres, by the arithmetic of the lookup (cell_center, pqp_env_core.cuh)."""
    res = m["resolution"]
    ox = m["center_x"] + (0.5 * (m["rows"] * res) - 0.5 * res)
    oy = m["center_y"] + (0.5 * (m["cols"] * res) - 0.5 * res)
    return ox + res * -np.arange(m["rows"], dtype=np.float64), oy + res * -np.arange(m["cols"], dtype=np.float64)


def border_points(m, k=9):
    """Points on and just either side of the four borders of a map and at its corners: [n, 2]."""
    lx, ly = m["rows"] * m["resolution"], m["cols"] * m["resolution"]
    cx, cy = m["center_x"], m["center_y"]
    pts = []
    for t in np.linspace(-0.5, 0.5, k):
        for e in (-0.5, 0.5):
            for d in (-1e-3, 0.0, 1e-3, -0.07, 0.07):
                pts.append((cx + e * lx + d, cy + t * ly))
                pts.append((cx + t * lx, cy + e * ly + d))
    return np.array(pts, dtype=np.float64)


def xy_tol(x, y, base=1e-8):
    """The bar on a Cartesian output: base + 4 ulp of the larger coordinate (1 ulp of 1e7 is 1.9e-9 m)."""
    return base + 4 * np.spacing(np.maximum(np.abs(x), np.abs(y)))


def angle_diff(a, b):
    """a - b modulo 2 pi, in [-pi, pi]."""
    d = np.asarray(a, dtype=LD) - np.asarray(b, dtype=LD)
    return (d - TWO_PI * np.round(d / TWO_PI)).astype(np.float64)


# ---- lines the generators cannot make ------------------------------------------------------------------------------
def _pieces(*parts):
    """kappa(s) of consecutive pieces (length, curvature)."""
    ends = np.cumsum([p[0] for p in parts])
    ks = np.array([p[1] for p in parts] + [parts[-1][1]])
    return lambda s: ks[np.searchsorted(ends, s, side="right")]


def turning_lines(n_long=400, first_path=0):
    """name -> one-path batch, headings wrapped into (-pi, pi]: a U-turn at kappa 0.18 between straight ends; a full
    circle and a figure of eight on n_long stations (the heading passes +-pi in the middle of the path); an S-bend at
    kappa +-0.19, just inside the steering limit tan(30 deg) / 2.85 = 0.2026."""
    half = np.pi / 0.18
    length = 0.3 * (n_long - 1)
    lines = {
        "u-turn": (int((20.0 + half) / 0.3) + 1, _pieces((10.0, 0.0), (half, 0.18), (10.0, 0.0))),
        "circle": (n_long, _pieces((length + 1.0, 2 * np.pi / length))),
        "figure of eight": (n_long, _pieces((length / 2, 4 * np.pi / length), (length, -4 * np.pi / length))),
        "s-bend": (int(26.0 / 0.3) + 1, _pieces((5.0, 0.0), (8.0, 0.19), (8.0, -0.19), (5.0, 0.0))),
    }
    out = {}
    for k, (name, (n, kap)) in enumerate(lines.items()):
        b = spacing.corridors([synth._accumulate_s(n)], [kap], first_path=first_path + k)
        out[name] = move(b, 0.0, 0.0, 0.0)
    return out


# last heading, goal heading, what the end-heading row must do (end_psi = constraintAngle(goal - last) < 70 deg)
WRAP_GOALS = [
    (np.pi - 0.02, -np.pi + 0.03, "constrained through a wrap"),          # end_psi 0.05 after + 2 pi ... - 2 pi
    (np.pi - 0.02, np.pi - 0.02 + 1.2 - 2 * np.pi, "constrained through a wrap"),       # 1.2 < 70 deg
    (np.pi - 0.02, np.pi - 0.02 - 1.3, "negative below -70 deg"),         # no fabs in the reference: constrained
    (np.pi - 0.02, np.pi - 0.02 + 1.23 - 2 * np.pi, "unconstrained"),     # 1.23 > 70 deg through a wrap
    (-np.pi + 0.02, np.pi - 0.03, "constrained through a wrap"),          # from the negative side: end_psi -0.05
    (-np.pi + 0.02, -np.pi + 0.02 - 1.3 + 2 * np.pi, "negative below -70 deg"),
]


def wrap_goal_lines(n=60, first_path=40):
    """One gently curved line per entry of WRAP_GOALS, turned so that its last heading is the entry's, with the entry's
    goal heading."""
    b = spacing.corridors([synth._accumulate_s(n)] * len(WRAP_GOALS), first_path=first_path,
                          kappa_list=[spacing.sine_kappa(0.05, 30.0, 0.4 * k) for k in range(len(WRAP_GOALS))])
    o = b["offsets"]
    b = move_each(b, [(last - b["ref"]["z"][o[i + 1] - 1], 3.0 * i, -2.0 * i) for i, (last, _, _) in enumerate(WRAP_GOALS)])
    b["end_heading"][:] = [goal for _, goal, _ in WRAP_GOALS]
    return b


def end_psi(b):
    """constraintAngle(end_heading - last heading) of every path, from the long double difference."""
    o = b["offsets"]
    return angle_diff(b["end_heading"], b["ref"]["z"][o[1:] - 1])


def concat(batches):
    """Batches joined into one, in order."""
    out = {k: np.concatenate([b[k] for b in batches]) for k in ("n_points", "ref", "bounds", "x0", "end_heading")}
    out["offsets"] = np.concatenate([[0], np.cumsum(out["n_points"])]).astype(np.int32)
    return out
