"""Reference lines for the spline-fit tests, shared by the CPU and GPU modules (like tests/spacing.py): evenly spaced
lines, the uneven spacings of tests/spacing.py (dynamic segmentation, the same jittered, step profiles, chord-length s),
the shortest fittable path (3 stations), a 416-station path, and paths pqp_fit_splines_device refuses (fewer than 3
stations, and every degenerate spacing of tests/spacing.py applied to the s of an otherwise good line)."""
import numpy as np

from path_optimizer_b200.abi import STATE_DTYPE
from tests import spacing

LENGTHS = (3, 4, 9, 50, 200, 416)


def _line(s, first_path=0):
    """One consistent line on the stations s (x, y, heading and curvature integrated from s)."""
    return spacing.corridors([np.asarray(s, dtype=np.float64)], first_path=first_path)["ref"].copy()


def batch_of(refs):
    """A batch (n_points, offsets, ref, x0, end_heading) of the given per-path state arrays, in order."""
    n = np.array([len(r) for r in refs], dtype=np.int32)
    off = np.zeros(len(n) + 1, dtype=np.int32)
    np.cumsum(n, out=off[1:])
    ref = np.concatenate([np.asarray(r, dtype=STATE_DTYPE) for r in refs] + [np.zeros(0, dtype=STATE_DTYPE)])
    x0 = np.zeros((len(n), 3))
    end = np.zeros(len(n))
    for i, r in enumerate(refs):
        if len(r):
            x0[i, 2] = r["k"][0]
            end[i] = r["z"][-1]
    return dict(n_points=n, offsets=off, ref=ref, x0=x0, end_heading=end)


def good_lines():
    """name -> state array of every fittable line."""
    out = {}
    for n in LENGTHS:
        out[f"even 0.3 n{n}"] = _line(0.3 * np.arange(n), n)
        out[f"even 1.1 n{n}"] = _line(5.0 + 1.1 * np.arange(n), n + 1)
        if n >= 9:
            for name, s in spacing.profiles(n, seed=n).items():
                out[f"{name} n{n}"] = _line(s, n + 2)
            first = _line(spacing.dynamic_s(n, spacing.sine_kappa(0.12, 25.0)), n + 3)
            out[f"chord n{n}"] = _line(spacing.chord_s(first["x"], first["y"]), n + 4)
    return out


def refused_lines():
    """name -> (state array, whether pqp_spline_fit accepts its s) of every line pqp_fit_splines_device refuses.
    pqp_spline_fit tests only that every interval is positive, so it accepts an infinite first or last knot."""
    out = {}
    base = _line(0.3 * np.arange(3))
    for n in (0, 1, 2):
        out[f"n{n}"] = (base[:n].copy(), False)
    for n in (3, 12, 60):
        good = _line(0.25 * np.arange(n) + 0.05 * np.sin(np.arange(n)), 50 + n)
        for kind in spacing.DEGENERATE:
            r = good.copy()
            try:
                r["s"] = spacing.degenerate(good["s"], kind)
            except IndexError:      # the kind needs more stations than n
                continue
            t = r["s"]
            end_inf = np.isinf(t[0]) or np.isinf(t[-1])
            host_accepts = bool(end_inf and np.isfinite(t[1:-1]).all() and (np.diff(t) > 0).all())
            out[f"{kind} n{n}"] = (r, host_accepts)
    return out
