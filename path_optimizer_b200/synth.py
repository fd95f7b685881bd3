"""Synthetic corridor batches for the BASELINE.json configs (SURVEY.md section 8d).

Counter-based RNG (splitmix64 of a key built from seed/config/path/field/point) so that any shard
of any batch can be regenerated independently on any rank.  Pure numpy; no CUDA, no oracle.

A batch is a dict:
  n_points  int32 [B]            stations per path
  offsets   int32 [B+1]          exclusive prefix sum
  ref       STATE_DTYPE [sum N]  reference states (x, y, z=heading, k, s)
  bounds    BOUNDS_DTYPE [sum N] clearance bounds of the four covering circles
  x0        float64 [B,3]        (init offset, init heading error, start curvature)
  end_heading float64 [B]        goal heading (VehicleState end state z)
"""
import numpy as np

from .abi import BOUNDS_DTYPE, STATE_DTYPE

BASE_SEED = 20260923
_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def splitmix64(x):
    """splitmix64 finaliser on a uint64 array (wrap-around arithmetic)."""
    x = np.asarray(x, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = x + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return z


def uniform(seed, config, path_id, field, point=0):
    """U[0,1) doubles; arguments broadcast like numpy arrays."""
    key = (np.uint64(seed)
           ^ (np.asarray(config, dtype=np.uint64) << np.uint64(56))
           ^ (np.asarray(path_id, dtype=np.uint64) << np.uint64(24))
           ^ (np.asarray(field, dtype=np.uint64) << np.uint64(16))
           ^ np.asarray(point, dtype=np.uint64))
    return (splitmix64(key) >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)


def _accumulate_s(n, ds=0.3):
    """s_i accumulated in double by += ds, as a resampler would produce them (this is what makes
    keep_control_steps_ = int(1.2/0.3000..4) = 3, SURVEY.md section 7)."""
    s = np.empty(n, dtype=np.float64)
    acc = 0.0
    for i in range(n):
        s[i] = acc
        acc += ds
    return s


def _pack(n_points, ref, bounds, x0, end_heading):
    n_points = np.ascontiguousarray(n_points, dtype=np.int32)
    offsets = np.zeros(len(n_points) + 1, dtype=np.int32)
    np.cumsum(n_points, out=offsets[1:])
    return dict(n_points=n_points, offsets=offsets, ref=np.ascontiguousarray(ref),
                bounds=np.ascontiguousarray(bounds), x0=np.ascontiguousarray(x0, dtype=np.float64),
                end_heading=np.ascontiguousarray(end_heading, dtype=np.float64))


def straight_corridors(batch, n=100, seed=BASE_SEED, first_path=0, config=2, wide_fraction=0.0):
    """BASELINE config 2 / 4: straight reference, constant symmetric corridor per path.

    ref[i] = (s_i, 0, 0, 0, s_i); half clearance w ~ U(0.5, 1.2) quantised down to 0.1 m (the
    reference's ray-march resolution, reference_path_impl.cpp:288,444); all four circles
    (lb, ub) = (-w, +w); x0 = (U(-0.3,0.3), U(-0.05,0.05), 0); goal heading 0.
    `wide_fraction` > 0 marks that share of paths as wide (w ~ U(1.5, 3)): ill-conditioned regime.
    """
    pid = np.arange(first_path, first_path + batch, dtype=np.uint64)
    s = _accumulate_s(n)
    ref = np.zeros((batch, n), dtype=STATE_DTYPE)
    ref["x"] = s[None, :]
    ref["s"] = s[None, :]
    w = 0.5 + 0.7 * uniform(seed, config, pid, 1)
    if wide_fraction > 0:
        wide = uniform(seed, config, pid, 5) < wide_fraction
        w = np.where(wide, 1.5 + 1.5 * uniform(seed, config, pid, 6), w)
    w = np.floor(w * 10.0 + 1e-9) / 10.0
    bounds = np.zeros((batch, n), dtype=BOUNDS_DTYPE)
    for c in range(4):
        bounds[f"c{c}_ub"] = w[:, None]
        bounds[f"c{c}_lb"] = -w[:, None]
    x0 = np.zeros((batch, 3))
    x0[:, 0] = -0.3 + 0.6 * uniform(seed, config, pid, 2)
    x0[:, 1] = -0.05 + 0.1 * uniform(seed, config, pid, 3)
    end_heading = np.zeros(batch)
    return _pack(np.full(batch, n), ref.reshape(-1), bounds.reshape(-1), x0, end_heading)


def curvy_corridors(batch, n=100, seed=BASE_SEED, first_path=0, config=3, n_points=None, path_ids=None):
    """Analytic curved corridors (config 5 / "config 3-lite"): kappa_ref(s) = A sin(2 pi s / L),
    A ~ U(0, 0.05), L ~ U(30, 80) m integrated to (x, y, heading); corridor centre follows a smooth
    lateral wave c(s) of amplitude U(0, 0.6) m, half widths per circle U(0.6, 1.6) quantised to
    0.1 m, so bounds differ per station and per circle (some above the 1.3 m soft margin).
    `n_points` (int array [batch]) gives mixed lengths; otherwise every path has n stations.  `path_ids` (int array
    [batch]) names the global ids of the paths to generate (a rank's shard of a work-balanced split); default
    first_path .. first_path + batch - 1."""
    if n_points is None:
        n_points = np.full(batch, n, dtype=np.int32)
    n_points = np.asarray(n_points, dtype=np.int32)
    total = int(n_points.sum())
    ref = np.zeros(total, dtype=STATE_DTYPE)
    bounds = np.zeros(total, dtype=BOUNDS_DTYPE)
    x0 = np.zeros((batch, 3))
    end_heading = np.zeros(batch)
    off = 0
    for b in range(batch):
        nb = int(n_points[b])
        pid = np.uint64(first_path + b if path_ids is None else int(path_ids[b]))
        s = _accumulate_s(nb)
        A = 0.05 * uniform(seed, config, pid, 1)
        L = 30.0 + 50.0 * uniform(seed, config, pid, 2)
        k = A * np.sin(2 * np.pi * s / L)
        theta = np.concatenate([[0.0], np.cumsum(0.5 * (k[1:] + k[:-1]) * np.diff(s))])
        x = np.concatenate([[0.0], np.cumsum(np.cos(0.5 * (theta[1:] + theta[:-1])) * np.diff(s))])
        y = np.concatenate([[0.0], np.cumsum(np.sin(0.5 * (theta[1:] + theta[:-1])) * np.diff(s))])
        r = ref[off:off + nb]
        r["x"], r["y"], r["z"], r["k"], r["s"] = x, y, theta, k, s
        amp = 0.6 * uniform(seed, config, pid, 3)
        lam = 20.0 + 40.0 * uniform(seed, config, pid, 4)
        ph = 2 * np.pi * uniform(seed, config, pid, 5)
        centre = amp * (np.sin(2 * np.pi * s / lam + ph) - np.sin(ph)) * np.minimum(s / 6.0, 1.0)
        bb = bounds[off:off + nb]
        for c in range(4):
            hw = 0.6 + 1.0 * uniform(seed, config, pid, 8 + c, np.arange(nb, dtype=np.uint64) // np.uint64(10))
            hw = np.floor(hw * 10.0 + 1e-9) / 10.0
            bb[f"c{c}_ub"] = np.round(centre + hw, 1)
            bb[f"c{c}_lb"] = np.round(centre - hw, 1)
        x0[b, 0] = -0.2 + 0.4 * uniform(seed, config, pid, 6)
        x0[b, 1] = -0.04 + 0.08 * uniform(seed, config, pid, 7)
        x0[b, 2] = k[0]
        end_heading[b] = theta[-1]
        off += nb
    return _pack(n_points, ref, bounds, x0, end_heading)


def mixed_lengths(batch, lo=50, hi=400, seed=BASE_SEED, first_path=0, config=5):
    """BASELINE config 5 station counts: N ~ U{lo..hi} per global path id."""
    pid = np.arange(first_path, first_path + batch, dtype=np.uint64)
    return (lo + np.floor((hi - lo + 1) * uniform(seed, config, pid, 30))).astype(np.int32)


def take_paths(batch, idx):
    """Paths `idx` (index array) of a batch as a new batch (copies)."""
    o = batch["offsets"]
    idx = np.asarray(idx, dtype=np.int64)
    sel = np.concatenate([np.arange(o[i], o[i + 1]) for i in idx]) if len(idx) else np.zeros(0, dtype=np.int64)
    out = dict(n_points=batch["n_points"][idx].copy(), ref=batch["ref"][sel].copy(), bounds=batch["bounds"][sel].copy(),
               x0=batch["x0"][idx].copy(), end_heading=batch["end_heading"][idx].copy())
    offsets = np.zeros(len(idx) + 1, dtype=np.int32)
    np.cumsum(out["n_points"], out=offsets[1:])
    out["offsets"] = offsets
    return out


def slice_batch(batch, begin, end):
    """Paths [begin, end) of a batch as a new batch (views where possible)."""
    o = batch["offsets"]
    lo, hi = int(o[begin]), int(o[end])
    out = dict(n_points=batch["n_points"][begin:end].copy(),
               ref=batch["ref"][lo:hi], bounds=batch["bounds"][lo:hi],
               x0=batch["x0"][begin:end], end_heading=batch["end_heading"][begin:end])
    offsets = np.zeros(end - begin + 1, dtype=np.int32)
    np.cumsum(out["n_points"], out=offsets[1:])
    out["offsets"] = offsets
    return out


# ---------------------------------------------------------------------------------------------
# Config 3: obstacle field + distance map (the input of the clearance-bounds stage)
# ---------------------------------------------------------------------------------------------

def disc_field_map(rows=1100, cols=250, resolution=0.2, n_discs=300, seed=BASE_SEED, config=3,
                   center=(0.0, 0.0), keep_clear_halfwidth=1.7):
    """Synthetic 0.2 m occupancy grid with random discs (radius U(0.5, 2) m) and its Euclidean
    distance transform in metres -- what the reference builds with cv::distanceTransform(L2,
    MASK_PRECISE) * resolution (path_optimizer_benchmark.cpp:39-43).  Discs whose edge would come
    within `keep_clear_halfwidth` of the map's x axis are pushed out so that a corridor exists.
    grid_map index convention: cell (i, j) centred at x = cx + L_x/2 - (i+0.5) res,
    y = cy + L_y/2 - (j+0.5) res.  Returns dict(distance float32 [rows, cols], rows, cols,
    resolution, center_x, center_y)."""
    from scipy import ndimage
    lx, ly = rows * resolution, cols * resolution
    xs = center[0] + lx / 2 - (np.arange(rows) + 0.5) * resolution
    ys = center[1] + ly / 2 - (np.arange(cols) + 0.5) * resolution
    free = np.ones((rows, cols), dtype=bool)
    idx = np.arange(n_discs, dtype=np.uint64)
    cx = center[0] - lx / 2 + lx * uniform(seed, config, 0xFFFFF0, 1, idx)
    cy = center[1] - ly / 2 + ly * uniform(seed, config, 0xFFFFF0, 2, idx)
    rad = 0.5 + 1.5 * uniform(seed, config, 0xFFFFF0, 3, idx)
    for k in range(n_discs):
        y0 = cy[k]
        gap = abs(y0 - center[1]) - rad[k]
        if gap < keep_clear_halfwidth:
            y0 = center[1] + np.sign(y0 - center[1] if y0 != center[1] else 1.0) * (keep_clear_halfwidth + rad[k])
        free &= ((xs[:, None] - cx[k]) ** 2 + (ys[None, :] - y0) ** 2) > rad[k] ** 2
    dist = ndimage.distance_transform_edt(free).astype(np.float32) * np.float32(resolution)
    return dict(distance=np.ascontiguousarray(dist), rows=rows, cols=cols, resolution=float(resolution),
                center_x=float(center[0]), center_y=float(center[1]))


def map_reference_paths(batch, n=200, seed=BASE_SEED, first_path=0, config=3, n_points=None,
                        x_range=(-100.0, 40.0), y_range=(-0.5, 0.5), heading_range=0.02, curvature_amp=0.004):
    """Reference lines for config 3: kappa_ref(s) = A sin(2 pi s / L), A ~ U(0, curvature_amp), L ~ U(30, 80) m,
    integrated to (x, y, heading) from a random start pose near the map's x axis.  No bounds: those
    come from the clearance stage.  x0 = (0, 0, k_0) as solveWithoutSmoothing sets it
    (path_optimizer.cpp:97); end heading = heading of the last station."""
    if n_points is None:
        n_points = np.full(batch, n, dtype=np.int32)
    n_points = np.asarray(n_points, dtype=np.int32)
    total = int(n_points.sum())
    ref = np.zeros(total, dtype=STATE_DTYPE)
    x0 = np.zeros((batch, 3))
    end_heading = np.zeros(batch)
    off = 0
    for b in range(batch):
        nb = int(n_points[b])
        pid = np.uint64(first_path + b)
        s = _accumulate_s(nb)
        A = curvature_amp * uniform(seed, config, pid, 1)
        L = 30.0 + 50.0 * uniform(seed, config, pid, 2)
        k = A * np.sin(2 * np.pi * s / L)
        th0 = heading_range * (2 * uniform(seed, config, pid, 20) - 1)
        theta = th0 + np.concatenate([[0.0], np.cumsum(0.5 * (k[1:] + k[:-1]) * np.diff(s))])
        xs = x_range[0] + (x_range[1] - x_range[0]) * uniform(seed, config, pid, 21)
        ys = y_range[0] + (y_range[1] - y_range[0]) * uniform(seed, config, pid, 22)
        x = xs + np.concatenate([[0.0], np.cumsum(np.cos(0.5 * (theta[1:] + theta[:-1])) * np.diff(s))])
        y = ys + np.concatenate([[0.0], np.cumsum(np.sin(0.5 * (theta[1:] + theta[:-1])) * np.diff(s))])
        r = ref[off:off + nb]
        r["x"], r["y"], r["z"], r["k"], r["s"] = x, y, theta, k, s
        x0[b, 2] = k[0]
        end_heading[b] = theta[-1]
        off += nb
    out = _pack(n_points, ref, np.zeros(total, dtype=BOUNDS_DTYPE), x0, end_heading)
    return out


def infeasible_corridors(batch, n=60, seed=BASE_SEED, first_path=0, config=6):
    """Corridors no path can satisfy (the reference logs "QP failed", path_optimizer.cpp:184): the
    vehicle starts ON the reference line (x0 offset 0 is an equality row) but from some station on
    the hard rows of circles 0 and 2 demand a lateral offset the dynamics cannot reach, or demand
    two incompatible offsets at once.  Every second path stays feasible as a control."""
    b = curvy_corridors(batch, n, seed=seed, first_path=first_path, config=config)
    off = b["offsets"]
    for p in range(batch):
        if p % 2 == 1:
            continue
        lo, hi = off[p], off[p + 1]
        kind = (p // 2) % 3
        bb = b["bounds"][lo:hi]
        if kind == 0:       # offset >= 0.6 m demanded from station 0 while e_y(0) = x0
            bb["c0_lb"], bb["c0_ub"] = 0.6, 1.5
            bb["c2_lb"], bb["c2_ub"] = 0.6, 1.5
            b["x0"][p, 0] = 0.0
        elif kind == 1:     # a 3 m jump between stations 1 and 2 (ds = 0.3 m, |kappa| bounded)
            bb["c0_lb"][2:], bb["c0_ub"][2:] = 3.0, 4.0
            bb["c2_lb"][2:], bb["c2_ub"][2:] = 3.0, 4.0
        else:               # rear circle pushed left, front circle pushed right by more than the wheelbase allows
            bb["c0_lb"][10:], bb["c0_ub"][10:] = 2.0, 2.5
            bb["c2_lb"][10:], bb["c2_ub"][10:] = -2.5, -2.0
    return b


# ---------------------------------------------------------------------------------------------
# Many scenes in one batch (pqp_set_maps + a map index per path)
# ---------------------------------------------------------------------------------------------

def scene_map(k, seed=BASE_SEED):
    """Scene k of a many-scene batch: disc_field_map with its own seed.  Every fourth scene (k % 4 == 1) has a 0.25 m
    resolution and a centre away from the origin, so that a set mixes map geometries."""
    if k % 4 == 1:
        return disc_field_map(resolution=0.25, seed=seed + k, center=(35.0 + 10.0 * (k % 7), -20.0 + 3.0 * (k % 5)))
    return disc_field_map(seed=seed + k)


def multi_map_batch(n_maps, n_candidates, n=200, seed=BASE_SEED, first_maps=(), order="grouped", mapper=map, **line_kw):
    """A batch planned over several maps: `first_maps` (e.g. the config-1 fixture map) followed by scene_map(k) for the
    remaining scenes up to `n_maps`, and `n_candidates` reference lines of `n` stations per map, placed in that map's
    frame (map_reference_paths shifted to the map's centre, starting 5 m inside its -x edge or at x = -100 m from the
    centre, whichever is further in).  `order`: "grouped" (the paths of map 0, then map 1, ...) or "interleaved" (one
    path of every map in turn).  `mapper` builds the generated maps (e.g. a process pool's map).
    Returns (maps, batch, map_index int32 [n_maps * n_candidates])."""
    first_maps = list(first_maps)
    maps = first_maps + list(mapper(scene_map, range(len(first_maps), n_maps), [seed] * (n_maps - len(first_maps))))
    parts = []
    for m, mp in enumerate(maps):
        lx = mp["rows"] * mp["resolution"]
        x_lo = max(-lx / 2 + 5.0, -100.0)
        x_hi = max(x_lo, min(40.0, lx / 2 - 5.0 - 0.3 * n))
        kw = dict(x_range=(mp["center_x"] + x_lo, mp["center_x"] + x_hi), y_range=(-0.5, 0.5))
        kw.update(line_kw)
        kw["y_range"] = (mp["center_y"] + kw["y_range"][0], mp["center_y"] + kw["y_range"][1])
        parts.append(map_reference_paths(n_candidates, n, seed=seed, first_path=m * n_candidates, **kw))
    b = dict(n_points=np.concatenate([p["n_points"] for p in parts]), ref=np.concatenate([p["ref"] for p in parts]),
             bounds=np.concatenate([p["bounds"] for p in parts]), x0=np.concatenate([p["x0"] for p in parts]),
             end_heading=np.concatenate([p["end_heading"] for p in parts]))
    b["offsets"] = np.concatenate([[0], np.cumsum(b["n_points"])]).astype(np.int32)
    map_index = np.repeat(np.arange(n_maps, dtype=np.int32), n_candidates)
    if order == "interleaved":
        perm = np.arange(n_maps * n_candidates).reshape(n_maps, n_candidates).T.reshape(-1)
        b, map_index = take_paths(b, perm), map_index[perm]
    elif order != "grouped":
        raise ValueError(f"order: 'grouped' or 'interleaved', got {order!r}")
    return maps, b, np.ascontiguousarray(map_index, dtype=np.int32)
