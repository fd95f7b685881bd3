"""Host-side mirror of the stages either side of the QP, on top of include/pqp_env.h.

Reference interfaces being mirrored:
  Map(grid_map) / getObstacleDistance                    src/tools/Map.cpp:8-22
  ReferencePath::updateBounds(map)                       src/data_struct/reference_path.cpp:77-79
  CollisionChecker::isSingleStateCollisionFreeImproved   src/tools/collision_checker.cpp:41-59
  PathOptimizer::optimizePath tails                      src/path_optimizer/path_optimizer.cpp:191-230
  PathOptimizer::solveWithoutSmoothing                   src/path_optimizer/path_optimizer.cpp:87-117
  tk::spline set_points / operator() / deriv             src/tools/spline.cpp:161-318

All numerics run in libpqp.so's sm_90a kernels (spline_fit / spline_eval are host helpers of the
same library); this module only marshals buffers.
"""
import ctypes as C

import numpy as np

from . import _lib
from .abi import (BOUNDS_DTYPE, FORMULATIONS, OK, SOLVED, STATE_DTYPE, DistanceMap, Stats, ptr)
from .solver import BatchPathSolver, PqpError

BOUNDS_IMPROVED, BOUNDS_SIMPLE = 0, 1
OUTPUT_RAW, OUTPUT_DENSIFY = 0, 1


def update_limits(params, ref, from_spline=False):
    """ReferencePathImpl::updateLimits (reference_path_impl.cpp:203-235): (max_k, max_kp) of the KPC formulation from the
    v, a fields of the reference states.  Host helper of libpqp.so."""
    ref = np.ascontiguousarray(ref, dtype=STATE_DTYPE)
    mk, mkp = np.zeros(len(ref)), np.zeros(len(ref))
    rc = _lib.load().pqp_update_limits(C.byref(params), int(bool(from_spline)), len(ref), ptr(ref), ptr(mk), ptr(mkp))
    if rc != OK:
        raise PqpError(f"pqp_update_limits failed (rc={rc}): {_lib.last_error()}")
    return mk, mkp


def spline_fit(t, y):
    """Natural cubic spline coefficients [n, 4] = (a, b, c, y) per knot (tk::spline layout)."""
    t = np.ascontiguousarray(t, dtype=np.float64)
    y = np.ascontiguousarray(y, dtype=np.float64)
    coef = np.zeros((len(t), 4))
    rc = _lib.load().pqp_spline_fit(len(t), ptr(t), ptr(y), ptr(coef))
    if rc != OK:
        raise PqpError(f"pqp_spline_fit failed (rc={rc}): {_lib.last_error()}")
    return coef


def spline_eval(t, coef, at, order=0):
    t = np.ascontiguousarray(t, dtype=np.float64)
    coef = np.ascontiguousarray(coef, dtype=np.float64)
    L = _lib.load()
    return np.array([L.pqp_spline_eval(len(t), ptr(t), ptr(coef), int(order), float(a)) for a in np.atleast_1d(at)])


def reference_splines(batch):
    """x(s), y(s) natural splines through the stations of every path of a batch: the x_s_/y_s_ pair
    updateBoundsImproved projects onto.  Returns dict(n_knots, knots, x_coef, y_coef)."""
    off = batch["offsets"]
    knots, xc, yc = [], [], []
    for b in range(len(batch["n_points"])):
        r = batch["ref"][off[b]:off[b + 1]]
        knots.append(np.array(r["s"]))
        xc.append(spline_fit(r["s"], r["x"]))
        yc.append(spline_fit(r["s"], r["y"]))
    return dict(n_knots=np.ascontiguousarray(batch["n_points"], dtype=np.int32),
                knots=np.concatenate(knots), x_coef=np.concatenate(xc), y_coef=np.concatenate(yc))


class PathPlanner(BatchPathSolver):
    """BatchPathSolver + map-based stages: bounds generation, collision check, output tails and
    the chained planner iteration."""

    def set_map(self, m):
        """m: dict(distance float32 [rows, cols], resolution, center_x, center_y)."""
        dist = np.ascontiguousarray(m["distance"], dtype=np.float32)
        dm = DistanceMap(ptr(dist), dist.shape[0], dist.shape[1], float(m["resolution"]),
                         float(m["center_x"]), float(m["center_y"]))
        rc = self._L.pqp_set_map(self._h, C.byref(dm))
        if rc != OK:
            raise PqpError(f"pqp_set_map failed (rc={rc}): {_lib.last_error()}")

    def set_maps(self, maps):
        """Replace the map set with several maps (pqp_set_maps), each a dict in the form set_map takes; plan() and
        plan_device() pick a path's map with `map_index`.  The single-stage calls and plan() without an index use
        map 0."""
        maps = list(maps)
        dists = [np.ascontiguousarray(m["distance"], dtype=np.float32) for m in maps]
        dms = (DistanceMap * max(len(maps), 1))()
        for i, (m, d) in enumerate(zip(maps, dists)):
            dms[i] = DistanceMap(ptr(d), d.shape[0], d.shape[1], float(m["resolution"]), float(m["center_x"]),
                                 float(m["center_y"]))
        rc = self._L.pqp_set_maps(self._h, len(maps), dms)
        if rc != OK:
            raise PqpError(f"pqp_set_maps failed (rc={rc}): {_lib.last_error()}")

    def map_distance(self, xy):
        xy = np.ascontiguousarray(xy, dtype=np.float64).reshape(-1, 2)
        out = np.zeros(len(xy))
        rc = self._L.pqp_map_distance(self._h, len(xy), ptr(xy), ptr(out))
        if rc != OK:
            raise PqpError(f"pqp_map_distance failed (rc={rc}): {_lib.last_error()}")
        return out

    @staticmethod
    def _spl(splines):
        if splines is None:
            return None, None, None, None
        return (np.ascontiguousarray(splines["n_knots"], dtype=np.int32),
                np.ascontiguousarray(splines["knots"], dtype=np.float64),
                np.ascontiguousarray(splines["x_coef"], dtype=np.float64),
                np.ascontiguousarray(splines["y_coef"], dtype=np.float64))

    def update_bounds(self, batch, mode=BOUNDS_SIMPLE, splines=None):
        """ReferencePath::updateBounds for every path.  Returns dict(bounds, n_valid, stats)."""
        n_points = np.ascontiguousarray(batch["n_points"], dtype=np.int32)
        ref = np.ascontiguousarray(batch["ref"], dtype=STATE_DTYPE)
        nk, kn, xc, yc = self._spl(splines)
        bounds = np.zeros(len(ref), dtype=BOUNDS_DTYPE)
        n_valid = np.zeros(len(n_points), dtype=np.int32)
        stats = Stats()
        rc = self._L.pqp_update_bounds_batch(self._h, int(mode), len(n_points), ptr(n_points), ptr(ref), ptr(nk),
                                             ptr(kn), ptr(xc), ptr(yc), ptr(bounds), ptr(n_valid), C.byref(stats))
        if rc != OK:
            raise PqpError(f"pqp_update_bounds_batch failed (rc={rc}): {_lib.last_error()}")
        return dict(bounds=bounds, n_valid=n_valid, stats=stats)

    def check_states(self, states):
        states = np.ascontiguousarray(states, dtype=STATE_DTYPE)
        ok = np.zeros(len(states), dtype=np.int32)
        rc = self._L.pqp_check_states(self._h, len(states), ptr(states), ptr(ok))
        if rc != OK:
            raise PqpError(f"pqp_check_states failed (rc={rc}): {_lib.last_error()}")
        return ok

    def finish_raw(self, n_points, paths, collision_check=True):
        n_points = np.ascontiguousarray(n_points, dtype=np.int32)
        paths = np.array(paths, dtype=STATE_DTYPE)
        n_kept = np.zeros(len(n_points), dtype=np.int32)
        ok = np.zeros(len(n_points), dtype=np.int32)
        stats = Stats()
        rc = self._L.pqp_finish_raw_batch(self._h, len(n_points), ptr(n_points), ptr(paths), int(collision_check),
                                          ptr(n_kept), ptr(ok), C.byref(stats))
        if rc != OK:
            raise PqpError(f"pqp_finish_raw_batch failed (rc={rc}): {_lib.last_error()}")
        return dict(states=paths, n_kept=n_kept, ok=ok, stats=stats)

    def densify(self, n_points, paths, output_spacing=0.3, collision_check=True, max_out=512):
        n_points = np.ascontiguousarray(n_points, dtype=np.int32)
        paths = np.ascontiguousarray(paths, dtype=STATE_DTYPE)
        B = len(n_points)
        out = np.zeros((B, max_out), dtype=STATE_DTYPE)
        n_out = np.zeros(B, dtype=np.int32)
        ok = np.zeros(B, dtype=np.int32)
        stats = Stats()
        rc = self._L.pqp_densify_batch(self._h, B, ptr(n_points), ptr(paths), float(output_spacing),
                                       int(collision_check), int(max_out), ptr(out), ptr(n_out), ptr(ok), C.byref(stats))
        if rc != OK:
            raise PqpError(f"pqp_densify_batch failed (rc={rc}): {_lib.last_error()}")
        return dict(states=out, n_out=n_out, ok=ok, stats=stats)

    def plan(self, batch, formulation="KP", bounds_mode=BOUNDS_SIMPLE, splines=None, output_mode=OUTPUT_RAW,
             output_spacing=0.3, collision_check=True, max_out=512, want_bounds=False, out=None, map_index=None):
        """PathOptimizer::solveWithoutSmoothing for every path of the batch (bounds -> QP -> tail).
        `out` may carry a preallocated (e.g. pinned) `states` array of the output shape.  `map_index`: int32 [B], the
        map of the set (set_maps) every path is planned on (pqp_plan_batch_maps); None: map 0 (pqp_plan_batch).  A path
        whose index is outside the set reports status -100 (invalid problem), 0 iterations, n_out = 0 and ok = 0."""
        form = FORMULATIONS[formulation] if isinstance(formulation, str) else int(formulation)
        n_points = np.ascontiguousarray(batch["n_points"], dtype=np.int32)
        B = len(n_points)
        ref = np.ascontiguousarray(batch["ref"], dtype=STATE_DTYPE)
        x0 = np.ascontiguousarray(batch["x0"], dtype=np.float64)
        end_heading = np.ascontiguousarray(batch["end_heading"], dtype=np.float64)
        nk, kn, xc, yc = self._spl(splines)
        shape = (len(ref),) if output_mode == OUTPUT_RAW else (B, max_out)
        if out is not None and "states" in out:
            states = out["states"]
            assert states.dtype == STATE_DTYPE and states.shape == shape and states.flags["C_CONTIGUOUS"]
        else:
            states = np.zeros(shape, dtype=STATE_DTYPE)
        n_out = np.zeros(B, dtype=np.int32)
        ok = np.zeros(B, dtype=np.int32)
        status = np.zeros(B, dtype=np.int32)
        iters = np.zeros(B, dtype=np.int32)
        bounds = np.zeros(len(ref), dtype=BOUNDS_DTYPE) if want_bounds else None
        stats = Stats()
        head = (self._h, form, int(bounds_mode), int(output_mode), B, ptr(n_points), ptr(ref))
        tail = (ptr(nk), ptr(kn), ptr(xc), ptr(yc), ptr(x0), ptr(end_heading), float(output_spacing),
                int(collision_check), int(max_out), ptr(states), ptr(n_out), ptr(ok), ptr(status), ptr(iters),
                ptr(bounds), C.byref(stats))
        if map_index is None:
            name, rc = "pqp_plan_batch", self._L.pqp_plan_batch(*head, *tail)
        else:
            mi = np.asarray(map_index)
            if mi.shape != (B,) or mi.dtype.kind not in "iu":
                raise ValueError(f"map_index: expected an integer array of shape ({B},), got {mi.dtype} {mi.shape}")
            mi = np.ascontiguousarray(mi, dtype=np.int32)
            name, rc = "pqp_plan_batch_maps", self._L.pqp_plan_batch_maps(*head, ptr(mi), *tail)
        if rc != OK:
            raise PqpError(f"{name} failed (rc={rc}): {_lib.last_error()}")
        return dict(states=states, n_out=n_out, ok=ok, status=status, iters=iters, bounds=bounds,
                    solved=(status == SOLVED), stats=stats)

    def plan_device(self, n_points, offsets, ref, x0, end_heading, max_n_points=0, formulation="KP",
                    bounds_mode=BOUNDS_SIMPLE, splines=None, output_mode=OUTPUT_RAW, output_spacing=0.3,
                    collision_check=True, max_out=512, want_bounds=False, out=None, stats=False, map_index=None):
        """plan() on torch CUDA tensors of the planner's device (path_optimizer_b200.device): n_points int32 [B],
        offsets int32 [B + 1], ref float64 [T, 7], x0 float64 [B, 3], end_heading float64 [B]; `splines` (IMPROVED)
        a dict of knot_offsets int32 [B + 1], knots [K], x_coef / y_coef [K, 4] (device.splines_to_device).  The whole
        chain runs on the device (pqp_plan_batch_device) on torch.cuda.current_stream() with plan()'s results bit for
        bit and no host synchronisation (unless `stats`): after one warm-up call it can be captured in a CUDA graph.
        max_n_points >= every n_points (0: the longest path any kernel class takes).  `out` may carry the output
        tensors (states: [T, 7] RAW or [B, max_out, 7] DENSIFY; n_out, ok, status, iters; bounds [T, 8]).
        `map_index`: int32 [B] on the device, the map of the set every path is planned on (pqp_plan_batch_device_maps,
        as plan(map_index=...)); None: map 0.  A graph replay reads the index from the captured tensor."""
        import torch
        from . import device as D
        form = FORMULATIONS[formulation] if isinstance(formulation, str) else int(formulation)
        dev = self._cuda_device()
        B, T = int(n_points.shape[0]), int(ref.shape[0])
        f64, i32 = torch.float64, torch.int32
        out = dict(out or {})
        shape = (T, D.STATE_COLS) if output_mode == OUTPUT_RAW else (B, int(max_out), D.STATE_COLS)

        def buf(name, shp, dtype):
            return out[name] if out.get(name) is not None else torch.empty(shp, dtype=dtype, device=dev)
        states = buf("states", shape, f64)
        n_out, ok, status, iters = buf("n_out", (B,), i32), buf("ok", (B,), i32), buf("status", (B,), i32), buf("iters", (B,), i32)
        bounds = buf("bounds", (T, D.BOUNDS_COLS), f64) if want_bounds else None
        spl = splines or {}
        K = int(spl["knots"].shape[0]) if splines is not None else 0
        args = [D.check(n_points, "n_points", i32, (B,), dev), D.check(offsets, "offsets", i32, (B + 1,), dev),
                D.check(ref, "ref", f64, (T, D.STATE_COLS), dev),
                D.check(spl.get("knot_offsets"), "knot_offsets", i32, (B + 1,), dev),
                D.check(spl.get("knots"), "knots", f64, (K,), dev), D.check(spl.get("x_coef"), "x_coef", f64, (K, 4), dev),
                D.check(spl.get("y_coef"), "y_coef", f64, (K, 4), dev),
                D.check(x0, "x0", f64, (B, 3), dev), D.check(end_heading, "end_heading", f64, (B,), dev)]
        outs = [D.check(states, "states", f64, shape, dev), D.check(n_out, "n_out", i32, (B,), dev),
                D.check(ok, "ok", i32, (B,), dev), D.check(status, "status", i32, (B,), dev),
                D.check(iters, "iters", i32, (B,), dev), D.check(bounds, "bounds", f64, (T, D.BOUNDS_COLS), dev)]
        st = Stats()
        head = (self._h, form, int(bounds_mode), int(output_mode), B, T, int(max_n_points))
        tail = (float(output_spacing), int(collision_check), int(max_out), *outs,
                torch.cuda.current_stream(dev).cuda_stream, C.byref(st) if stats else None)
        if map_index is None:
            name, rc = "pqp_plan_batch_device", self._L.pqp_plan_batch_device(*head, *args, *tail)
        else:
            mi = D.check(map_index, "map_index", i32, (B,), dev)
            name, rc = "pqp_plan_batch_device_maps", self._L.pqp_plan_batch_device_maps(*head, *args[:3], mi, *args[3:],
                                                                                        *tail)
        if rc != OK:
            raise PqpError(f"{name} failed (rc={rc}): {_lib.last_error()}")
        return dict(states=states, n_out=n_out, ok=ok, status=status, iters=iters, bounds=bounds,
                    stats=st if stats else None)
