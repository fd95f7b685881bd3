"""Host-side mirror of the stages either side of the QP, on top of include/pqp_env.h.

Reference interfaces being mirrored:
  Map(grid_map) / getObstacleDistance                    src/tools/Map.cpp:8-22
  ReferencePath::updateBounds(map)                       src/data_struct/reference_path.cpp:77-79
  CollisionChecker::isSingleStateCollisionFreeImproved   src/tools/collision_checker.cpp:41-59
  PathOptimizer::optimizePath tails                      src/path_optimizer/path_optimizer.cpp:191-230
  PathOptimizer::solveWithoutSmoothing                   src/path_optimizer/path_optimizer.cpp:87-117
  PathOptimizer::segmentSmoothedPath                     src/path_optimizer/path_optimizer.cpp:119-178
  tk::spline set_points / operator() / deriv             src/tools/spline.cpp:161-318

All numerics run in libpqp.so's sm_90a kernels (spline_fit / spline_eval are host helpers of the
same library); this module only marshals buffers.
"""
import ctypes as C

import numpy as np

from . import _lib
from .abi import (BOUNDS_DTYPE, FORMULATIONS, OK, SOLVED, STATE_DTYPE, DistanceMap, OccupancyMap, Stats, ptr)
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
        self._map_shapes = [dist.shape]

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
        self._map_shapes = [d.shape for d in dists]

    @staticmethod
    def _occupancy_descriptors(maps, cells):
        oms = (OccupancyMap * max(len(maps), 1))()
        for i, (m, (p, rows, cols)) in enumerate(zip(maps, cells)):
            oms[i] = OccupancyMap(p, rows, cols, float(m["resolution"]), float(m["center_x"]), float(m["center_y"]))
        return oms

    def set_maps_occupancy(self, maps):
        """Replace the map set with layers the device builds from occupancy grids (pqp_set_maps_occupancy): each map a
        dict of `occupancy` uint8 [rows, cols] (0 = obstacle, anything else free), resolution, center_x, center_y.  A
        layer is the exact Euclidean distance transform in metres, bit for bit
        ndimage.distance_transform_edt(occupancy != 0).astype(float32) * float32(resolution) (synth.distance_layer)."""
        maps = list(maps)
        occ = [np.ascontiguousarray(m["occupancy"], dtype=np.uint8) for m in maps]
        if any(o.ndim != 2 for o in occ):
            raise ValueError("occupancy: expected uint8 arrays of shape [rows, cols]")
        oms = self._occupancy_descriptors(maps, [(o.ctypes.data, o.shape[0], o.shape[1]) for o in occ])
        rc = self._L.pqp_set_maps_occupancy(self._h, len(maps), oms)
        if rc != OK:
            raise PqpError(f"pqp_set_maps_occupancy failed (rc={rc}): {_lib.last_error()}")
        self._map_shapes = [o.shape for o in occ]

    def set_maps_occupancy_device(self, maps):
        """set_maps_occupancy with `occupancy` as torch uint8 CUDA tensors [rows, cols] on the planner's device
        (pqp_set_maps_occupancy_device), on torch.cuda.current_stream().  With the geometry of the current set (after
        one such call) it only launches the transform and can be captured in a CUDA graph with plan_device; a new layout
        synchronises and is refused while the stream is capturing."""
        import torch
        from . import device as D
        dev = self._cuda_device()
        maps = list(maps)
        cells = []
        for m in maps:
            t = m["occupancy"]
            shape = tuple(t.shape) if isinstance(t, torch.Tensor) else ()
            if len(shape) != 2:
                raise ValueError("occupancy: expected uint8 CUDA tensors of shape [rows, cols]")
            cells.append((D.check(t, "occupancy", torch.uint8, shape, dev), shape[0], shape[1]))
        oms = self._occupancy_descriptors(maps, cells)
        rc = self._L.pqp_set_maps_occupancy_device(self._h, len(maps), oms, torch.cuda.current_stream(dev).cuda_stream)
        if rc != OK:
            raise PqpError(f"pqp_set_maps_occupancy_device failed (rc={rc}): {_lib.last_error()}")
        self._map_shapes = [(rows, cols) for _, rows, cols in cells]

    def get_map(self, m):
        """Layer of map m of the set (pqp_get_map): float32 [rows, cols].  Synchronise the stream of a
        set_maps_occupancy_device call first."""
        shapes = getattr(self, "_map_shapes", [])
        out = np.empty(shapes[m] if 0 <= m < len(shapes) else (0, 0), dtype=np.float32)
        rc = self._L.pqp_get_map(self._h, int(m), ptr(out))
        if rc != OK:
            raise PqpError(f"pqp_get_map failed (rc={rc}): {_lib.last_error()}")
        return out

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
             output_spacing=0.3, collision_check=True, max_out=512, want_bounds=False, out=None, map_index=None,
             param_index=None):
        """PathOptimizer::solveWithoutSmoothing for every path of the batch (bounds -> QP -> tail).
        `out` may carry a preallocated (e.g. pinned) `states` array of the output shape.  `map_index`: int32 [B], the
        map of the set (set_maps) every path is planned on (pqp_plan_batch_maps); None: map 0 (pqp_plan_batch).  A path
        whose index is outside the set reports status -100 (invalid problem), 0 iterations, n_out = 0 and ok = 0.
        `param_index`: int32 [B], the parameter set (set_param_sets) every path is planned with (pqp_plan_batch_sets);
        None: set 0.  An index outside the sets fails its path the same way.
        `formulation`: a name for the whole batch, or one per path (pqp_plan_batch_forms): an int32 array [B] of
        PQP_FORM_* values or a list of names; a value that is not a formulation fails its path the same way."""
        n_points = np.ascontiguousarray(batch["n_points"], dtype=np.int32)
        B = len(n_points)
        forms = self._forms(formulation, B)
        form = 0 if forms is not None else FORMULATIONS[formulation] if isinstance(formulation, str) else int(formulation)
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
        mi = None
        if map_index is not None:
            mi = np.asarray(map_index)
            if mi.shape != (B,) or mi.dtype.kind not in "iu":
                raise ValueError(f"map_index: expected an integer array of shape ({B},), got {mi.dtype} {mi.shape}")
            mi = np.ascontiguousarray(mi, dtype=np.int32)
        if forms is not None:
            pi = None if param_index is None else self._param_index(param_index, B)
            name = "pqp_plan_batch_forms"
            rc = self._L.pqp_plan_batch_forms(self._h, *head[2:], ptr(mi), ptr(pi), ptr(forms), *tail)
        elif param_index is not None:
            pi = self._param_index(param_index, B)
            name, rc = "pqp_plan_batch_sets", self._L.pqp_plan_batch_sets(*head, ptr(mi), ptr(pi), *tail)
        elif map_index is None:
            name, rc = "pqp_plan_batch", self._L.pqp_plan_batch(*head, *tail)
        else:
            name, rc = "pqp_plan_batch_maps", self._L.pqp_plan_batch_maps(*head, ptr(mi), *tail)
        if rc != OK:
            raise PqpError(f"{name} failed (rc={rc}): {_lib.last_error()}")
        return dict(states=states, n_out=n_out, ok=ok, status=status, iters=iters, bounds=bounds,
                    solved=(status == SOLVED), stats=stats)

    def fit_splines_device(self, offsets, ref, out=None):
        """reference_splines() on the device (pqp_fit_splines_device): the x(s), y(s) splines of every path of a batch
        from torch CUDA tensors offsets int32 [B + 1] and ref float64 [T, 7], on torch.cuda.current_stream().  Returns
        dict(knot_offsets, knots [T], x_coef [T, 4], y_coef [T, 4], ok int32 [B]), ready for plan_device(splines=...):
        knot_offsets is `offsets` itself, and the coefficients equal spline_fit's bit for bit.  A path with fewer than 3
        stations or an s that is not finite and strictly increasing gets ok = 0 and NaN knots and rows; fail it in
        plan_device with map_index = torch.where(ok != 0, map_index, -1).  No host synchronisation; after one warm-up
        call on the planner it can be captured in a CUDA graph.  `out` may carry the output tensors (knots, x_coef,
        y_coef, ok), e.g. those of an earlier call, so that a captured graph writes where the plan reads."""
        import torch
        from . import device as D
        dev = self._cuda_device()
        B, T = int(offsets.shape[0]) - 1, int(ref.shape[0])
        out = dict(out or {})

        def buf(name, shp, dtype):
            return out[name] if out.get(name) is not None else torch.empty(shp, dtype=dtype, device=dev)
        knots, xc, yc = buf("knots", (T,), torch.float64), buf("x_coef", (T, 4), torch.float64), buf("y_coef", (T, 4), torch.float64)
        ok = buf("ok", (B,), torch.int32)
        rc = self._L.pqp_fit_splines_device(
            self._h, B, T, D.check(offsets, "offsets", torch.int32, (B + 1,), dev),
            D.check(ref, "ref", torch.float64, (T, D.STATE_COLS), dev), D.check(knots, "knots", torch.float64, (T,), dev),
            D.check(xc, "x_coef", torch.float64, (T, 4), dev), D.check(yc, "y_coef", torch.float64, (T, 4), dev),
            D.check(ok, "ok", torch.int32, (B,), dev), torch.cuda.current_stream(dev).cuda_stream)
        if rc != OK:
            raise PqpError(f"pqp_fit_splines_device failed (rc={rc}): {_lib.last_error()}")
        return dict(knot_offsets=offsets, knots=knots, x_coef=xc, y_coef=yc, ok=ok)

    def segment_device(self, splines, max_s, start, goal, max_n_points, capacity=None, delta_s_smaller=0.15,
                       delta_s_larger=0.3, dynamic_segmentation=True, search_delta_s=0.5, out=None):
        """PathOptimizer::segmentSmoothedPath for every path of a batch on the device (pqp_segment_reference_device):
        smoothed lines in, the reference states plan_device reads out.  `splines` a dict of knot_offsets int32 [B + 1],
        knots [K], x_coef / y_coef [K, 4] (fit_splines_device's output or device.splines_to_device), max_s float64 [B]
        the lines' lengths, start / goal float64 [B, 7] states, all torch CUDA tensors; on torch.cuda.current_stream().
        The defaults are the reference's flags: raw output with output_spacing 0.3 (spacings 0.15 and 0.3; without raw
        output 0.5 and 1.0), dynamic segmentation on, exact position off (search step 0.5; 0.1 with it).  capacity:
        stations the output holds (default the planner's max_total_points), the total_points to plan with.
        Returns dict(n_points int32 [B], offsets int32 [B + 1], ref float64 [capacity, 7], x0 [B, 3], end_heading [B],
        ok int32 [B]).  A refused path (heading error over 75 degrees, max_s <= 0 or not finite, more than
        max_n_points stations, past the capacity in index order, or a spline that is not usable) gets ok = 0 and 0
        stations; fail it in plan_device with map_index = torch.where(ok != 0, map_index, -1).  No host
        synchronisation; after one call on the planner it can be captured in a CUDA graph.  `out` may carry the output
        tensors, e.g. those of an earlier call, so that a captured graph writes where the plan reads."""
        import torch
        from . import device as D
        dev = self._cuda_device()
        B = int(max_s.shape[0])
        cap = int(self.max_total_points if capacity is None else capacity)
        K = int(splines["knots"].shape[0])
        f64, i32 = torch.float64, torch.int32
        out = dict(out or {})

        def buf(name, shp, dtype):
            return out[name] if out.get(name) is not None else torch.empty(shp, dtype=dtype, device=dev)
        n_points, offsets, ok = buf("n_points", (B,), i32), buf("offsets", (B + 1,), i32), buf("ok", (B,), i32)
        ref, x0, end_heading = buf("ref", (cap, D.STATE_COLS), f64), buf("x0", (B, 3), f64), buf("end_heading", (B,), f64)
        rc = self._L.pqp_segment_reference_device(
            self._h, B, D.check(splines["knot_offsets"], "knot_offsets", i32, (B + 1,), dev),
            D.check(splines["knots"], "knots", f64, (K,), dev), D.check(splines["x_coef"], "x_coef", f64, (K, 4), dev),
            D.check(splines["y_coef"], "y_coef", f64, (K, 4), dev), D.check(max_s, "max_s", f64, (B,), dev),
            D.check(start, "start", f64, (B, D.STATE_COLS), dev), D.check(goal, "goal", f64, (B, D.STATE_COLS), dev),
            float(delta_s_smaller), float(delta_s_larger), int(bool(dynamic_segmentation)), float(search_delta_s),
            int(max_n_points), cap, D.check(n_points, "n_points", i32, (B,), dev),
            D.check(offsets, "offsets", i32, (B + 1,), dev), D.check(ref, "ref", f64, (cap, D.STATE_COLS), dev),
            D.check(x0, "x0", f64, (B, 3), dev), D.check(end_heading, "end_heading", f64, (B,), dev),
            D.check(ok, "ok", i32, (B,), dev), torch.cuda.current_stream(dev).cuda_stream)
        if rc != OK:
            raise PqpError(f"pqp_segment_reference_device failed (rc={rc}): {_lib.last_error()}")
        return dict(n_points=n_points, offsets=offsets, ref=ref, x0=x0, end_heading=end_heading, ok=ok)

    def plan_device(self, n_points, offsets, ref, x0, end_heading, max_n_points=0, formulation="KP",
                    bounds_mode=BOUNDS_SIMPLE, splines=None, output_mode=OUTPUT_RAW, output_spacing=0.3,
                    collision_check=True, max_out=512, want_bounds=False, out=None, stats=False, map_index=None,
                    param_index=None, n_param_sets=0, form_mask=0):
        """plan() on torch CUDA tensors of the planner's device (path_optimizer_b200.device): n_points int32 [B],
        offsets int32 [B + 1], ref float64 [T, 7], x0 float64 [B, 3], end_heading float64 [B]; `splines` (IMPROVED)
        a dict of knot_offsets int32 [B + 1], knots [K], x_coef / y_coef [K, 4] (device.splines_to_device).  The whole
        chain runs on the device (pqp_plan_batch_device) on torch.cuda.current_stream() with plan()'s results bit for
        bit and no host synchronisation (unless `stats`): after one warm-up call it can be captured in a CUDA graph.
        max_n_points >= every n_points (0: the longest path any kernel class takes).  `out` may carry the output
        tensors (states: [T, 7] RAW or [B, max_out, 7] DENSIFY; n_out, ok, status, iters; bounds [T, 8]).
        `map_index`: int32 [B] on the device, the map of the set every path is planned on (pqp_plan_batch_device_maps,
        as plan(map_index=...)); None: map 0.  A graph replay reads the index from the captured tensor.
        `param_index`: int32 [B] on the device, the parameter set of every path (pqp_plan_batch_device_sets, as
        plan(param_index=...)); None: set 0.  n_param_sets > 0 bounds the sets launched (an index at or past it fails
        its path).  A graph replays with the sets it was captured with.
        `formulation` one per path (pqp_plan_batch_device_forms): an int32 CUDA tensor [B] of PQP_FORM_* values (a
        graph replay reads the captured tensor), or an array / list of names, uploaded per call.  `form_mask`
        (1 << PQP_FORM_* or a list of names; 0: all three) bounds the formulations launched; a path outside it fails."""
        import torch
        from . import device as D
        dev = self._cuda_device()
        B, T = int(n_points.shape[0]), int(ref.shape[0])
        forms = self._forms_device(formulation, B, dev)
        form = 0 if forms is not None else FORMULATIONS[formulation] if isinstance(formulation, str) else int(formulation)
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
        if forms is not None:
            mi = D.check(map_index, "map_index", i32, (B,), dev)
            pi = D.check(param_index, "param_index", i32, (B,), dev)
            fm = D.check(forms, "formulation", i32, (B,), dev)
            name = "pqp_plan_batch_device_forms"
            rc = self._L.pqp_plan_batch_device_forms(self._h, *head[2:], int(n_param_sets), self._form_mask(form_mask),
                                                     *args[:3], mi, pi, fm, *args[3:], *tail)
        elif param_index is not None:
            mi = D.check(map_index, "map_index", i32, (B,), dev)
            pi = D.check(param_index, "param_index", i32, (B,), dev)
            name = "pqp_plan_batch_device_sets"
            rc = self._L.pqp_plan_batch_device_sets(*head, int(n_param_sets), *args[:3], mi, pi, *args[3:], *tail)
        elif map_index is None:
            name, rc = "pqp_plan_batch_device", self._L.pqp_plan_batch_device(*head, *args, *tail)
        else:
            mi = D.check(map_index, "map_index", i32, (B,), dev)
            name, rc = "pqp_plan_batch_device_maps", self._L.pqp_plan_batch_device_maps(*head, *args[:3], mi, *args[3:],
                                                                                        *tail)
        if rc != OK:
            raise PqpError(f"{name} failed (rc={rc}): {_lib.last_error()}")
        return dict(states=states, n_out=n_out, ok=ok, status=status, iters=iters, bounds=bounds,
                    stats=st if stats else None)
