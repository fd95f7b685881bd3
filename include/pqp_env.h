/*
 * pqp_env.h -- C ABI of the stages either side of the path QP ("next" rows N2-N4 of the scope
 * table): clearance-bounds generation on a distance map, the post-solve collision check with arc
 * length re-accumulation, spline densification, and the solveWithoutSmoothing-shaped driver that
 * chains  bounds -> QP -> tail  on the device with one upload and one download per batch.
 *
 * Same rules as pqp.h: plain C, POD structs, caller-owned buffers, nothing throws, no CPU
 * fallback.  Every entry point cites the reference interface it replaces.
 */
#ifndef PQP_ENV_H_
#define PQP_ENV_H_

#include "pqp.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ROS-free stand-in for the "distance" layer of the grid_map::GridMap the reference wraps in
 * PathOptimizationNS::Map (src/tools/Map.cpp:8-14).  Index convention of grid_map_core (third
 * party, not vendored): cell (i, j) is centred at
 *     x = center_x + rows*resolution/2 - (i + 0.5)*resolution
 *     y = center_y + cols*resolution/2 - (j + 0.5)*resolution
 * i.e. (0,0) is the +x/+y corner, rows run along -x, columns along -y.  `distance` is ROW-major
 * here ([i*cols + j], metres to the nearest obstacle, float like grid_map's Eigen::MatrixXf). */
typedef struct pqp_distance_map {
    const float *distance;
    int32_t rows, cols;
    double resolution;
    double center_x, center_y;
} pqp_distance_map;

/* Bounds-generation variants (ReferencePath::updateBounds dispatches to the first one,
 * reference_path.cpp:77-79). */
enum pqp_bounds_mode {
    PQP_BOUNDS_IMPROVED = 0, /* updateBoundsImproved, reference_path_impl.cpp:142-201: circle centres
                              * re-projected onto the reference spline (needs the spline arguments) */
    PQP_BOUNDS_SIMPLE   = 1  /* updateBounds, reference_path_impl.cpp:237-281: circle centres on the
                              * heading line, exact == for the blocked test */
};

/* Output modes of the optimizePath tail (path_optimizer.cpp:191-230). */
enum pqp_output_mode {
    PQP_OUTPUT_RAW     = 0,  /* FLAGS_enable_raw_output = true (default): re-accumulate s, check, truncate */
    PQP_OUTPUT_DENSIFY = 1   /* false: tk::spline through (s,x),(s,y), resample every output_spacing */
};

/* Upload a distance map to the handle's device (kept until replaced or the handle is destroyed;
 * a planner reuses one map for many paths): the same as pqp_set_maps with one map.  Replaces:
 * Map::Map(grid_map) (Map.cpp:8-14) as constructed by PathOptimizer (path_optimizer.cpp:24-27). */
int pqp_set_map(pqp_handle *h, const pqp_distance_map *map);

/* Replace the handle's map set with `n_maps` >= 1 maps, each with its own rows, cols, resolution
 * and centre, so that one plan call can batch paths of several scenes (pqp_plan_batch_maps,
 * pqp_plan_batch_device_maps).  Every descriptor is checked first, with the rules of pqp_set_map:
 * a bad argument returns PQP_ERR_ARG and leaves the previous set in place.  The cells are copied
 * into one library-owned, grow-only device buffer, and the descriptors into a grow-only device
 * table (one row per map); no caller pointer is kept.  Synchronous, like pqp_set_map.  If the
 * device allocation fails the handle has no map set.  Do not call it while a device entry of the
 * handle that reads the maps is in flight.
 * The single-stage entries (pqp_update_bounds_batch, pqp_check_states, pqp_finish_raw_batch,
 * pqp_densify_batch, pqp_map_distance) and the plan entries without a map index read map 0.
 * The plan chain reads the descriptors from device memory, not from launch arguments: a CUDA
 * graph captured from pqp_plan_batch_device(_maps) follows a later pqp_set_maps as long as the
 * new set has no more maps than the largest set uploaded before the capture (the table is
 * reallocated otherwise, and the graph must be captured again).
 * Replaces: one Map(grid_map) per scene.  The reference plans against one map at a time; there
 * is no reference counterpart for several maps. */
int pqp_set_maps(pqp_handle *h, int n_maps, const pqp_distance_map *maps);

/* An occupancy grid from which the device builds a distance layer: the `binary` matrix the reference passes to
 * cv::distanceTransform.  `cells` is ROW-major [rows][cols] in the index convention of pqp_distance_map; a cell value of
 * 0 is an obstacle, any other value is free.  Geometry as pqp_distance_map. */
typedef struct pqp_occupancy_map {
    const uint8_t *cells;
    int32_t rows, cols;
    double resolution;
    double center_x, center_y;
} pqp_occupancy_map;

/* Replace the handle's map set with `n_maps` >= 1 layers built on the device from occupancy grids, as pqp_set_maps
 * replaces it from finished layers: every descriptor is checked first (NULL cells, rows or cols < 1, resolution <= 0:
 * PQP_ERR_ARG, the previous set stays), the layers go into the same grow-only cell buffer and table, and afterwards every
 * entry sees an ordinary map set.  Only the uint8 cells are uploaded (a quarter of the bytes of a layer).  Synchronous.
 * Layer of a map: the exact Euclidean distance transform.  With d2 the squared distance, in cells, from a cell's centre
 * to the nearest obstacle cell's centre (64-bit integers), the cell holds (float)sqrt((double)d2) * (float)resolution,
 * one float multiply; obstacle cells hold 0, and cells outside the grid are not obstacles.  That is bit for bit
 * ndimage.distance_transform_edt(cells != 0).astype(float32) * float32(resolution), and within 1 ulp of
 * cv::distanceTransform(CV_DIST_L2, CV_DIST_MASK_PRECISE) * resolution.  A grid with no obstacle gets OpenCV's value on
 * every cell: 2^64 * resolution.
 * Replaces: cv::distanceTransform(binary, CV_DIST_L2, CV_DIST_MASK_PRECISE) * resolution and Map(grid_map) per scene
 * (path_optimizer_benchmark.cpp:28-43, demo.cpp:103-110). */
int pqp_set_maps_occupancy(pqp_handle *h, int n_maps, const pqp_occupancy_map *maps);

/* pqp_set_maps_occupancy with DEVICE `cells` pointers (a host array of descriptors), asynchronous on `stream` (NULL: the
 * handle's stream).
 *   Same layout: when n_maps and every map's rows, cols, resolution and centre equal the handle's current set, and an
 *   earlier occupancy call has sized the transform's scratch for that set, the call only launches the transform (two
 *   kernels per 256 maps): no allocation, no copy, no host synchronisation.  It can then be captured in a CUDA graph
 *   together with pqp_plan_batch_device(_maps, _sets).
 *   Otherwise it lays the set out anew and synchronises.  If `stream` is capturing it returns PQP_ERR_ARG instead, before
 *   it touches the stream, so the capture stays valid.
 *   Replay: a replayed build writes map m only if table row m still has the cell address, rows and cols it was captured
 *   with; otherwise that map's build does nothing.  A replay after a later layout change leaves the current set as it
 *   is, and a plan in the same graph reads the current set (the table-growth rule of pqp_set_maps applies).
 * No reference counterpart: the reference builds its layer on the host. */
int pqp_set_maps_occupancy_device(pqp_handle *h, int n_maps, const pqp_occupancy_map *maps, void *stream);

/* Copy map m's layer (rows * cols floats, row-major) of the handle's set into the host buffer `out`, synchronously on
 * the handle's stream (synchronise the stream of a pqp_set_maps_occupancy_device call first).  PQP_ERR_ARG when m is
 * outside [0, n_maps) or `out` is NULL.  No reference counterpart (grid_map's layer is host memory there). */
int pqp_get_map(pqp_handle *h, int m, float *out);

/* Map::getObstacleDistance (Map.cpp:16-22) for `n` positions xy[n][2] on the device: bilinear
 * interpolation of the four surrounding cell centres, nearest cell when a neighbour falls outside
 * the grid, 0 outside the map; result rounded to float like grid_map's atPosition.  Map 0 of the
 * set. */
int pqp_map_distance(pqp_handle *h, int n, const double *xy, double *out);

/* Curvature and curvature-rate limits of the "KPC" formulation from the speed profile carried by the reference
 * states (v, a fields): friction circle  max_k = sqrt((mu g)^2 - a^2) / v^2  and rate limit
 * max_kp = max_curvature_rate / v, both DBL_MAX where v <= 1e-4; when the reference states were rebuilt from splines
 * (`from_spline` != 0: no speed information) max_k = tan(max_steering_angle) / wheel_base and max_kp = DBL_MAX.
 * g = 9.8 as in the reference.  Host arrays, n entries each (what pqp_solve_batch takes as max_k / max_kp).
 * pqp_update_limits_device does the same on device arrays of the handle's device, asynchronously on `stream`
 * (NULL: the handle's stream).  Replaces: ReferencePathImpl::updateLimits (reference_path_impl.cpp:203-235). */
int pqp_update_limits(const pqp_params *params, int from_spline, int n, const pqp_state *ref,
                      double *max_k, double *max_kp);
int pqp_update_limits_device(pqp_handle *h, int from_spline, int n, const pqp_state *d_ref,
                             double *d_max_k, double *d_max_kp, void *stream);

/* Natural cubic spline through (t_i, y_i), i < n (n >= 3, t strictly increasing), in the
 * piecewise form tk::spline keeps (src/tools/spline.cpp:161-249, default boundary = zero second
 * derivative, quadratic extrapolation):  f(t) = ((a_i h + b_i) h + c_i) h + y_i,  h = t - t_i.
 * coef[i] = {a_i, b_i, c_i, y_i}.  Host-side helper (O(n)); the device has its own copy for the
 * densify tail.  Replaces: tk::spline::set_points. */
int pqp_spline_fit(int n, const double *t, const double *y, double *coef /* [n][4] */);

/* pqp_spline_fit for every path of a batch on DEVICE arrays of the handle's device: the x(s) and y(s) splines
 * updateBoundsImproved projects onto (ReferencePathImpl::x_s_, y_s_), in the layout pqp_plan_batch_device* takes with
 * PQP_BOUNDS_IMPROVED: pass d_offsets as d_knot_offsets and the three outputs as d_knots, d_x_coef, d_y_coef.
 *   d_offsets          [batch+1] exclusive prefix of the station counts; d_offsets[batch] = total_points
 *   d_ref              [total_points] reference states; the knots are their s, the values their x and y
 *   d_knots            [total_points] out: the stations' s, copied as they are
 *   d_x_coef, d_y_coef [total_points][4] out: pqp_spline_fit's rows for (s, x) and (s, y), bit for bit
 *   d_ok               [batch] out: 1 when the path was fitted, 0 when it was refused
 * A path is refused when it has fewer than 3 stations or its s is not strictly increasing or not finite; its knots
 * and coefficient rows are then NaN, and no other path changes.  (pqp_spline_fit refuses the same paths, except that
 * it accepts an infinite first or last knot and returns non-finite rows for it.)  To fail a refused path in a plan
 * call without a host round trip, give it a map index outside the map set on the device, e.g.
 * map_index[b] = d_ok[b] ? map_index[b] : -1: pqp_plan_batch_device_maps then reports it as PQP_INVALID_PROBLEM with
 * 0 iterations, out_n = 0 and ok = 0 and no other path changes.
 * NULL pointers (with batch > 0) or a negative batch or total_points return PQP_ERR_ARG; a batch or total_points
 * above the handle's capacity PQP_ERR_CAPACITY; nothing is launched then.  Asynchronous on `stream` (NULL: the
 * handle's stream), no host synchronisation; the scratch (4 doubles per station of the handle's max_total_points) is
 * allocated by the first call, after which the call allocates nothing and can be captured in a CUDA graph together
 * with the plan entries.  No map set is needed.
 * Replaces: tk::spline::set_points through the reference line's (s, x) and (s, y), the splines handed to
 * ReferencePathImpl::setSpline (reference_path_impl.cpp:36-41), once per path. */
int pqp_fit_splines_device(pqp_handle *h, int batch, int total_points, const int32_t *d_offsets, const pqp_state *d_ref,
                           double *d_knots, double *d_x_coef, double *d_y_coef, int32_t *d_ok, void *stream);

/* Segment smoothed reference lines into reference states for every path of a batch, on DEVICE arrays of the handle's
 * device: what segmentSmoothedPath (path_optimizer.cpp:119-178) does between the smoother and the QP, with outputs in
 * the layout pqp_plan_batch_device* takes.
 *   d_knot_offsets, d_knots, d_x_coef, d_y_coef   every path's x(s), y(s) splines, the layout pqp_fit_splines_device
 *                      writes and pqp_plan_batch_device* reads with PQP_BOUNDS_IMPROVED
 *   d_max_s            [batch] every line's length, what ReferencePathImpl::setSpline receives
 *   d_start, d_goal    [batch] VehicleState's start and end states
 *   delta_s_smaller, delta_s_larger   the spacings of :168-173: (0.15, FLAGS_output_spacing) with
 *                      FLAGS_enable_raw_output, else (0.5, 1.0)
 *   dynamic_segmentation   FLAGS_enable_dynamic_segmentation
 *   search_delta_s     the goal-search step: 0.1 with FLAGS_enable_exact_position, else 0.5
 *   max_n_points       stations a path may have at most
 *   capacity           stations d_ref holds (the total_points to plan with)
 *   d_n_points         [batch] out: stations of every path (0 when refused)
 *   d_offsets          [batch+1] out: their exclusive prefix; d_offsets[batch] <= capacity (with batch = 0 the
 *                      one entry 0 is written when d_offsets is not NULL)
 *   d_ref              [capacity] out: the stations, x, y, z, k, s filled, v = a = 0; entries past d_offsets[batch]
 *                      are not written
 *   d_x0               [batch][3] out: (initial offset, initial heading error, start.k), written for every path
 *   d_end_heading      [batch] out: goal.z
 *   d_ok               [batch] out: 1 when the path was segmented, 0 when it was refused
 * Per path: the initial offset is the distance from the start to the spline's first point, positive when that point
 * lies right of the start's heading, and the heading error constraintAngle(start.z - heading at s = 0) (:125-141);
 * when the goal is not within 1e-6 of the point at max_s, the length is cut to the sample closest to the goal on the
 * lattice max_s - i * search_delta_s (accumulated), searched backwards until a sample lies more than 8 m from the goal
 * while the closest lies within 8 m (:143-166); then ReferencePathImpl::buildReferenceFromSpline (reference_path_impl.cpp
 * :474-499) samples s = 0, s1, ... <= the cut length, each step delta_s_larger, or with dynamic segmentation shortened
 * towards delta_s_smaller as |k| goes from 0.08 to 0.2.  Heading and curvature come from the splines' derivatives as
 * getHeading and getCurvature compute them (tools.cpp:32-44), in the arithmetic of the densifying tail.
 * A path is refused (ok = 0, 0 stations; no other path changes) when:
 *   - its splines have fewer than 3 knots, its initial offset is not finite, or start.z minus the heading at s = 0 is
 *     not finite or exceeds 2^20 rad in magnitude (e.g. the NaN rows of a line pqp_fit_splines_device refused, or a
 *     NaN start);
 *   - |initial heading error| > 75 degrees (:137-140);
 *   - max_s <= 0 or is not finite, or max_s > search_delta_s * 2^22 (a goal search too long to walk).  The guard
 *     still admits long searches: a goal that is NaN or more than 8 m from every sample visits every lattice sample,
 *     about 1.1 us each on one thread of an H100, so up to about 4.6 s for one path at the limit;
 *   - it needs more than max_n_points stations;
 *   - the running total of stations, in index order, would pass capacity: path b is refused when the stations of paths
 *     0..b, refused ones counting 0, exceed capacity, and so is every later path with stations.
 * To fail a refused path in the plan without a host round trip, give it a map index outside the map set on the device
 * (map_index[b] = d_ok[b] ? map_index[b] : -1), as for pqp_fit_splines_device.
 * NULL pointers (with batch > 0), a negative batch or capacity, max_n_points < 1, or spacings that are not positive and
 * finite or with delta_s_larger < delta_s_smaller return PQP_ERR_ARG; a batch above the handle's max_batch or a
 * capacity above its max_total_points PQP_ERR_CAPACITY; nothing is launched then.  Asynchronous on `stream` (NULL: the
 * handle's stream), no host synchronisation; the scratch (one int32 per path of the handle's max_batch) is allocated by
 * the first call, after which the call allocates nothing and can be captured in a CUDA graph between
 * pqp_fit_splines_device and the plan entries.  No map set is needed.
 * Replaces: PathOptimizer::segmentSmoothedPath (path_optimizer.cpp:119-173) up to buildReferenceFromSpline, once per
 * path; the bounds and limits it goes on to compute are the plan entries' stages. */
int pqp_segment_reference_device(pqp_handle *h, int batch, const int32_t *d_knot_offsets, const double *d_knots,
                                 const double *d_x_coef, const double *d_y_coef, const double *d_max_s,
                                 const pqp_state *d_start, const pqp_state *d_goal, double delta_s_smaller,
                                 double delta_s_larger, int dynamic_segmentation, double search_delta_s,
                                 int max_n_points, int capacity, int32_t *d_n_points, int32_t *d_offsets,
                                 pqp_state *d_ref, double *d_x0, double *d_end_heading, int32_t *d_ok, void *stream);

/* Search a corridor around every smoothed reference line of a batch and post-smooth the line inside it, on DEVICE
 * arrays of the handle's device: what ReferencePathSmoother::solve does after its smoother (graphSearchDp, then
 * postSmooth), with outputs in the layout pqp_segment_reference_device takes.
 *   d_knot_offsets, d_knots, d_x_coef, d_y_coef, d_max_s   every path's smoothed x(s), y(s) splines and length, the
 *                      layout pqp_segment_reference_device takes
 *   d_start            [batch] VehicleState's start state
 *   d_map_index        [batch] every path's map in the handle's set, or NULL for map 0
 *   search_lateral_range, search_lateral_spacing, search_longitudial_spacing   FLAGS_search_* (10, 0.6, 1.5)
 *   max_layers         layers a path may have at most (>= 4)
 *   capacity           knot rows the outputs hold
 *   d_knot_offsets_out [batch+1] out: exclusive prefix of every path's knots (0 when refused); d_knot_offsets_out[batch]
 *                      <= capacity (with batch = 0 the one entry 0 is written when the array is not NULL)
 *   d_knots_out, d_x_coef_out [capacity][4], d_y_coef_out [capacity][4]   out: the post-smoothed lines' splines;
 *                      rows past d_knot_offsets_out[batch] are not written
 *   d_max_s_out        [batch] out: every line's new length, NaN when refused
 *   d_ok               [batch] out: 1 when the path was post-smoothed, 0 when it was refused
 *   d_status, d_iters  [batch] out: the post-smoothing QP's status and iterations; a path refused before its QP reports
 *                      PQP_INVALID_PROBLEM and 0 iterations, as an empty problem does
 *   d_layers           [capacity][3] out, or NULL: (layer s, lower bound, upper bound) of every kept layer, the
 *                      reference's layers_s_list_ / layers_bounds_, in the knot rows of the path
 * Per path, graphSearchDp (reference_path_smoother.cpp:145-301): the start's closest point on the line
 * (findClosestPoint, tools.cpp:66-110: a 0.5 m grid scan and up to 20 Newton steps, clamped above by max_s only), the
 * layers s += search_longitudial_spacing from it while below max_s, then max_s (0.5 m spacing for a line of 6 m or
 * less); the start's lateral offset vehicle_l; a lattice of lateral nodes cur_l += spacing from -range while <= range
 * per layer, a node feasible inside the map at distance >= 1.45 m and not past the turning radius on the inside, layer 0
 * holding the start node alone; the DP of calculateCostAt (:110-143, weights 1, 0.5, 16 and 0.5, safe distance 3 m),
 * its min over predecessors taken in index order with a strict '<'; the search stops at the first layer with no
 * reachable node, backtracks from the cheapest node of the last layer reached, and marches each chosen node's bounds
 * outwards in 0.2 m steps up to 6 m (layer 0: -10, 10).  Then postSmooth (:534-644): the QP with weights 1, 100 and
 * 1000 on (offset, dx, ddx) of every layer, row 0 pinned to vehicle_l, solved with the handle's OSQP settings (the
 * reference's OsqpEigen solvers set only verbosity and warm start, so under the default settings these are the
 * settings postSmooth runs with); the points ref + offset * (cos, sin)(heading + pi/2), s accumulated, and the natural
 * splines x(s), y(s) of tk::spline fitted through them.  The generic core's epilogue wraps heading + pi/2 into
 * [-pi, pi] before its cosine and sine, so a point may differ from postSmooth's in the last bits.
 * A path is refused (ok = 0, 0 knots, NaN max_s; no other path changes) when:
 *   - its splines have fewer than 3 knots, or max_s <= 0, is not finite or exceeds 2^20 m (a grid scan too long);
 *   - its start heading is not finite or exceeds 2^20 rad, or its closest point or vehicle_l is not finite;
 *   - |vehicle_l| > search_lateral_range;
 *   - it has more than max_layers layers, or the lateral lattice has more than 64 nodes;
 *   - it reaches fewer than 4 layers;
 *   - its QP does not end PQP_SOLVED, or its post-smoothed s is not strictly increasing;
 *   - its map index lies outside the map set;
 *   - the running total of knots, in index order, would pass capacity (as pqp_segment_reference_device's stations).
 * NULL pointers (with batch > 0), a negative batch or capacity, max_layers < 4, flags that are not positive and finite,
 * or no map set return PQP_ERR_ARG; a batch above the handle's max_batch, a capacity above its max_total_points or a
 * max_layers whose QP does not fit one SM's shared memory (about 740 layers on an H100) PQP_ERR_CAPACITY; nothing is
 * launched then.  Asynchronous on `stream` (NULL: the handle's stream), no host synchronisation; the scratch (about
 * 0.6 KB per layer of max_layers per path of the handle's max_batch, and the kept points) is allocated by the first call
 * and grows only with a larger max_layers, so after one call with the largest max_layers the call allocates nothing and
 * can be captured in a CUDA graph ahead of pqp_segment_reference_device.
 * Replaces: ReferencePathSmoother::graphSearchDp + ReferencePathSmoother::postSmooth (reference_path_smoother.cpp
 * :145-301, :534-644), once per path. */
int pqp_post_smooth_device(pqp_handle *h, int batch, const int32_t *d_knot_offsets, const double *d_knots,
                           const double *d_x_coef, const double *d_y_coef, const double *d_max_s,
                           const pqp_state *d_start, const int32_t *d_map_index, double search_lateral_range,
                           double search_lateral_spacing, double search_longitudial_spacing, int max_layers,
                           int capacity, int32_t *d_knot_offsets_out, double *d_knots_out, double *d_x_coef_out,
                           double *d_y_coef_out, double *d_max_s_out, int32_t *d_ok, int32_t *d_status,
                           int32_t *d_iters, double *d_layers, void *stream);

/* Smooth every raw reference polyline of a batch on DEVICE arrays of the handle's device: what
 * ReferencePathSmoother::solve does before graphSearchDp under the default flags (smoothing_method TENSION2,
 * tension_solver OSQP) -- the B-spline pre-pass, segmentRawReference and TensionSmoother2's smoothing QP -- with outputs
 * in the layout pqp_post_smooth_device takes.
 *   d_point_offsets    [batch+1] exclusive prefix of every path's input points
 *   d_points           [d_point_offsets[batch]] the raw polylines; x and y are read
 *   deviation_w, curvature_w, curvature_rate_w   FLAGS_tension_2_deviation_weight, _curvature_weight and
 *                      _curvature_rate_weight (0.005, 1, 10)
 *   max_raw_samples    B-spline samples a path may have at most (about its length in metres + 2)
 *   max_points         resampled stations a path may have at most (ceil of its sampled length + 1)
 *   capacity           knot rows the outputs hold
 *   d_knot_offsets_out [batch+1] out: exclusive prefix of every path's knots (0 when refused); d_knot_offsets_out[batch]
 *                      <= capacity (with batch = 0 the one entry 0 is written)
 *   d_knots_out, d_x_coef_out [capacity][4], d_y_coef_out [capacity][4]   out: the smoothed lines' splines; rows past
 *                      d_knot_offsets_out[batch] are not written
 *   d_max_s_out        [batch] out: every smoothed line's length s.back() + 3, NaN when refused
 *   d_ok               [batch] out: 1 when the path was smoothed, 0 when it was refused
 *   d_status, d_iters  [batch] out: the smoothing QP's status and iterations; a path refused before its QP reports
 *                      PQP_INVALID_PROBLEM and 0 iterations, as an empty problem does
 * Per path: bSpline (reference_path_smoother.cpp:498-532) -- the length as the serial sum of distance() (tools.cpp:46),
 * the degree 3, 4 or 5 from the average segment length (> 10, > 5, else), the clamped B-spline of that degree with the
 * points as control points (tinyspline's BSpline(n, 2, degree), restated: clamped uniform knots and de Boor's
 * algorithm), sampled at t += 1 / length (accumulated) while t < 1 and at t = 1, and s the serial sum of the sample
 * distances; segmentRawReference (:50-88) -- the natural splines x(s), y(s) of tk::spline through the samples, sampled
 * at s = 0, 1, 2, ... while s.back() < max_s (the last one extrapolated), with the heading atan2(dy, dx) and curvature
 * (dx ddy - dy ddx) / pow(dx^2 + dy^2, 1.5); TensionSmoother2::osqpSmooth (tension_smoother_2.cpp:163-301) -- the QP in
 * x, y, theta of every station and k of all but the last, with the three weights, the update rows and the pins of x_0,
 * y_0, solved with the handle's OSQP settings (the reference's OsqpEigen solver sets only verbosity and warm start, so
 * under the default settings these are the settings it runs with); and TensionSmoother::smooth's tail
 * (tension_smoother.cpp:84-96) -- s accumulated from the solution's x, y, the natural splines x(s), y(s) fitted through
 * them, max_s = s.back() + 3.  The TENSION method is pqp_smooth_reference_tension_device below; the IPOPT solver and
 * the ANGLE_DIFF method are not restated.
 * A path is refused (ok = 0, 0 knots, NaN max_s; no other path changes) when:
 *   - it has fewer than 4 points (:36-39);
 *   - the B-spline's degree is not below its point count (tinyspline refuses such a spline and the reference throws;
 *     here it is a refusal), e.g. 4 or 5 points less than 5 m apart on average;
 *   - its length is not positive and finite (a NaN or infinite coordinate);
 *   - it has more than max_raw_samples B-spline samples, or more than max_points stations;
 *   - its samples are fewer than 3 or their s is not strictly increasing, or it has fewer than 3 stations
 *     (tk::spline::set_points asserts both, spline.cpp:164-165);
 *   - its QP does not end PQP_SOLVED, or its smoothed s is not strictly increasing and finite;
 *   - the running total of knots, in index order, would pass capacity (as pqp_segment_reference_device's stations).
 * NULL pointers (with batch > 0), a negative batch or capacity, max_raw_samples or max_points below 3, or a weight that
 * is negative or not finite return PQP_ERR_ARG; a batch above the handle's max_batch, a capacity above its
 * max_total_points or a max_points whose QP does not fit one SM's shared memory (507 stations on an H100, 227 KB)
 * PQP_ERR_CAPACITY; nothing is launched then.  Asynchronous on `stream` (NULL: the handle's stream), no host
 * synchronisation; the scratch (about 0.2 KB per raw sample of max_raw_samples and 0.6 KB per station of max_points, per
 * path of the handle's max_batch, and the kept points) is allocated by the first call and grows only with a larger
 * max_raw_samples or max_points, so after one call with the largest caps the call allocates nothing and can be captured
 * in a CUDA graph ahead of pqp_post_smooth_device.
 * Replaces: ReferencePathSmoother::bSpline + TensionSmoother2::smooth (TENSION2, OSQP), once per path. */
int pqp_smooth_reference_device(pqp_handle *h, int batch, const int32_t *d_point_offsets, const pqp_state *d_points,
                                double deviation_w, double curvature_w, double curvature_rate_w, int max_raw_samples,
                                int max_points, int capacity, int32_t *d_knot_offsets_out, double *d_knots_out,
                                double *d_x_coef_out, double *d_y_coef_out, double *d_max_s_out, int32_t *d_ok,
                                int32_t *d_status, int32_t *d_iters, void *stream);

/* pqp_smooth_reference_device with smoothing_method TENSION (tension_solver OSQP): the same B-spline pre-pass,
 * segmentRawReference, tail, outputs and reservation, with TensionSmoother's clearance-bounded smoothing QP in place of
 * TensionSmoother2's.  Parameters as pqp_smooth_reference_device, plus
 *   deviation_w, curvature_w, curvature_rate_w   FLAGS_cartesian_deviation_weight, _curvature_weight and
 *                      _curvature_rate_weight (0, 1, 50)
 *   d_map_index        [batch] the map of every path in the handle's map set (pqp_set_map / pqp_set_maps), or NULL for
 *                      map 0
 * Per path, TensionSmoother::osqpSmooth (tension_smoother.cpp:186-237) with setHessianMatrix (:239-263) and
 * setConstraintMatrix (:265-314): over the N stations (x_i, y_i, heading_i) of segmentRawReference, the unknowns x_i,
 * y_i and the lateral offsets d_i; q = 0; P the dds blocks (1, -2, 1)(1, -2, 1)' curvature_w and the ddds blocks
 * (-1, 3, -3, 1)(-1, 3, -3, 1)' curvature_rate_w of the x and y chains, and deviation_w on every d_i; the rows
 * x_i - cos(theta_i) d_i = x_ref_i, y_i - sin(theta_i) d_i = y_ref_i with theta_i = heading_i + pi/2, and d_i with
 * d_0 = 0, |d_{N-1}| <= 0.5 and |d_i| <= min(clearance_i, 2) between, clearance_i being Map::getObstacleDistance
 * (Map.cpp:16-22) at the station in the path's map (bilinear in the distance layer, 0 outside the map); exact zeros of
 * P and A dropped as Eigen's sparseView drops them; solved with the handle's OSQP settings.  The smoothed line is the
 * solution's x_i, y_i, followed by TensionSmoother::smooth's tail (:84-96) as above.
 * A path is refused for the reasons of pqp_smooth_reference_device, and when its map index lies outside the map set.
 * Errors as pqp_smooth_reference_device, and PQP_ERR_ARG when the handle has no map set; the QP fits one SM's shared
 * memory up to 277 stations on an H100 (227 KB), so a larger max_points returns PQP_ERR_CAPACITY.  The scratch is the
 * smoothing stage's, sized for whichever of the two QPs asked for more.
 * Replaces: ReferencePathSmoother::bSpline + TensionSmoother::smooth (TENSION, OSQP), once per path. */
int pqp_smooth_reference_tension_device(pqp_handle *h, int batch, const int32_t *d_point_offsets,
                                        const pqp_state *d_points, double deviation_w, double curvature_w,
                                        double curvature_rate_w, const int32_t *d_map_index, int max_raw_samples,
                                        int max_points, int capacity, int32_t *d_knot_offsets_out, double *d_knots_out,
                                        double *d_x_coef_out, double *d_y_coef_out, double *d_max_s_out, int32_t *d_ok,
                                        int32_t *d_status, int32_t *d_iters, void *stream);

/* tk::spline::operator() / deriv (spline.cpp:250-318) on a fitted spline; order 0..2. */
double pqp_spline_eval(int n, const double *t, const double *coef, int order, double at);

/* Clearance bounds for a batch of reference paths against the uploaded map (map 0 of the set).
 *   mode             pqp_bounds_mode
 *   n_points, ref    as pqp_solve_batch
 *   n_knots          [batch]            } IMPROVED only: the x(s), y(s) splines of each path
 *   knots            [sum n_knots]      } (ReferencePathImpl::x_s_, y_s_), concatenated; coefficient
 *   x_coef, y_coef   [sum n_knots][4]   } layout of pqp_spline_fit.  NULL for SIMPLE.
 *   out_bounds       [sum n_points]; entries at and after a path's blocked station are undefined
 *   out_n_valid      [batch] number of leading stations with usable bounds = the size the
 *                    reference resizes reference_states_/bounds_ to when the path is blocked
 *                    (reference_path_impl.cpp:183-199); == n_points[b] when nothing is blocked
 * Replaces: ReferencePath::updateBounds(map) (reference_path.cpp:77-79) once per path. */
int pqp_update_bounds_batch(pqp_handle *h, int mode, int batch, const int32_t *n_points,
                            const pqp_state *ref,
                            const int32_t *n_knots, const double *knots,
                            const double *x_coef, const double *y_coef,
                            pqp_station_bounds *out_bounds, int32_t *out_n_valid,
                            pqp_stats *stats);

/* Footprint check of `n` states against the uploaded map (map 0 of the set): bounding circle first, then the six
 * covering circles.  ok[i] = 1 when collision free.
 * Replaces: CollisionChecker::isSingleStateCollisionFreeImproved (collision_checker.cpp:41-59)
 * with CarGeometry's circles (car_geometry.cpp:38-57). */
int pqp_check_states(pqp_handle *h, int n, const pqp_state *states, int32_t *ok);

/* The raw-output tail of optimizePath for a batch of solved paths, in place: s re-accumulated from
 * chord lengths, each state checked against map 0 of the set, path cut at the first colliding state.
 *   paths            [sum n_points] in/out (s rewritten)
 *   out_n_kept       [batch] states kept (== n_points[b] when no collision)
 *   out_ok           [batch] the reference's return value: 1 if nothing collided, else
 *                    (s of the last kept state >= 20 m); 0 when even the first state collides
 * Replaces: path_optimizer.cpp:191-202. */
int pqp_finish_raw_batch(pqp_handle *h, int batch, const int32_t *n_points, pqp_state *paths,
                         int collision_check, int32_t *out_n_kept, int32_t *out_ok,
                         pqp_stats *stats);

/* The densifying tail: spline through the solved path, resampled every `output_spacing` metres
 * (heading and curvature from the spline derivatives), cut at the first colliding sample (map 0
 * of the set).
 *   out_states       [batch][max_out] (path b starts at b*max_out)
 *   out_n            [batch] samples written (a path that needs more than max_out reports
 *                    max_out and ok = 0)
 *   out_ok           [batch] as above
 * Replaces: path_optimizer.cpp:203-230. */
int pqp_densify_batch(pqp_handle *h, int batch, const int32_t *n_points, const pqp_state *paths,
                      double output_spacing, int collision_check, int max_out,
                      pqp_state *out_states, int32_t *out_n, int32_t *out_ok, pqp_stats *stats);

/* One whole planner iteration per path, batched:  bounds (N2) -> QP -> tail (N3/N4), chained on the
 * device; host buffers in and out.  Inputs as pqp_update_bounds_batch + pqp_solve_batch (x0 of
 * the reference's solveWithoutSmoothing is (0,0,start.k): pass what VehicleState would hold).
 *   out_states       RAW: [sum n_points]; DENSIFY: [batch][max_out]
 *   out_n            [batch] states of the final path (after blocked-truncation and collision cut)
 *   out_ok           [batch] the reference's bool: QP solved and tail ok
 *   status, iters    as pqp_solve_batch (optional)
 *   out_bounds       optional [sum n_points] the bounds that were used
 * Replaces: PathOptimizer::solveWithoutSmoothing (path_optimizer.cpp:87-117) once per path. */
int pqp_plan_batch(pqp_handle *h, int formulation, int bounds_mode, int output_mode, int batch,
                   const int32_t *n_points, const pqp_state *ref,
                   const int32_t *n_knots, const double *knots,
                   const double *x_coef, const double *y_coef,
                   const double *x0, const double *end_heading,
                   double output_spacing, int collision_check, int max_out,
                   pqp_state *out_states, int32_t *out_n, int32_t *out_ok,
                   int32_t *status, int32_t *iters, pqp_station_bounds *out_bounds,
                   pqp_stats *stats);

/* The same planner iteration on DEVICE arrays of the handle's device, e.g. reference paths another CUDA stage produced:
 * nothing crosses to the host.  Arguments as pqp_plan_batch, with these differences:
 *   d_offsets          [batch+1] exclusive prefix of d_n_points; total_points = d_offsets[batch]
 *   max_n_points       >= every n_points[b]: sizes the bounds grid and bounds the class dispatch (0: the longest path
 *                      any kernel class of the formulation takes).  A longer path reports PQP_INVALID_PROBLEM unless
 *                      blocking cut it within its first max_n_points stations.
 *   d_knot_offsets     [batch+1] exclusive prefix of the knot counts (IMPROVED only), instead of n_knots
 *   d_out_states .. d_out_bounds   the caller's device buffers (d_iters, d_out_bounds optional; d_status required)
 * The QP step picks every path's kernel class on the device (as pqp_solve_batch_device_dispatch), so each path runs on
 * the class pqp_plan_batch would choose and the results equal pqp_plan_batch's bit for bit.  "KPC" derives its limits
 * on the device as pqp_plan_batch does; stations past a cut read as zeros (RAW).  Asynchronous on `stream` (NULL: the
 * handle's stream); no host synchronisation unless `stats` is non-NULL (then only kernel_ms and kernel_launches are
 * filled); no allocation once an earlier call on the handle has sized its buffers: make one warm-up call, then the call
 * can be captured into a CUDA graph and replayed after new inputs are copied into the captured buffers.  One call in
 * flight per handle.  pqp_set_order_hint is not applied.  No reference counterpart. */
int pqp_plan_batch_device(pqp_handle *h, int formulation, int bounds_mode, int output_mode, int batch,
                          int total_points, int max_n_points,
                          const int32_t *d_n_points, const int32_t *d_offsets, const pqp_state *d_ref,
                          const int32_t *d_knot_offsets, const double *d_knots,
                          const double *d_x_coef, const double *d_y_coef,
                          const double *d_x0, const double *d_end_heading,
                          double output_spacing, int collision_check, int max_out,
                          pqp_state *d_out_states, int32_t *d_out_n, int32_t *d_out_ok,
                          int32_t *d_status, int32_t *d_iters, pqp_station_bounds *d_out_bounds,
                          void *stream, pqp_stats *stats);

/* pqp_plan_batch and pqp_plan_batch_device over the handle's map set (pqp_set_maps): the same
 * arguments plus one map index per path, on the host (`map_index`) or on the device
 * (`d_map_index`), both int32 [batch].
 *   Path b uses map map_index[b] for its clearance bounds and for the collision check of its raw
 *   or densified tail.  A NULL index means map 0 for every path: pqp_plan_batch and
 *   pqp_plan_batch_device are these entries with a NULL index.
 *   An index outside [0, n_maps) makes that path report PQP_INVALID_PROBLEM with 0 iterations,
 *   out_n = 0 and ok = 0 (its bounds are undefined, its RAW states read as zeros); no other path's
 *   results change.  The index is checked before the map table is read.
 * Each path gets the results pqp_plan_batch gives it on its own map, bit for bit.  The device
 * entry keeps every promise of pqp_plan_batch_device: asynchronous on `stream`, no allocation
 * after a warm-up call, capturable in a CUDA graph (replays read the index from the captured
 * buffer).
 * Replaces: PathOptimizer::solveWithoutSmoothing (path_optimizer.cpp:87-117) once per path, each
 * path with the PathOptimizer of its own scene.  No reference counterpart for several maps. */
int pqp_plan_batch_maps(pqp_handle *h, int formulation, int bounds_mode, int output_mode, int batch,
                        const int32_t *n_points, const pqp_state *ref, const int32_t *map_index,
                        const int32_t *n_knots, const double *knots,
                        const double *x_coef, const double *y_coef,
                        const double *x0, const double *end_heading,
                        double output_spacing, int collision_check, int max_out,
                        pqp_state *out_states, int32_t *out_n, int32_t *out_ok,
                        int32_t *status, int32_t *iters, pqp_station_bounds *out_bounds,
                        pqp_stats *stats);
int pqp_plan_batch_device_maps(pqp_handle *h, int formulation, int bounds_mode, int output_mode,
                               int batch, int total_points, int max_n_points,
                               const int32_t *d_n_points, const int32_t *d_offsets,
                               const pqp_state *d_ref, const int32_t *d_map_index,
                               const int32_t *d_knot_offsets, const double *d_knots,
                               const double *d_x_coef, const double *d_y_coef,
                               const double *d_x0, const double *d_end_heading,
                               double output_spacing, int collision_check, int max_out,
                               pqp_state *d_out_states, int32_t *d_out_n, int32_t *d_out_ok,
                               int32_t *d_status, int32_t *d_iters,
                               pqp_station_bounds *d_out_bounds, void *stream, pqp_stats *stats);

/* pqp_plan_batch_maps and pqp_plan_batch_device_maps over the handle's parameter sets (pqp_set_param_sets) as well: the
 * same arguments plus one set index per path (`param_index` on the host, `d_param_index` on the device, int32 [batch])
 * and, for the device entry, `n_param_sets`, an upper bound on the indices used (0: the handle's set count).
 *   Path b runs every stage with set param_index[b]: circle radius and d1..d4 of its bounds, the footprint of its
 *   collision check, the "KPC" limits (mu, curvature rate) and everything the QP reads.  Its results -- status,
 *   iterations, states, bounds, out_n and ok -- equal, bit for bit, those pqp_plan_batch_maps gives it on a handle whose
 *   only set is that one.  A NULL index means set 0: the _maps entries are these with a NULL index.
 *   An index outside [0, n_sets), or for the device entry at or past n_param_sets, makes that path report
 *   PQP_INVALID_PROBLEM with 0 iterations, out_n = 0 and ok = 0; no other path's results change.  The index is checked
 *   before the sets are read.
 * The QP step launches one grid per (set, kernel class) pair (pqp_solve_batch_sets,
 * pqp_solve_batch_device_dispatch_sets).  The device entry keeps every promise of pqp_plan_batch_device_maps; a CUDA
 * graph replays with the sets it was captured with, at every stage (the map rule differs: the chain reads the map
 * descriptors from device memory, so a replay follows a later pqp_set_maps).
 * Replaces: PathOptimizer::solveWithoutSmoothing (path_optimizer.cpp:87-117) once per path, with that path's FLAGS_*
 * (and the PathOptimizer of its own scene). */
int pqp_plan_batch_sets(pqp_handle *h, int formulation, int bounds_mode, int output_mode, int batch,
                        const int32_t *n_points, const pqp_state *ref, const int32_t *map_index,
                        const int32_t *param_index,
                        const int32_t *n_knots, const double *knots,
                        const double *x_coef, const double *y_coef,
                        const double *x0, const double *end_heading,
                        double output_spacing, int collision_check, int max_out,
                        pqp_state *out_states, int32_t *out_n, int32_t *out_ok,
                        int32_t *status, int32_t *iters, pqp_station_bounds *out_bounds,
                        pqp_stats *stats);
int pqp_plan_batch_device_sets(pqp_handle *h, int formulation, int bounds_mode, int output_mode,
                               int batch, int total_points, int max_n_points, int n_param_sets,
                               const int32_t *d_n_points, const int32_t *d_offsets,
                               const pqp_state *d_ref, const int32_t *d_map_index,
                               const int32_t *d_param_index,
                               const int32_t *d_knot_offsets, const double *d_knots,
                               const double *d_x_coef, const double *d_y_coef,
                               const double *d_x0, const double *d_end_heading,
                               double output_spacing, int collision_check, int max_out,
                               pqp_state *d_out_states, int32_t *d_out_n, int32_t *d_out_ok,
                               int32_t *d_status, int32_t *d_iters,
                               pqp_station_bounds *d_out_bounds, void *stream, pqp_stats *stats);

/* pqp_plan_batch_sets and pqp_plan_batch_device_sets with one formulation per path in place of the scalar:
 * `formulation` (host) or `d_formulation` (device), int32 [batch] of PQP_FORM_* values; the array is required.
 *   Path b's results -- status, iterations, states, bounds, out_n and ok -- equal, bit for bit, those the _sets entry
 *   gives it when called with formulation = formulation[b], for any mix of maps, sets and lengths in the batch.
 *   A formulation outside {0, 1, 2}, or for the device entry outside `form_mask`, makes only that path report
 *   PQP_INVALID_PROBLEM with 0 iterations, out_n = 0 and ok = 0; no other path changes.  Map and set indices keep
 *   their rules.
 *   form_mask      device entry: bitmask of 1 << PQP_FORM_*, 0 = all three; it only bounds what is launched.
 *   max_n_points   device entry: 0 = the longest path any class of any formulation in the mask takes.  Each path stays
 *                  limited by its own formulation's classes, as in its _sets call; a longer one reports
 *                  PQP_INVALID_PROBLEM (its bounds past that limit are then computed, where the _sets call leaves them
 *                  unwritten).
 * The "KPC" limits are derived on the device, as the chain does for a "KPC" call, whenever some path is "KPC" (host
 * entry) or the mask holds "KPC" (device entry); "KP" and "K" paths do not read them.  The bounds and tail stages do
 * not depend on the formulation.  The device entry keeps every promise of pqp_plan_batch_device_sets (no allocation
 * after a warm-up call with the same or a larger mask and set count; a CUDA graph replay reads the formulations from
 * the captured array).
 * Replaces: PathOptimizer::solveWithoutSmoothing (path_optimizer.cpp:87-117) once per path, with that path's
 * FLAGS_optimization_method. */
int pqp_plan_batch_forms(pqp_handle *h, int bounds_mode, int output_mode, int batch,
                         const int32_t *n_points, const pqp_state *ref, const int32_t *map_index,
                         const int32_t *param_index, const int32_t *formulation,
                         const int32_t *n_knots, const double *knots,
                         const double *x_coef, const double *y_coef,
                         const double *x0, const double *end_heading,
                         double output_spacing, int collision_check, int max_out,
                         pqp_state *out_states, int32_t *out_n, int32_t *out_ok,
                         int32_t *status, int32_t *iters, pqp_station_bounds *out_bounds,
                         pqp_stats *stats);
int pqp_plan_batch_device_forms(pqp_handle *h, int bounds_mode, int output_mode,
                                int batch, int total_points, int max_n_points, int n_param_sets,
                                int form_mask,
                                const int32_t *d_n_points, const int32_t *d_offsets,
                                const pqp_state *d_ref, const int32_t *d_map_index,
                                const int32_t *d_param_index, const int32_t *d_formulation,
                                const int32_t *d_knot_offsets, const double *d_knots,
                                const double *d_x_coef, const double *d_y_coef,
                                const double *d_x0, const double *d_end_heading,
                                double output_spacing, int collision_check, int max_out,
                                pqp_state *d_out_states, int32_t *d_out_n, int32_t *d_out_ok,
                                int32_t *d_status, int32_t *d_iters,
                                pqp_station_bounds *d_out_bounds, void *stream, pqp_stats *stats);

#ifdef __cplusplus
} /* extern "C" */
#endif
#endif /* PQP_ENV_H_ */
