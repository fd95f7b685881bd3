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

#ifdef __cplusplus
} /* extern "C" */
#endif
#endif /* PQP_ENV_H_ */
