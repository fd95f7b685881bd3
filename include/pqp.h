/*
 * pqp.h -- C ABI of the H100-native batched path-QP solver ("pqp").
 *
 * This is the drop-in boundary for the ONE hot path of LiJiangnanBit/path_optimizer:
 *   OsqpSolver::create(type, reference_path, vehicle_state, horizon)->solve(&path)
 *   (reference: include/path_optimizer/solver/solver.hpp:31-36, src/solver/solver.cpp:30-77),
 * reached from PathOptimizer::optimizePath (src/path_optimizer/path_optimizer.cpp:180-186).
 *
 * Everything here is plain C: POD structs, pointers and sizes.  No torch / Eigen /
 * STL types cross this boundary, nothing throws, the caller owns every buffer it
 * passes and the library retains no pointer after a call returns.
 *
 * Each entry point cites the reference interface it replaces (file:line relative to
 * the reference tree).
 */
#ifndef PQP_H_
#define PQP_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PQP_ABI_VERSION 1

/* ------------------------------------------------------------------------- */
/* Records (mirror the reference's I/O types field for field).               */
/* ------------------------------------------------------------------------- */

/* PathOptimizationNS::State, include/path_optimizer/data_struct/data_struct.hpp:13-30.
 * z = heading, k = curvature, s = arc length; v, a only read by the "KPC" limits. */
typedef struct pqp_state {
    double x, y, z, k, s, v, a;
} pqp_state;

/* CoveringCircleBounds::SingleCircleBounds {ub, lb}, data_struct.hpp:72-91
 * (ub = left clearance, lb = right clearance, lateral offsets of circle centre j).
 * Only ub/lb are read by the QP (solver_kp_as_input.cpp:166-187); x/y/heading of the
 * reference struct are display-only and not part of the boundary. */
typedef struct pqp_station_bounds {
    double c0_ub, c0_lb;
    double c1_ub, c1_lb;
    double c2_ub, c2_lb;
    double c3_ub, c3_lb;
} pqp_station_bounds;

/* Snapshot of the gflags the hot path reads at call time (src/config/planning_flags.cpp)
 * plus the OSQP settings the reference leaves at library defaults (solver.cpp:48-49).
 * The reference reads mutable process globals inside the solve; a batched solver must
 * snapshot them once per handle. */
typedef struct pqp_params {
    /* vehicle geometry, planning_flags.cpp:18-43 */
    double car_width;              /* 2.0  */
    double car_length;             /* 4.9  */
    double safety_margin;          /* 0.0  */
    double wheel_base;             /* 2.85 */
    double rear_axle_to_center;    /* 1.45 */
    double max_steering_angle;     /* 30 deg in rad */
    double mu;                     /* 0.4  (KPC limits) */
    double max_curvature_rate;     /* 0.1  (KPC limits) */
    /* derived by updateConfig(), planning_flags.cpp:8-14 */
    double circle_radius;
    double d1, d2, d3, d4;
    /* weights, planning_flags.cpp:102-116 */
    double K_curvature_weight;     /* 50  */
    double K_curvature_rate_weight;/* 200 */
    double K_deviation_weight;     /* 0   */
    double KP_curvature_weight;    /* 10  */
    double KP_curvature_rate_weight;/* 200 */
    double KP_deviation_weight;    /* 0   */
    double KP_slack_weight;        /* 3   */
    double expected_safety_margin; /* 1.3 */
    int32_t constraint_end_heading;/* true */
    /* OSQP settings: library defaults of the OSQP 0.6.x the reference links
     * (solver.cpp:48-49 only changes verbosity and warm start). */
    double rho;                    /* 0.1  */
    double sigma;                  /* 1e-6 */
    double alpha;                  /* 1.6  */
    double eps_abs;                /* 1e-3 */
    double eps_rel;                /* 1e-3 */
    double eps_prim_inf;           /* 1e-4 */
    double eps_dual_inf;           /* 1e-4 */
    int32_t max_iter;              /* 4000 */
    int32_t scaling;               /* 10 Ruiz sweeps */
    int32_t check_termination;     /* 25 */
    int32_t adaptive_rho;          /* 1 */
    /* OSQP's default interval (0 = automatic) is chosen from wall-clock timing -- the first
     * iteration at which solve time exceeds 0.4 x setup time, rounded to a multiple of
     * check_termination, at least 25 -- and is therefore not reproducible.  Here it is an
     * explicit iteration count.  Default 25: for this problem class (KKT dimension ~1.7k-4.5k,
     * nnz(L) ~ 2.5 per column) OSQP's setup costs roughly 20-30 ADMM iterations, so its rule
     * lands on 25 (see DESIGN.md).  100 = OSQP's fallback when built without PROFILING. */
    int32_t adaptive_rho_interval; /* 25 */
    double adaptive_rho_tolerance; /* 5 */
    int32_t reserved_[3];
} pqp_params;

/* Formulations = the three type strings of OsqpSolver::create (solver.cpp:34-43). */
enum pqp_formulation {
    PQP_FORM_KP  = 0,   /* "KP"  SolverKpAsInput            (default, planning_flags.cpp:93) */
    PQP_FORM_K   = 1,   /* "K"   SolverKAsInput                                              */
    PQP_FORM_KPC = 2    /* "KPC" SolverKpAsInputConstrained                                  */
};

/* Per-problem status: the OSQP status_val the reference would have seen.  The reference's
 * bool is (status == PQP_SOLVED): osqp-eigen's solve() returns false for anything else. */
enum pqp_status {
    PQP_SOLVED                 = 1,
    PQP_SOLVED_INACCURATE      = 2,
    PQP_MAX_ITER_REACHED       = -2,
    PQP_PRIMAL_INFEASIBLE      = -3,
    PQP_DUAL_INFEASIBLE        = -4,
    PQP_NON_CVX                = -7,
    PQP_UNSOLVED               = -10,
    PQP_INVALID_PROBLEM        = -100  /* osqp_setup would have refused: l > u, n < 2, ... */
};
/* Open corridor sides.  A circle bound of +-1e30 (OSQP_INFTY) or beyond is accepted on a box row.  On the open side of
 * ONE row of a slack pair (KP: c1_lb or c3_lb opened below, c1_ub or c3_ub above; K: c1; KPC: c2) it makes that row free
 * while its partner is not: OSQP would weigh the two rows differently (RHO_MIN against rho), and the thread-per-station
 * kernels, which eliminate the slack on the premise of equal weights, refuse such a path with PQP_INVALID_PROBLEM
 * (0 iterations, NaN output).  Both rows of a pair opened together are solved. */
/* Station spacing.  The stations' s need not be evenly spaced; these are refused with PQP_INVALID_PROBLEM (0 iterations,
 * NaN output):
 *  - a NaN or infinite s, in every formulation.  This is a stated rule: the reference would hand the resulting NaN /
 *    inf matrix entries to OSQP;
 *  - "KP" and "KPC": a zero-length interval anywhere (a duplicate waypoint, or every station at one s).  The reference's
 *    dynamics-row constant ds (c - a ref - b ref_kp) with ref_kp = dkappa / ds (solver_kp_as_input.cpp:86-97) is NaN
 *    there, and osqp_setup refuses l = u = NaN.  "K" has no such division and solves zero-length intervals.
 * A negative interval is solved as the reference would solve it. */

/* Library-level return codes (never exceptions). */
enum pqp_rc {
    PQP_OK = 0,
    PQP_ERR_ARG = 1,          /* null pointer, negative size, unknown formulation */
    PQP_ERR_CAPACITY = 2,     /* batch / station count exceeds what the handle was created for */
    PQP_ERR_CUDA = 3,         /* a CUDA runtime call failed; see pqp_last_error() */
    PQP_ERR_UNSUPPORTED = 4   /* e.g. n_points too large for one SM's shared memory */
};

/* Timing/diagnostics filled by the solve calls (all optional: pass NULL). */
typedef struct pqp_stats {
    float h2d_ms;             /* host->device copies (host-buffer entry point only) */
    float kernel_ms;          /* solve kernel(s), CUDA events on the handle's stream */
    float d2h_ms;
    int64_t h2d_bytes;
    int64_t d2h_bytes;
    int32_t kernel_launches;  /* number of this library's kernels launched by the call */
    int32_t max_iters;        /* max ADMM iterations over the batch */
    int64_t total_iters;      /* sum of ADMM iterations over the batch */
    int32_t n_solved;         /* problems with status == PQP_SOLVED */
    int32_t reserved_;
} pqp_stats;

typedef struct pqp_handle pqp_handle;

/* ------------------------------------------------------------------------- */
/* Entry points                                                               */
/* ------------------------------------------------------------------------- */

/* Fill *p with the reference's flag defaults (planning_flags.cpp:18-119) and run
 * pqp_params_update_config on it.  Replaces: gflags DEFINE_* + updateConfig(). */
int pqp_params_default(pqp_params *p);

/* Recompute circle_radius and d1..d4 from the geometry fields.
 * Replaces: updateConfig(), planning_flags.cpp:8-14 (called from the PathOptimizer
 * constructor, path_optimizer.cpp:30). */
int pqp_params_update_config(pqp_params *p);

/* keep_control_steps_ of one path, computed in double exactly as the reference does:
 * reference_interval_ = max ds over the first <= 9 intervals (solver.cpp:21-27), then
 * max(int(1.2 / reference_interval_), 1) (solver_kp_as_input.cpp:17).  KPC fixes it at 4
 * (solver_kp_as_input_constrained.cpp:17); K has no hold (returns 1).  The maximum has std::max semantics, so a NaN
 * interval is skipped; a maximum of 0 (or one so small that 1.2 / it exceeds INT_MAX, where the reference's int() is
 * undefined) gives INT_MAX, which no kernel class takes; paths of fewer than 2 stations give 1.  The kernels, the
 * device dispatch and the test oracle all follow this one rule. */
int pqp_keep_control_steps(int formulation, const pqp_state *ref, int n_points);

/* Number of QP variables / constraints for (formulation, n_points, keep):
 * solver_kp_as_input.cpp:18-23, solver_k_as_input.cpp:18-19,
 * solver_kp_as_input_constrained.cpp:18-24. Returns PQP_ERR_ARG on bad input. */
int pqp_problem_size(int formulation, int n_points, int keep, int *n_var, int *n_con);

/* Create a solver bound to CUDA device `device`, able to take up to `max_batch` paths and
 * `max_total_points` stations (sum over the batch) per call.  Fails (PQP_ERR_CUDA) when no
 * CUDA device / kernel image is usable -- there is no CPU fallback.
 * Replaces: OsqpSolver::create (solver.cpp:30-44) + the OsqpEigen::Solver member
 * (solver.hpp:52) that every reference solve constructs from scratch. */
int pqp_create(pqp_handle **out, const pqp_params *params, int device,
               int max_batch, int max_total_points);

void pqp_destroy(pqp_handle *h);

/* Replace the parameter snapshot of an existing handle (the reference re-reads FLAGS_* on
 * every solve, e.g. solver_kp_as_input.cpp:48-51): pqp_set_param_sets(h, 1, params). */
int pqp_set_params(pqp_handle *h, const pqp_params *params);

/* Most parameter sets one handle holds. */
#define PQP_MAX_PARAM_SETS 64

/* Replace the handle's parameter sets with `n_sets` (1..PQP_MAX_PARAM_SETS) snapshots, so that one call can batch paths
 * of several vehicles, weight sweeps or solver tolerances (pqp_solve_batch_sets, pqp_solve_batch_device_dispatch_sets,
 * pqp_plan_batch_sets, pqp_plan_batch_device_sets: one set index per path).  Every set is given already run through
 * pqp_params_update_config, as for pqp_set_params.  Every argument is checked before anything changes: a bad one returns
 * PQP_ERR_ARG and leaves the previous sets in place.  Synchronous; no caller pointer is kept.  The params given to
 * pqp_create are set 0; the entries without a set index, and the single-stage entries of pqp_env.h, read set 0.
 * Every stage takes the sets by value at launch: a CUDA graph captured before this call keeps, at every stage, the sets
 * it was captured with; capture again to follow the new ones.
 * Replaces: the FLAGS_* globals the reference reads at call time (solver_kp_as_input.cpp:48-51, 111-127, 155-158;
 * reference_path_impl.cpp:203-235; updateConfig() from the PathOptimizer constructor), one value set per path. */
int pqp_set_param_sets(pqp_handle *h, int n_sets, const pqp_params *sets);

/* Solve `batch` independent path QPs.  HOST buffers; H2D / D2H copies happen inside.
 *
 *   n_points[b]      stations of path b (>= 2); paths are concatenated in `ref`/`bounds`/outputs
 *   ref              [sum n_points] reference states  (ReferencePath::getReferenceStates())
 *   bounds           [sum n_points] clearance bounds  (ReferencePath::getBounds())
 *   x0               [batch][3] = {init offset, init heading error, start curvature}
 *                    (VehicleState::getInitError(), getStartState().k; solver_kp_as_input.cpp:143-147)
 *   end_heading      [batch] goal heading, VehicleState::getEndState().z (:196)
 *   max_k, max_kp    [sum n_points] each, KPC only (ReferencePath::getMaxKList / getMaxKpList, one entry per
 *                    station; like the reference the solver reads the first ch entries of a path's max_kp); else NULL.
 *                    pqp_update_limits (pqp_env.h) derives them from the v, a fields of the reference states.
 * All three formulations are assembled inside thread-per-station kernel classes ("KP" up to 408 stations per path,
 * "KPC" up to 256, "K" up to 416; a longer path reports PQP_INVALID_PROBLEM for itself).
 *   out_states       [sum n_points] optimized path: x, y, z(heading), k, s filled exactly as
 *                    getOptimizedPath does (solver_kp_as_input.cpp:26-43); v = a = 0
 *   out_frenet       optional [sum n_points][3] = (e_y, e_phi, kappa) raw QP solution
 *   status           [batch] pqp_status; the reference's `bool solve()` is status == PQP_SOLVED
 *   iters            optional [batch] ADMM iterations used
 *
 * Replaces: OsqpSolver::solve (solver.cpp:46-77) called once per path. */
int pqp_solve_batch(pqp_handle *h, int formulation, int batch,
                    const int32_t *n_points,
                    const pqp_state *ref,
                    const pqp_station_bounds *bounds,
                    const double *x0,
                    const double *end_heading,
                    const double *max_k,
                    const double *max_kp,
                    pqp_state *out_states,
                    double *out_frenet,
                    int32_t *status,
                    int32_t *iters,
                    pqp_stats *stats);

/* Same solve with every array already resident in DEVICE memory of the handle's device
 * (e.g. produced by the clearance kernel or owned by the host framework).  `offsets` is the
 * exclusive prefix sum of n_points with offsets[batch] = sum.  The host cannot see the device-side
 * n_points, so the caller states upper bounds used to size shared memory: `max_n_points` >= every
 * n_points[b], and `min_keep` <= keep_control_steps <= `max_keep` for every path (pass 0, 0 for
 * "unknown": 1..4 is assumed).  ONE kernel class is chosen that takes every (n_points, keep) inside those bounds
 * (PQP_ERR_UNSUPPORTED when no single class does: tighten them, or use pqp_solve_batch_device_classes); only a path
 * that exceeds the stated bounds reports PQP_INVALID_PROBLEM.  Asynchronous on `stream`
 * (a cudaStream_t, or NULL for the handle's own stream); no host synchronisation is done
 * unless `stats` is non-NULL.  Formulations: "KP", and "KPC" (d_max_k / d_max_kp then required, every path <= 256
 * stations; keep bounds are ignored: KPC holds a control for 4 stations), "K" (every path <= 416 stations; keep bounds
 * ignored: one steering control per station).
 * No reference counterpart (the reference has no device). */
int pqp_solve_batch_device(pqp_handle *h, int formulation, int batch, int total_points,
                           int max_n_points, int min_keep, int max_keep,
                           const int32_t *d_n_points, const int32_t *d_offsets,
                           const pqp_state *d_ref,
                           const pqp_station_bounds *d_bounds,
                           const double *d_x0,
                           const double *d_end_heading,
                           const double *d_max_k,
                           const double *d_max_kp,
                           pqp_state *d_out_states,
                           double *d_out_frenet,
                           int32_t *d_status,
                           int32_t *d_iters,
                           void *stream,
                           pqp_stats *stats);

/* Device-resident solve of a MIXED-LENGTH batch: as pqp_solve_batch_device, but the caller passes HOST copies of the
 * per-path station counts (`h_n_points`, equal to the device-side d_n_points) and keep_control_steps (`h_keep`, from
 * pqp_keep_control_steps), so that every path runs on the kernel class of its own (length, keep) -- what
 * pqp_solve_batch does for host buffers -- instead of one class sized for the longest path.  The classes are launched
 * on internal lanes forked from / joined into `stream`, the class of the longest paths first (BASELINE config 5:
 * "length-bucketed").  The class plan is cached while (h_n_points, h_keep) stay the same; when they change the call
 * synchronises `stream` once before re-planning.  No reference counterpart. */
int pqp_solve_batch_device_classes(pqp_handle *h, int formulation, int batch, int total_points,
                                   const int32_t *h_n_points, const int32_t *h_keep,
                                   const int32_t *d_n_points, const int32_t *d_offsets,
                                   const pqp_state *d_ref,
                                   const pqp_station_bounds *d_bounds,
                                   const double *d_x0,
                                   const double *d_end_heading,
                                   const double *d_max_k,
                                   const double *d_max_kp,
                                   pqp_state *d_out_states,
                                   double *d_out_frenet,
                                   int32_t *d_status,
                                   int32_t *d_iters,
                                   void *stream,
                                   pqp_stats *stats);

/* Device-resident solve of a MIXED-LENGTH batch whose station counts exist on the device only: the arguments of
 * pqp_solve_batch_device, and every path runs on the kernel class pqp_solve_batch would choose for it, with the same
 * results bit for bit.  A dispatch kernel reads d_n_points, computes keep_control_steps from d_ref exactly as
 * pqp_keep_control_steps does, looks the class up in the table pqp_create built with the host's own selection and sorts
 * the paths into per-class launch order (longest first); every class the bounds can reach is then launched on internal
 * lanes forked from / joined into `stream`.  The bounds only narrow what is launched: `max_n_points` >= every
 * n_points[b] and, for "KP", `min_keep` <= keep_control_steps <= `max_keep` (each 0 = unknown).  A path outside the
 * stated bounds reports PQP_INVALID_PROBLEM (0 iterations, NaN states); `total_points` must be offsets[batch].
 * Asynchronous on `stream`; no host synchronisation unless `stats` is non-NULL; no allocation: after one warm-up call
 * the call can be captured into a CUDA graph.  One call in flight per handle.  pqp_set_order_hint is not applied (the
 * order inside a class is longest path first).  No reference counterpart. */
int pqp_solve_batch_device_dispatch(pqp_handle *h, int formulation, int batch, int total_points,
                                    int max_n_points, int min_keep, int max_keep,
                                    const int32_t *d_n_points, const int32_t *d_offsets,
                                    const pqp_state *d_ref,
                                    const pqp_station_bounds *d_bounds,
                                    const double *d_x0,
                                    const double *d_end_heading,
                                    const double *d_max_k,
                                    const double *d_max_kp,
                                    pqp_state *d_out_states,
                                    double *d_out_frenet,
                                    int32_t *d_status,
                                    int32_t *d_iters,
                                    void *stream,
                                    pqp_stats *stats);

/* pqp_solve_batch and pqp_solve_batch_device_dispatch over the handle's parameter sets (pqp_set_param_sets): the same
 * arguments plus one set index per path, on the host (`param_index`) or on the device (`d_param_index`), both int32
 * [batch].  Path b is solved with set param_index[b]: its results equal, bit for bit, those of a handle whose only set
 * is that one.  A NULL index means set 0 for every path: pqp_solve_batch and pqp_solve_batch_device_dispatch are these
 * entries with a NULL index.  An index outside [0, n_sets), or for the device entry at or past `n_param_sets`, makes only
 * that path report PQP_INVALID_PROBLEM (0 iterations, NaN states); the index is checked before the sets are read, and
 * no other path's results change.
 *   n_param_sets   device entry: an upper bound on the indices used (0: the handle's set count).  Like max_n_points it
 *                  bounds what is launched: one grid per (set, kernel class) pair the bounds reach.
 * The host entry plans one launch segment per (set, class), longest path first inside a segment (pqp_set_order_hint and
 * the input-derived order still apply inside a segment).  The device entry keeps every promise of
 * pqp_solve_batch_device_dispatch (asynchronous, no allocation after a warm-up call with the same or a larger
 * n_param_sets, capturable); its sort needs device scratch that grows with n_param_sets.  With PQP_GENERIC_K /
 * PQP_GENERIC_KPC set, a non-NULL index returns PQP_ERR_UNSUPPORTED.
 * Replaces: OsqpSolver::solve (solver.cpp:46-77) once per path, with that path's FLAGS_*. */
int pqp_solve_batch_sets(pqp_handle *h, int formulation, int batch,
                         const int32_t *n_points,
                         const pqp_state *ref,
                         const pqp_station_bounds *bounds,
                         const double *x0,
                         const double *end_heading,
                         const double *max_k,
                         const double *max_kp,
                         const int32_t *param_index,
                         pqp_state *out_states,
                         double *out_frenet,
                         int32_t *status,
                         int32_t *iters,
                         pqp_stats *stats);
int pqp_solve_batch_device_dispatch_sets(pqp_handle *h, int formulation, int batch, int total_points,
                                         int max_n_points, int min_keep, int max_keep, int n_param_sets,
                                         const int32_t *d_n_points, const int32_t *d_offsets,
                                         const pqp_state *d_ref,
                                         const pqp_station_bounds *d_bounds,
                                         const double *d_x0,
                                         const double *d_end_heading,
                                         const double *d_max_k,
                                         const double *d_max_kp,
                                         const int32_t *d_param_index,
                                         pqp_state *d_out_states,
                                         double *d_out_frenet,
                                         int32_t *d_status,
                                         int32_t *d_iters,
                                         void *stream,
                                         pqp_stats *stats);

/* pqp_solve_batch_sets and pqp_solve_batch_device_dispatch_sets with one formulation per path in place of the scalar:
 * `formulation` (host) or `d_formulation` (device), int32 [batch] of PQP_FORM_* values, so that one call can mix
 * "KP", "K" and "KPC" paths (e.g. vehicles configured for "KPC" beside vehicles on "KP", or the three formulations of
 * the same scenes side by side).  The array is required.
 *   Path b's results -- status, iterations, states and Frenet states -- equal, bit for bit, those the _sets entry gives
 *   it when called with formulation = formulation[b], for any mix of parameter sets and lengths in the batch.
 *   A formulation outside {0, 1, 2}, or for the device entry outside `form_mask`, makes only that path report
 *   PQP_INVALID_PROBLEM (0 iterations, NaN states); no other path changes.  Set indices keep their rules.
 *   form_mask      device entry: bitmask of 1 << PQP_FORM_*, 0 = all three.  Like n_param_sets it only bounds what is
 *                  launched: one grid per reachable (set, kernel class) pair of the formulations in the mask.
 *   max_n_points   device entry: as for the _sets entry, for every formulation (0: unknown); each path stays limited
 *                  by its own formulation's classes ("KPC" 256 stations, "KP" 408 at keep 3..4, "K" 416).
 *   max_k, max_kp  the "KPC" limits: PQP_ERR_ARG when NULL and some path is "KPC" (host entry) or the mask holds
 *                  "KPC" (device entry).  "KP" and "K" paths do not read them.
 * The host entry plans one launch segment per (set, kernel class), with each path on the class of its own formulation.
 * The device entry keeps every promise of pqp_solve_batch_device_dispatch_sets: asynchronous on `stream`, no host
 * synchronisation unless `stats` is non-NULL, no allocation after a warm-up call with the same or a larger mask and set
 * count, capturable in a CUDA graph (a replay reads the formulations from the captured array).  Its sort needs device
 * scratch of its own.  With PQP_GENERIC_K / PQP_GENERIC_KPC set and a path of that formulation, the host entry
 * returns PQP_ERR_UNSUPPORTED.
 * Replaces: OsqpSolver::create(FLAGS_optimization_method, ...) + solve (solver.cpp:30-77) once per path, with that
 * path's FLAGS_optimization_method. */
int pqp_solve_batch_forms(pqp_handle *h, int batch,
                          const int32_t *n_points,
                          const pqp_state *ref,
                          const pqp_station_bounds *bounds,
                          const double *x0,
                          const double *end_heading,
                          const double *max_k,
                          const double *max_kp,
                          const int32_t *param_index,
                          const int32_t *formulation,
                          pqp_state *out_states,
                          double *out_frenet,
                          int32_t *status,
                          int32_t *iters,
                          pqp_stats *stats);
int pqp_solve_batch_device_dispatch_forms(pqp_handle *h, int batch, int total_points,
                                          int max_n_points, int min_keep, int max_keep, int n_param_sets,
                                          int form_mask,
                                          const int32_t *d_n_points, const int32_t *d_offsets,
                                          const pqp_state *d_ref,
                                          const pqp_station_bounds *d_bounds,
                                          const double *d_x0,
                                          const double *d_end_heading,
                                          const double *d_max_k,
                                          const double *d_max_kp,
                                          const int32_t *d_param_index,
                                          const int32_t *d_formulation,
                                          pqp_state *d_out_states,
                                          double *d_out_frenet,
                                          int32_t *d_status,
                                          int32_t *d_iters,
                                          void *stream,
                                          pqp_stats *stats);

/* Last error text for this thread (CUDA error strings etc.); never NULL. */
/* Launch-order hint for the next solves of a batch of `batch` paths: expected ADMM iterations per path, e.g. the
 * `iters` the previous planning cycle reported for the same candidates.  Inside a kernel class the paths are then
 * launched longest expected work (stations x iterations) first instead of longest path first, which shortens the tail of
 * a launch whose paths outnumber the resident CTA slots only a few times (1024 x 100 on one H100: 5.16 ms in index order,
 * 4.43 ms with an exact hint; DESIGN.md section 6).  Results do not depend on the order.  NULL or batch 0 clears
 * the hint; a hint whose length differs from a call's batch is ignored by that call.  No reference counterpart. */
int pqp_set_order_hint(pqp_handle *h, int batch, const int32_t *expected_iters);

const char *pqp_last_error(void);

/* "pqp <abi> sm_90a <build info>" */
const char *pqp_version(void);

/* Largest n_points a path may have on this device (one path must fit one SM's shared memory; longer paths report
 * PQP_INVALID_PROBLEM).  The limit depends on keep_control_steps: pqp_max_points_keep gives it for one value
 * (1..10; e.g. 408 at keep = 3 on the thread-per-station classes, then the one-warp kernel up to 414), pqp_max_points
 * the minimum over keep = 1..10, i.e. a length every spacing can take.  KPC: 256 stations, K: 416 (their largest
 * classes; keep does not matter for them). */
int pqp_max_points(pqp_handle *h, int formulation);
int pqp_max_points_keep(pqp_handle *h, int formulation, int keep);

/* Diagnostics (no device needed): which kernel class the library selects.  pqp_class_info: for ONE path of
 * (n_points, keep) as pqp_solve_batch / pqp_solve_batch_device_classes / pqp_plan_batch choose it -- index into the
 * class table (order of preference), CTA size and dynamic shared memory; PQP_ERR_UNSUPPORTED when no class takes the
 * path (it would report PQP_INVALID_PROBLEM).  pqp_device_class_info: the single class pqp_solve_batch_device picks for
 * the caller's bounds.  smem_optin = the device's opt-in shared memory per block (0: H100's 232448). */
int pqp_class_info(int n_points, int keep, int smem_optin, int *variant, int *threads, int64_t *smem_bytes);
int pqp_class_info_kpc(int n_points, int smem_optin, int *variant, int *threads, int64_t *smem_bytes);   /* the same for a "KPC" path (keep_control_steps is 4); PQP_ERR_UNSUPPORTED: longer than the largest KPC class (256 stations) */
int pqp_class_info_form(int formulation, int n_points, int keep, int smem_optin, int *variant, int *threads, int64_t *smem_bytes);   /* any formulation ("K": keep ignored) */
const char *pqp_class_name(int variant);   /* kernel name of a class-table index, as profilers print it ("" if out of range) */
int pqp_device_class_info(int max_n_points, int min_keep, int max_keep, int smem_optin, int *variant, int *threads,
                          int64_t *smem_bytes);
/* The class table the device dispatch looks paths up in (pqp_solve_batch_device_dispatch), built by the same selection
 * as pqp_class_info_form: 11 rows (keep_control_steps 1..10, then keep > 10) of *ncols class indices each, entry
 * [keep - 1][n_points]; the last column is one station past the longest path any class of the formulation takes and
 * stands for every longer path.  table = NULL: only *ncols.  PQP_ERR_CAPACITY when `capacity` < 11 * *ncols. */
int pqp_class_table(int formulation, int smem_optin, int8_t *table, int capacity, int *ncols);

#ifdef __cplusplus
} /* extern "C" */
#endif
#endif /* PQP_H_ */
