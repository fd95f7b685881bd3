/*
 * pqp_oracle.h -- CPU ORACLE (test infrastructure, NOT product code).
 *
 * A plain-C, fp64, single-path restatement of the reference hot path
 *   OsqpSolver::solve()  (reference src/solver/solver.cpp:46-77)
 * = QP assembly (src/solver/solver_kp_as_input.cpp, solver_k_as_input.cpp,
 *   solver_kp_as_input_constrained.cpp) + the OSQP ADMM algorithm the reference calls through
 *   osqp-eigen + state extraction (getOptimizedPath).
 *
 * PARITY UNPINNED: the reference ships no tests, golden vectors or known-answer fixtures for this
 * path (SURVEY.md section 4 / 8c) and its solver dependency -- OSQP (github.com/oxfordcontrol/osqp)
 * and osqp-eigen (github.com/robotology/osqp-eigen), both cloned un-pinned at HEAD by
 * scripts/install_deps.sh:102,116, OSQP 0.6.x era -- is not vendored under /root/reference and is
 * not installable here (no network, no Eigen).  The ADMM part below therefore restates OSQP's
 * PUBLISHED algorithm (Stellato et al., "OSQP: an operator splitting solver for quadratic
 * programs", Math. Prog. Comp. 2020, and the documented behaviour of OSQP 0.6.x: Ruiz
 * equilibration, rho vector, termination and adaptive-rho rules); it is cross-checked against an
 * independent numpy/scipy twin (oracle/twin.py) and a KKT optimality certificate, not against a
 * real OSQP binary.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may
 * use this code, and only as the checker / the CPU baseline.
 */
#ifndef PQP_ORACLE_H_
#define PQP_ORACLE_H_

#include "../include/pqp.h"
#include "../include/pqp_env.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Sparse QP in triplet form:  min 1/2 x'Px + q'x  s.t.  l <= Ax <= u.
 * P holds the UPPER triangle only (i <= j), as osqp-eigen passes it to OSQP. */
typedef struct oqp_problem {
    int n, m;
    int p_nnz, a_nnz;
    int *p_i, *p_j; double *p_v;
    int *a_i, *a_j; double *a_v;
    double *q, *l, *u;
} oqp_problem;

typedef struct oqp_info {
    int status;            /* pqp_status */
    int iters;
    int rho_updates;
    double rho_final;
    double pri_res, dua_res;
    double obj_val;
    int kkt_n, kkt_lnz;    /* size of the KKT system and nnz(L) */
    double margin;         /* the deciding check(s) -- the one that stopped the run, or the last one and the 10x
                              re-check at max_iter: smallest relative gap |a - b| / max(|a|, |b|) of a residual or
                              certificate value a from its threshold b (0 when nothing was checked) */
} oqp_info;

/* Flag defaults, restated from src/config/planning_flags.cpp:18-119 + updateConfig() :8-14,
 * and OSQP 0.6.x default settings. */
void oracle_params_default(pqp_params *p);

/* keep_control_steps_ (solver.cpp:21-27, solver_kp_as_input.cpp:17,
 * solver_kp_as_input_constrained.cpp:17). */
int oracle_keep_control_steps(int formulation, const pqp_state *ref, int n);

/* Assemble the QP of one path exactly as the reference's setHessianMatrix /
 * setConstraintMatrix do (structural entries are kept even when numerically zero; Eigen's
 * sparseView() would drop exact zeros, which does not change any product).
 * max_k/max_kp are read for PQP_FORM_KPC only.  Returns NULL on bad input. */
oqp_problem *oracle_assemble(const pqp_params *prm, int formulation, int n,
                             const pqp_state *ref, const pqp_station_bounds *bounds,
                             const double x0[3], double end_heading,
                             const double *max_k, const double *max_kp);
void oracle_problem_free(oqp_problem *qp);

/* OSQP-algorithm restatement on a generic sparse QP.  x (n) and y (m) receive the unscaled
 * primal/dual solution (NaN when the status carries no solution, as OSQP does).
 * trace, if non-NULL, receives the UNSCALED primal iterate after every check_termination
 * interval: trace[(k-1)*n .. k*n) = x at iteration k*check_termination, up to trace_cap rows. */
int oracle_osqp_solve(const pqp_params *prm, const oqp_problem *qp,
                      double *x, double *y, oqp_info *info,
                      double *trace, int trace_cap);

/* getOptimizedPath (solver_kp_as_input.cpp:26-43, solver_k_as_input.cpp:22-44,
 * solver_kp_as_input_constrained.cpp:26-43): QP solution -> n states; frenet (optional)
 * gets (e_y, e_phi, k) per station. */
void oracle_extract(int formulation, int n, const pqp_state *ref, const double *x,
                    pqp_state *out, double *frenet);

/* One whole hot-path call: assemble -> solve -> extract.  Returns the pqp_status. */
int oracle_solve_path(const pqp_params *prm, int formulation, int n,
                      const pqp_state *ref, const pqp_station_bounds *bounds,
                      const double x0[3], double end_heading,
                      const double *max_k, const double *max_kp,
                      pqp_state *out, double *frenet, oqp_info *info);

/* Batch driver used as the CPU baseline: same argument layout as pqp_solve_batch, run on
 * `threads` host threads (pthreads, static partition).  Returns wall seconds spent. */
double oracle_solve_batch(const pqp_params *prm, int formulation, int batch,
                          const int32_t *n_points, const pqp_state *ref,
                          const pqp_station_bounds *bounds, const double *x0,
                          const double *end_heading, const double *max_k, const double *max_kp,
                          pqp_state *out, double *frenet, int32_t *status, int32_t *iters,
                          int threads);

/* ---- stages either side of the QP (pqp_oracle_env.c; rows N2-N4 of the scope table) ---- */

/* Map::getObstacleDistance / isInside, src/tools/Map.cpp:16-26 over grid_map geometry. */
int oracle_map_inside(const pqp_distance_map *m, double x, double y);
double oracle_map_distance(const pqp_distance_map *m, double x, double y);

/* tk::spline::set_points / operator() / deriv, src/tools/spline.cpp:161-318 (re-derived). */
int oracle_spline_fit(int n, const double *t, const double *y, double *coef);
double oracle_spline_eval(int n, const double *t, const double *coef, int order, double at);

/* getClearanceWithDirectionStrict, reference_path_impl.cpp:283-472; out = {left, right}. */
void oracle_clearance_strict(const pqp_params *prm, const pqp_distance_map *map, double sx,
                             double sy, double sz, double out[2]);

/* updateBoundsImproved / updateBounds, reference_path_impl.cpp:142-201 / 237-281. */
int oracle_update_bounds(const pqp_params *prm, const pqp_distance_map *map, int mode, int n,
                         const pqp_state *ref, int n_knots, const double *knots,
                         const double *x_coef, const double *y_coef, pqp_station_bounds *out);

/* CarGeometry circles + CollisionChecker, car_geometry.cpp:38-57, collision_checker.cpp:17-59. */
void oracle_car_circles(const pqp_params *prm, double c[7][3]);
/* ReferencePathImpl::updateLimits (reference_path_impl.cpp:203-235) */
void oracle_update_limits(const pqp_params *prm, int from_spline, int n, const pqp_state *ref, double *max_k, double *max_kp);
int oracle_state_collision_free(const pqp_params *prm, const pqp_distance_map *map,
                                const pqp_state *s);

/* optimizePath tails, path_optimizer.cpp:191-202 and :203-230. */
int oracle_finish_raw(const pqp_params *prm, const pqp_distance_map *map, int n, pqp_state *path,
                      int collision_check, int *n_kept);
int oracle_densify(const pqp_params *prm, const pqp_distance_map *map, int n, const pqp_state *path,
                   double spacing, int collision_check, int max_out, pqp_state *out, int *n_out);

/* solveWithoutSmoothing, path_optimizer.cpp:87-117, one path. */
int oracle_plan_path(const pqp_params *prm, const pqp_distance_map *map, int formulation,
                     int bounds_mode, int output_mode, int n, const pqp_state *ref, int n_knots,
                     const double *knots, const double *x_coef, const double *y_coef,
                     const double x0[3], double end_heading, double spacing, int collision_check,
                     int max_out, pqp_state *out, int *n_out, int *status, int *iters,
                     pqp_station_bounds *bounds_out);

#ifdef __cplusplus
}
#endif
#endif
