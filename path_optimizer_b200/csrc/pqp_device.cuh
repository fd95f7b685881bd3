// pqp_device.cuh -- shared definitions for the batched path-QP kernels (sm_90a).
//
// Hot path being replaced: OsqpSolver::solve() of LiJiangnanBit/path_optimizer
// (reference src/solver/solver.cpp:46-77): QP assembly (solver_kp_as_input.cpp:45-203), the
// OSQP ADMM solve behind osqp-eigen, and getOptimizedPath (solver_kp_as_input.cpp:26-43).
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/pqp.h"
#include "pqp_warp.cuh"

namespace pqp {

// OSQP 0.6.x constants (upstream; see include/pqp.h and DESIGN.md)
constexpr double kOsqpInfty = 1e30;
constexpr double kRhoMin = 1e-6;
constexpr double kRhoMax = 1e6;
constexpr double kRhoEqOverIneq = 1e3;
constexpr double kRhoTol = 1e-4;
constexpr double kMinScaling = 1e-4;
constexpr double kMaxScaling = 1e4;

constexpr int kMaxBand = 16;  // max half-bandwidth of the reduced KKT (keep_control_steps <= 10)

// Device-side snapshot of what the kernels need from pqp_params (plus host-precomputed values).
struct DevParams {
    double d1, d2, d3, d4;
    double w_c, w_cr, w_pq, w_s;     // KP_curvature / curvature_rate / deviation / slack weights
    double kmax;                     // tan(max_steering_angle) / wheel_base
    double k_w_c, k_w_cr, k_w_pq;    // "K" formulation: K_curvature / curvature_rate / deviation weights (solver_k_as_input.cpp:50-53)
    double wheel_base, max_steer;    // "K": steering-angle control (setDynamicMatrix :89-103, bounds :180-183)
    double margin;                   // expected_safety_margin
    int constraint_end_heading;
    double rho, sigma, alpha, eps_abs, eps_rel, eps_prim_inf, eps_dual_inf;
    int max_iter, scaling, check_termination, adaptive_rho, adaptive_rho_interval;
    double adaptive_rho_tolerance;
};

// Problem batch as seen by a kernel: every pointer is a device pointer.
struct BatchView {
    int batch;
    const int32_t *n_points;           // [B]
    const int32_t *offsets;            // [B+1]
    const pqp_state *ref;              // [sum N]
    const pqp_station_bounds *bounds;  // [sum N]
    const double *x0;                  // [B][3]
    const double *end_heading;         // [B]
    const double *max_k = nullptr;     // [sum N] KPC only: ReferencePath::getMaxKList (per station)
    const double *max_kp = nullptr;    // [sum N] KPC only: getMaxKpList; like the reference the solver reads entry j of a path for control j
    pqp_state *out_states;             // [sum N]
    double *out_frenet;                // [sum N][3] or nullptr
    int32_t *status;                   // [B]
    int32_t *iters;                    // [B] or nullptr
    double *workspace;                 // global scratch: 32*sum(N) + 2048*B doubles (kp2_ws_doubles)
    long long *debug;                  // phase-timing dump (PQP_PHASE_TIMING builds only), else nullptr
};


// Host-side snapshot of the flags the KP path reads (solver_kp_as_input.cpp:48-51,111-127,155-158).
inline DevParams dev_params_from(const pqp_params &p) {
    DevParams d;
    d.d1 = p.d1; d.d2 = p.d2; d.d3 = p.d3; d.d4 = p.d4;
    d.w_c = p.KP_curvature_weight; d.w_cr = p.KP_curvature_rate_weight;
    d.w_pq = p.KP_deviation_weight; d.w_s = p.KP_slack_weight;
    d.kmax = tan(p.max_steering_angle) / p.wheel_base;
    d.k_w_c = p.K_curvature_weight; d.k_w_cr = p.K_curvature_rate_weight; d.k_w_pq = p.K_deviation_weight;
    d.wheel_base = p.wheel_base; d.max_steer = p.max_steering_angle;
    d.margin = p.expected_safety_margin;
    d.constraint_end_heading = p.constraint_end_heading;
    d.rho = p.rho; d.sigma = p.sigma; d.alpha = p.alpha;
    d.eps_abs = p.eps_abs; d.eps_rel = p.eps_rel;
    d.eps_prim_inf = p.eps_prim_inf; d.eps_dual_inf = p.eps_dual_inf;
    d.max_iter = p.max_iter; d.scaling = p.scaling; d.check_termination = p.check_termination;
    d.adaptive_rho = p.adaptive_rho; d.adaptive_rho_interval = p.adaptive_rho_interval;
    d.adaptive_rho_tolerance = p.adaptive_rho_tolerance;
    return d;
}

// tools.hpp:24-35 (constraintAngle), iterative form
PQP_DEV double constraint_angle(double a) {
    const double pi = 3.14159265358979323846;
    while (a > pi) a -= 2 * pi;
    while (a < -pi) a += 2 * pi;
    return a;
}

PQP_DEV double limit_scaling(double v) {
    v = v < kMinScaling ? 1.0 : v;
    v = v > kMaxScaling ? kMaxScaling : v;
    return v;
}

PQP_DEV double clampd(double v, double lo, double hi) { return fmin(fmax(v, lo), hi); }
// Same projection for lo <= hi, with the two compares independent of each other (a dependent
// fmin(fmax()) on doubles costs ~50 cycles on sm_90: DSETP + SEL + SEL, twice).
PQP_DEV double clamp2(double v, double lo, double hi) {
    double z = v;
    z = (v < lo) ? lo : z;
    z = (v > hi) ? hi : z;
    return z;
}

// OSQP's rho vector entry for a row with SCALED bounds (El, Eu) [upstream set_rho_vec].
PQP_DEV double rho_bar(double El, double Eu, double rho) {
    if (El < -kOsqpInfty * kMinScaling && Eu > kOsqpInfty * kMinScaling) return kRhoMin;
    if (Eu - El < kRhoTol) return kRhoEqOverIneq * rho;
    return rho;
}

// OSQP is_primal_infeasible on the certificate (||E dy||, u'dy+ + l'dy-, ||D^-1 A'dy||), all in
// unscaled terms (see the kernels): dy is a certificate when it is non-trivial, separates the
// bounds and is (nearly) orthogonal to the range of A.
PQP_DEV bool primal_infeasible(double nrm, double lhs, double cert, double eps) {
    return nrm > eps && lhs < -eps * nrm && cert < eps * nrm;
}

}  // namespace pqp
