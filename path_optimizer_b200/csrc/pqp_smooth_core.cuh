// pqp_smooth_core.cuh -- per-thread device functions of pqp_smooth_reference_device and
// pqp_smooth_reference_tension_device: the B-spline pre-pass of ReferencePathSmoother::bSpline, the resampling of
// segmentRawReference, the TENSION2 smoothing QP of TensionSmoother2::osqpSmooth and the TENSION smoothing QP of
// TensionSmoother::osqpSmooth, assembled in the band order of the generic core (pqp_gen_core.cuh, 4-unknown
// separators for TENSION2, 9-unknown separators for TENSION).  Like pqp_corridor_core.cuh, every function is a straight per-thread restatement, so the test-only host
// build (-DPQP_HOST_EMU, tests/emu/) calls them in a loop where the kernel spreads them over a warp.
//
// Reference behaviour being replaced (file:line in the reference tree):
//   ReferencePathSmoother::solve, input check          src/reference_path_smoother/reference_path_smoother.cpp:36-39
//   ReferencePathSmoother::bSpline                     :498-532
//   ReferencePathSmoother::segmentRawReference         :50-88
//   TensionSmoother2::osqpSmooth / setHessianMatrix / setConstraintMatrix / setGradient
//                                                      src/reference_path_smoother/tension_smoother_2.cpp:163-301
//   TensionSmoother::osqpSmooth / setHessianMatrix / setConstraintMatrix
//                                                      src/reference_path_smoother/tension_smoother.cpp:186-314
//   TensionSmoother::smooth tail                       src/reference_path_smoother/tension_smoother.cpp:84-96
//   distance                                           src/tools/tools.cpp:46-48
//
// The B-spline is tinyspline's clamped BSpline(n, 2, degree) with the input points as control points.  tinyspline is
// not part of the reference tree; the clamped uniform knot vector and de Boor's algorithm are restated from their
// published definitions (de Boor, "A Practical Guide to Splines"), so parity with tinyspline itself is not pinned.
// Arithmetic: every product and sum rounded alone (mul / add), pow(d, 2) as d * d, the reference's serial
// accumulations (tmp_t += delta_t, the s sums) kept as accumulations in its order.
#pragma once
#include "pqp_env_core.cuh"

namespace pqp {

// Refusal reasons (0: accepted); the C ABI reports them all as ok = 0.
enum SmoothRefusal {
    SM_OK = 0,
    SM_FEW = 1,          // fewer than 4 input points (:36-39)
    SM_DEGREE = 2,       // degree >= points: tinyspline refuses the B-spline, the reference throws
    SM_LENGTH = 3,       // the polyline's length is not positive and finite
    SM_RAW_MANY = 4,     // more B-spline samples than max_raw_samples
    SM_RAW_ORDER = 5,    // fewer than 3 B-spline samples, or their s not strictly increasing (tk::spline::set_points)
    SM_MANY = 6,         // more resampled stations than max_points
    SM_SHORT = 7,        // fewer than 3 resampled stations (the smoothed spline's tk::spline::set_points)
    SM_QP = 8,           // the smoothing QP did not end SOLVED
    SM_S_ORDER = 9,      // the smoothed s is not strictly increasing or not finite (tk::spline::set_points)
    SM_CAPACITY = 10,    // the running knot total would pass the capacity (decided by the reservation)
    SM_MAP = 11          // TENSION: the path's map index lies outside the map set
};

constexpr int kSmoothMaxDegree = 5;

// distance (tools.cpp:46-48)
PQP_HD double smooth_distance(double x0, double y0, double x1, double y1) {
    const double dx = x0 - x1, dy = y0 - y1;
    return sqrt(add(mul(dx, dx), mul(dy, dy)));
}

// bSpline's length and degree (:499-508) of the n points (px[i], py[i]) at a stride of `stride` doubles.  Returns the
// degree; *length the serial sum of the segment lengths.
PQP_HD int smooth_degree(int n, const double *px, const double *py, int stride, double *length) {
    double len = 0;
    for (int i = 0; i + 1 < n; ++i)
        len = add(len, smooth_distance(px[stride * i], py[stride * i], px[stride * (i + 1)], py[stride * (i + 1)]));
    *length = len;
    const double avg = len / (double)(n - 1);
    return avg > 10 ? 3 : avg > 5 ? 4 : 5;
}

// Knot j of the clamped uniform knot vector of n control points and degree p: 0 for j <= p, 1 for j >= n, and
// (j - p) / (n - p) between.
PQP_HD double smooth_knot(int n, int p, int j) {
    if (j <= p) return 0.0;
    if (j >= n) return 1.0;
    return (double)(j - p) / (double)(n - p);
}

// The B-spline at t in [0, 1] by de Boor's algorithm: the knot span k (p <= k <= n - 1) with knot k <= t < knot k + 1,
// t = 1 in the last span, then p rounds of affine combinations of control points k - p .. k.
PQP_HD void smooth_bspline_eval(int n, int p, const double *px, const double *py, int stride, double t, double *x,
                                double *y) {
    int k = p;
    while (k + 1 < n && smooth_knot(n, p, k + 1) <= t) ++k;
    double dx[kSmoothMaxDegree + 1], dy[kSmoothMaxDegree + 1];
    for (int j = 0; j <= p; ++j) {
        dx[j] = px[stride * (j + k - p)];
        dy[j] = py[stride * (j + k - p)];
    }
    for (int r = 1; r <= p; ++r)
        for (int j = p; j >= r; --j) {
            const double lo = smooth_knot(n, p, j + k - p), hi = smooth_knot(n, p, j + 1 + k - r);
            const double a = (t - lo) / (hi - lo);
            dx[j] = add(mul(1.0 - a, dx[j - 1]), mul(a, dx[j]));
            dy[j] = add(mul(1.0 - a, dy[j - 1]), mul(a, dy[j]));
        }
    *x = dx[p];
    *y = dy[p];
}

// Samples of bSpline (:518-526): t = 0, delta_t, 2 delta_t, ... (accumulated) while t < 1, then t = 1.  Counts at most
// cap + 1 samples; with t != nullptr writes the first min(count, cap) parameters.
PQP_HD int smooth_sample_params(double length, int cap, double *t) {
    const double delta_t = 1.0 / length;
    int k = 0;
    for (double tmp_t = 0; tmp_t < 1 && k <= cap; tmp_t = add(tmp_t, delta_t), ++k)
        if (t && k < cap) t[k] = tmp_t;
    if (k <= cap) {
        if (t && k < cap) t[k] = 1.0;
        ++k;
    }
    return k;
}

// One s step of bSpline (:527-531) and of osqpSmooth's output (tension_smoother_2.cpp:213-217).
PQP_HD double smooth_step(double x0, double y0, double x1, double y1) {
    const double dx = x1 - x0, dy = y1 - y0;
    return sqrt(add(mul(dx, dx), mul(dy, dy)));
}

// segmentRawReference's station count (:61-68): s = 0, 1, 2, ... while s.back() < max_s (the pushed s are exact
// integers, and max_s - s.back() > 1 never holds after the loop).  max_s is finite and at most 2^30 here.
PQP_HD int smooth_station_count(double max_s) { return max_s > 0 ? (int)ceil(max_s) + 1 : 1; }

// The TENSION2 QP (setHessianMatrix / setGradient / setConstraintMatrix, tension_smoother_2.cpp:221-301) in the band
// order of the generic core: station i's unknowns (x_i, y_i, theta_i, k_i) at 4i .. 4i + 3 (the last station has no
// k), n = 4N - 1; rows in the reference's order -- x update (row i), y update (N - 1 + i), theta update (2N - 2 + i),
// the x and y pins (3N - 3, 3N - 2), m = 3N - 1.  Every row has at most 3 entries, P couples only k_i and k_{i+1}, and
// the reduced KKT has bandwidth 4.  Weights: w = (deviation, curvature, curvature rate).
struct SmoothWeights {
    double dev, curv, rate;
};

// Station i's entries: its rows (the three updates when i < N - 1, the pins when i = 0), its P and q entries and its
// CSC columns.  st: the resampled state of station i (x, y, heading z, curvature k); ds = s_{i+1} - s_i.  A_col / A_val
// / l / u point at the path's rows, Pd / Po_idx / Po_val / q at its n-arrays, ptr / row / val at its CSC arrays.
PQP_HD void smooth_qp_station(int N, int i, const pqp_state &st, double ds, double x0, double y0, const SmoothWeights &w,
                              int32_t *A_col, double *A_val, double *l, double *u, double *Pd, int32_t *Po_idx,
                              double *Po_val, double *q, int32_t *ptr, int32_t *row, double *val) {
    auto put = [&](int r, double b, int c0, double v0, int c1, double v1, int c2, double v2) {
        A_col[4 * r] = c0; A_col[4 * r + 1] = c1; A_col[4 * r + 2] = c2; A_col[4 * r + 3] = -1;
        A_val[4 * r] = v0; A_val[4 * r + 1] = v1; A_val[4 * r + 2] = v2; A_val[4 * r + 3] = 0.0;
        l[r] = b; u[r] = b;
    };
    const bool next = i + 1 < N;
    const int g = 4 * i;
    const double sn = sin(st.z), cs = cos(st.z);
    if (next) {
        put(i, mul(ds, cs), g, -1.0, g + 2, mul(ds, sn), g + 4, 1.0);
        put(N - 1 + i, mul(ds, sn), g + 1, -1.0, g + 2, mul(-ds, cs), g + 5, 1.0);
        put(2 * N - 2 + i, mul(-ds, st.k), g + 2, -1.0, g + 3, -ds, g + 6, 1.0);
    }
    if (i == 0) {
        put(3 * N - 3, x0, 0, 1.0, -1, 0.0, -1, 0.0);
        put(3 * N - 2, y0, 1, 1.0, -1, 0.0, -1, 0.0);
    }
    // P: x and y 2 w_dev; k_i 2 w_curv, plus 2 w_rate (1, -1; -1, 1) on (k_i, k_{i+1}) for i <= N - 3, added in the
    // reference's order; q: -2 w_dev (x, y)
    const double pdev = mul(w.dev, 2.0), prate = mul(2.0, w.rate);
    for (int t = 0; t < 4 && g + t < 4 * N - 1; ++t) {
        Pd[g + t] = t < 2 ? pdev : 0.0;
        Po_idx[2 * (g + t)] = Po_idx[2 * (g + t) + 1] = -1;
        Po_val[2 * (g + t)] = Po_val[2 * (g + t) + 1] = 0.0;
        q[g + t] = t == 0 ? mul(mul(-2.0, w.dev), st.x) : t == 1 ? mul(mul(-2.0, w.dev), st.y) : 0.0;
    }
    if (next) {
        double pk = mul(w.curv, 2.0);
        if (i >= 1) pk = add(pk, prate);          // block i - 1's (1, 1) entry
        if (i + 2 < N) pk = add(pk, prate);       // block i's (0, 0) entry
        Pd[g + 3] = pk;
        int qn = 0;
        if (i >= 1) { Po_idx[2 * (g + 3) + qn] = g - 1; Po_val[2 * (g + 3) + qn] = -prate; ++qn; }
        if (i + 2 < N) { Po_idx[2 * (g + 3) + qn] = g + 7; Po_val[2 * (g + 3) + qn] = -prate; }
    }
    // CSC, rows ascending.  Station 0 holds 8 entries, an inner station 9, the last 3: station i's start at 9i - 1.
    int e = i == 0 ? 0 : 9 * i - 1;
    ptr[g] = e;                                          // x_i: x update i-1 (+1), x update i (-1), x pin
    if (i > 0) { row[e] = i - 1; val[e++] = 1.0; }
    if (next) { row[e] = i; val[e++] = -1.0; }
    if (i == 0) { row[e] = 3 * N - 3; val[e++] = 1.0; }
    ptr[g + 1] = e;                                      // y_i: y update i-1 (+1), y update i (-1), y pin
    if (i > 0) { row[e] = N - 2 + i; val[e++] = 1.0; }
    if (next) { row[e] = N - 1 + i; val[e++] = -1.0; }
    if (i == 0) { row[e] = 3 * N - 2; val[e++] = 1.0; }
    ptr[g + 2] = e;                                      // theta_i: x update i, y update i, theta updates i-1, i
    if (next) { row[e] = i; val[e++] = mul(ds, sn); }
    if (next) { row[e] = N - 1 + i; val[e++] = mul(-ds, cs); }
    if (i > 0) { row[e] = 2 * N - 3 + i; val[e++] = 1.0; }
    if (next) { row[e] = 2 * N - 2 + i; val[e++] = -1.0; }
    if (next) {
        ptr[g + 3] = e;                                  // k_i: theta update i (-ds)
        row[e] = 2 * N - 2 + i; val[e++] = -ds;
    } else {
        ptr[g + 3] = e;                                  // closes ptr[n] = 9N - 7
    }
}

// The generic core's separators: station e's (x, y, theta, k) for e = 0, L, 2L, ... < N - 1, at most 32, with
// L = max(2, (N - 2) / 31 + 1).  Returns M.
PQP_HD int smooth_qp_separators(int N, int32_t *sep) {
    int L = (N - 2) / 31 + 1;
    if (L < 2) L = 2;
    int M = 0;
    for (int e = 0; e < N - 1 && M < 32; e += L) sep[M++] = 4 * e;
    return M;
}

// The TENSION QP (TensionSmoother::setHessianMatrix / setConstraintMatrix, tension_smoother.cpp:239-314; q = 0) in the
// band order of the generic core: station i's unknowns (x_i, y_i, d_i) at 3i .. 3i + 2, n = 3N; rows in the
// reference's order -- x_i - cos(theta_i) d_i = x_ref_i (row i), y_i - sin(theta_i) d_i = y_ref_i (N + i), d_i (2N + i),
// m = 3N, theta_i = heading_i + pi/2 unwrapped.  The x and y chains of P couple each unknown to three neighbours on each
// side, so the reduced KKT has half-bandwidth 9 and a separator is three stations (9 unknowns).  Weights: w = (deviation,
// curvature, curvature rate) = FLAGS_cartesian_deviation_weight, _curvature_weight, _curvature_rate_weight.  Exact zeros
// of P and A are dropped, as Eigen's sparseView drops them.
constexpr int kTensionPartners = 6;
constexpr double kTensionHalfPi = 1.57079632679489661923;   // M_PI_2
constexpr double kTensionMaxClearance = 2.0;                  // default_clearance (:300)

// (1, -2, 1) and (-1, 3, -3, 1), the dds and ddds vectors of setHessianMatrix
PQP_HD double tension_dds(int k) { return k == 1 ? -2.0 : 1.0; }
PQP_HD double tension_ddds(int k) { return k == 0 ? -1.0 : k == 1 ? 3.0 : k == 2 ? -3.0 : 1.0; }

// Entry (a, b), |a - b| <= 3, of the x (or y) chain of setHessianMatrix (:245-257): the dds block (v_a v_b) w_curv at
// i = 0 .. N - 3 and the ddds block (u_a u_b) w_rate at i = 0 .. N - 4, added into a zero matrix in the reference's
// order (block i's dds, then its ddds), each block entry rounded once.
PQP_HD double tension_chain_hess(int N, int a, int b, const SmoothWeights &w) {
    const int lo = a < b ? a : b, hi = a < b ? b : a;
    double h = 0.0;
    for (int i = hi - 3 > 0 ? hi - 3 : 0; i <= lo && i <= N - 3; ++i) {
        if (hi - i <= 2) h = add(h, mul(mul(tension_dds(a - i), tension_dds(b - i)), w.curv));
        if (i <= N - 4) h = add(h, mul(mul(tension_ddds(a - i), tension_ddds(b - i)), w.rate));
    }
    return h;
}

// The d_i column's cos / sin entries of rows x_i and y_i: -cos(theta_i), -sin(theta_i) (:283-285).
PQP_HD void tension_normal(const pqp_state &st, double *nc, double *ns) {
    const double theta = add(st.z, kTensionHalfPi);
    *nc = -cos(theta);
    *ns = -sin(theta);
}

// Station i's CSC entries: x_i and y_i one each, d_i its kept cos / sin entries and its own row.
PQP_HD int tension_qp_csc_count(const pqp_state &st) {
    double nc, ns;
    tension_normal(st, &nc, &ns);
    return 3 + (nc != 0.0) + (ns != 0.0);
}

// Station i's entries: its rows x_i, y_i, d_i, its P entries and its CSC columns.  st: the resampled station (x, y,
// heading z); clearance: Map::getObstacleDistance at (st.x, st.y), read for 0 < i < N - 1 only; e: the CSC entries of
// stations 0 .. i - 1 (tension_qp_csc_count summed).  A_col / A_val / l / u point at the path's rows, Pd / Po_idx /
// Po_val [kTensionPartners] at its n-arrays (partners in ascending band position, unused slots -1), ptr / row / val at
// its CSC arrays; the last station also closes ptr[3N].
PQP_HD void tension_qp_station(int N, int i, const pqp_state &st, double clearance, const SmoothWeights &w, int e,
                               int32_t *A_col, double *A_val, double *l, double *u, double *Pd, int32_t *Po_idx,
                               double *Po_val, int32_t *ptr, int32_t *row, double *val) {
    double nc, ns;
    tension_normal(st, &nc, &ns);
    const int g = 3 * i;
    auto put = [&](int r, int c0, int c1, double v1, double lo, double up) {
        A_col[4 * r] = c0; A_val[4 * r] = 1.0;
        const bool keep = c1 >= 0 && v1 != 0.0;
        A_col[4 * r + 1] = keep ? c1 : -1; A_val[4 * r + 1] = keep ? v1 : 0.0;
        A_col[4 * r + 2] = A_col[4 * r + 3] = -1;
        A_val[4 * r + 2] = A_val[4 * r + 3] = 0.0;
        l[r] = lo; u[r] = up;
    };
    put(i, g, g + 2, nc, st.x, st.x);
    put(N + i, g + 1, g + 2, ns, st.y, st.y);
    // d bounds (:296-313): d_0 = 0, |d_{N-1}| <= 0.5, otherwise |d_i| <= std::min(clearance, 2)
    double dl = 0.0, du = 0.0;
    if (i == N - 1) { dl = -0.5; du = 0.5; }
    else if (i > 0) {
        const double c = kTensionMaxClearance < clearance ? kTensionMaxClearance : clearance;
        dl = -c; du = c;
    }
    put(2 * N + i, g + 2, -1, 0.0, dl, du);
    // P: the x and y chains (x_k at 3k, y_k at 3k + 1), then d_i's diagonal w_dev (:258-261)
    for (int t = 0; t < 2; ++t) {
        const int j = g + t;
        Pd[j] = tension_chain_hess(N, i, i, w);
        int q = 0;
        for (int k = i - 3; k <= i + 3; ++k) {
            if (k < 0 || k >= N || k == i) continue;
            const double h = tension_chain_hess(N, i, k, w);
            if (h != 0.0) { Po_idx[kTensionPartners * j + q] = 3 * k + t; Po_val[kTensionPartners * j + q] = h; ++q; }
        }
        for (; q < kTensionPartners; ++q) { Po_idx[kTensionPartners * j + q] = -1; Po_val[kTensionPartners * j + q] = 0.0; }
    }
    Pd[g + 2] = w.dev;
    for (int q = 0; q < kTensionPartners; ++q) {
        Po_idx[kTensionPartners * (g + 2) + q] = -1;
        Po_val[kTensionPartners * (g + 2) + q] = 0.0;
    }
    // CSC, rows ascending: x_i (row i), y_i (row N + i), d_i (rows i, N + i, 2N + i)
    ptr[g] = e;
    row[e] = i; val[e++] = 1.0;
    ptr[g + 1] = e;
    row[e] = N + i; val[e++] = 1.0;
    ptr[g + 2] = e;
    if (nc != 0.0) { row[e] = i; val[e++] = nc; }
    if (ns != 0.0) { row[e] = N + i; val[e++] = ns; }
    row[e] = 2 * N + i; val[e++] = 1.0;
    if (i == N - 1) ptr[3 * N] = e;
}

// The generic core's separators for the TENSION QP: stations e, e + 1, e + 2 (band positions 3e .. 3e + 8) for e = 0,
// L, 2L, ... with e + 2 < N - 1, at most 32, L = max(6, (N - 4) / 31 + 1).  L >= 6 leaves at least three stations (9
// unknowns, the half-bandwidth) between two separators, so no entry of the reduced KKT couples two separators; the first
// always starts at 0.  Returns M.
PQP_HD int tension_qp_separators(int N, int32_t *sep) {
    int L = (N - 4) / 31 + 1;
    if (L < 6) L = 6;
    int M = 0;
    sep[M++] = 0;
    for (int e = L; e + 3 <= N - 1 && M < 32; e += L) sep[M++] = 3 * e;
    return M;
}

}  // namespace pqp
