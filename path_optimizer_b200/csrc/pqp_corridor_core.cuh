// pqp_corridor_core.cuh -- per-thread device functions of pqp_post_smooth_device: the lattice DP that picks a corridor
// around a smoothed reference line (graphSearchDp) and the bounds and QP rows of the post-smoothing that follows it
// (postSmooth).  Like pqp_segment_core.cuh, every function is a straight per-thread restatement, so the test-only host
// build (-DPQP_HOST_EMU, tests/emu/) calls them in a loop where the kernel spreads them over a warp.
//
// Reference behaviour being replaced (file:line in the reference tree):
//   ReferencePathSmoother::graphSearchDp              src/reference_path_smoother/reference_path_smoother.cpp:145-301
//     closest point, layer lattice, vehicle_l         :151-172
//     node sampling and feasibility, rough bounds     :174-229
//     DP and backtrack, 0.2 m bound march             :231-293
//   ReferencePathSmoother::calculateCostAt            :110-143
//   ReferencePathSmoother::postSmooth / setPost*      :534-644
//   findClosestPoint / getHeading / global2Local      src/tools/tools.cpp:32-110
//
// Arithmetic: splines through pqp::spline_eval, heading and curvature through pqp::densify_sample (getHeading and
// getCurvature), every product and sum rounded alone (mul / add), the reference's serial accumulations (the lattice's
// tmp_s += search_ds, the lateral cur_l += spacing, the marches' += 0.2) kept as accumulations in its order.
#pragma once
#include "pqp_env_core.cuh"

namespace pqp {

// Lateral nodes per layer the kernel holds: two per lane of its warp.  The reference's defaults (range 10, spacing
// 0.6) give 34.
constexpr int kCorridorMaxLateral = 64;
// findClosestPoint scans the line every 0.5 m: a line longer than this is refused rather than scanned.
constexpr double kCorridorMaxLength = 1048576.0;   // 2^20 m, 2^21 samples
// The DP wraps direction - start.z with constraintAngle: a start heading beyond this is refused before it loops.
constexpr double kCorridorMaxHeading = 1048576.0;  // 2^20 rad
constexpr double kCorridorThreshold = 1.45;        // search_threshold, :176
constexpr double kDblMax = 1.7976931348623157e308;

// Refusal reasons (0: accepted); the C ABI reports them all as ok = 0.
enum CorridorRefusal {
    COR_OK = 0,
    COR_BAD_SPLINE = 1,    // fewer than 3 knots
    COR_BAD_LENGTH = 2,    // max_s <= 0, not finite, or above kCorridorMaxLength
    COR_BAD_START = 3,     // closest point or vehicle_l not finite, start.z not finite or beyond kCorridorMaxHeading
    COR_FAR = 4,           // |vehicle_l| > range (:167-170)
    COR_TOO_MANY = 5,      // more layers than max_layers
    COR_SHORT = 6,         // fewer than 4 layers reached (:535-539)
    COR_QP = 7,            // the post-smoothing QP did not end SOLVED
    COR_S_ORDER = 8,       // the post-smoothed s is not strictly increasing (tk::spline::set_points)
    COR_MAP = 9,           // the map index lies outside the map set
    COR_CAPACITY = 10,     // the running knot total would pass the capacity (decided by the reservation)
    COR_WIDE = 11          // the lateral lattice has more than kCorridorMaxLateral nodes
};

// The search flags, as call arguments.  lat[j] is the lateral lattice cur_l += spacing from -range while <= range
// (:186-212), accumulated once on the host.
struct CorridorFlags {
    double range, spacing, ds_long;
    int n_lat;
    double lat[kCorridorMaxLateral];
};

// One grid sample of findClosestPoint (tools.cpp:79-87): the distance from (x, y) to the line at s = 0.5 k.  Adding
// 0.5 to a multiple of 0.5 is exact, so sample k is the k-th of the reference's accumulated walk.
PQP_HD double corridor_grid_dist(const SplineView &xs, const SplineView &ys, long long k, double x, double y) {
    const double s = 0.5 * (double)k;
    const double dx = spline_eval(xs, 0, s) - x, dy = spline_eval(ys, 0, s) - y;
    return sqrt(add(mul(dx, dx), mul(dy, dy)));
}

// Samples of the grid scan: s = 0.5 k <= max_s.
PQP_HD long long corridor_grid_count(double max_s) { return (long long)floor(2.0 * max_s) + 1; }

// The Newton steps of findClosestPoint (tools.cpp:88-109) from the grid's best s, clamped above by max_s only.
PQP_HD double corridor_newton(const SplineView &xs, const SplineView &ys, double x, double y, double s0, double max_s) {
    double cur = s0, prev = s0;
    for (int i = 0; i < 20; ++i) {
        const double px = spline_eval(xs, 0, cur) - x, py = spline_eval(ys, 0, cur) - y;
        const double dx = spline_eval(xs, 1, cur), dy = spline_eval(ys, 1, cur);
        const double ddx = spline_eval(xs, 2, cur), ddy = spline_eval(ys, 2, cur);
        const double j = add(mul(px, dx), mul(py, dy));
        const double h = add(add(add(mul(dx, dx), mul(px, ddx)), mul(dy, dy)), mul(py, ddy));
        cur -= j / h;
        if (fabs(cur - prev) < 1e-5) break;
        prev = cur;
    }
    return max_s < cur ? max_s : cur;   // std::min(cur, max_s)
}

// global2Local(proj_point, start).y (:163-166, tools.cpp:57-64): the start's lateral offset from the line at s.
PQP_HD double corridor_vehicle_l(const SplineView &xs, const SplineView &ys, double s, const pqp_state &start) {
    const pqp_state p = densify_sample(xs, ys, s);
    const double dx = start.x - p.x, dy = start.y - p.y;
    return add(mul(-dx, sin(p.z)), mul(dy, cos(p.z)));
}

// One lattice node (:189-208): position, distance to the nearest obstacle (-1 outside the map) and feasibility.  r is
// the layer's sample (x, y, heading, curvature), c_n / s_n the cosine and sine of heading + pi/2.
struct CorridorNode {
    double x, y, dis;
    bool feasible;
};
PQP_HD CorridorNode corridor_node(const MapView &m, const pqp_state &r, double c_n, double s_n, double l) {
    CorridorNode nd;
    nd.x = add(r.x, mul(l, c_n));
    nd.y = add(r.y, mul(l, s_n));
    nd.dis = map_inside(m, nd.x, nd.y) ? map_distance(m, nd.x, nd.y) : -1.0;
    const double ref_r = 1 / r.k;
    nd.feasible = !((r.k < 0 && l < ref_r) || (r.k > 0 && l > ref_r) || nd.dis < kCorridorThreshold);
    return nd;
}

// calculateCostAt's own part (:122-125): obstacle within 3 m, weight 0.5, and the offset, weight 1.
PQP_HD double corridor_self_cost(double dis, double l, double range) {
    double c = 0;
    if (dis < 3.0) c = add(c, mul((3.0 - dis) / 3.0, 0.5));
    return add(c, mul(fabs(l) / range, 1.0));
}

// The previous layer as calculateCostAt reads it: per node its l, position, direction and cost, and whether it was
// reached (a feasible node with a parent, or layer 0's start node).  A feasible node without a parent has cost DBL_MAX
// and no direction in the reference; self + edge + DBL_MAX rounds to DBL_MAX there and never passes the strict '<', so
// it is skipped here.
struct CorridorPrev {
    const double *x, *y, *dir, *cost;
    const unsigned char *live;
};

// calculateCostAt for one feasible node (:127-142): the min over the previous layer in index order with a strict '<',
// so the first index wins a tie.  Returns the chosen predecessor (-1: none) with its cost and direction.
PQP_HD int corridor_relax(const CorridorFlags &f, const CorridorPrev &p, double prev_s, double s, double l, double heading,
                          double x, double y, double self, double *cost, double *dir) {
    double min_cost = kDblMax, best_dir = 0;
    int best = -1;
    for (int k = 0; k < f.n_lat; ++k) {
        if (!p.live[k]) continue;
        if (fabs(f.lat[k] - l) > s - prev_s) continue;
        const double direction = atan2(y - p.y[k], x - p.x[k]);
        const double edge = add(mul(fabs(wrap_angle(direction - p.dir[k])) / M_PI_2, 16.0),
                                mul(fabs(wrap_angle(direction - heading)) / M_PI_2, 0.5));
        const double total = add(add(self, edge), p.cost[k]);
        if (total < min_cost) {
            min_cost = total;
            best = k;
            best_dir = direction;
        }
    }
    *cost = best >= 0 ? min_cost : kDblMax;
    *dir = best_dir;
    return best;
}

// The rough bounds of a feasible node j (:213-228): the l of the first and last node of the run of feasible nodes that
// holds it.  feas: bit k set when node k is feasible.
PQP_HD void corridor_rough(const CorridorFlags &f, unsigned long long feas, int j, double *lo, double *hi) {
    int a = j, b = j;
    while (a > 0 && ((feas >> (a - 1)) & 1ull)) --a;
    while (b + 1 < f.n_lat && ((feas >> (b + 1)) & 1ull)) ++b;
    *lo = f.lat[a];
    *hi = f.lat[b];
}

// The 0.2 m bound march of one chosen node (:256-287), from its rough bounds outwards while the map is clear by more
// than 1.45 m, until 6 m either side.  r: the layer's sample.
PQP_HD void corridor_march(const MapView &m, const pqp_state &r, double rough_lo, double rough_hi, double *lo, double *hi) {
    const double check_s = 0.2, check_limit = 6.0;
    const double a = r.z + M_PI_2, c_n = cos(a), s_n = sin(a);
    double ub = add(check_s, rough_hi), lb = add(-check_s, rough_lo);
    while (ub < check_limit) {
        const double x = add(r.x, mul(ub, c_n)), y = add(r.y, mul(ub, s_n));
        if (map_inside(m, x, y) && map_distance(m, x, y) > kCorridorThreshold) {
            ub = add(ub, check_s);
        } else {
            ub = add(ub, -check_s);
            break;
        }
    }
    while (lb > -check_limit) {
        const double x = add(r.x, mul(lb, c_n)), y = add(r.y, mul(lb, s_n));
        if (map_inside(m, x, y) && map_distance(m, x, y) > kCorridorThreshold) {
            lb = add(lb, -check_s);
        } else {
            lb = add(lb, check_s);
            break;
        }
    }
    *lo = lb;
    *hi = ub;
}

// The post-smoothing QP (setPostHessianMatrix / setPostConstraintMatrix, :590-644) in the band order of the generic
// core: unknowns (x_i, dx_i, ddx_i) of layer i at 3i, 3i+1, 3i+2, rows in the reference's order -- x range (row i),
// dx - x (row R + i), ddx - dx (row 2R - 1 + i).  The entries of the rows that layer i owns: its x range row with
// bounds (lo, hi), and for i < R - 1 its two transition rows with ds = s_{i+1} - s_i.  A_col / A_val / l / u point at
// the path's rows.
PQP_HD void corridor_qp_rows(int R, int i, double lo, double hi, double ds, int32_t *A_col, double *A_val, double *l,
                             double *u) {
    auto row = [&](int r, double lr, double ur, int c0, double v0, int c1, double v1, int c2, double v2) {
        A_col[4 * r] = c0; A_col[4 * r + 1] = c1; A_col[4 * r + 2] = c2; A_col[4 * r + 3] = -1;
        A_val[4 * r] = v0; A_val[4 * r + 1] = v1; A_val[4 * r + 2] = v2; A_val[4 * r + 3] = 0.0;
        l[r] = lr; u[r] = ur;
    };
    row(i, lo, hi, 3 * i, 1.0, -1, 0.0, -1, 0.0);
    if (i + 1 < R) {
        row(R + i, 0.0, 0.0, 3 * i + 3, 1.0, 3 * i, -1.0, 3 * i + 1, -ds);
        row(2 * R - 1 + i, 0.0, 0.0, 3 * i + 4, 1.0, 3 * i + 1, -1.0, 3 * i + 2, -ds);
    }
}

// Layer i's three columns of that A in CSC with rows ascending, the order the generic core's host assembly emits
// (R >= 4).  Layer 0 holds 5 entries, an inner layer 7 and the last 3, so layer i's start at 7 i - 2 (i >= 1); ptr,
// row and val point at the path's arrays, and the last layer also closes ptr[3R] = 7R - 6.
PQP_HD void corridor_qp_columns(int R, int i, double ds, int32_t *ptr, int32_t *row, double *val) {
    int e = i == 0 ? 0 : 7 * i - 2;
    const bool next = i + 1 < R;
    ptr[3 * i] = e;                                  // x_i: x range i, dx-x i-1 (+1), dx-x i (-1)
    row[e] = i; val[e++] = 1.0;
    if (i > 0) { row[e] = R + i - 1; val[e++] = 1.0; }
    if (next) { row[e] = R + i; val[e++] = -1.0; }
    ptr[3 * i + 1] = e;                              // dx_i: dx-x i (-ds), ddx-dx i-1 (+1), ddx-dx i (-1)
    if (next) { row[e] = R + i; val[e++] = -ds; }
    if (i > 0) { row[e] = 2 * R - 2 + i; val[e++] = 1.0; }
    if (next) { row[e] = 2 * R - 1 + i; val[e++] = -1.0; }
    ptr[3 * i + 2] = e;                              // ddx_i: ddx-dx i (-ds)
    if (next) { row[e] = 2 * R - 1 + i; val[e++] = -ds; }
    if (!next) ptr[3 * R] = e;
}

// The generic core's separators: layer e's (x, dx, ddx) for e = 0, L, 2L, ... < R - 1, at most 32, with
// L = max(2, (R - 2) / 31 + 1), as the host assembly of "K" places them.  Returns M.
PQP_HD int corridor_qp_separators(int R, int32_t *sep) {
    int L = (R - 2) / 31 + 1;
    if (L < 2) L = 2;
    int M = 0;
    for (int e = 0; e < R - 1 && M < 32; e += L) sep[M++] = 3 * e;
    return M;
}

}  // namespace pqp
