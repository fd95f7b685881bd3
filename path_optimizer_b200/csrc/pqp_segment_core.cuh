// pqp_segment_core.cuh -- per-thread device functions of pqp_segment_reference_device: one smoothed reference line
// (its x(s), y(s) splines and length) turned into the reference states the plan chain reads.  Like pqp_env_core.cuh,
// every function is a straight per-thread restatement, so the test-only host build (-DPQP_HOST_EMU, tests/emu/) calls
// them in a loop.
//
// Reference behaviour being replaced (file:line in the reference tree):
//   PathOptimizer::segmentSmoothedPath                 src/path_optimizer/path_optimizer.cpp:119-178
//     initial offset and heading error, 75 deg test    :125-141
//     goal cut (closest lattice sample to the goal)     :143-166
//     spacings from FLAGS_enable_raw_output             :168-173
//   ReferencePathImpl::buildReferenceFromSpline        src/data_struct/reference_path_impl.cpp:474-499
//   getHeading / getCurvature / global2Local / distance src/tools/tools.cpp:32-64
//   constraintAngle / isEqual                          include/path_optimizer/tools/tools.hpp:24-35, tools.cpp:28-30
//
// Arithmetic: the spline is evaluated by pqp::spline_eval and heading and curvature come from pqp::densify_sample, the
// functions the densifying tail uses.  Every product and sum is rounded alone (mul / add), pow(v, 2) is the correctly
// rounded square mul(v, v), and the two serial accumulations of the reference (the goal search's  tmp_s -= search_ds
// and the walk's  tmp_s += ...) are kept as accumulations in its order.
#pragma once
#include "pqp_env_core.cuh"

namespace pqp {

// The flags segmentSmoothedPath reads, as call arguments.
struct SegmentFlags {
    double ds_small, ds_large;   // (0.15, FLAGS_output_spacing) with FLAGS_enable_raw_output, else (0.5, 1.0)
    double search_ds;            // 0.1 with FLAGS_enable_exact_position, else 0.5
    int dynamic;                 // FLAGS_enable_dynamic_segmentation
    int max_n;                   // a path that needs more stations is refused
};

// The goal search visits at most this many lattice samples: a longer search (max_s > search_ds * kSegmentMaxSearch) is
// refused rather than walked, so that no thread loops for minutes (or forever, once max_s - search_ds == max_s).
// At the limit a search that never breaks (a NaN goal, or one more than 8 m from every sample) still takes about
// 4.6 s on one H100 thread (1.1 us per sample, DESIGN.md §9).
constexpr double kSegmentMaxSearch = 4194304.0;   // 2^22
// start.z - (heading at s = 0) beyond this many radians is refused before constraintAngle wraps it.
constexpr double kSegmentMaxTurn = 1048576.0;     // 2^20

// Refusal reasons of segment_count (0: accepted); the C ABI reports them all as ok = 0.
enum SegmentRefusal {
    SEG_OK = 0,
    SEG_BAD_SPLINE = 1,     // fewer than 3 knots, the initial offset not finite, or start.z minus the heading at s = 0
                            // not finite or beyond kSegmentMaxTurn (NaN rows, a NaN or infinite start)
    SEG_HEADING = 2,        // |initial heading error| > 75 deg (path_optimizer.cpp:137-140)
    SEG_BAD_LENGTH = 3,     // max_s <= 0, not finite, or too long to search
    SEG_TOO_MANY = 4,       // more than max_n stations
    SEG_CAPACITY = 5        // the running station total would pass the capacity (decided by the scan)
};

// One step of the walk (reference_path_impl.cpp:490-496): the spacing after a sample of curvature k.
PQP_HD double segment_step(const SegmentFlags &f, double tmp_s, double k) {
    if (!f.dynamic) return add(tmp_s, f.ds_large);
    const double large_k = 0.2, small_k = 0.08;
    const double ak = fabs(k);
    const double k_share = ak > large_k ? 1.0 : ak < small_k ? 0.0 : (ak - small_k) / (large_k - small_k);
    return add(tmp_s, add(f.ds_large, -mul(k_share, f.ds_large - f.ds_small)));
}

// Count pass of one path (one thread): the initial error x0 = (offset, heading error, start.k), the length after the
// goal cut (*cut_s) and the number of stations (*n, 0 when refused).  Returns a SegmentRefusal.
PQP_HD int segment_count(const SegmentFlags &f, const SplineView &xs, const SplineView &ys, double max_s,
                         const pqp_state &start, const pqp_state &goal, double *x0, double *cut_s, int *n) {
    *n = 0;
    *cut_s = max_s;
    x0[0] = 0.0; x0[1] = 0.0; x0[2] = start.k;
    if (xs.n < 3 || ys.n < 3) return SEG_BAD_SPLINE;
    // initial error (:125-136): first point of the spline, its heading from the first derivatives
    const pqp_state first = densify_sample(xs, ys, 0.0);
    const double dx = first.x - start.x, dy = first.y - start.y;
    const double local_y = add(mul(-dx, sin(start.z)), mul(dy, cos(start.z)));   // global2Local(start, first).y
    const double ex = start.x - first.x, ey = start.y - first.y;
    const double min_distance = sqrt(add(mul(ex, ex), mul(ey, ey)));
    const double offset = local_y < 0 ? min_distance : -min_distance;
    const double turn = start.z - first.z;
    x0[0] = offset; x0[1] = turn;
    // constraintAngle subtracts 2 pi until the angle lies in [-pi, pi]: it never ends on an infinite angle, and takes
    // ages on a huge one, so those are refused before it runs
    if (!(fabs(offset) <= 1.7976931348623157e308) || !(fabs(turn) <= kSegmentMaxTurn)) return SEG_BAD_SPLINE;
    const double heading_error = wrap_angle(turn);
    x0[1] = heading_error;
    if (fabs(heading_error) > 75 * M_PI / 180) return SEG_HEADING;
    if (!(max_s > 0.0) || !(max_s <= f.search_ds * kSegmentMaxSearch)) return SEG_BAD_LENGTH;
    // goal cut (:143-166)
    double length = max_s;
    {
        const double gx = goal.x - spline_eval(xs, 0, length), gy = goal.y - spline_eval(ys, 0, length);
        const double end_distance = sqrt(add(mul(gx, gx), mul(gy, gy)));
        if (!(fabs(end_distance - 0.0) < 1e-6)) {      // !isEqual(end_distance, 0), FLAGS_epsilon
            double tmp_s = length - f.search_ds;
            double min_dis_to_goal = end_distance, min_dis_s = length;
            while (tmp_s > 0) {
                const double x = spline_eval(xs, 0, tmp_s) - goal.x, y = spline_eval(ys, 0, tmp_s) - goal.y;
                const double tmp_dis = sqrt(add(mul(x, x), mul(y, y)));
                if (tmp_dis < min_dis_to_goal) {
                    min_dis_to_goal = tmp_dis;
                    min_dis_s = tmp_s;
                }
                if (tmp_dis > 8 && min_dis_to_goal < 8) break;
                tmp_s -= f.search_ds;
            }
            length = min_dis_s;
        }
    }
    *cut_s = length;
    // buildReferenceFromSpline (:474-499): count the samples, stopping one past the cap
    int count = 0;
    double tmp_s = 0;
    while (tmp_s <= length) {
        if (count == f.max_n) return SEG_TOO_MANY;
        const double k = densify_sample(xs, ys, tmp_s).k;
        ++count;
        tmp_s = segment_step(f, tmp_s, k);
    }
    *n = count;
    return SEG_OK;
}

// Write pass of one accepted path (one thread): the same walk as segment_count on the cut length, n states
// (x, y, heading, curvature, s; v = a = 0) into out.  Bit for bit the samples the count pass visited.
PQP_HD void segment_write(const SegmentFlags &f, const SplineView &xs, const SplineView &ys, int n, pqp_state *out) {
    double tmp_s = 0;
    for (int i = 0; i < n; ++i) {
        const pqp_state st = densify_sample(xs, ys, tmp_s);
        out[i] = st;
        tmp_s = segment_step(f, tmp_s, st.k);
    }
}

// Station reservation in index order: path b, with `count` stations (0 when refused) and `before` the stations of
// every path before it (whether kept or not), keeps its stations when before + count <= capacity.  Once the running
// total passes the capacity it stays past it, so the refused paths are a suffix of the paths with stations.
PQP_HD bool segment_fits(long long before, int count, long long capacity) {
    return count > 0 && before + count <= capacity;
}

}  // namespace pqp
