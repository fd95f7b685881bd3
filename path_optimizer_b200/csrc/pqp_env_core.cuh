// pqp_env_core.cuh -- per-thread device functions of the stages either side of the QP:
// distance-map lookup, clearance ray march, covering-circle collision test, cubic-spline
// evaluation.  No warp collectives here: every function is a straight per-thread restatement, so
// the test-only host build (-DPQP_HOST_EMU, tests/emu/) just calls them in a loop.
//
// Reference behaviour being replaced (file:line in the reference tree):
//   Map::getObstacleDistance                       src/tools/Map.cpp:16-22 (over grid_map_core)
//   getClearanceWithDirectionStrict                src/data_struct/reference_path_impl.cpp:283-472
//   getApproxState / updateBounds[Improved]        reference_path_impl.cpp:120-140, 142-201, 237-281
//   CollisionChecker / CarGeometry                 src/tools/collision_checker.cpp:17-59, car_geometry.cpp:38-74
//   tk::spline::operator() / deriv                 src/tools/spline.cpp:250-318
//
// Arithmetic note: products that feed sums are written with mul()/add() so the device build does
// not contract them into FMAs; a lookup then rounds exactly as the reference's separate
// multiply/add sequence does and threshold decisions (clearance < radius) agree bit for bit with
// an IEEE host evaluation apart from the libm-vs-CUDA sin/cos last-ulp differences.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/pqp_env.h"

#if defined(PQP_HOST_EMU) || !defined(__CUDACC__)
#define PQP_HD inline
namespace pqp {
inline double mul(double a, double b) { return a * b; }
inline double add(double a, double b) { return a + b; }
inline float ldg(const float *p) { return *p; }
inline double ldg(const double *p) { return *p; }
}  // namespace pqp
#else
#define PQP_HD __host__ __device__ __forceinline__
namespace pqp {
PQP_HD double mul(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
PQP_HD double add(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
template <typename T> PQP_HD T ldg(const T *p) {
#ifdef __CUDA_ARCH__
    return __ldg(p);
#else
    return *p;
#endif
}
}  // namespace pqp
#endif

namespace pqp {

struct MapView {
    const float *d;     // [rows*cols] row-major, device memory
    int rows, cols;
    double res, cx, cy;
    double lx, ly;      // rows*res, cols*res
    double ox, oy;      // centre of cell 0 along x / y:  c + (0.5*len - 0.5*res)
};

PQP_HD MapView make_map_view(const float *d, int rows, int cols, double res, double cx, double cy) {
    MapView m;
    m.d = d; m.rows = rows; m.cols = cols; m.res = res; m.cx = cx; m.cy = cy;
    m.lx = rows * res; m.ly = cols * res;
    m.ox = cx + (0.5 * m.lx - 0.5 * res);
    m.oy = cy + (0.5 * m.ly - 0.5 * res);
    return m;
}

// The map set of a handle (pqp_set_maps) as the kernels see it: a device table with one descriptor per map, the number
// of maps, and an optional per-path index into the table (NULL: map 0 for every path).  The count is read from memory
// rather than passed by value, so that a captured launch follows a later upload of a set of another size.
struct MapTable {
    const MapView *maps;
    const int32_t *n_maps;
    const int32_t *index;
};

// Descriptor of path b's map, or NULL when its index lies outside [0, n_maps): the index is checked before the table
// is read.
PQP_HD const MapView *map_of(const MapTable &t, int b) {
    const int m = t.index ? t.index[b] : 0;
    return (m >= 0 && m < *t.n_maps) ? t.maps + m : nullptr;
}

// grid_map isInside: 0 <= -((p - c) - len/2) < len on both axes
PQP_HD bool map_inside(const MapView &m, double x, double y) {
    const double tx = -add(x - m.cx, -mul(0.5, m.lx));
    const double ty = -add(y - m.cy, -mul(0.5, m.ly));
    return tx >= 0.0 && ty >= 0.0 && tx < m.lx && ty < m.ly;
}

PQP_HD double cell_center(double o, double res, int idx) { return add(o, mul(res, (double)(-idx))); }

// Map::getObstacleDistance: bilinear over the four surrounding cell centres, nearest cell when a
// neighbour is off the grid, 0 outside the map; rounded to float as grid_map returns it.
PQP_HD double map_distance(const MapView &m, double x, double y) {
    if (!map_inside(m, x, y)) return 0.0;
    const int i0 = (int)(-((add(x, -mul(0.5, m.lx)) - m.cx) / m.res));
    const int j0 = (int)(-((add(y, -mul(0.5, m.ly)) - m.cy) / m.res));
    const double px = cell_center(m.ox, m.res, i0), py = cell_center(m.oy, m.res, j0);
    int i_lo, i_hi, j_lo, j_hi;   // lo/hi coordinate; a larger coordinate is a smaller index
    if (x >= px) { i_lo = i0; i_hi = i0 - 1; } else { i_lo = i0 + 1; i_hi = i0; }
    if (y >= py) { j_lo = j0; j_hi = j0 - 1; } else { j_lo = j0 + 1; j_hi = j0; }
    const bool ok = i_lo >= 0 && i_lo < m.rows && i_hi >= 0 && i_hi < m.rows &&
                    j_lo >= 0 && j_lo < m.cols && j_hi >= 0 && j_hi < m.cols;
    if (!ok) {
        if (i0 < 0 || i0 >= m.rows || j0 < 0 || j0 >= m.cols) return 0.0;
        return (double)ldg(m.d + (size_t)i0 * m.cols + j0);
    }
    const double f0 = ldg(m.d + (size_t)i_lo * m.cols + j_lo);
    const double f1 = ldg(m.d + (size_t)i_hi * m.cols + j_lo);
    const double f2 = ldg(m.d + (size_t)i_lo * m.cols + j_hi);
    const double f3 = ldg(m.d + (size_t)i_hi * m.cols + j_hi);
    const double rx = (x - cell_center(m.ox, m.res, i_lo)) / m.res;
    const double ry = (y - cell_center(m.oy, m.res, j_lo)) / m.res;
    const double fx = 1.0 - rx, fy = 1.0 - ry;
    const double v = add(add(add(mul(mul(f0, fx), fy), mul(mul(f1, rx), fy)), mul(mul(f2, fx), ry)),
                         mul(mul(f3, rx), ry));
    return (double)(float)v;
}

PQP_HD double wrap_angle(double a) {     // constraintAngle, tools.hpp:24-35
    while (a > M_PI) a -= 2 * M_PI;
    while (a < -M_PI) a += 2 * M_PI;
    return a;
}

// One ray: position at signed-free distance t along direction (ca, sa) from (sx, sy)
struct Ray {
    double sx, sy, ca, sa;
    PQP_HD double dist(const MapView &m, double t) const {
        return map_distance(m, add(sx, mul(t, ca)), add(sy, mul(t, sa)));
    }
};

// getClearanceWithDirectionStrict (:283-472) without the original-spline branch (:322-389, needs
// FLAGS_enable_simple_boundary_decision = false).  left/right are signed lateral offsets.
PQP_HD void clearance_strict(const MapView &m, double radius, double sx, double sy, double sz,
                             double &left_bound, double &right_bound) {
    const double delta_s = 0.5;
    const int n = (int)(5.0 / delta_s);
    const double left_angle = wrap_angle(sz + M_PI_2), right_angle = wrap_angle(sz - M_PI_2);
    const Ray L{sx, sy, cos(left_angle), sin(left_angle)};
    const Ray R{sx, sy, cos(right_angle), sin(right_angle)};
    const double original = map_distance(m, sx, sy);
    if (original > radius) {
        double right_s = 0;
        for (int j = 0; j != n; ++j) {
            right_s += delta_s;
            if (R.dist(m, right_s) < radius) break;
        }
        double left_s = 0;
        for (int j = 0; j != n; ++j) {
            left_s += delta_s;
            if (L.dist(m, left_s) < radius) break;
        }
        right_bound = -(right_s - delta_s);
        left_bound = left_s - delta_s;
    } else {
        double right_s = 0;
        for (int j = 0; j != n; ++j) {
            right_s += delta_s;
            if (R.dist(m, right_s) > radius) break;
        }
        double left_s = 0;
        for (int j = 0; j != n; ++j) {
            left_s += delta_s;
            if (L.dist(m, left_s) > radius) break;
        }
        if (left_s < right_s) {
            right_bound = left_s;
            for (int j = 0; j != n; ++j) {
                left_s += delta_s;
                if (L.dist(m, left_s) < radius) break;
            }
            left_bound = left_s - delta_s;
        } else {
            left_bound = -right_s;
            for (int j = 0; j != n; ++j) {
                right_s += delta_s;
                if (R.dist(m, right_s) < radius) break;
            }
            right_bound = -(right_s - delta_s);
        }
    }
    const double smaller_ds = 0.1;
    const int fine = (int)(delta_s / smaller_ds);
    for (int i = 1; i != fine; ++i) {
        left_bound += smaller_ds;
        if (L.dist(m, left_bound) < radius) { left_bound -= smaller_ds; break; }
    }
    for (int i = 1; i != fine; ++i) {
        right_bound -= smaller_ds;
        // the reference walks the RIGHT ray with a negative parameter: x = sx + right_bound*cos(right_angle)
        if (R.dist(m, right_bound) < radius) { right_bound += smaller_ds; break; }
    }
}

// Piecewise-cubic spline in tk::spline's layout: knots t[n], coef[n][4] = {a, b, c, y}.
struct SplineView {
    int n;
    const double *t, *c;
};

PQP_HD double spline_eval(const SplineView &s, int order, double at) {
    int lo = 0, hi = s.n;                       // lower_bound
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (ldg(s.t + mid) < at) lo = mid + 1; else hi = mid;
    }
    int idx = lo - 1;
    if (idx < 0) idx = 0;
    const double h = at - ldg(s.t + idx);
    if (at < ldg(s.t)) {
        const double b0 = ldg(s.c + 1), c0 = ldg(s.c + 2);
        if (order == 0) return add(mul(add(mul(b0, h), c0), h), ldg(s.c + 3));
        if (order == 1) return add(mul(mul(2.0, b0), h), c0);
        return mul(mul(2.0, b0), h);
    }
    const double *c = s.c + 4 * (size_t)idx;
    if (at > ldg(s.t + s.n - 1)) {
        const double *e = s.c + 4 * (size_t)(s.n - 1);
        if (order == 0) return add(mul(add(mul(ldg(e + 1), h), ldg(e + 2)), h), ldg(e + 3));
        if (order == 1) return add(mul(mul(2.0, ldg(e + 1)), h), ldg(e + 2));
        return mul(2.0, ldg(e + 1));
    }
    const double a3 = ldg(c), b2 = ldg(c + 1), c1 = ldg(c + 2), y0 = ldg(c + 3);
    if (order == 0) return add(mul(add(mul(add(mul(a3, h), b2), h), c1), h), y0);
    if (order == 1) return add(mul(add(mul(mul(3.0, a3), h), mul(2.0, b2)), h), c1);
    return add(mul(mul(6.0, a3), h), mul(2.0, b2));
}

// Bounds of one covering circle of one station (one thread).  Returns true when that circle is
// blocked (isEqual(ub, lb) in the improved variant, ub == lb in the simple one).
PQP_HD bool circle_bounds(const MapView &m, double radius, int mode, const pqp_state &st, double dj,
                          const SplineView &xs, const SplineView &ys, double &ub, double &lb) {
    const double cz = cos(st.z), sz = sin(st.z);
    const double cx = add(st.x, mul(dj, cz)), cy = add(st.y, mul(dj, sz));
    if (mode == PQP_BOUNDS_IMPROVED) {
        // getApproxState (:120-140)
        const double x = spline_eval(xs, 0, st.s + dj), y = spline_eval(ys, 0, st.s + dj);
        const double v1x = cx - st.x, v1y = cy - st.y, v2x = x - st.x, v2y = y - st.y;
        const double proj = add(mul(v1x, v2x), mul(v1y, v2y)) / fmax(0.001, sqrt(add(mul(v1x, v1x), mul(v1y, v1y))));
        const double move = fabs(dj) - proj;
        const double sgn = dj >= 0 ? 1.0 : -1.0;
        const double ax = add(x, mul(mul(sgn, move), cz)), ay = add(y, mul(mul(sgn, move), sz));
        clearance_strict(m, radius, ax, ay, st.z, ub, lb);
        const double dx = ax - cx, dy = ay - cy;
        const double offset = add(mul(-dx, sz), mul(dy, cz));          // global2Local(c_j, c_jj).y
        ub += offset;
        lb += offset;
        return fabs(ub - lb) < 1e-6;                                   // isEqual, FLAGS_epsilon
    }
    clearance_strict(m, radius, cx, cy, st.z, ub, lb);
    return ub == lb;
}

// CarGeometry::setCircles (car_geometry.cpp:38-57) with CollisionChecker's constructor arguments
// (collision_checker.cpp:9-15).  c[0] = bounding circle, c[1..6] = rr, rl, fr, fl, fm, rm.
struct CarCircles {
    double x[7], y[7], r[7];
};

inline CarCircles make_car_circles(const pqp_params &p) {
    CarCircles c;
    const double width = p.car_width;
    const double back = p.car_length / 2.0 - p.rear_axle_to_center;
    const double front = p.car_length / 2.0 + p.rear_axle_to_center;
    const double length = front + back;
    c.x[0] = (front - back) / 2.0; c.y[0] = 0;
    c.r[0] = sqrt(pow(length / 2, 2) + pow(width / 2, 2));
    const double shift = width / 4.0;
    const double small_r = sqrt(2 * pow(shift, 2));
    const double large_r = sqrt(pow(width, 2) + pow((length - width) / 2.0, 2)) / 2;
    c.x[1] = -back + shift; c.y[1] = -width / 2.0 + shift; c.r[1] = small_r;
    c.x[2] = -back + shift; c.y[2] = width / 2.0 - shift;  c.r[2] = small_r;
    c.x[3] = front - shift; c.y[3] = -width / 2.0 + shift; c.r[3] = small_r;
    c.x[4] = front - shift; c.y[4] = width / 2.0 - shift;  c.r[4] = small_r;
    c.x[5] = c.x[0] + (length - width) / 4; c.y[5] = 0; c.r[5] = large_r;
    c.x[6] = c.x[0] - (length - width) / 4; c.y[6] = 0; c.r[6] = large_r;
    return c;
}

// What the stages either side of the QP read of one parameter set (pqp_set_param_sets): the covering-circle radius and
// offsets d1..d4 of the bounds, the footprint of the collision check and the "KPC" limits (mu, curvature rate, and
// kmax = tan(max_steering_angle) / wheel_base for limits rebuilt from splines).
struct ParamRow {
    double radius, d[4];
    CarCircles car;
    double mu, rate, kmax;
};

inline ParamRow make_param_row(const pqp_params &p) {
    ParamRow r;
    r.radius = p.circle_radius;
    r.d[0] = p.d1; r.d[1] = p.d2; r.d[2] = p.d3; r.d[3] = p.d4;
    r.car = make_car_circles(p);
    r.mu = p.mu; r.rate = p.max_curvature_rate;
    r.kmax = tan(p.max_steering_angle) / p.wheel_base;
    return r;
}

// The parameter sets of a handle as the kernels see them, passed by value, so that a captured launch keeps the sets it
// was captured with (as the solve kernels keep their by-value pqp::DevParams): R rows of which the first n are in use,
// and an optional per-path index into them (NULL: row 0 for every path).  R = 1 without an index, PQP_MAX_PARAM_SETS
// with one.
template <int R> struct ParamTable {
    ParamRow row[R];
    int n;
    const int32_t *index;
};

// Path b's row, or NULL when its index lies outside [0, n): the index is checked before the rows are read.
template <int R> PQP_HD const ParamRow *param_of(const ParamTable<R> &t, int b) {
    const int k = t.index ? t.index[b] : 0;
    return (k >= 0 && k < t.n) ? &t.row[k] : nullptr;
}

// isSingleStateCollisionFreeImproved (:41-59) -> isSingleStateCollisionFree (:17-39)
PQP_HD bool state_collision_free(const MapView &m, const CarCircles &c, double sx, double sy, double sz) {
    const double cz = cos(sz), sn = sin(sz);
    // local2Global, tools.cpp:54-59: x*cos - y*sin + X, x*sin + y*cos + Y
    const double bx = add(add(mul(c.x[0], cz), -mul(c.y[0], sn)), sx);
    const double by = add(add(mul(c.x[0], sn), mul(c.y[0], cz)), sy);
    if (!map_inside(m, bx, by)) return false;
    if (!(map_distance(m, bx, by) < c.r[0])) return true;
    for (int k = 1; k < 7; ++k) {
        const double x = add(add(mul(c.x[k], cz), -mul(c.y[k], sn)), sx);
        const double y = add(add(mul(c.x[k], sn), mul(c.y[k], cz)), sy);
        if (!map_inside(m, x, y)) return false;
        if (map_distance(m, x, y) < c.r[k]) return false;
    }
    return true;
}

// tk::spline::set_points requires strictly increasing knots (an assert, spline.cpp:165): a path whose s repeats or
// goes back (a duplicate waypoint) or is NaN is not resampled -- the densifying tail reports it as failed.
PQP_HD bool knots_increasing(int n, const double *t) {
    for (int i = 1; i < n; ++i)
        if (!(t[i] > t[i - 1])) return false;
    return true;
}

// Natural cubic spline through (t_i, Y(i)): tk::spline::set_points with its default boundary
// (spline.cpp:146-249: zero second derivative at both ends), re-derived.  Unknowns b_i = f''/2
// from the tridiagonal continuity system (Thomas elimination, one thread), then a_i, c_i; the last
// knot carries the right-extrapolation polynomial.  coef[i] = {a, b, c, y}; diag/rhs: n scratch each.
template <typename F>
PQP_HD void spline_fit(int n, const double *t, F Y, double *coef, double *diag, double *rhs) {
    diag[0] = 2.0; rhs[0] = 0.0;
    double upper_prev = 0.0;
    for (int i = 1; i < n - 1; ++i) {
        const double hl = t[i] - t[i - 1], hr = t[i + 1] - t[i];
        const double lo = hl / 3.0, di = mul(2.0, t[i + 1] - t[i - 1]) / 3.0, up = hr / 3.0;
        const double r = (Y(i + 1) - Y(i)) / hr - (Y(i) - Y(i - 1)) / hl;
        const double w = lo / diag[i - 1];
        diag[i] = add(di, -mul(w, upper_prev));
        rhs[i] = add(r, -mul(w, rhs[i - 1]));
        upper_prev = up;
    }
    coef[4 * (n - 1) + 1] = 0.0;                 // b lives in coef[4i+1]
    for (int i = n - 2; i >= 1; --i) {
        const double up = (t[i + 1] - t[i]) / 3.0;
        coef[4 * i + 1] = add(rhs[i], -mul(up, coef[4 * (i + 1) + 1])) / diag[i];
    }
    coef[1] = 0.0;
    for (int i = 0; i < n - 1; ++i) {
        const double h = t[i + 1] - t[i];
        const double bi = coef[4 * i + 1], bn = coef[4 * (i + 1) + 1];
        coef[4 * i + 0] = (bn - bi) / mul(3.0, h);
        coef[4 * i + 2] = add((Y(i + 1) - Y(i)) / h, -(mul(add(mul(2.0, bi), bn), h) / 3.0));
        coef[4 * i + 3] = Y(i);
    }
    const int i = n - 2;
    const double h = t[n - 1] - t[n - 2];
    coef[4 * (n - 1) + 0] = 0.0;
    coef[4 * (n - 1) + 2] = add(add(mul(mul(mul(3.0, coef[4 * i]), h), h), mul(mul(2.0, coef[4 * i + 1]), h)), coef[4 * i + 2]);
    coef[4 * (n - 1) + 3] = Y(n - 1);
}

// The knots pqp_fit_splines_device fits a path's splines on: at least three, finite and strictly increasing.  A strictly
// increasing sequence lies between its ends, so only the ends need the finiteness test.
PQP_HD bool fit_knots_ok(int n, const double *t) {
    return n >= 3 && knots_increasing(n, t) && t[0] >= -1.7976931348623157e308 && t[n - 1] <= 1.7976931348623157e308;
}

// One thread of pqp_fit_splines_device: coordinate `coord` (0: x, 1: y) of the path whose n stations start at ref,
// on knots t that are already in place.  coef: that coordinate's n rows; scr: 4n doubles of scratch shared by the
// path's two threads (x: [0, 2n), y: [2n, 4n)).  A refused path gets NaN rows (the x thread also sets its knots to
// NaN, so the caller must have finished every read of t by the path's y thread first).
PQP_HD void fit_path_coord(int n, bool ok, int coord, const pqp_state *ref, double *t, double *coef, double *scr) {
    static_assert(sizeof(pqp_state) == 7 * sizeof(double), "pqp_state: seven doubles");
    if (!ok) {
        const double nan_v = nan("");
        for (int i = 0; i < 4 * n; ++i) coef[i] = nan_v;
        if (coord == 0)
            for (int i = 0; i < n; ++i) t[i] = nan_v;
        return;
    }
    const double *y = coord ? &ref[0].y : &ref[0].x;
    spline_fit(n, t, [&](int i) { return ldg(y + 7 * (size_t)i); }, coef, scr + 2 * (size_t)coord * n,
               scr + (2 * (size_t)coord + 1) * n);
}

// One resampled output state (path_optimizer.cpp:216-222): position from the splines, heading and
// curvature from their derivatives (getHeading / getCurvature, tools.cpp:34-46).
PQP_HD pqp_state densify_sample(const SplineView &xs, const SplineView &ys, double ts) {
    pqp_state st;
    st.x = spline_eval(xs, 0, ts);
    st.y = spline_eval(ys, 0, ts);
    const double x1 = spline_eval(xs, 1, ts), y1 = spline_eval(ys, 1, ts);
    const double x2 = spline_eval(xs, 2, ts), y2 = spline_eval(ys, 2, ts);
    st.z = atan2(y1, x1);
    st.k = add(mul(x1, y2), -mul(y1, x2)) / pow(add(mul(x1, x1), mul(y1, y1)), 1.5);
    st.s = ts;
    st.v = 0; st.a = 0;
    return st;
}

// s re-accumulation of the raw tail (path_optimizer.cpp:192-195), in the reference's serial order
PQP_HD void accumulate_s(int n, pqp_state *p) {
    double s = 0, px = 0, py = 0;
    for (int i = 0; i < n; ++i) {
        const double x = p[i].x, y = p[i].y;
        if (i != 0) {
            const double dx = px - x, dy = py - y;
            s = add(s, sqrt(add(mul(dx, dx), mul(dy, dy))));
        }
        p[i].s = s;
        px = x; py = y;
    }
}

}  // namespace pqp
