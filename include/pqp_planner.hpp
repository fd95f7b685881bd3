// pqp_planner.hpp -- C++ host side above include/pqp_env.h, header only: the stages either side of
// the QP with the reference's call shapes.
//   reference                                                            here
//   Map(grid_map) / getObstacleDistance            (Map.cpp:8-22)         pqp::DistanceMap + PathOptimizerGpu::getObstacleDistance
//   tk::spline set_points / operator() / deriv     (spline.cpp:161-318)   pqp::Spline
//   CollisionChecker::isSingleStateCollisionFreeImproved (collision_checker.cpp:41-59)   PathOptimizerGpu::isCollisionFree
//   ReferencePath::updateBounds(map)               (reference_path.cpp:77-79)            PathOptimizerGpu::updateBounds
//   PathOptimizer::solveWithoutSmoothing(ref, &path)  (path_optimizer.cpp:87-117)        PathOptimizerGpu::solveWithoutSmoothing
// A PathOptimizerGpu may hold several maps (scenes) at once, with one map index per reference in the batched
// solveWithoutSmoothing; the reference has one map per PathOptimizer and no counterpart for this.
// The single-path overloads keep the reference's signatures; the vector-of-paths overloads are the
// batched forms the GPU is for.  FLAGS_enable_raw_output / enable_collision_check / output_spacing
// (planning_flags.cpp:127-133) are members with the same defaults.  Nothing throws; a bool result
// means what the reference's bool means.
#ifndef PQP_PLANNER_HPP_
#define PQP_PLANNER_HPP_

#include <vector>

#include "pqp_env.h"
#include "pqp_solver.hpp"

namespace pqp {

// Row-major copy of a grid_map "distance" layer (see pqp_distance_map for the index convention).
struct DistanceMap {
    std::vector<float> distance;
    int rows = 0, cols = 0;
    double resolution = 0, center_x = 0, center_y = 0;
    pqp_distance_map view() const { return pqp_distance_map{distance.data(), rows, cols, resolution, center_x, center_y}; }
};

// tk::spline's interface (natural boundary, quadratic extrapolation): set_points, operator(), deriv.
class Spline {
 public:
    bool set_points(const std::vector<double> &x, const std::vector<double> &y) {
        if (x.size() != y.size() || x.size() < 3) return false;
        x_ = x;
        coef_.assign(4 * x.size(), 0.0);
        return pqp_spline_fit((int)x.size(), x_.data(), y.data(), coef_.data()) == PQP_OK;
    }
    double operator()(double at) const { return pqp_spline_eval((int)x_.size(), x_.data(), coef_.data(), 0, at); }
    double deriv(int order, double at) const { return pqp_spline_eval((int)x_.size(), x_.data(), coef_.data(), order, at); }
    const std::vector<double> &knots() const { return x_; }
    const std::vector<double> &coefficients() const { return coef_; }   // [n][4] = a, b, c, y

 private:
    std::vector<double> x_, coef_;
};

class PathOptimizerGpu {
 public:
    bool enable_raw_output = true;        // FLAGS_enable_raw_output
    bool enable_collision_check = true;   // FLAGS_enable_collision_check
    double output_spacing = 0.3;          // FLAGS_output_spacing
    int bounds_mode = PQP_BOUNDS_SIMPLE;  // PQP_BOUNDS_IMPROVED needs the splines argument
    int max_output_states = 1024;         // room per path for the densified output

    // PathOptimizer(start, end, map) (path_optimizer.cpp:19-31): start/end states per path are passed
    // with each call instead (a batch has one pair per path).
    static std::unique_ptr<PathOptimizerGpu> create(const DistanceMap &map, int max_batch, int max_total_points,
                                                    const pqp_params *params = nullptr, int device = 0) {
        return create(std::vector<DistanceMap>{map}, max_batch, max_total_points, params, device);
    }

    // Several scenes on one handle: maps[m] is map m of the batched solveWithoutSmoothing's map index.  The
    // single-path calls (getObstacleDistance, isCollisionFree, updateBounds, solveWithoutSmoothing without an index)
    // use maps[0].
    static std::unique_ptr<PathOptimizerGpu> create(const std::vector<DistanceMap> &maps, int max_batch,
                                                    int max_total_points, const pqp_params *params = nullptr,
                                                    int device = 0) {
        std::unique_ptr<PathOptimizerGpu> p(new PathOptimizerGpu);
        if (!p->handle_.open(params, device, max_batch, max_total_points)) {
            std::fprintf(stderr, "pqp_create failed: %s\n", pqp_last_error());
            return nullptr;
        }
        std::vector<pqp_distance_map> v;
        for (const DistanceMap &m : maps) v.push_back(m.view());
        if (pqp_set_maps(p->handle_.get(), (int)v.size(), v.data()) != PQP_OK) {
            std::fprintf(stderr, "pqp_set_maps failed: %s\n", pqp_last_error());
            return nullptr;
        }
        return p;
    }

    double getObstacleDistance(double x, double y) const {
        const double xy[2] = {x, y};
        double d = 0;
        pqp_map_distance(handle_.get(), 1, xy, &d);
        return d;
    }

    bool isCollisionFree(const State &s) const {
        int32_t ok = 0;
        pqp_check_states(handle_.get(), 1, reinterpret_cast<const pqp_state *>(&s), &ok);
        return ok != 0;
    }

    // ReferencePath::updateBounds for a batch; n_valid[b] = stations that keep their bounds.
    bool updateBounds(const std::vector<std::vector<State>> &references, std::vector<std::vector<CoveringCircleBounds>> *bounds,
                      std::vector<int32_t> *n_valid, const std::vector<Spline> *x_s = nullptr,
                      const std::vector<Spline> *y_s = nullptr) {
        Packed in;
        if (!pack(references, x_s, y_s, &in)) return false;
        std::vector<CoveringCircleBounds> flat(in.ref.size());
        n_valid->assign(references.size(), 0);
        const int rc = pqp_update_bounds_batch(handle_.get(), in.mode, (int)references.size(), in.n.data(),
                                               reinterpret_cast<const pqp_state *>(in.ref.data()), in.nk_ptr(), in.knots_ptr(),
                                               in.xc_ptr(), in.yc_ptr(), reinterpret_cast<pqp_station_bounds *>(flat.data()),
                                               n_valid->data(), nullptr);
        if (rc != PQP_OK) return false;
        bounds->assign(references.size(), {});
        size_t off = 0;
        for (size_t b = 0; b < references.size(); ++b) {
            (*bounds)[b].assign(flat.begin() + off, flat.begin() + off + (*n_valid)[b]);   // bounds_ is cut at the blocked station
            off += references[b].size();
        }
        return true;
    }

    // Batched PathOptimizer::solveWithoutSmoothing: ok[b] is the reference's return value for path b and
    // (*final_paths)[b] what it would have left in *final_path.
    bool solveWithoutSmoothing(const std::vector<std::vector<State>> &references, const std::vector<VehicleStateView> &vehicle,
                               std::vector<std::vector<State>> *final_paths, std::vector<char> *ok,
                               const std::vector<Spline> *x_s = nullptr, const std::vector<Spline> *y_s = nullptr,
                               std::vector<int32_t> *status = nullptr) {
        return plan(references, vehicle, nullptr, final_paths, ok, x_s, y_s, status);
    }

    // The same with map_index[b] naming the map (of those the optimizer was created with) reference b is planned on.
    // A reference whose index names no map gets ok = 0, an empty path and status PQP_INVALID_PROBLEM.
    bool solveWithoutSmoothing(const std::vector<std::vector<State>> &references, const std::vector<VehicleStateView> &vehicle,
                               const std::vector<int32_t> &map_index, std::vector<std::vector<State>> *final_paths,
                               std::vector<char> *ok, const std::vector<Spline> *x_s = nullptr,
                               const std::vector<Spline> *y_s = nullptr, std::vector<int32_t> *status = nullptr) {
        if (map_index.size() != references.size()) return false;
        return plan(references, vehicle, map_index.data(), final_paths, ok, x_s, y_s, status);
    }

    // The reference's single-path signature (path_optimizer.cpp:87-88).
    bool solveWithoutSmoothing(const std::vector<State> &reference_points, const VehicleStateView &vehicle,
                               std::vector<State> *final_path) {
        if (!final_path || reference_points.empty()) return false;   // "Empty input, quit path optimization!"
        std::vector<std::vector<State>> out;
        std::vector<char> ok;
        if (!solveWithoutSmoothing({reference_points}, {vehicle}, &out, &ok)) return false;
        *final_path = out[0];
        return ok[0] != 0;
    }

    pqp_handle *handle() const { return handle_.get(); }

 private:
    // Batched solveWithoutSmoothing (pqp_plan_batch_maps; map_index NULL: map 0 for every reference).
    bool plan(const std::vector<std::vector<State>> &references, const std::vector<VehicleStateView> &vehicle,
              const int32_t *map_index, std::vector<std::vector<State>> *final_paths, std::vector<char> *ok,
              const std::vector<Spline> *x_s, const std::vector<Spline> *y_s, std::vector<int32_t> *status) {
        const int B = (int)references.size();
        Packed in;
        if (!final_paths || !ok || (int)vehicle.size() < B || !pack(references, x_s, y_s, &in)) return false;
        std::vector<double> x0(3 * (size_t)B), endh((size_t)B);
        for (int b = 0; b < B; ++b) {
            x0[3 * b] = vehicle[b].init_offset;           // setInitError(0, 0) in the reference (path_optimizer.cpp:97)
            x0[3 * b + 1] = vehicle[b].init_heading_error;
            x0[3 * b + 2] = vehicle[b].start_k;
            endh[b] = vehicle[b].end_heading;
        }
        const bool raw = enable_raw_output;
        std::vector<State> out(raw ? in.ref.size() : (size_t)B * max_output_states);
        std::vector<int32_t> n_out(B), okv(B), st(B);
        const int rc = pqp_plan_batch_maps(handle_.get(), PQP_FORM_KP, in.mode, raw ? PQP_OUTPUT_RAW : PQP_OUTPUT_DENSIFY,
                                           B, in.n.data(), reinterpret_cast<const pqp_state *>(in.ref.data()), map_index,
                                           in.nk_ptr(), in.knots_ptr(), in.xc_ptr(), in.yc_ptr(), x0.data(), endh.data(),
                                           output_spacing, enable_collision_check ? 1 : 0, max_output_states,
                                           reinterpret_cast<pqp_state *>(out.data()), n_out.data(), okv.data(), st.data(),
                                           nullptr, nullptr, nullptr);
        if (rc != PQP_OK) {
            std::fprintf(stderr, "pqp_plan_batch_maps failed: %s\n", pqp_last_error());
            return false;
        }
        final_paths->assign(B, {});
        ok->assign(B, 0);
        size_t off = 0;
        for (int b = 0; b < B; ++b) {
            const size_t base = raw ? off : (size_t)b * max_output_states;
            (*final_paths)[b].assign(out.begin() + base, out.begin() + base + n_out[b]);
            (*ok)[b] = (char)(okv[b] != 0);
            off += references[b].size();
        }
        if (status) *status = st;
        return true;
    }

    struct Packed {
        std::vector<int32_t> n, nk;
        std::vector<State> ref;
        std::vector<double> knots, xc, yc;
        int mode = PQP_BOUNDS_SIMPLE;
        const int32_t *nk_ptr() const { return mode == PQP_BOUNDS_IMPROVED ? nk.data() : nullptr; }
        const double *knots_ptr() const { return mode == PQP_BOUNDS_IMPROVED ? knots.data() : nullptr; }
        const double *xc_ptr() const { return mode == PQP_BOUNDS_IMPROVED ? xc.data() : nullptr; }
        const double *yc_ptr() const { return mode == PQP_BOUNDS_IMPROVED ? yc.data() : nullptr; }
    };
    bool pack(const std::vector<std::vector<State>> &references, const std::vector<Spline> *x_s,
              const std::vector<Spline> *y_s, Packed *p) const {
        p->mode = (bounds_mode == PQP_BOUNDS_IMPROVED && x_s && y_s) ? PQP_BOUNDS_IMPROVED : PQP_BOUNDS_SIMPLE;
        if (bounds_mode == PQP_BOUNDS_IMPROVED && p->mode != PQP_BOUNDS_IMPROVED) return false;
        for (size_t b = 0; b < references.size(); ++b) {
            p->n.push_back((int32_t)references[b].size());
            p->ref.insert(p->ref.end(), references[b].begin(), references[b].end());
            if (p->mode == PQP_BOUNDS_IMPROVED) {
                if (b >= x_s->size() || b >= y_s->size()) return false;
                const Spline &sx = (*x_s)[b], &sy = (*y_s)[b];
                if (sx.knots().size() != sy.knots().size()) return false;
                p->nk.push_back((int32_t)sx.knots().size());
                p->knots.insert(p->knots.end(), sx.knots().begin(), sx.knots().end());
                p->xc.insert(p->xc.end(), sx.coefficients().begin(), sx.coefficients().end());
                p->yc.insert(p->yc.end(), sy.coefficients().begin(), sy.coefficients().end());
            }
        }
        return true;
    }
    PathOptimizerGpu() = default;
    Handle handle_;
};

}  // namespace pqp
#endif  // PQP_PLANNER_HPP_
