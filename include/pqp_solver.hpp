// pqp_solver.hpp -- C++ host side above the C ABI (include/pqp.h), header only.
//
// Mirrors the reference's solver interface for the hot path so that the call sites read the same:
//   reference                                                      here
//   PathOptimizationNS::State                (data_struct.hpp:13)  pqp::State   (layout == pqp_state)
//   CoveringCircleBounds                     (data_struct.hpp:72)  pqp::CoveringCircleBounds
//   OsqpSolver::create(type, ref, veh, N)    (solver.cpp:30-44)    pqp::GpuOsqpSolver::create(...)
//   bool OsqpSolver::solve(vector<State>*)   (solver.cpp:46-77)    bool GpuOsqpSolver::solve(vector<State>*)
//   -- (the reference has no batched form) --                      pqp::BatchPathSolver::solve(...)
// Error behaviour follows the reference: create() returns nullptr for an unknown type string
// (solver.cpp:41-43, "No such solver!"), solve() returns false unless the QP status is SOLVED
// (osqp-eigen semantics) and leaves *optimized_path cleared in that case.  Nothing throws.
//
// ROS-free: depends only on the C++17 standard library and libpqp.so.
#ifndef PQP_SOLVER_HPP_
#define PQP_SOLVER_HPP_

#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "pqp.h"

namespace pqp {

// PathOptimizationNS::State (data_struct.hpp:13-30): same field order, same defaults.
struct State {
    State() = default;
    State(double x, double y, double z = 0, double k = 0, double s = 0, double v = 0, double a = 0)
        : x(x), y(y), z(z), k(k), s(s), v(v), a(a) {}
    double x{}, y{}, z{} /* heading */, k{} /* curvature */, s{}, v{}, a{};
};
static_assert(sizeof(State) == sizeof(pqp_state), "State must alias pqp_state");

// CoveringCircleBounds (data_struct.hpp:72-91): ub = left, lb = right, per covering circle.
struct CoveringCircleBounds {
    struct SingleCircleBounds {
        double ub{}, lb{};
    } c0, c1, c2, c3;
};
static_assert(sizeof(CoveringCircleBounds) == sizeof(pqp_station_bounds), "bounds must alias pqp_station_bounds");

// What the solver reads from VehicleState (vehicle_state_frenet.hpp): getInitError(), getStartState().k,
// getEndState().z.
struct VehicleStateView {
    double init_offset{};        // getInitError()[0]
    double init_heading_error{}; // getInitError()[1]
    double start_k{};            // getStartState().k
    double end_heading{};        // getEndState().z
};

inline int formulation_from_type(const std::string &type) {
    if (type == "KP") return PQP_FORM_KP;
    if (type == "K") return PQP_FORM_K;
    if (type == "KPC") return PQP_FORM_KPC;  // NB the gflags validator says "KCP" (planning_flags.cpp:96-99)
    return -1;
}

// RAII owner of a pqp_handle.
class Handle {
 public:
    Handle() = default;
    ~Handle() { reset(); }
    Handle(const Handle &) = delete;
    Handle &operator=(const Handle &) = delete;
    bool open(const pqp_params *params, int device, int max_batch, int max_total_points) {
        reset();
        pqp_params def;
        if (!params) {
            pqp_params_default(&def);
            params = &def;
        }
        return pqp_create(&h_, params, device, max_batch, max_total_points) == PQP_OK;
    }
    void reset() {
        if (h_) pqp_destroy(h_);
        h_ = nullptr;
    }
    pqp_handle *get() const { return h_; }
    explicit operator bool() const { return h_ != nullptr; }

 private:
    pqp_handle *h_ = nullptr;
};

// Batched form: `batch` independent paths, concatenated station arrays.
class BatchPathSolver {
 public:
    struct Result {
        std::vector<State> states;        // [sum N] optimized paths (x, y, heading, k, s)
        std::vector<double> frenet;       // [sum N][3] (e_y, e_phi, kappa)
        std::vector<int32_t> status;      // [batch] pqp_status
        std::vector<int32_t> iters;       // [batch]
        pqp_stats stats{};
        int rc = PQP_OK;
    };

    static std::unique_ptr<BatchPathSolver> create(const std::string &type, int max_batch, int max_total_points,
                                                   const pqp_params *params = nullptr, int device = 0) {
        const int form = formulation_from_type(type);
        if (form < 0) {
            std::fprintf(stderr, "No such solver!\n");
            return nullptr;
        }
        std::unique_ptr<BatchPathSolver> s(new BatchPathSolver);
        s->form_ = form;
        if (!s->handle_.open(params, device, max_batch, max_total_points)) {
            std::fprintf(stderr, "pqp_create failed: %s\n", pqp_last_error());
            return nullptr;
        }
        return s;
    }

    // Several parameter sets on one handle (pqp_set_param_sets): param_sets[k] is set k of solve()'s param_index,
    // param_sets[0] the set of a solve without one.
    static std::unique_ptr<BatchPathSolver> create(const std::string &type, int max_batch, int max_total_points,
                                                   const std::vector<pqp_params> &param_sets, int device = 0) {
        if (param_sets.empty()) return nullptr;
        std::unique_ptr<BatchPathSolver> s = create(type, max_batch, max_total_points, &param_sets[0], device);
        if (s && pqp_set_param_sets(s->handle_.get(), (int)param_sets.size(), param_sets.data()) != PQP_OK) {
            std::fprintf(stderr, "pqp_set_param_sets failed: %s\n", pqp_last_error());
            return nullptr;
        }
        return s;
    }

    // n_points[b] stations per path; reference_states / bounds concatenated; vehicle[b] per path.
    bool solve(const std::vector<int32_t> &n_points, const std::vector<State> &reference_states,
               const std::vector<CoveringCircleBounds> &bounds, const std::vector<VehicleStateView> &vehicle,
               Result *out) {
        return solve(n_points, reference_states, bounds, vehicle, nullptr, out);
    }

    // The same with param_index[b] naming the parameter set path b is solved with (pqp_solve_batch_sets): OsqpSolver::solve
    // once per path with that path's FLAGS_*.  A path whose index names no set reports PQP_INVALID_PROBLEM.
    bool solve(const std::vector<int32_t> &n_points, const std::vector<State> &reference_states,
               const std::vector<CoveringCircleBounds> &bounds, const std::vector<VehicleStateView> &vehicle,
               const std::vector<int32_t> &param_index, Result *out) {
        if (param_index.size() != n_points.size()) return false;
        return solve(n_points, reference_states, bounds, vehicle, param_index.data(), out);
    }

    // The same with method[b] ("KP", "K" or "KPC") the FLAGS_optimization_method path b is solved with
    // (pqp_solve_batch_forms): OsqpSolver::create(method[b], ...) and solve once per path.  An empty param_index means
    // set 0 for every path.  A path whose method is no formulation reports PQP_INVALID_PROBLEM, as the reference's
    // create returns nullptr for it.  "KPC" paths read max_k / max_kp (concatenated like reference_states;
    // ReferencePath::getMaxKList / getMaxKpList); without them a batch with a "KPC" path fails with PQP_ERR_ARG.
    bool solve(const std::vector<int32_t> &n_points, const std::vector<State> &reference_states,
               const std::vector<CoveringCircleBounds> &bounds, const std::vector<VehicleStateView> &vehicle,
               const std::vector<int32_t> &param_index, const std::vector<std::string> &method, Result *out,
               const std::vector<double> *max_k = nullptr, const std::vector<double> *max_kp = nullptr) {
        if ((!param_index.empty() && param_index.size() != n_points.size()) || method.size() != n_points.size())
            return false;
        std::vector<int32_t> forms(method.size());
        for (size_t b = 0; b < method.size(); ++b) forms[b] = formulation_from_type(method[b]);
        return solve(n_points, reference_states, bounds, vehicle, param_index.empty() ? nullptr : param_index.data(), out,
                     forms.data(), max_k ? max_k->data() : nullptr, max_kp ? max_kp->data() : nullptr);
    }

    pqp_handle *handle() const { return handle_.get(); }

 private:
    // forms NULL: pqp_solve_batch_sets with the solver's type; else pqp_solve_batch_forms
    bool solve(const std::vector<int32_t> &n_points, const std::vector<State> &reference_states,
               const std::vector<CoveringCircleBounds> &bounds, const std::vector<VehicleStateView> &vehicle,
               const int32_t *param_index, Result *out, const int32_t *forms = nullptr, const double *max_k = nullptr,
               const double *max_kp = nullptr) {
        const int batch = (int)n_points.size();
        size_t total = 0;
        for (int n : n_points) total += (size_t)n;
        if (!out || reference_states.size() < total || bounds.size() < total || (int)vehicle.size() < batch) return false;
        std::vector<double> x0(3 * (size_t)batch), endh((size_t)batch);
        for (int b = 0; b < batch; ++b) {
            x0[3 * b] = vehicle[b].init_offset;            // solver_kp_as_input.cpp:143-147
            x0[3 * b + 1] = vehicle[b].init_heading_error;
            x0[3 * b + 2] = vehicle[b].start_k;
            endh[b] = vehicle[b].end_heading;              // :196
        }
        out->states.assign(total, State());
        out->frenet.assign(3 * total, 0.0);
        out->status.assign(batch, PQP_UNSOLVED);
        out->iters.assign(batch, 0);
        const pqp_state *ref = reinterpret_cast<const pqp_state *>(reference_states.data());
        const pqp_station_bounds *bnd = reinterpret_cast<const pqp_station_bounds *>(bounds.data());
        pqp_state *states = reinterpret_cast<pqp_state *>(out->states.data());
        if (forms)
            out->rc = pqp_solve_batch_forms(handle_.get(), batch, n_points.data(), ref, bnd, x0.data(), endh.data(), max_k,
                                            max_kp, param_index, forms, states, out->frenet.data(), out->status.data(),
                                            out->iters.data(), &out->stats);
        else
            out->rc = pqp_solve_batch_sets(handle_.get(), form_, batch, n_points.data(), ref, bnd, x0.data(), endh.data(),
                                           nullptr, nullptr, param_index, states, out->frenet.data(), out->status.data(),
                                           out->iters.data(), &out->stats);
        if (out->rc != PQP_OK)
            std::fprintf(stderr, "%s failed: %s\n", forms ? "pqp_solve_batch_forms" : "pqp_solve_batch_sets", pqp_last_error());
        return out->rc == PQP_OK;
    }

    BatchPathSolver() = default;
    Handle handle_;
    int form_ = PQP_FORM_KP;
};

// Single-path adaptor with the reference's call shape; this is what replaces
// `OsqpSolver::create(FLAGS_optimization_method, *reference_path_, *vehicle_state_, size_)`
// at path_optimizer.cpp:182 (see INTEGRATION.md).
class GpuOsqpSolver {
 public:
    static std::unique_ptr<GpuOsqpSolver> create(const std::string &type, const std::vector<State> &reference_states,
                                                 const std::vector<CoveringCircleBounds> &bounds,
                                                 const VehicleStateView &vehicle_state, const size_t &horizon,
                                                 const pqp_params *params = nullptr, int device = 0) {
        if (reference_states.size() < horizon || bounds.size() < horizon) return nullptr;
        std::unique_ptr<GpuOsqpSolver> s(new GpuOsqpSolver(reference_states, bounds, vehicle_state, horizon));
        s->batch_ = BatchPathSolver::create(type, 1, (int)(horizon > 2 ? horizon : 2), params, device);
        if (!s->batch_) return nullptr;
        return s;
    }

    // bool OsqpSolver::solve(std::vector<State>*): true iff OSQP status == SOLVED.
    bool solve(std::vector<State> *optimized_path) {
        if (!optimized_path) return false;
        BatchPathSolver::Result r;
        std::vector<int32_t> n{(int32_t)horizon_};
        std::vector<VehicleStateView> v{vehicle_};
        if (!batch_->solve(n, ref_, bounds_, v, &r)) return false;
        last_status_ = r.status[0];
        last_iters_ = r.iters[0];
        if (r.status[0] != PQP_SOLVED) return false;
        optimized_path->clear();  // solver_kp_as_input.cpp:29
        optimized_path->assign(r.states.begin(), r.states.end());
        return true;
    }
    int last_status() const { return last_status_; }
    int last_iters() const { return last_iters_; }

 private:
    GpuOsqpSolver(const std::vector<State> &ref, const std::vector<CoveringCircleBounds> &b,
                  const VehicleStateView &v, size_t horizon)
        : ref_(ref), bounds_(b), vehicle_(v), horizon_(horizon) {}
    // like the reference (solver.hpp:50-51) the solver holds references: both must outlive it
    const std::vector<State> &ref_;
    const std::vector<CoveringCircleBounds> &bounds_;
    VehicleStateView vehicle_;
    size_t horizon_;
    std::unique_ptr<BatchPathSolver> batch_;
    int last_status_ = PQP_UNSOLVED, last_iters_ = 0;
};

}  // namespace pqp
#endif  // PQP_SOLVER_HPP_
