// pqp_dispatch.h -- per-path kernel-class selection that host and device evaluate alike: keep_control_steps from the
// reference states, the caller's bounds, and one lookup in the class table pqp_create builds with class_for
// (pqp_capi.cu).  The table is the only description of the selection, so the device dispatch
// (pqp_solve_batch_device_dispatch, pqp_plan_batch_device) picks the class pqp_solve_batch would pick for every path.
// Plain C++ as well: tests/emu/dispatch_emu.cpp compiles it with g++.
#pragma once
#include <stdint.h>

#include "../../include/pqp.h"

#if defined(__CUDACC__) && !defined(PQP_HOST_EMU)
#define PQP_HD __host__ __device__ __forceinline__
#else
#define PQP_HD inline
#endif

namespace pqp {

// rows of a class table: keep_control_steps 1..10, then one row for every keep > 10
constexpr int kTableKeepRows = 11;

// keep_control_steps_ of one path, in double as the reference computes it: reference_interval_ = max ds over the first
// <= 9 intervals (solver.cpp:21-27, std::max: a NaN interval leaves the maximum as it was), then
// max(int(1.2 / reference_interval_), 1) (solver_kp_as_input.cpp:17).  KPC holds a control for 4 stations
// (solver_kp_as_input_constrained.cpp:17); K has no hold.  pqp_keep_control_steps is this function.
PQP_HD int keep_control_steps(int formulation, const pqp_state *ref, int n_points) {
    if (formulation == PQP_FORM_K) return 1;
    if (formulation == PQP_FORM_KPC) return 4;
    if (!ref || n_points < 2) return 1;
    double interval = 0;
    for (int i = 1; i < n_points && i < 10; ++i) {
        const double ds = ref[i].s - ref[i - 1].s;
        interval = interval < ds ? ds : interval;
    }
    const double q = 1.2 / interval;
    const int keep = (q == q && q < 2147483647.0) ? (int)q : (q == q ? 2147483647 : 0);
    return keep > 1 ? keep : 1;
}

// Class-table index of a path of n stations at keep_control_steps = keep, or -1 when the path lies outside the bounds
// the caller stated (max_n = 0, min_keep = 0, max_keep = 0: unknown; keep bounds apply to "KP" only).  `table` is the
// formulation's table: kTableKeepRows rows of `ncols` entries, entry [keep - 1][n] for n < ncols; column ncols - 1 is
// one station past the longest path any class takes, where every longer path lands too.
PQP_HD int dispatch_class(const int8_t *table, int ncols, int formulation, int n, int keep, int max_n, int min_keep,
                          int max_keep) {
    if (max_n > 0 && n > max_n) return -1;
    if (formulation == PQP_FORM_KP && ((min_keep > 0 && keep < min_keep) || (max_keep > 0 && keep > max_keep))) return -1;
    const int row = keep > 10 ? kTableKeepRows - 1 : (keep < 1 ? 0 : keep - 1);
    const int col = n < 0 ? 0 : (n >= ncols ? ncols - 1 : n);
    return table[row * ncols + col];
}

}  // namespace pqp
