// dispatch_emu.cpp -- TEST HARNESS: the per-path class selection of the device dispatch (keep_control_steps, the
// caller's bounds, the class-table lookup of pqp_dispatch.h) compiled with plain g++, so that the CPU suite can hold it
// against the host selection (pqp_keep_control_steps + pqp_class_info_form) without a GPU.  Never linked into libpqp.so.
#include "../../path_optimizer_b200/csrc/pqp_dispatch.h"

extern "C" int dispatch_emu_class(const int8_t *table, int ncols, int formulation, const pqp_state *ref, int n_points,
                                  int max_n, int min_keep, int max_keep, int *keep_out) {
    const int keep = pqp::keep_control_steps(formulation, ref, n_points);
    if (keep_out) *keep_out = keep;
    return pqp::dispatch_class(table, ncols, formulation, n_points, keep, max_n, min_keep, max_keep);
}
