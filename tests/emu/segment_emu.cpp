// segment_emu.cpp -- TEST HARNESS: pqp_segment_reference_device on the CPU, compiled with plain g++ (-DPQP_HOST_EMU)
// into a library of its own (tests/emu/segment_emu.py).  It runs the per-thread functions of csrc/pqp_segment_core.cuh
// in the order of the kernel's three launches: every path's count pass, the reservation in index order (the warp scan
// done serially, with the same pqp::segment_fits rule), then every kept path's write pass.  Never linked into
// libpqp.so.
#define PQP_HOST_EMU 1
#include "../../path_optimizer_b200/csrc/pqp_segment_core.cuh"

extern "C" {

// Inputs and outputs as pqp_segment_reference_device; also every path's refusal reason (pqp::SegmentRefusal, with
// SEG_CAPACITY for a path the reservation refused) and its length after the goal cut.
void segment_emu(int batch, const int32_t *koff, const double *knots, const double *xc, const double *yc,
                 const double *max_s, const pqp_state *start, const pqp_state *goal, double ds_small, double ds_large,
                 int dynamic, double search_ds, int max_n, int capacity, int32_t *n_points, int32_t *offsets,
                 pqp_state *ref, double *x0, double *end_heading, int32_t *ok, int32_t *reason, double *cut_s) {
    const pqp::SegmentFlags f{ds_small, ds_large, search_ds, dynamic ? 1 : 0, max_n};
    for (int b = 0; b < batch; ++b) {
        const int o = koff[b], n = koff[b + 1] - o;
        const pqp::SplineView xs{n, knots + o, xc + 4 * (size_t)o}, ys{n, knots + o, yc + 4 * (size_t)o};
        reason[b] = pqp::segment_count(f, xs, ys, max_s[b], start[b], goal[b], x0 + 3 * (size_t)b, cut_s + b,
                                       n_points + b);
        end_heading[b] = goal[b].z;
    }
    long long all = 0;
    offsets[0] = 0;
    for (int b = 0; b < batch; ++b) {
        const int c = n_points[b];
        const bool keep = pqp::segment_fits(all, c, capacity);
        all += c;
        if (!keep && c > 0) reason[b] = pqp::SEG_CAPACITY;
        n_points[b] = keep ? c : 0;
        offsets[b + 1] = offsets[b] + n_points[b];
        ok[b] = keep ? 1 : 0;
    }
    for (int b = 0; b < batch; ++b) {
        if (!ok[b]) continue;
        const int o = koff[b], n = koff[b + 1] - o;
        const pqp::SplineView xs{n, knots + o, xc + 4 * (size_t)o}, ys{n, knots + o, yc + 4 * (size_t)o};
        pqp::segment_write(f, xs, ys, n_points[b], ref + offsets[b]);
    }
}

}  // extern "C"
