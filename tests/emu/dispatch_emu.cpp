// dispatch_emu.cpp -- TEST HARNESS: the device dispatch of pqp_dispatch.h compiled with plain g++, so that the CPU suite
// can hold it against the host selection (pqp_keep_control_steps + pqp_class_info_form) without a GPU: the per-path
// class selection (keep_control_steps, the caller's bounds, the class-table lookup) and the sort pqp_dispatch_kernel
// (pqp_capi.cu) builds on it.  Never linked into libpqp.so.
#include <vector>

#include "../../path_optimizer_b200/csrc/pqp_dispatch.h"

static pqp::FormTables tables_of(const int8_t *const table[3], const int ncols[3], const int max_n[3]) {
    pqp::FormTables t;
    for (int f = 0; f < 3; ++f) { t.table[f] = table[f]; t.ncols[f] = ncols[f]; t.max_n[f] = max_n[f]; }
    return t;
}

extern "C" {

int dispatch_emu_class(const int8_t *table, int ncols, int formulation, const pqp_state *ref, int n_points, int max_n,
                       int min_keep, int max_keep, int *keep_out) {
    const int keep = pqp::keep_control_steps(formulation, ref, n_points);
    if (keep_out) *keep_out = keep;
    return pqp::dispatch_class(table, ncols, formulation, n_points, keep, max_n, min_keep, max_keep);
}

// The kernel's sort, serially: every path's formulation (form[b]; form NULL: the one formulation of a one-bit
// form_mask), its keep_control_steps and key pqp::dispatch_key_forms over the layout (the classes [v_lo, v_lo + nv),
// `stride` length buckets each), a histogram over the keys, its exclusive prefix and the scatter into order segments of
// `batch` entries each (segment set * nv + class - v_lo, pre-filled with `batch`).  A path with key -1 gets no entry.
// table / ncols / max_n: [3], indexed by PQP_FORM_* (only the mask's formulations are read); order: [n_sets * nv *
// batch]; key: [batch].
void dispatch_sort_emu(const int8_t *const table[3], const int ncols[3], const int max_n[3], int form_mask,
                       const int32_t *form, int v_lo, int nv, int stride, int n_sets, int batch, const int32_t *n_points,
                       const int32_t *offsets, const pqp_state *ref, const int32_t *set_index, int min_keep,
                       int max_keep, int32_t *order, int32_t *key) {
    const pqp::FormTables t = tables_of(table, ncols, max_n);
    const int nsv = n_sets * nv, nb = nsv * stride;
    std::vector<int32_t> hist((size_t)nb, 0), base((size_t)nsv, 0);
    for (size_t i = 0; i < (size_t)nsv * batch; ++i) order[i] = batch;
    for (int b = 0; b < batch; ++b) {
        const int n = n_points[b], s = set_index ? set_index[b] : 0;
        const int f = form ? form[b] : pqp::mask_form(form_mask);
        const bool ok = pqp::form_in_mask(f, form_mask) && s >= 0 && s < n_sets;
        const int keep = ok ? pqp::keep_control_steps(f, ref + offsets[b], n) : 0;
        key[b] = pqp::dispatch_key_forms(t, form_mask, f, s, n_sets, n, keep, min_keep, max_keep, nv, stride, v_lo);
        if (key[b] >= 0) hist[key[b]]++;
    }
    int run = 0;
    for (int i = 0; i < nb; ++i) { const int c = hist[i]; hist[i] = run; run += c; }
    for (int r = 0; r < nsv; ++r) base[r] = hist[(size_t)r * stride];
    for (int b = 0; b < batch; ++b) {
        if (key[b] < 0) continue;
        const int r = key[b] / stride;
        order[(size_t)r * batch + (hist[key[b]]++ - base[r])] = b;
    }
}

}  // extern "C"
