// forms_emu.cpp -- TEST HARNESS: the per-path-formulation dispatch of pqp_dispatch.h (pqp::dispatch_key_forms) and
// the sort pqp_dispatch_forms_kernel builds on it (pqp_capi.cu), compiled with plain g++ so that the CPU suite can hold
// them against the host selection (pqp_keep_control_steps + pqp_class_info_form) without a GPU.  Never linked into
// libpqp.so.
#include <vector>

#include "../../path_optimizer_b200/csrc/pqp_dispatch.h"

namespace {
pqp::FormTables tables_of(const int8_t *const table[3], const int ncols[3], const int max_n[3]) {
    pqp::FormTables t;
    for (int f = 0; f < 3; ++f) { t.table[f] = table[f]; t.ncols[f] = ncols[f]; t.max_n[f] = max_n[f]; }
    return t;
}
}  // namespace

extern "C" {

// The key of one path (-1: none), keep given.
int forms_emu_key(const int8_t *const table[3], const int ncols[3], const int max_n[3], int form_mask, int form,
                  int set, int n_sets, int n, int keep, int min_keep, int max_keep, int n_variants, int stride) {
    return pqp::dispatch_key_forms(tables_of(table, ncols, max_n), form_mask, form, set, n_sets, n, keep, min_keep,
                                   max_keep, n_variants, stride);
}

// The kernel's sort, serially: keep_control_steps of every path in its own formulation, its key, a histogram over the
// keys, its exclusive prefix and the scatter into order segments of `batch` entries each (segment set * n_variants +
// class, pre-filled with `batch`).  order: [n_sets * n_variants * batch]; key: [batch].
void forms_dispatch_emu(const int8_t *const table[3], const int ncols[3], const int max_n[3], int form_mask,
                        int n_variants, int stride, int n_sets, int batch, const int32_t *n_points,
                        const int32_t *offsets, const pqp_state *ref, const int32_t *set_index, const int32_t *form,
                        int min_keep, int max_keep, int32_t *order, int32_t *key) {
    const pqp::FormTables t = tables_of(table, ncols, max_n);
    const int nsv = n_sets * n_variants, nb = nsv * stride;
    std::vector<int32_t> hist((size_t)nb, 0), base((size_t)nsv, 0);
    for (size_t i = 0; i < (size_t)nsv * batch; ++i) order[i] = batch;
    for (int b = 0; b < batch; ++b) {
        const int n = n_points[b], f = form[b], s = set_index ? set_index[b] : 0;
        const int keep = pqp::form_in_mask(f, form_mask) ? pqp::keep_control_steps(f, ref + offsets[b], n) : 0;
        key[b] = pqp::dispatch_key_forms(t, form_mask, f, s, n_sets, n, keep, min_keep, max_keep, n_variants, stride);
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
