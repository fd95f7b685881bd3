// forms_emu.cpp -- TEST HARNESS: the per-path-formulation dispatch of pqp_dispatch.h (pqp::dispatch_key_forms) and
// the sort pqp_dispatch_kernel builds on it (pqp_capi.cu, serially in dispatch_emu.cpp), compiled with plain g++ so that
// the CPU suite can hold them against the host selection (pqp_keep_control_steps + pqp_class_info_form) without a GPU.
// Never linked into libpqp.so.
#include "dispatch_emu.cpp"

extern "C" {

// The key of one path (-1: none), keep given, in the order that spans every class from the first.
int forms_emu_key(const int8_t *const table[3], const int ncols[3], const int max_n[3], int form_mask, int form,
                  int set, int n_sets, int n, int keep, int min_keep, int max_keep, int n_variants, int stride) {
    return pqp::dispatch_key_forms(tables_of(table, ncols, max_n), form_mask, form, set, n_sets, n, keep, min_keep,
                                   max_keep, n_variants, stride);
}

// dispatch_sort_emu over per-path formulations, in the order that spans every class from the first (v_lo = 0).
void forms_dispatch_emu(const int8_t *const table[3], const int ncols[3], const int max_n[3], int form_mask,
                        int n_variants, int stride, int n_sets, int batch, const int32_t *n_points,
                        const int32_t *offsets, const pqp_state *ref, const int32_t *set_index, const int32_t *form,
                        int min_keep, int max_keep, int32_t *order, int32_t *key) {
    dispatch_sort_emu(table, ncols, max_n, form_mask, form, 0, n_variants, stride, n_sets, batch, n_points, offsets, ref,
                      set_index, min_keep, max_keep, order, key);
}

}  // extern "C"
