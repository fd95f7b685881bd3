// fit_emu.cpp -- TEST HARNESS: pqp_fit_splines_device on the CPU, compiled with plain g++ (-DPQP_HOST_EMU) into a
// library of its own (tests/emu/fit_emu.py).  It runs the per-thread functions of csrc/pqp_env_core.cuh in the order the
// kernel's barriers allow: every knot copied, then every path's refusal decided, then every (path, coordinate) thread's
// fit_path_coord, with the scratch layout of the kernel.  Never linked into libpqp.so.
#define PQP_HOST_EMU 1
#include <vector>

#include "../../path_optimizer_b200/csrc/pqp_env_core.cuh"

extern "C" {

// offsets [batch+1], ref [total] -> knots [total], x_coef / y_coef [total][4], ok [batch]
void fit_emu(int batch, const int32_t *offsets, const pqp_state *ref, double *knots, double *xc, double *yc,
             int32_t *ok) {
    const int total = offsets[batch];
    std::vector<double> scr(4 * (size_t)(total > 0 ? total : 0));
    for (int k = offsets[0]; k < total; ++k) knots[k] = ref[k].s;
    std::vector<char> fit((size_t)batch);
    for (int b = 0; b < batch; ++b) fit[b] = pqp::fit_knots_ok(offsets[b + 1] - offsets[b], knots + offsets[b]);
    for (int b = 0; b < batch; ++b) {
        const int off = offsets[b], n = offsets[b + 1] - off;
        for (int coord = 0; coord < 2; ++coord)
            pqp::fit_path_coord(n > 0 ? n : 0, fit[b], coord, ref + off, knots + off, (coord ? yc : xc) + 4 * (size_t)off,
                                scr.data() + 4 * (size_t)off);
        ok[b] = fit[b] ? 1 : 0;
    }
}

}  // extern "C"
