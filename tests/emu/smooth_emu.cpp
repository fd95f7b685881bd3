// smooth_emu.cpp -- TEST HARNESS: the per-path work of pqp_smooth_reference_device on the CPU, compiled with plain g++
// (-DPQP_HOST_EMU) into a library of its own (tests/emu/smooth_emu.py).  smooth_emu_stage calls the per-thread
// functions of csrc/pqp_smooth_core.cuh in the kernels' order -- degree and length, the sample parameters, de Boor per
// sample, the s sum, the raw fit (pqp::spline_fit, as pqp_fit_splines_kernel), the station count, the resampling
// (pqp::densify_sample) and the QP of every station with its separators -- with the warp's lanes run one after the
// other.  smooth_emu_solve runs the width-4 generic core (pqp_gen_core.cuh, gen_solve_qp<4, true>) on such a QP with
// one host thread per lane (pqp_warp.cuh).  Never linked into libpqp.so.
#define PQP_HOST_EMU 1
#include <pthread.h>

#include <vector>

#include "../../path_optimizer_b200/csrc/pqp_gen_core.cuh"
#include "../../path_optimizer_b200/csrc/pqp_smooth_core.cuh"

extern "C" {

// One path up to its QP.  Outputs: *K raw samples t / x / y / s [max_raw], the raw fit's rows xc / yc [max_raw][4],
// *N stations st [max_points], and for an accepted path the QP in the assemble kernel's layout: A_col / A_val
// [3N - 1][4], l / u [3N - 1], Pd / q [4N - 1], Po_idx / Po_val [4N - 1][2], csc_ptr [4N], csc_row / csc_val [9N - 7],
// sep [32] with *M separators.  Returns the pqp::SmoothRefusal up to SM_SHORT.
int smooth_emu_stage(int n, const double *px, const double *py, double w_dev, double w_curv, double w_rate, int max_raw,
                     int max_points, int *K_out, double *t, double *x, double *y, double *s, double *xc, double *yc,
                     int *N_out, pqp_state *st, int32_t *A_col, double *A_val, double *l, double *u, double *Pd,
                     double *q, int32_t *Po_idx, double *Po_val, int32_t *csc_ptr, int32_t *csc_row, double *csc_val,
                     int32_t *sep, int *M) {
    using namespace pqp;
    *K_out = 0;
    *N_out = 0;
    *M = 0;
    if (n < 4) return SM_FEW;
    double length;
    const int deg = smooth_degree(n, px, py, 1, &length);
    if (deg >= n) return SM_DEGREE;
    if (!(length > 0 && length <= 1.7976931348623157e308)) return SM_LENGTH;
    const int K = smooth_sample_params(length, max_raw, t);
    if (K > max_raw) return SM_RAW_MANY;
    *K_out = K;
    double acc = 0;
    for (int k = 0; k < K; ++k) {
        smooth_bspline_eval(n, deg, px, py, 1, t[k], &x[k], &y[k]);
        if (k > 0) acc = add(acc, smooth_step(x[k - 1], y[k - 1], x[k], y[k]));
        s[k] = acc;
    }
    if (!fit_knots_ok(K, s)) return SM_RAW_ORDER;
    std::vector<double> diag(K), rhs(K);
    spline_fit(K, s, [&](int i) { return x[i]; }, xc, diag.data(), rhs.data());
    spline_fit(K, s, [&](int i) { return y[i]; }, yc, diag.data(), rhs.data());
    const SplineView xs{K, s, xc}, ys{K, s, yc};
    const double max_s = s[K - 1];
    if (!(max_s <= (double)max_points)) return SM_MANY;
    const int N = smooth_station_count(max_s);
    if (N > max_points) return SM_MANY;
    if (N < 3) return SM_SHORT;
    *N_out = N;
    const double x0 = spline_eval(xs, 0, 0.0), y0 = spline_eval(ys, 0, 0.0);
    const SmoothWeights w{w_dev, w_curv, w_rate};
    for (int i = 0; i < N; ++i) {
        st[i] = densify_sample(xs, ys, (double)i);
        smooth_qp_station(N, i, st[i], (double)(i + 1) - (double)i, x0, y0, w, A_col, A_val, l, u, Pd, Po_idx, Po_val, q,
                          csc_ptr, csc_row, csc_val);
    }
    *M = smooth_qp_separators(N, sep);
    return SM_OK;
}

}  // extern "C"

namespace {
struct LaneArgs {
    pqp::EmuShared *sh;
    int lane;
    const pqp::DevParams *prm;
    const pqp::GenView *gv;
    double *smem;
    size_t cap;
    const double *q;
};
void *lane_main(void *p) {
    LaneArgs *a = (LaneArgs *)p;
    pqp::Warp w{a->lane, a->sh};
    pqp::gen_solve_qp<4, true>(w, *a->prm, *a->gv, 0, a->smem, a->cap, a->q);
    return nullptr;
}
}  // namespace

extern "C" {

// The width-4 generic core on one path's QP (the layout of smooth_emu_stage).  Outputs: frenet [N][3] the solution's
// (x_i, y_i, theta_i), *status, *iters.
int smooth_emu_solve(const pqp_params *params, int N, int M, const int32_t *A_col, const double *A_val, const double *l,
                     const double *u, const double *Pd, const double *q, const int32_t *Po_idx, const double *Po_val,
                     const int32_t *csc_ptr, const int32_t *csc_row, const double *csc_val, const int32_t *sep,
                     const pqp_state *st, double *frenet, int32_t *status, int32_t *iters) {
    const pqp::DevParams prm = pqp::dev_params_from(*params);
    const int n = 4 * N - 1, m = 3 * N - 1;
    int32_t meta[pqp::kGenMeta] = {n, m, n, 4, M, N, 0, 0, 0, 0, 0};
    std::vector<int32_t> out_idx(3 * (size_t)N);
    for (int i = 0; i < N; ++i)
        for (int t = 0; t < 3; ++t) out_idx[3 * i + t] = 4 * i + t;
    std::vector<pqp_state> out_states(N);
    pqp::GenView gv;
    gv.batch = 1; gv.meta = meta;
    gv.A_col = A_col; gv.A_val = A_val; gv.l = l; gv.u = u; gv.Pd = Pd; gv.Po_idx = Po_idx; gv.Po_val = Po_val;
    gv.csc_ptr = csc_ptr; gv.csc_row = csc_row; gv.csc_val = csc_val; gv.sep = sep; gv.out_idx = out_idx.data();
    gv.ref = st; gv.out_states = out_states.data(); gv.out_frenet = frenet; gv.status = status; gv.iters = iters;
    const size_t cap = pqp::gen_smem_doubles<4>(n, m, 4);
    std::vector<double> smem(cap, nan(""));
    pqp::EmuShared sh;
    pthread_barrier_init(&sh.bar, nullptr, 32);
    pthread_t th[32];
    LaneArgs args[32];
    for (int k = 0; k < 32; ++k) {
        args[k] = LaneArgs{&sh, k, &prm, &gv, smem.data(), cap, q};
        pthread_create(&th[k], nullptr, lane_main, &args[k]);
    }
    for (int k = 0; k < 32; ++k) pthread_join(th[k], nullptr);
    pthread_barrier_destroy(&sh.bar);
    return 0;
}

}  // extern "C"
