// kp_emu.cpp -- TEST HARNESS ONLY: runs the product's warp-synchronous solver source
// (path_optimizer_b200/csrc/pqp_kp_core.cuh) on the CPU by backing each of the 32 lanes with a host
// thread (see pqp_warp.cuh, PQP_HOST_EMU).  It exists so that the kernel logic can be checked against
// the oracle on a machine without a GPU.  It is NOT part of libpqp.so and the product never calls it.
#define PQP_HOST_EMU 1
#include <pthread.h>
#include <stdlib.h>
#include <string.h>

#include "../../path_optimizer_b200/csrc/pqp_kp_core3.cuh"
#include "../../path_optimizer_b200/csrc/pqp_kk_core.cuh"

namespace {
struct LaneArgs {
    pqp::EmuShared *sh;
    pqp::EmuCta *cta;
    int lane, wid, nw;
    const pqp::DevParams *prm;
    const pqp::BatchView *bv;
    int prob;
    double *smem;
    size_t smem_doubles;
    int variant;  // 0: one-warp generic core; 5..: thread-per-station classes (tests/emu/emu.py: VARIANTS)
};
void *lane_main(void *p) {
    LaneArgs *a = (LaneArgs *)p;
    pqp::Warp w{a->lane, a->sh};
    pqp::Cta c{w, pqp::CtaSync{a->cta}, a->wid, a->nw, a->smem};
    // leading doubles: CTA reduction scratch (16 per warp) of the thread-per-station kernels (kCtaScratch); the one-warp
    // kernel gets the whole allocation (pqp_k1_generic.cu), which its longest paths need
    const int res = a->variant == 0 ? 0 : a->nw > 8 ? 256 : 128;
    double *sm = a->smem + res;
    const size_t cap = a->smem_doubles - res;
    switch (a->variant) {
    case 5: pqp::Kp3<17, 6, 4>::solve_path(c, *a->prm, *a->bv, a->prob, sm, cap); break;
    case 6: pqp::Kp3<23, 7, 4>::solve_path(c, *a->prm, *a->bv, a->prob, sm, cap); break;
    case 7: pqp::Kp3<27, 7, 8, 34>::solve_path(c, *a->prm, *a->bv, a->prob, sm, cap); break;
    case 8: pqp::Kp3<17, 6, 8, 34>::solve_path(c, *a->prm, *a->bv, a->prob, sm, cap); break;
    case 9: pqp::Kp3<23, 7, 8, 34>::solve_path(c, *a->prm, *a->bv, a->prob, sm, cap); break;
    case 10: pqp::Kp3<37, 7, 13, 34>::solve_path(c, *a->prm, *a->bv, a->prob, sm, cap); break;
    case 11: pqp::Kp3<37, 7, 12, 34>::solve_path(c, *a->prm, *a->bv, a->prob, sm, cap); break;
    case 12: pqp::Kp3<27, 7, 10, 34>::solve_path(c, *a->prm, *a->bv, a->prob, sm, cap); break;
    case 20: pqp::Kp3<23, 7, 4, 17, 2>::solve_path(c, *a->prm, *a->bv, a->prob, sm, cap); break;    // "KPC" classes
    case 21: pqp::Kp3<23, 7, 8, 34, 2>::solve_path(c, *a->prm, *a->bv, a->prob, sm, cap); break;
    case 22: pqp::Kp3<13, 7, 8, 34, 2>::solve_path(c, *a->prm, *a->bv, a->prob, sm, cap); break;
    case 30: pqp::Kk<4>::solve_path(c, *a->prm, *a->bv, a->prob, sm, cap); break;                      // "K" classes
    case 31: pqp::Kk<8>::solve_path(c, *a->prm, *a->bv, a->prob, sm, cap); break;
    case 32: pqp::Kk<13>::solve_path(c, *a->prm, *a->bv, a->prob, sm, cap); break;
    default: pqp::kp_solve_path(w, *a->prm, *a->bv, a->prob, sm, cap);   // generic core: one warp
    }
    return nullptr;
}
}  // namespace

static const double *g_emu_max_k = nullptr, *g_emu_max_kp = nullptr;
extern "C" void kp_emu_set_limits(const double *max_k, const double *max_kp) { g_emu_max_k = max_k; g_emu_max_kp = max_kp; }

extern "C" int kp_emu_solve_batch(const pqp_params *params, int batch, const int32_t *n_points,
                                  const int32_t *offsets, const pqp_state *ref,
                                  const pqp_station_bounds *bounds, const double *x0,
                                  const double *end_heading, pqp_state *out_states, double *out_frenet,
                                  int32_t *status, int32_t *iters, int smem_bytes, int variant, int nwarps) {
    if (variant == 0 || nwarps < 1) nwarps = 1;
    if (variant == 5 || variant == 6) nwarps = 4;
    if (variant >= 7) nwarps = 8;
    if (variant == 10) nwarps = 13;
    if (variant == 11) nwarps = 12;
    if (variant == 12) nwarps = 10;
    if (variant == 20) nwarps = 4;
    if (variant == 21 || variant == 22) nwarps = 8;
    if (variant == 30) nwarps = 4;
    if (variant == 31) nwarps = 8;
    if (variant == 32) nwarps = 13;
    pqp::DevParams prm = pqp::dev_params_from(*params);
    pqp::BatchView bv;
    bv.batch = batch; bv.n_points = n_points; bv.offsets = offsets; bv.ref = ref; bv.bounds = bounds;
    bv.x0 = x0; bv.end_heading = end_heading; bv.out_states = out_states; bv.out_frenet = out_frenet;
    bv.status = status; bv.iters = iters; bv.debug = nullptr;
    bv.max_k = g_emu_max_k; bv.max_kp = g_emu_max_kp;
    const size_t ws_n = pqp::kp2_ws_doubles((size_t)offsets[batch], (size_t)batch);
    bv.workspace = (double *)malloc(ws_n * sizeof(double));
    for (size_t k = 0; k < ws_n; ++k) bv.workspace[k] = nan("");
    const size_t smem_doubles = (size_t)smem_bytes / sizeof(double);
    double *smem = (double *)malloc(smem_doubles * sizeof(double));
    for (int prob = 0; prob < batch; ++prob) {
        // poison the scratch so that reads of uninitialised shared memory show up as NaN
        for (size_t k = 0; k < smem_doubles; ++k) smem[k] = nan("");
        const int nth = 32 * nwarps;
        pqp::EmuShared sh[16];
        pqp::EmuCta cta;
        cta.nthreads = nth;
        pthread_barrier_init(&cta.bar, nullptr, nth);
        for (int k = 0; k < nwarps; ++k) pthread_barrier_init(&sh[k].bar, nullptr, 32);
        pthread_t th[512];
        LaneArgs args[512];
        for (int t = 0; t < nth; ++t) {
            args[t] = LaneArgs{&sh[t / 32], &cta, t % 32, t / 32, nwarps, &prm, &bv, prob, smem, smem_doubles, variant};
            pthread_create(&th[t], nullptr, lane_main, &args[t]);
        }
        for (int t = 0; t < nth; ++t) pthread_join(th[t], nullptr);
        for (int k = 0; k < nwarps; ++k) pthread_barrier_destroy(&sh[k].bar);
        pthread_barrier_destroy(&cta.bar);
    }
    free(smem);
    free(bv.workspace);
    return 0;
}

// ---- generic banded kernel ("K" / "KPC") under the same warp emulator -------------------------------
#include "../../path_optimizer_b200/csrc/pqp_gen_core.cuh"
#include "../../path_optimizer_b200/csrc/pqp_forms.h"
#include <vector>

namespace {
struct GenLaneArgs {
    pqp::EmuShared *sh;
    int lane;
    const pqp::DevParams *prm;
    const pqp::GenView *gv;
    double *smem;
    size_t cap;
};
void *gen_lane_main(void *p) {
    GenLaneArgs *a = (GenLaneArgs *)p;
    pqp::Warp w{a->lane, a->sh};
    pqp::gen_solve_qp(w, *a->prm, *a->gv, 0, a->smem, a->cap);
    return nullptr;
}
}  // namespace

extern "C" int gen_emu_solve_batch(const pqp_params *params, int formulation, int batch, const int32_t *n_points,
                                   const int32_t *offsets, const pqp_state *ref, const pqp_station_bounds *bounds,
                                   const double *x0, const double *end_heading, const double *max_k, const double *max_kp,
                                   pqp_state *out_states, double *out_frenet, int32_t *status, int32_t *iters) {
    pqp::DevParams prm = pqp::dev_params_from(*params);
    for (int b = 0; b < batch; ++b) {
        const int o = offsets[b], N = n_points[b];
        pqp::GenProblem g;
        bool ok = formulation == PQP_FORM_K
                      ? pqp::assemble_k(*params, N, ref + o, bounds + o, x0 + 3 * b, end_heading[b], g)
                      : pqp::assemble_kpc(*params, N, ref + o, bounds + o, x0 + 3 * b, end_heading[b], max_k + o, max_kp + o, g);
        if (!ok) { status[b] = PQP_INVALID_PROBLEM; iters[b] = 0; continue; }
        int32_t meta[pqp::kGenMeta] = {g.n, g.m, g.n_den, g.bw, g.M, N, 0, 0, 0, 0, 0};
        pqp::GenView gv;
        gv.batch = 1; gv.meta = meta;
        gv.A_col = g.A_col.data(); gv.A_val = g.A_val.data(); gv.l = g.l.data(); gv.u = g.u.data();
        gv.Pd = g.Pd.data(); gv.Po_idx = g.Po_idx.data(); gv.Po_val = g.Po_val.data();
        gv.csc_ptr = g.csc_ptr.data(); gv.csc_row = g.csc_row.data(); gv.csc_val = g.csc_val.data();
        gv.sep = g.sep; gv.out_idx = g.out_idx.data();
        gv.ref = ref + o; gv.out_states = out_states + o; gv.out_frenet = out_frenet + 3 * (size_t)o;
        gv.status = status + b; gv.iters = iters + b;
        const size_t cap = pqp::gen_smem_doubles(g.n, g.m, g.bw);
        std::vector<double> smem(cap, nan(""));
        pqp::EmuShared sh;
        pthread_barrier_init(&sh.bar, nullptr, 32);
        pthread_t th[32];
        GenLaneArgs args[32];
        for (int l = 0; l < 32; ++l) {
            args[l] = GenLaneArgs{&sh, l, &prm, &gv, smem.data(), cap};
            pthread_create(&th[l], nullptr, gen_lane_main, &args[l]);
        }
        for (int l = 0; l < 32; ++l) pthread_join(th[l], nullptr);
        pthread_barrier_destroy(&sh.bar);
    }
    return 0;
}
