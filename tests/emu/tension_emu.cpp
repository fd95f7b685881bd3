// tension_emu.cpp -- TEST HARNESS: the per-path work of pqp_smooth_reference_tension_device on the CPU, compiled with
// plain g++ (-DPQP_HOST_EMU) into a library of its own (tests/emu/tension_emu.py).  tension_emu_stage runs the front of
// the smoothing stage (smooth_emu_stage of smooth_emu.cpp: B-spline, raw fit, stations), then the TENSION QP of every
// station with its clearance (pqp::map_distance on the path's map) and its separators, the stations one after the other
// as the assemble kernel's lanes take them.  tension_emu_solve runs the width-9 generic core (pqp_gen_core.cuh,
// gen_solve_qp<9, false, 6>) on such a QP with one host thread per lane (pqp_warp.cuh).  Never linked into libpqp.so.
#include "smooth_emu.cpp"

extern "C" {

// One path up to its QP.  dmap: the path's distance map, NULL for a map index outside the set.  Outputs: *N stations st
// [max_points], their clearances clear [max_points] (0 at both ends, which are not looked up), and for an accepted path
// the QP in the assemble kernel's layout: A_col / A_val [3N][4], l / u [3N], Pd [3N], Po_idx / Po_val [3N][6], csc_ptr
// [3N + 1], csc_row / csc_val [<= 5N], sep [32] with *M separators.  Returns the pqp::SmoothRefusal up to SM_SHORT, or
// SM_MAP, in the kernels' order.
int tension_emu_stage(int n, const double *px, const double *py, const pqp_distance_map *dmap, double w_dev,
                      double w_curv, double w_rate, int max_raw, int max_points, int *N_out, pqp_state *st,
                      double *clear, int32_t *A_col, double *A_val, double *l, double *u, double *Pd, int32_t *Po_idx,
                      double *Po_val, int32_t *csc_ptr, int32_t *csc_row, double *csc_val, int32_t *sep, int *M) {
    using namespace pqp;
    *N_out = 0;
    *M = 0;
    // the front, with scratch for what the TENSION2 QP would take
    const size_t Km = (size_t)max_raw + 1, Nm = (size_t)max_points;
    std::vector<double> t(Km), x(Km), y(Km), s(Km), xc(4 * Km), yc(4 * Km);
    std::vector<int32_t> a2c(12 * Nm), po2(8 * Nm), cp2(4 * Nm + 1), cr2(9 * Nm);
    std::vector<double> a2v(12 * Nm), l2(3 * Nm), u2(3 * Nm), pd2(4 * Nm), q2(4 * Nm), pv2(8 * Nm), cv2(9 * Nm);
    int K = 0, N = 0, M2 = 0;
    int32_t sep2[32];
    int reason = smooth_emu_stage(n, px, py, w_dev, w_curv, w_rate, max_raw, max_points, &K, t.data(), x.data(),
                                  y.data(), s.data(), xc.data(), yc.data(), &N, st, a2c.data(), a2v.data(), l2.data(),
                                  u2.data(), pd2.data(), q2.data(), po2.data(), pv2.data(), cp2.data(), cr2.data(),
                                  cv2.data(), sep2, &M2);
    // the sample kernel's refusals come first, then the assemble kernel's map check, then the rest of the front
    if (reason == SM_FEW || reason == SM_DEGREE || reason == SM_LENGTH || reason == SM_RAW_MANY) return reason;
    if (!dmap) return SM_MAP;
    if (reason != SM_OK) return reason;
    *N_out = N;
    const MapView mv = make_map_view(dmap->distance, dmap->rows, dmap->cols, dmap->resolution, dmap->center_x,
                                     dmap->center_y);
    const SmoothWeights w{w_dev, w_curv, w_rate};
    int e = 0;
    for (int i = 0; i < N; ++i) {
        clear[i] = (i > 0 && i < N - 1) ? map_distance(mv, st[i].x, st[i].y) : 0.0;
        tension_qp_station(N, i, st[i], clear[i], w, e, A_col, A_val, l, u, Pd, Po_idx, Po_val, csc_ptr, csc_row,
                           csc_val);
        e += tension_qp_csc_count(st[i]);
    }
    *M = tension_qp_separators(N, sep);
    return SM_OK;
}

}  // extern "C"

namespace {
void *tension_lane_main(void *p) {
    LaneArgs *a = (LaneArgs *)p;
    pqp::Warp w{a->lane, a->sh};
    pqp::gen_solve_qp<9, false, pqp::kTensionPartners>(w, *a->prm, *a->gv, 0, a->smem, a->cap);
    return nullptr;
}
}  // namespace

extern "C" {

// The width-9 generic core on one path's QP (the layout of tension_emu_stage).  Outputs: frenet [N][3] the solution's
// (x_i, y_i, d_i), *status, *iters.
int tension_emu_solve(const pqp_params *params, int N, int M, const int32_t *A_col, const double *A_val,
                      const double *l, const double *u, const double *Pd, const int32_t *Po_idx, const double *Po_val,
                      const int32_t *csc_ptr, const int32_t *csc_row, const double *csc_val, const int32_t *sep,
                      const pqp_state *st, double *frenet, int32_t *status, int32_t *iters) {
    const pqp::DevParams prm = pqp::dev_params_from(*params);
    const int n = 3 * N, m = 3 * N;
    int32_t meta[pqp::kGenMeta] = {n, m, n, 9, M, N, 0, 0, 0, 0, 0};
    std::vector<int32_t> out_idx(3 * (size_t)N);
    for (int i = 0; i < 3 * N; ++i) out_idx[i] = i;
    std::vector<pqp_state> out_states(N);
    pqp::GenView gv;
    gv.batch = 1; gv.meta = meta;
    gv.A_col = A_col; gv.A_val = A_val; gv.l = l; gv.u = u; gv.Pd = Pd; gv.Po_idx = Po_idx; gv.Po_val = Po_val;
    gv.csc_ptr = csc_ptr; gv.csc_row = csc_row; gv.csc_val = csc_val; gv.sep = sep; gv.out_idx = out_idx.data();
    gv.ref = st; gv.out_states = out_states.data(); gv.out_frenet = frenet; gv.status = status; gv.iters = iters;
    const size_t cap = pqp::gen_smem_doubles<9>(n, m, 9);
    std::vector<double> smem(cap, nan(""));
    pqp::EmuShared sh;
    pthread_barrier_init(&sh.bar, nullptr, 32);
    pthread_t th[32];
    LaneArgs args[32];
    for (int k = 0; k < 32; ++k) {
        args[k] = LaneArgs{&sh, k, &prm, &gv, smem.data(), cap, nullptr};
        pthread_create(&th[k], nullptr, tension_lane_main, &args[k]);
    }
    for (int k = 0; k < 32; ++k) pthread_join(th[k], nullptr);
    pthread_barrier_destroy(&sh.bar);
    return 0;
}

}  // extern "C"
