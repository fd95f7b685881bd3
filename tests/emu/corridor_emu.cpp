// corridor_emu.cpp -- TEST HARNESS: the per-path work of pqp_post_smooth_device's search kernel on the CPU, compiled with
// plain g++ (-DPQP_HOST_EMU) into a library of its own (tests/emu/corridor_emu.py).  It calls the per-thread functions
// of csrc/pqp_corridor_core.cuh in the kernel's order -- grid scan and Newton, layer lattice, vehicle_l, layer 0, the DP
// layer by layer (corridor_node, corridor_self_cost, corridor_relax), the last layer's argmin, the backtrack with
// corridor_rough, the bound march, and the QP rows, columns and separators -- with the warp's lanes run one after the
// other.  Never linked into libpqp.so.
#define PQP_HOST_EMU 1
#include <vector>

#include "../../path_optimizer_b200/csrc/pqp_corridor_core.cuh"

extern "C" {

// One path.  Outputs: reason (pqp::CorridorRefusal up to COR_SHORT), R layers (0 when refused), s / lo / hi / chain
// [max_layers], vehicle_l, and for an accepted path the QP in the search kernel's layout: A_col / A_val [3R - 2][4],
// l / u [3R - 2], csc_ptr [3R + 1], csc_row / csc_val [7R - 6], sep [32] with *M separators.
int corridor_emu(int nk, const double *knots, const double *xc, const double *yc, double max_s, const pqp_state *start,
                 const float *dist, int rows, int cols, double res, double cx, double cy, double range, double spacing,
                 double ds_long, int max_layers, int *R_out, double *s, double *lo, double *hi, int *chain,
                 double *vehicle_l, int32_t *A_col, double *A_val, double *l, double *u, int32_t *csc_ptr,
                 int32_t *csc_row, double *csc_val, int32_t *sep, int *M) {
    using namespace pqp;
    *R_out = 0;
    *M = 0;
    CorridorFlags f;
    f.range = range; f.spacing = spacing; f.ds_long = ds_long;
    int n = 0;
    for (double c = -range; c <= range && n <= kCorridorMaxLateral; c += spacing, ++n)   // the host's lattice
        if (n < kCorridorMaxLateral) f.lat[n] = c;
    f.n_lat = n;
    if (f.n_lat > kCorridorMaxLateral) return COR_WIDE;
    const MapView m = make_map_view(dist, rows, cols, res, cx, cy);
    const SplineView xs{nk, knots, xc}, ys{nk, knots, yc};
    if (nk < 3) return COR_BAD_SPLINE;
    if (!(max_s > 0.0 && max_s <= kCorridorMaxLength)) return COR_BAD_LENGTH;
    if (!(fabs(start->z) <= kCorridorMaxHeading)) return COR_BAD_START;
    double best = kDblMax;
    long long bk = 0;
    const long long K = corridor_grid_count(max_s);
    for (long long k = 0; k < K; ++k) {
        const double d = corridor_grid_dist(xs, ys, k, start->x, start->y);
        if (d < best) { best = d; bk = k; }
    }
    const double s0 = corridor_newton(xs, ys, start->x, start->y, 0.5 * (double)bk, max_s);
    if (!isfinite(s0)) return COR_BAD_START;
    const double search_ds = max_s > 6 ? ds_long : 0.5;
    std::vector<double> lay;
    for (double t = s0; t < max_s && (int)lay.size() <= max_layers; t = add(t, search_ds)) lay.push_back(t);
    lay.push_back(max_s);
    if ((int)lay.size() > max_layers) return COR_TOO_MANY;
    const double vl = corridor_vehicle_l(xs, ys, s0, *start);
    *vehicle_l = vl;
    if (!isfinite(vl)) return COR_BAD_START;
    if (fabs(vl) > range) return COR_FAR;
    const int start_idx = (int)((range + vl) / spacing);
    const int L = (int)lay.size();
    std::vector<int8_t> pred((size_t)L * kCorridorMaxLateral, -1);
    std::vector<unsigned long long> feas(L, 0);
    double px[kCorridorMaxLateral], py[kCorridorMaxLateral], pdir[kCorridorMaxLateral], pcost[kCorridorMaxLateral];
    unsigned char live[kCorridorMaxLateral];
    {
        const pqp_state r = densify_sample(xs, ys, s0);
        const double an = r.z + M_PI_2, c_n = cos(an), s_n = sin(an);
        for (int j = 0; j < n; ++j) {
            px[j] = add(r.x, mul(f.lat[j], c_n));
            py[j] = add(r.y, mul(f.lat[j], s_n));
            live[j] = j == start_idx;
            pdir[j] = start->z;
            pcost[j] = j == start_idx ? 0.0 : kDblMax;
        }
        feas[0] = (start_idx >= 0 && start_idx < n) ? 1ull << start_idx : 0ull;
    }
    int max_layer = 0;
    for (int i = 1; i < L; ++i) {
        const pqp_state r = densify_sample(xs, ys, lay[i]);
        const double an = r.z + M_PI_2, c_n = cos(an), s_n = sin(an);
        double nx[kCorridorMaxLateral], ny[kCorridorMaxLateral], nd[kCorridorMaxLateral], nc[kCorridorMaxLateral];
        int np[kCorridorMaxLateral];
        const CorridorPrev prev{px, py, pdir, pcost, live};
        bool reached = false;
        unsigned long long mask = 0;
        for (int j = 0; j < n; ++j) {
            const CorridorNode node = corridor_node(m, r, c_n, s_n, f.lat[j]);
            nx[j] = node.x; ny[j] = node.y; np[j] = -1;
            if (node.feasible) {
                mask |= 1ull << j;
                const double self = corridor_self_cost(node.dis, f.lat[j], range);
                np[j] = corridor_relax(f, prev, lay[i - 1], lay[i], f.lat[j], r.z, node.x, node.y, self, &nc[j], &nd[j]);
            }
            pred[(size_t)i * kCorridorMaxLateral + j] = (int8_t)np[j];
            reached = reached || np[j] >= 0;
        }
        feas[i] = mask;
        if (!reached) break;
        for (int j = 0; j < n; ++j) {
            px[j] = nx[j]; py[j] = ny[j]; live[j] = np[j] >= 0;
            pdir[j] = np[j] >= 0 ? nd[j] : 0.0;
            pcost[j] = np[j] >= 0 ? nc[j] : kDblMax;
        }
        max_layer = i;
    }
    double mc = kDblMax;
    int j = -1;
    for (int k = 0; k < n; ++k)
        if (pcost[k] < mc) { mc = pcost[k]; j = k; }
    if (j < 0) return COR_SHORT;
    const int R = max_layer + 1;
    for (int i = max_layer; i >= 0; --i) {
        chain[i] = j;
        s[i] = lay[i];
        if (i > 0) {
            corridor_rough(f, feas[i], j, &lo[i], &hi[i]);
            j = pred[(size_t)i * kCorridorMaxLateral + j];
        }
    }
    if (R < 4) return COR_SHORT;
    for (int i = 0; i < R; ++i) {
        const pqp_state r = densify_sample(xs, ys, s[i]);
        double a = -10.0, b = 10.0;
        if (i > 0) corridor_march(m, r, lo[i], hi[i], &a, &b);
        lo[i] = a; hi[i] = b;
    }
    for (int i = 0; i < R; ++i) {
        const double ds = i + 1 < R ? s[i + 1] - s[i] : 0.0;
        corridor_qp_rows(R, i, i == 0 ? vl : lo[i], i == 0 ? vl : hi[i], ds, A_col, A_val, l, u);
        corridor_qp_columns(R, i, ds, csc_ptr, csc_row, csc_val);
    }
    *M = corridor_qp_separators(R, sep);
    *R_out = R;
    return COR_OK;
}

}  // extern "C"
