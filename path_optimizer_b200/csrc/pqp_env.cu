// pqp_env.cu -- kernels and extern "C" entry points (include/pqp_env.h) of the stages either side
// of the path QP: clearance-bounds generation, collision check + s re-accumulation, spline
// densification, and the solveWithoutSmoothing-shaped chain  bounds -> QP -> tail  that keeps a
// whole planner iteration of a batch of paths on the device.  No CPU fallback.
//
// These kernels are gathers on a float distance map (4 B loads, L2-resident for planner-sized
// maps: 1100x250 cells = 1.1 MB); one thread owns one (station, circle) ray march or one state's
// footprint, grids are sized from the batch.
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <new>
#include <vector>

#include "pqp_edt_core.cuh"
#include "pqp_env_core.cuh"
#include "pqp_segment_core.cuh"
#include "pqp_dispatch.h"
#include "pqp_handle.h"

namespace {

using pqp::CarCircles;
using pqp::MapTable;
using pqp::MapView;
using pqp::ParamRow;
using pqp::ParamTable;
using pqp::SplineView;

struct EnvState {
    // the map set (pqp_set_maps): every map's cells one after the other, a device table of one descriptor per map and
    // the device copy of the count; all grow-only, so that a captured chain keeps reading the current set
    float *d_map = nullptr;
    size_t map_cap = 0;
    MapView *d_maps = nullptr;
    size_t maps_cap = 0;
    int32_t *d_nmaps = nullptr;
    int n_maps = 0;                // 0: no map set
    std::vector<MapView> h_maps;   // host copy of the table (n_maps rows)
    // occupancy builds (pqp_set_maps_occupancy*): the uploaded cells of the host entry, and the transform's scratch
    // (3 int32 per cell, at three times a map's cell offset).  An outgrown scratch goes to the handle's retired list: a
    // graph captured before still writes it.
    uint8_t *d_occ = nullptr;
    size_t occ_cap = 0;
    int32_t *d_edt = nullptr;
    size_t edt_cap = 0;
    // per-batch scratch (sized from the handle's capacity at first use)
    int32_t *d_nvalid = nullptr, *d_nkept = nullptr, *d_ok = nullptr, *d_koff = nullptr;
    int32_t *d_mapidx = nullptr;   // pqp_plan_batch_maps: the uploaded map index
    int32_t *d_setidx = nullptr;   // pqp_plan_batch_sets: the uploaded parameter-set index
    double *d_spl = nullptr;       // densify workspace: 13 doubles per station
    pqp_state *d_dense = nullptr;  // densify output [batch][max_out] (grow-only)
    size_t dense_cap = 0;
    // spline inputs (grow-only): knots + x/y coefficients
    double *d_knots = nullptr, *d_xc = nullptr, *d_yc = nullptr;
    size_t knot_cap = 0;
    // pqp_fit_splines_device: diag and rhs of both coordinates, 4 doubles per station (max_total, at first use)
    double *d_fit = nullptr;
    // pqp_segment_reference_device: every path's station count between its launches (max_batch, at first use)
    int32_t *d_seg = nullptr;
    // generic scratch for pqp_map_distance / pqp_check_states (grow-only)
    char *d_tmp = nullptr;
    size_t tmp_cap = 0;
    cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
};

void env_free(void *p) {
    EnvState *e = (EnvState *)p;
    cudaFree(e->d_map); cudaFree(e->d_maps); cudaFree(e->d_nmaps); cudaFree(e->d_mapidx); cudaFree(e->d_setidx);
    cudaFree(e->d_nvalid); cudaFree(e->d_nkept); cudaFree(e->d_ok); cudaFree(e->d_koff);
    cudaFree(e->d_spl); cudaFree(e->d_dense); cudaFree(e->d_knots); cudaFree(e->d_xc); cudaFree(e->d_yc);
    cudaFree(e->d_tmp); cudaFree(e->d_occ); cudaFree(e->d_edt); cudaFree(e->d_fit); cudaFree(e->d_seg);
    for (auto &ev : e->ev) if (ev) cudaEventDestroy(ev);
    delete e;
}

int env_get(pqp_handle *h, EnvState **out) {
    if (!h->env) {
        EnvState *e = new (std::nothrow) EnvState;
        if (!e) return PQP_ERR_ARG;
        h->env = e;
        h->env_free = env_free;
        PQP_CUDA(cudaSetDevice(h->device));
        const size_t B = (size_t)h->max_batch, T = (size_t)h->max_total;
        PQP_CUDA(cudaMalloc(&e->d_nvalid, B * sizeof(int32_t)));
        PQP_CUDA(cudaMalloc(&e->d_nkept, B * sizeof(int32_t)));
        PQP_CUDA(cudaMalloc(&e->d_ok, B * sizeof(int32_t)));
        PQP_CUDA(cudaMalloc(&e->d_koff, (B + 1) * sizeof(int32_t)));
        PQP_CUDA(cudaMalloc(&e->d_mapidx, B * sizeof(int32_t)));
        PQP_CUDA(cudaMalloc(&e->d_setidx, B * sizeof(int32_t)));
        PQP_CUDA(cudaMalloc(&e->d_nmaps, sizeof(int32_t)));
        PQP_CUDA(cudaMemset(e->d_nmaps, 0, sizeof(int32_t)));
        PQP_CUDA(cudaMalloc(&e->d_spl, T * 13 * sizeof(double)));
        for (auto &ev : e->ev) PQP_CUDA(cudaEventCreate(&ev));
    }
    *out = (EnvState *)h->env;
    return PQP_OK;
}

template <typename T>
int grow(T **p, size_t *cap, size_t need_bytes) {
    if (need_bytes <= *cap) return PQP_OK;
    cudaFree(*p);
    *p = nullptr;
    *cap = 0;
    PQP_CUDA(cudaMalloc(p, need_bytes));
    *cap = need_bytes;
    return PQP_OK;
}

// ---------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------

// The env kernels take the handle's parameter sets by value (pqp::ParamTable): R = 1 row (set 0) for the entries without
// a set index, kSetRows with one.
constexpr int kSetRows = PQP_MAX_PARAM_SETS;
static_assert(sizeof(ParamTable<kSetRows>) + 512 <= 32764, "the parameter table must fit a kernel's parameter space");

template <int R> struct BoundsArgs {
    MapTable maps;
    ParamTable<R> prm;
    int mode;
    const int32_t *n_points, *offsets;
    const pqp_state *ref;
    const int32_t *koff;           // [batch+1] knot offsets (IMPROVED), else null
    const double *knots, *xc, *yc;
    pqp_station_bounds *out;
    int32_t *n_valid;              // pre-set to n_points; atomicMin with the first blocked station
    int first_path;                // grid.y is capped at 65535: a larger batch is launched in tiles of paths
};

// grid (ceil(4*maxN/128), batch): thread = (station, circle) of path blockIdx.y
template <int R>
__global__ void __launch_bounds__(128)
pqp_bounds_kernel(const __grid_constant__ BoundsArgs<R> a) {
    const int b = a.first_path + blockIdx.y;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    const int i = t >> 2, j = t & 3;
    const int n = a.n_points[b];
    if (i >= n) return;
    const MapView *mp = pqp::map_of(a.maps, b);
    const ParamRow *pr = pqp::param_of(a.prm, b);
    if (!mp || !pr) {              // map or set index outside its set: no usable station, the QP reports PQP_INVALID_PROBLEM
        if (t == 0) a.n_valid[b] = 0;
        return;
    }
    const MapView map = *mp;
    const int off = a.offsets[b];
    const pqp_state st = a.ref[off + i];
    SplineView xs{0, nullptr, nullptr}, ys{0, nullptr, nullptr};
    if (a.mode == PQP_BOUNDS_IMPROVED) {
        const int k0 = a.koff[b], nk = a.koff[b + 1] - k0;
        xs = SplineView{nk, a.knots + k0, a.xc + 4 * (size_t)k0};
        ys = SplineView{nk, a.knots + k0, a.yc + 4 * (size_t)k0};
    }
    double ub, lb;
    const bool blocked = pqp::circle_bounds(map, pr->radius, a.mode, st, pr->d[j], xs, ys, ub, lb);
    double *o = &a.out[off + i].c0_ub + 2 * j;
    o[0] = ub;
    o[1] = lb;
    if (blocked) atomicMin(&a.n_valid[b], i);
}

// The single-stage lookups read map 0 of the set (the entry points check that a set is in place).
__global__ void pqp_map_distance_kernel(const MapView *maps, int n, const double *xy, double *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const MapView map = maps[0];
    out[i] = pqp::map_distance(map, xy[2 * i], xy[2 * i + 1]);
}

__global__ void pqp_check_states_kernel(const MapView *maps, const __grid_constant__ CarCircles car, int n,
                                        const pqp_state *s, int32_t *ok) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const MapView map = maps[0];
    ok[i] = pqp::state_collision_free(map, car, s[i].x, s[i].y, s[i].z) ? 1 : 0;
}

// The tails look their path's map and parameter set up once per CTA (thread 0, into shared memory).  Without a
// collision check neither is read, and no map set is needed.
template <int R> struct TailArgs {
    MapTable maps;
    ParamTable<R> prm;
    const int32_t *n_points, *offsets;
    const int32_t *status;   // optional: tail only for PQP_SOLVED paths (plan chain)
    pqp_state *paths;
    int collision_check;
    int32_t *n_kept, *ok;
};

// Raw tail (path_optimizer.cpp:191-202): one CTA per path.  Thread 0 re-accumulates s in the
// reference's serial order while every thread checks footprints; the cut is the first failure.
template <int R>
__global__ void __launch_bounds__(128)
pqp_finish_raw_kernel(const __grid_constant__ TailArgs<R> a) {
    __shared__ int first_fail, has_map, row_s;
    __shared__ MapView map_s;
    const int b = blockIdx.x;
    const int n = a.n_points[b];
    pqp_state *p = a.paths + a.offsets[b];
    if (a.status && a.status[b] != PQP_SOLVED) {
        if (threadIdx.x == 0) { a.n_kept[b] = 0; a.ok[b] = 0; }
        return;
    }
    if (threadIdx.x == 0) {
        first_fail = n;
        const MapView *mp = a.collision_check ? pqp::map_of(a.maps, b) : nullptr;
        const ParamRow *pr = a.collision_check ? pqp::param_of(a.prm, b) : nullptr;
        has_map = mp != nullptr && pr != nullptr;
        map_s = mp ? *mp : MapView{};
        row_s = pr ? (int)(pr - a.prm.row) : 0;
    }
    __syncthreads();
    if (a.collision_check && !has_map) {   // map or set index outside its set
        if (threadIdx.x == 0) { a.n_kept[b] = 0; a.ok[b] = 0; }
        return;
    }
    if (a.collision_check) {
        const MapView map = map_s;
        const CarCircles &car = a.prm.row[row_s].car;
        for (int i = threadIdx.x; i < n; i += blockDim.x)
            if (!pqp::state_collision_free(map, car, p[i].x, p[i].y, p[i].z)) atomicMin(&first_fail, i);
    }
    if (threadIdx.x == 0) {
        pqp::accumulate_s(n, p);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int f = first_fail;
        a.n_kept[b] = f;
        a.ok[b] = (f >= n) ? 1 : (f > 0 ? (p[f - 1].s >= 20 ? 1 : 0) : 0);
    }
}

template <int R> struct DensifyArgs {
    MapTable maps;
    ParamTable<R> prm;
    const int32_t *n_points, *offsets, *status;
    const pqp_state *paths;
    double *ws;              // 13 doubles per station: t, x/y coef (4 each), 4 scratch
    double spacing;
    int collision_check, max_out;
    pqp_state *out;          // [batch][max_out]
    int32_t *n_out, *ok;
};

// Densifying tail (path_optimizer.cpp:203-230): one CTA per path; threads 0 and 32 fit x(s), y(s),
// then all threads evaluate / check the samples.
template <int R>
__global__ void __launch_bounds__(128)
pqp_densify_kernel(const __grid_constant__ DensifyArgs<R> a) {
    __shared__ int first_fail, has_map, knots_ok, row_s;
    __shared__ MapView map_s;
    const int b = blockIdx.x;
    const int n = a.n_points[b];
    const int off = a.offsets[b];
    const pqp_state *p = a.paths + off;
    pqp_state *out = a.out + (size_t)b * a.max_out;
    if ((a.status && a.status[b] != PQP_SOLVED) || n < 3) {
        if (threadIdx.x == 0) { a.n_out[b] = 0; a.ok[b] = 0; }
        return;
    }
    double *ws = a.ws + 13 * (size_t)off;
    double *t = ws, *xc = ws + n, *yc = ws + 5 * (size_t)n, *scr = ws + 9 * (size_t)n;
    for (int i = threadIdx.x; i < n; i += blockDim.x) t[i] = p[i].s;
    if (threadIdx.x == 0) {
        first_fail = 0x7fffffff;
        const MapView *mp = a.collision_check ? pqp::map_of(a.maps, b) : nullptr;
        const ParamRow *pr = a.collision_check ? pqp::param_of(a.prm, b) : nullptr;
        has_map = mp != nullptr && pr != nullptr;
        map_s = mp ? *mp : MapView{};
        row_s = pr ? (int)(pr - a.prm.row) : 0;
    }
    __syncthreads();
    if (a.collision_check && !has_map) {   // map or set index outside its set
        if (threadIdx.x == 0) { a.n_out[b] = 0; a.ok[b] = 0; }
        return;
    }
    const MapView map = map_s;
    const CarCircles &car = a.prm.row[row_s].car;
    // threads 0 and 32 fit x(s) and y(s) side by side (diag / rhs scratch: 2n doubles each)
    if (threadIdx.x == 0) {
        knots_ok = pqp::knots_increasing(n, t);
        pqp::spline_fit(n, t, [&](int i) { return p[i].x; }, xc, scr, scr + n);
    }
    if (threadIdx.x == 32) pqp::spline_fit(n, t, [&](int i) { return p[i].y; }, yc, scr + 2 * (size_t)n, scr + 3 * (size_t)n);
    __syncthreads();
    if (!knots_ok) {
        if (threadIdx.x == 0) { a.n_out[b] = 0; a.ok[b] = 0; }
        return;
    }
    const double s_end = t[n - 1];
    // number of samples: i*spacing <= s_end, i = 0, 1, ...
    long long cnt = 0;
    if (s_end >= 0.0 && a.spacing > 0.0) {
        cnt = (long long)(s_end / a.spacing) + 1;
        while (cnt > 0 && !(pqp::mul((double)(cnt - 1), a.spacing) <= s_end)) --cnt;
        while (pqp::mul((double)cnt, a.spacing) <= s_end) ++cnt;
    }
    const SplineView xs{n, t, xc}, ys{n, t, yc};
    const long long lim = cnt < (long long)a.max_out + 1 ? cnt : (long long)a.max_out + 1;   // samples that matter
    for (long long i = threadIdx.x; i < lim; i += blockDim.x) {
        const pqp_state st = pqp::densify_sample(xs, ys, pqp::mul((double)i, a.spacing));
        if (a.collision_check && !pqp::state_collision_free(map, car, st.x, st.y, st.z)) atomicMin(&first_fail, (int)i);
        if (i < a.max_out) out[i] = st;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const long long f = first_fail;
        if (f < lim) {                       // collision seen before any overflow
            a.n_out[b] = (int)f;
            a.ok[b] = f > 0 ? (pqp::mul((double)(f - 1), a.spacing) >= 20 ? 1 : 0) : 0;
        } else if (cnt > a.max_out) {
            a.n_out[b] = a.max_out;
            a.ok[b] = 0;
        } else {
            a.n_out[b] = (int)cnt;
            a.ok[b] = 1;
        }
    }
}

// Occupancy builds (pqp_edt_core.cuh): one launch per pass covers up to kEdtMaps maps, blockIdx.y = map of the launch.
// The builds are passed by value, so a captured launch keeps the occupancy and destination it was captured with; before
// it writes anything a map's threads check that table row `index` still describes that destination (address, rows,
// cols), so a replay after a later layout change leaves the current set alone.
constexpr int kEdtMaps = 256;
struct EdtMap {
    const uint8_t *occ;      // [rows][cols], 0 = obstacle
    float *dst;              // the layer's cells in the map buffer
    int32_t *scratch;        // 3 * rows * cols
    int rows, cols;
    float res;
    int index;               // row of the table
};
struct EdtArgs {
    const MapView *table;
    const int32_t *n_maps;
    EdtMap map[kEdtMaps];
};
static_assert(sizeof(EdtArgs) <= 32764, "the build descriptors must fit a kernel's parameter space");

__device__ __forceinline__ bool edt_current(const EdtArgs &a, const EdtMap &m) {
    if (m.index >= *a.n_maps) return false;
    const MapView &v = a.table[m.index];
    return v.d == m.dst && v.rows == m.rows && v.cols == m.cols;
}

// grid (ceil(max cols / 128), maps): thread = column
__global__ void __launch_bounds__(128)
pqp_edt_column_kernel(const __grid_constant__ EdtArgs a) {
    const EdtMap &m = a.map[blockIdx.y];
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m.cols || !edt_current(a, m)) return;
    pqp::edt_column(m.occ, m.rows, m.cols, j, m.scratch + (size_t)j * m.rows, 1);
}

// grid (ceil(max rows / 128), maps): thread = row
__global__ void __launch_bounds__(128)
pqp_edt_row_kernel(const __grid_constant__ EdtArgs a) {
    const EdtMap &m = a.map[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m.rows || !edt_current(a, m)) return;
    const size_t R = (size_t)m.rows, n = R * (size_t)m.cols;
    pqp::edt_row(m.scratch + i, R, m.cols, m.scratch + n + i, m.scratch + 2 * n + i, R, m.res,
                 m.dst + (size_t)i * m.cols);
}

// pqp_fit_splines_device: one CTA per kFitPaths paths, one thread per (path, coordinate), a path's x and y threads on
// adjacent lanes.  The CTA first copies the knots of its paths (one range of stations, the offsets being an exclusive
// prefix), so that no fit reads a knot before it is written; after a barrier every thread decides its path's refusal
// from the knots, and only after a second barrier may a refused path's x thread overwrite them with NaN.
constexpr int kFitPaths = 32;
struct FitArgs {
    int batch;
    const int32_t *offsets;
    const pqp_state *ref;
    double *knots, *xc, *yc;
    double *scr;             // 4 doubles per station: diag and rhs of x, then of y
    int32_t *ok;
};

__global__ void __launch_bounds__(2 * kFitPaths)
pqp_fit_splines_kernel(const __grid_constant__ FitArgs a) {
    const int b0 = blockIdx.x * kFitPaths;
    const int nb = min(kFitPaths, a.batch - b0);
    const int lo = a.offsets[b0], hi = a.offsets[b0 + nb];
    for (int k = lo + (int)threadIdx.x; k < hi; k += blockDim.x) a.knots[k] = a.ref[k].s;
    __syncthreads();
    const int p = threadIdx.x >> 1, coord = threadIdx.x & 1;
    const int b = b0 + p;
    const bool active = p < nb;
    int off = 0, n = 0;
    bool ok = false;
    if (active) {
        off = a.offsets[b];
        n = a.offsets[b + 1] - off;
        ok = pqp::fit_knots_ok(n, a.knots + off);
    }
    __syncthreads();
    if (!active) return;
    const size_t o = (size_t)off;
    pqp::fit_path_coord(max(n, 0), ok, coord, a.ref + o, a.knots + o, (coord ? a.yc : a.xc) + 4 * o, a.scr + 4 * o);
    if (coord == 0) a.ok[b] = ok ? 1 : 0;
}

// pqp_segment_reference_device: three launches on the caller's stream.  (1) one thread per path walks its line once to
// count its stations (pqp::segment_count) and writes x0 and end_heading; (2) one warp reserves the stations in index
// order and writes n_points, offsets and ok; (3) one thread per kept path walks its line again and writes its states
// (pqp::segment_write), the same samples bit for bit.  The counts sit in the handle's scratch between the launches.
struct SegmentArgs {
    pqp::SegmentFlags f;
    int batch;
    long long capacity;
    const int32_t *koff;
    const double *knots, *xc, *yc;
    const double *max_s;
    const pqp_state *start, *goal;
    int32_t *count;          // scratch [batch]: stations of every path, 0 when refused
    int32_t *n_points, *offsets, *ok;
    pqp_state *ref;
    double *x0, *end_heading;
};
constexpr int kSegmentThreads = 128;

__device__ __forceinline__ void segment_splines(const SegmentArgs &a, int b, SplineView &xs, SplineView &ys) {
    const int o = a.koff[b], n = a.koff[b + 1] - o;
    xs = SplineView{n, a.knots + o, a.xc + 4 * (size_t)o};
    ys = SplineView{n, a.knots + o, a.yc + 4 * (size_t)o};
}

__global__ void __launch_bounds__(kSegmentThreads)
pqp_segment_count_kernel(const __grid_constant__ SegmentArgs a) {
    const int b = blockIdx.x * kSegmentThreads + threadIdx.x;
    if (b >= a.batch) return;
    SplineView xs, ys;
    segment_splines(a, b, xs, ys);
    const pqp_state start = a.start[b], goal = a.goal[b];
    double x0[3], cut_s;
    int n;
    pqp::segment_count(a.f, xs, ys, a.max_s[b], start, goal, x0, &cut_s, &n);
    a.count[b] = n;
    a.x0[3 * (size_t)b + 0] = x0[0];
    a.x0[3 * (size_t)b + 1] = x0[1];
    a.x0[3 * (size_t)b + 2] = x0[2];
    a.end_heading[b] = goal.z;
}

__device__ __forceinline__ long long warp_inclusive_sum(long long v) {
    const int lane = threadIdx.x & 31;
    for (int d = 1; d < 32; d <<= 1) {
        const long long u = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v += u;
    }
    return v;
}

__global__ void __launch_bounds__(32)
pqp_segment_scan_kernel(const __grid_constant__ SegmentArgs a) {
    const int lane = threadIdx.x;
    long long all = 0, kept = 0;      // stations of every path before the tile, and of the kept ones
    if (lane == 0) a.offsets[0] = 0;
    for (int b0 = 0; b0 < a.batch; b0 += 32) {
        const int b = b0 + lane;
        const int c = b < a.batch ? a.count[b] : 0;
        const long long ia = warp_inclusive_sum(c);
        const bool keep = pqp::segment_fits(all + ia - c, c, a.capacity);
        const int ck = keep ? c : 0;
        const long long ik = warp_inclusive_sum(ck);
        if (b < a.batch) {
            a.n_points[b] = ck;
            a.offsets[b + 1] = (int32_t)(kept + ik);
            a.ok[b] = keep ? 1 : 0;
        }
        all += __shfl_sync(0xffffffffu, ia, 31);
        kept += __shfl_sync(0xffffffffu, ik, 31);
    }
}

__global__ void __launch_bounds__(kSegmentThreads)
pqp_segment_write_kernel(const __grid_constant__ SegmentArgs a) {
    const int b = blockIdx.x * kSegmentThreads + threadIdx.x;
    if (b >= a.batch || !a.ok[b]) return;
    SplineView xs, ys;
    segment_splines(a, b, xs, ys);
    pqp::segment_write(a.f, xs, ys, a.n_points[b], a.ref + a.offsets[b]);
}

// ---------------------------------------------------------------------------------------------
// host helpers
// ---------------------------------------------------------------------------------------------

// Lays out a set of n_maps geometries (each map's cells start on a 256-byte boundary of the one cell buffer): grows the
// cell buffer and the table, and writes the table and the count on `st`.  The caller fills the cells, synchronises and
// then publishes the set (e->n_maps, e->h_maps); until then the handle has none.  `Desc`: pqp_distance_map or
// pqp_occupancy_map.
template <typename Desc>
int lay_out_maps(EnvState *e, int n_maps, const Desc *maps, cudaStream_t st, std::vector<MapView> *table) {
    constexpr size_t kAlign = 256 / sizeof(float);
    std::vector<size_t> first((size_t)n_maps);
    size_t cells = 0;
    for (int m = 0; m < n_maps; ++m) {
        first[m] = cells;
        cells += ((size_t)maps[m].rows * (size_t)maps[m].cols + kAlign - 1) / kAlign * kAlign;
    }
    e->n_maps = 0;   // no set until the new one is in place
    e->h_maps.clear();
    int rc = grow(&e->d_map, &e->map_cap, cells * sizeof(float));
    if (rc != PQP_OK) return rc;
    rc = grow(&e->d_maps, &e->maps_cap, (size_t)n_maps * sizeof(MapView));
    if (rc != PQP_OK) return rc;
    table->resize((size_t)n_maps);
    for (int m = 0; m < n_maps; ++m) {
        const Desc &d = maps[m];
        (*table)[m] = pqp::make_map_view(e->d_map + first[m], d.rows, d.cols, d.resolution, d.center_x, d.center_y);
    }
    const int32_t count = n_maps;
    PQP_CUDA(cudaMemcpyAsync(e->d_maps, table->data(), table->size() * sizeof(MapView), cudaMemcpyHostToDevice, st));
    PQP_CUDA(cudaMemcpyAsync(e->d_nmaps, &count, sizeof(int32_t), cudaMemcpyHostToDevice, st));
    return PQP_OK;
}

// Bytes of transform scratch a table needs: 3 int32 per cell of the map buffer up to the end of its last map.
size_t edt_need(const EnvState *e, const std::vector<MapView> &table) {
    size_t end = 0;
    for (const MapView &v : table) end = std::max(end, (size_t)(v.d - e->d_map) + (size_t)v.rows * v.cols);
    return 3 * end * sizeof(int32_t);
}

// Launches the build of every map of `table` from the occupancy grids occ[m] (device pointers).
int launch_edt(EnvState *e, const std::vector<MapView> &table, const uint8_t *const *occ, cudaStream_t st) {
    const int n_maps = (int)table.size();
    for (int first = 0; first < n_maps; first += kEdtMaps) {
        EdtArgs a;
        a.table = e->d_maps;
        a.n_maps = e->d_nmaps;
        const int n = std::min(kEdtMaps, n_maps - first);
        int max_rows = 0, max_cols = 0;
        for (int k = 0; k < n; ++k) {
            const MapView &v = table[first + k];
            const size_t off = (size_t)(v.d - e->d_map);
            a.map[k] = EdtMap{occ[first + k], const_cast<float *>(v.d), e->d_edt + 3 * off, v.rows, v.cols, (float)v.res,
                              first + k};
            max_rows = std::max(max_rows, v.rows);
            max_cols = std::max(max_cols, v.cols);
        }
        pqp_edt_column_kernel<<<dim3((unsigned)((max_cols + 127) / 128), (unsigned)n), 128, 0, st>>>(a);
        PQP_CUDA(cudaGetLastError());
        pqp_edt_row_kernel<<<dim3((unsigned)((max_rows + 127) / 128), (unsigned)n), 128, 0, st>>>(a);
        PQP_CUDA(cudaGetLastError());
    }
    return PQP_OK;
}

// Checks occupancy descriptors as pqp_set_maps checks its own.
bool occupancy_ok(int n_maps, const pqp_occupancy_map *maps) {
    if (n_maps < 1 || !maps) return false;
    for (int m = 0; m < n_maps; ++m) {
        const pqp_occupancy_map &d = maps[m];
        if (!d.cells || d.rows < 1 || d.cols < 1 || !(d.resolution > 0.0)) return false;
    }
    return true;
}

// Lays out an occupancy set and sizes the transform's scratch (an outgrown one is retired, not freed).
int lay_out_occupancy(pqp_handle *h, EnvState *e, int n_maps, const pqp_occupancy_map *maps, cudaStream_t st,
                      std::vector<MapView> *table) {
    int rc = lay_out_maps(e, n_maps, maps, st, table);
    if (rc != PQP_OK) return rc;
    const size_t need = edt_need(e, *table);
    if (need > e->edt_cap) {
        if (e->d_edt) h->retired.push_back(e->d_edt);
        e->d_edt = nullptr;
        e->edt_cap = 0;
        PQP_CUDA(cudaMalloc(&e->d_edt, need));
        e->edt_cap = need;
    }
    return PQP_OK;
}

int need_map(pqp_handle *h, EnvState **e) {
    int rc = env_get(h, e);
    if (rc != PQP_OK) return rc;
    if ((*e)->n_maps < 1) {
        pqp_set_err("no distance map: call pqp_set_map or pqp_set_maps first");
        return PQP_ERR_ARG;
    }
    return PQP_OK;
}

// The handle's map set for the kernels; `index` [batch] on the device, or NULL for map 0.
MapTable map_table(const EnvState *e, const int32_t *index) { return MapTable{e->d_maps, e->d_nmaps, index}; }

// uploads n_points/offsets/ref (+ splines) into the handle's buffers; returns total and max n
int upload_paths(pqp_handle *h, EnvState *e, int batch, const int32_t *n_points, const pqp_state *ref, int mode,
                 const int32_t *n_knots, const double *knots, const double *x_coef, const double *y_coef,
                 long long *total_out, int *max_n_out, int64_t *bytes, cudaStream_t st) {
    if (batch > h->max_batch) { pqp_set_err("batch exceeds the handle's max_batch"); return PQP_ERR_CAPACITY; }
    long long total = 0;
    int max_n = 0;
    h->h_off[0] = 0;
    for (int b = 0; b < batch; ++b) {
        if (n_points[b] < 0) { pqp_set_err("negative n_points"); return PQP_ERR_ARG; }
        total += n_points[b];
        if (total > h->max_total) { pqp_set_err("station count exceeds the handle's max_total_points"); return PQP_ERR_CAPACITY; }
        h->h_off[b + 1] = (int32_t)total;
        max_n = std::max(max_n, (int)n_points[b]);
    }
    const size_t B = (size_t)batch, T = (size_t)total;
    PQP_CUDA(cudaMemcpyAsync(h->d_n, n_points, B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    PQP_CUDA(cudaMemcpyAsync(h->d_off, h->h_off, (B + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    PQP_CUDA(cudaMemcpyAsync(h->d_ref, ref, T * sizeof(pqp_state), cudaMemcpyHostToDevice, st));
    *bytes += (int64_t)(B * 2 * sizeof(int32_t) + sizeof(int32_t) + T * sizeof(pqp_state));
    if (mode == PQP_BOUNDS_IMPROVED) {
        if (!n_knots || !knots || !x_coef || !y_coef) {
            pqp_set_err("PQP_BOUNDS_IMPROVED needs the reference splines (n_knots, knots, x_coef, y_coef)");
            return PQP_ERR_ARG;
        }
        // knot offsets (a small host vector; see the note on pageable copies below)
        std::vector<int32_t> koff(B + 1, 0);
        for (int b = 0; b < batch; ++b) {
            if (n_knots[b] < 3) { pqp_set_err("a reference spline needs >= 3 knots"); return PQP_ERR_ARG; }
            koff[b + 1] = koff[b] + n_knots[b];
        }
        const size_t K = (size_t)koff[B];
        if (K * 4 * sizeof(double) > e->knot_cap) {
            cudaFree(e->d_knots); cudaFree(e->d_xc); cudaFree(e->d_yc);
            e->d_knots = e->d_xc = e->d_yc = nullptr;
            e->knot_cap = 0;
            PQP_CUDA(cudaMalloc(&e->d_knots, K * sizeof(double)));
            PQP_CUDA(cudaMalloc(&e->d_xc, K * 4 * sizeof(double)));
            PQP_CUDA(cudaMalloc(&e->d_yc, K * 4 * sizeof(double)));
            e->knot_cap = K * 4 * sizeof(double);
        }
        // pageable source: the copy is staged before the call returns, so the local vector is safe
        PQP_CUDA(cudaMemcpyAsync(e->d_koff, koff.data(), (B + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        PQP_CUDA(cudaMemcpyAsync(e->d_knots, knots, K * sizeof(double), cudaMemcpyHostToDevice, st));
        PQP_CUDA(cudaMemcpyAsync(e->d_xc, x_coef, K * 4 * sizeof(double), cudaMemcpyHostToDevice, st));
        PQP_CUDA(cudaMemcpyAsync(e->d_yc, y_coef, K * 4 * sizeof(double), cudaMemcpyHostToDevice, st));
        *bytes += (int64_t)((B + 1) * sizeof(int32_t) + K * 9 * sizeof(double));
    }
    *total_out = total;
    *max_n_out = max_n;
    return PQP_OK;
}

// Device arrays of one batch of paths: what upload_paths leaves in the handle's buffers, or the caller's own
// (pqp_plan_batch_device).
struct PathsView {
    const int32_t *n_points, *offsets;
    const pqp_state *ref;
    const int32_t *koff;           // [batch+1] knot offsets (IMPROVED), else null
    const double *knots, *xc, *yc;
};

PathsView handle_paths(pqp_handle *h, EnvState *e) {
    return PathsView{h->d_n, h->d_off, h->d_ref, e->d_koff, e->d_knots, e->d_xc, e->d_yc};
}

// The handle's first n_sets parameter sets for the kernels; `index` [batch] on the device, or NULL for set 0.
template <int R> ParamTable<R> param_table(const pqp_handle *h, const int32_t *index, int n_sets) {
    ParamTable<R> t;
    t.n = n_sets;
    t.index = index;
    for (int s = 0; s < n_sets; ++s) t.row[s] = pqp::make_param_row(h->sets[s]);
    return t;
}

// A stage's parameter sets: the path index on the device (NULL: set 0 for every path, one row) and the number of sets
// an index may name.
struct SetIndex {
    const int32_t *index;
    int n_sets;
};
constexpr SetIndex kSet0{nullptr, 1};

template <int R>
int launch_bounds_impl(pqp_handle *h, EnvState *e, int mode, int batch, int max_n, const PathsView &p,
                       const int32_t *map_index, SetIndex set, pqp_station_bounds *out, cudaStream_t st) {
    BoundsArgs<R> a;
    a.maps = map_table(e, map_index);
    a.prm = param_table<R>(h, set.index, set.n_sets);
    a.mode = mode;
    a.n_points = p.n_points; a.offsets = p.offsets; a.ref = p.ref;
    a.koff = p.koff; a.knots = p.knots; a.xc = p.xc; a.yc = p.yc;
    a.out = out;
    a.n_valid = e->d_nvalid;
    PQP_CUDA(cudaMemcpyAsync(e->d_nvalid, p.n_points, (size_t)batch * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    for (int first = 0; max_n > 0 && first < batch; first += 65535) {
        a.first_path = first;
        dim3 grid((unsigned)((4 * max_n + 127) / 128), (unsigned)std::min(65535, batch - first));
        pqp_bounds_kernel<R><<<grid, 128, 0, st>>>(a);
        PQP_CUDA(cudaGetLastError());
    }
    return PQP_OK;
}

int launch_bounds_kernel(pqp_handle *h, EnvState *e, int mode, int batch, int max_n, const PathsView &p,
                         const int32_t *map_index, SetIndex set, pqp_station_bounds *out, cudaStream_t st) {
    return set.index ? launch_bounds_impl<kSetRows>(h, e, mode, batch, max_n, p, map_index, set, out, st)
                     : launch_bounds_impl<1>(h, e, mode, batch, max_n, p, map_index, kSet0, out, st);
}

template <int R>
int launch_finish_raw_impl(pqp_handle *h, EnvState *e, int batch, const int32_t *d_n, const int32_t *d_off,
                           const int32_t *d_status, const int32_t *map_index, SetIndex set, pqp_state *d_paths,
                           int collision_check, int32_t *d_n_kept, int32_t *d_ok, cudaStream_t st) {
    TailArgs<R> a;
    a.maps = map_table(e, map_index); a.prm = param_table<R>(h, set.index, set.n_sets);
    a.n_points = d_n; a.offsets = d_off; a.status = d_status; a.paths = d_paths;
    a.collision_check = collision_check ? 1 : 0;
    a.n_kept = d_n_kept; a.ok = d_ok;
    pqp_finish_raw_kernel<R><<<batch, 128, 0, st>>>(a);
    PQP_CUDA(cudaGetLastError());
    return PQP_OK;
}

int launch_finish_raw(pqp_handle *h, EnvState *e, int batch, const int32_t *d_n, const int32_t *d_off,
                      const int32_t *d_status, const int32_t *map_index, SetIndex set, pqp_state *d_paths,
                      int collision_check, int32_t *d_n_kept, int32_t *d_ok, cudaStream_t st) {
    return set.index ? launch_finish_raw_impl<kSetRows>(h, e, batch, d_n, d_off, d_status, map_index, set, d_paths,
                                                        collision_check, d_n_kept, d_ok, st)
                     : launch_finish_raw_impl<1>(h, e, batch, d_n, d_off, d_status, map_index, kSet0, d_paths,
                                                 collision_check, d_n_kept, d_ok, st);
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
extern "C" {

int pqp_set_maps(pqp_handle *h, int n_maps, const pqp_distance_map *maps) {
    if (!h || n_maps < 1 || !maps) {
        pqp_set_err("pqp_set_maps: bad argument (needs a handle and n_maps >= 1 descriptors)");
        return PQP_ERR_ARG;
    }
    // every descriptor is checked before any device state changes: a bad one leaves the previous set in place
    for (int m = 0; m < n_maps; ++m) {
        const pqp_distance_map &d = maps[m];
        if (!d.distance || d.rows < 1 || d.cols < 1 || !(d.resolution > 0.0)) {
            pqp_set_err("pqp_set_maps: bad map descriptor (NULL distance, rows or cols < 1, or resolution <= 0)");
            return PQP_ERR_ARG;
        }
    }
    EnvState *e;
    int rc = env_get(h, &e);
    if (rc != PQP_OK) return rc;
    PQP_CUDA(cudaSetDevice(h->device));
    std::vector<MapView> table;
    rc = lay_out_maps(e, n_maps, maps, h->stream, &table);
    if (rc != PQP_OK) return rc;
    for (int m = 0; m < n_maps; ++m) {
        const pqp_distance_map &d = maps[m];
        PQP_CUDA(cudaMemcpyAsync(const_cast<float *>(table[m].d), d.distance, (size_t)d.rows * d.cols * sizeof(float),
                                 cudaMemcpyHostToDevice, h->stream));
    }
    PQP_CUDA(cudaStreamSynchronize(h->stream));
    e->n_maps = n_maps;
    e->h_maps.swap(table);
    return PQP_OK;
}

int pqp_set_map(pqp_handle *h, const pqp_distance_map *map) { return pqp_set_maps(h, 1, map); }

int pqp_set_maps_occupancy(pqp_handle *h, int n_maps, const pqp_occupancy_map *maps) {
    // every descriptor is checked before any device state changes: a bad one leaves the previous set in place
    if (!h || !occupancy_ok(n_maps, maps)) {
        pqp_set_err("pqp_set_maps_occupancy: bad argument (needs a handle and n_maps >= 1 descriptors with cells, rows "
                    "and cols >= 1 and resolution > 0)");
        return PQP_ERR_ARG;
    }
    EnvState *e;
    int rc = env_get(h, &e);
    if (rc != PQP_OK) return rc;
    PQP_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = h->stream;
    std::vector<MapView> table;
    rc = lay_out_occupancy(h, e, n_maps, maps, st, &table);
    if (rc != PQP_OK) return rc;
    // the cells go to the upload buffer at the maps' cell offsets
    const MapView &last = table.back();
    rc = grow(&e->d_occ, &e->occ_cap, (size_t)(last.d - e->d_map) + (size_t)last.rows * last.cols);
    if (rc != PQP_OK) return rc;
    std::vector<const uint8_t *> occ((size_t)n_maps);
    for (int m = 0; m < n_maps; ++m) {
        uint8_t *dst = e->d_occ + (table[m].d - e->d_map);
        PQP_CUDA(cudaMemcpyAsync(dst, maps[m].cells, (size_t)maps[m].rows * maps[m].cols, cudaMemcpyHostToDevice, st));
        occ[m] = dst;
    }
    rc = launch_edt(e, table, occ.data(), st);
    if (rc != PQP_OK) return rc;
    PQP_CUDA(cudaStreamSynchronize(st));
    e->n_maps = n_maps;
    e->h_maps.swap(table);
    return PQP_OK;
}

int pqp_set_maps_occupancy_device(pqp_handle *h, int n_maps, const pqp_occupancy_map *maps, void *stream) {
    if (!h || !occupancy_ok(n_maps, maps)) {
        pqp_set_err("pqp_set_maps_occupancy_device: bad argument (needs a handle and n_maps >= 1 descriptors with cells, "
                    "rows and cols >= 1 and resolution > 0)");
        return PQP_ERR_ARG;
    }
    cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
    std::vector<const uint8_t *> occ((size_t)n_maps);
    for (int m = 0; m < n_maps; ++m) occ[m] = maps[m].cells;
    EnvState *e = (EnvState *)h->env;
    bool same = e && e->n_maps == n_maps && (int)e->h_maps.size() == n_maps;
    for (int m = 0; same && m < n_maps; ++m) {
        const MapView &v = e->h_maps[m];
        const pqp_occupancy_map &d = maps[m];
        same = v.rows == d.rows && v.cols == d.cols && v.res == d.resolution && v.cx == d.center_x && v.cy == d.center_y;
    }
    if (same && edt_need(e, e->h_maps) <= e->edt_cap) {
        PQP_CUDA(cudaSetDevice(h->device));
        return launch_edt(e, e->h_maps, occ.data(), st);
    }
    // a new layout allocates and synchronises, which a capture must not see
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    PQP_CUDA(cudaStreamIsCapturing(st, &cs));
    if (cs != cudaStreamCaptureStatusNone) {
        pqp_set_err("pqp_set_maps_occupancy_device: the map layout changes (count, rows, cols, resolution or centre), "
                    "which cannot be captured; make one call with this layout before capturing");
        return PQP_ERR_ARG;
    }
    int rc = env_get(h, &e);
    if (rc != PQP_OK) return rc;
    PQP_CUDA(cudaSetDevice(h->device));
    std::vector<MapView> table;
    rc = lay_out_occupancy(h, e, n_maps, maps, st, &table);
    if (rc != PQP_OK) return rc;
    rc = launch_edt(e, table, occ.data(), st);
    if (rc != PQP_OK) return rc;
    PQP_CUDA(cudaStreamSynchronize(st));
    e->n_maps = n_maps;
    e->h_maps.swap(table);
    return PQP_OK;
}

int pqp_get_map(pqp_handle *h, int m, float *out) {
    if (!h || !out || m < 0 || !h->env || m >= ((EnvState *)h->env)->n_maps) {
        pqp_set_err("pqp_get_map: bad argument (needs a handle, an output buffer and a map of the set)");
        return PQP_ERR_ARG;
    }
    const MapView &v = ((EnvState *)h->env)->h_maps[m];
    PQP_CUDA(cudaSetDevice(h->device));
    PQP_CUDA(cudaMemcpyAsync(out, v.d, (size_t)v.rows * v.cols * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    PQP_CUDA(cudaStreamSynchronize(h->stream));
    return PQP_OK;
}

int pqp_map_distance(pqp_handle *h, int n, const double *xy, double *out) {
    if (!h || n < 0 || (n > 0 && (!xy || !out))) { pqp_set_err("pqp_map_distance: bad argument"); return PQP_ERR_ARG; }
    EnvState *e;
    int rc = need_map(h, &e);
    if (rc != PQP_OK || n == 0) return rc;
    PQP_CUDA(cudaSetDevice(h->device));
    rc = grow(&e->d_tmp, &e->tmp_cap, (size_t)n * 3 * sizeof(double));
    if (rc != PQP_OK) return rc;
    double *d_xy = (double *)e->d_tmp, *d_out = d_xy + 2 * (size_t)n;
    cudaStream_t st = h->stream;
    PQP_CUDA(cudaMemcpyAsync(d_xy, xy, (size_t)n * 2 * sizeof(double), cudaMemcpyHostToDevice, st));
    pqp_map_distance_kernel<<<(n + 127) / 128, 128, 0, st>>>(e->d_maps, n, d_xy, d_out);
    PQP_CUDA(cudaGetLastError());
    PQP_CUDA(cudaMemcpyAsync(out, d_out, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, st));
    PQP_CUDA(cudaStreamSynchronize(st));
    return PQP_OK;
}

// Natural cubic spline on the host (helper for callers that hold plain arrays): same recurrences
// as the device fit.
int pqp_spline_fit(int n, const double *t, const double *y, double *coef) {
    if (n < 3 || !t || !y || !coef) { pqp_set_err("pqp_spline_fit: need n >= 3"); return PQP_ERR_ARG; }
    std::vector<double> diag((size_t)n), rhs((size_t)n), b((size_t)n);
    diag[0] = 2.0; rhs[0] = 0.0;
    double upper_prev = 0.0;
    for (int i = 1; i < n - 1; ++i) {
        const double hl = t[i] - t[i - 1], hr = t[i + 1] - t[i];
        if (!(hl > 0.0) || !(hr > 0.0)) { pqp_set_err("pqp_spline_fit: knots must increase strictly"); return PQP_ERR_ARG; }
        const double lo = hl / 3.0, di = 2.0 * (t[i + 1] - t[i - 1]) / 3.0, up = hr / 3.0;
        const double r = (y[i + 1] - y[i]) / hr - (y[i] - y[i - 1]) / hl;
        const double w = lo / diag[i - 1];
        diag[i] = di - w * upper_prev;
        rhs[i] = r - w * rhs[i - 1];
        upper_prev = up;
    }
    b[n - 1] = 0.0;
    for (int i = n - 2; i >= 1; --i) b[i] = (rhs[i] - (t[i + 1] - t[i]) / 3.0 * b[i + 1]) / diag[i];
    b[0] = 0.0;
    for (int i = 0; i < n - 1; ++i) {
        const double hh = t[i + 1] - t[i];
        coef[4 * i + 0] = (b[i + 1] - b[i]) / (3.0 * hh);
        coef[4 * i + 1] = b[i];
        coef[4 * i + 2] = (y[i + 1] - y[i]) / hh - (2.0 * b[i] + b[i + 1]) * hh / 3.0;
        coef[4 * i + 3] = y[i];
    }
    const int i = n - 2;
    const double hh = t[n - 1] - t[n - 2];
    coef[4 * (n - 1) + 0] = 0.0;
    coef[4 * (n - 1) + 1] = b[n - 1];
    coef[4 * (n - 1) + 2] = 3.0 * coef[4 * i] * hh * hh + 2.0 * coef[4 * i + 1] * hh + coef[4 * i + 2];
    coef[4 * (n - 1) + 3] = y[n - 1];
    return PQP_OK;
}

double pqp_spline_eval(int n, const double *t, const double *coef, int order, double at) {
    if (n < 1 || !t || !coef || order < 0 || order > 2) return nan("");
    return pqp::spline_eval(SplineView{n, t, coef}, order, at);
}

int pqp_fit_splines_device(pqp_handle *h, int batch, int total_points, const int32_t *d_offsets, const pqp_state *d_ref,
                           double *d_knots, double *d_x_coef, double *d_y_coef, int32_t *d_ok, void *stream) {
    if (!h || batch < 0 || total_points < 0 ||
        (batch > 0 && (!d_offsets || !d_ref || !d_knots || !d_x_coef || !d_y_coef || !d_ok))) {
        pqp_set_err("pqp_fit_splines_device: bad argument");
        return PQP_ERR_ARG;
    }
    if (batch > h->max_batch || total_points > h->max_total) {
        pqp_set_err("batch / total_points exceed what the handle was created for (workspace size)");
        return PQP_ERR_CAPACITY;
    }
    EnvState *e;
    int rc = env_get(h, &e);
    if (rc != PQP_OK || batch == 0) return rc;
    PQP_CUDA(cudaSetDevice(h->device));
    if (!e->d_fit) PQP_CUDA(cudaMalloc(&e->d_fit, (size_t)h->max_total * 4 * sizeof(double)));
    cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
    const FitArgs a{batch, d_offsets, d_ref, d_knots, d_x_coef, d_y_coef, e->d_fit, d_ok};
    pqp_fit_splines_kernel<<<(batch + kFitPaths - 1) / kFitPaths, 2 * kFitPaths, 0, st>>>(a);
    PQP_CUDA(cudaGetLastError());
    return PQP_OK;
}

int pqp_segment_reference_device(pqp_handle *h, int batch, const int32_t *d_knot_offsets, const double *d_knots,
                                 const double *d_x_coef, const double *d_y_coef, const double *d_max_s,
                                 const pqp_state *d_start, const pqp_state *d_goal, double delta_s_smaller,
                                 double delta_s_larger, int dynamic_segmentation, double search_delta_s,
                                 int max_n_points, int capacity, int32_t *d_n_points, int32_t *d_offsets,
                                 pqp_state *d_ref, double *d_x0, double *d_end_heading, int32_t *d_ok, void *stream) {
    const bool spacing_ok = delta_s_smaller > 0 && delta_s_larger >= delta_s_smaller && isfinite(delta_s_larger) &&
                            search_delta_s > 0 && isfinite(search_delta_s);
    if (!h || batch < 0 || capacity < 0 || max_n_points < 1 || !spacing_ok ||
        (batch > 0 && (!d_knot_offsets || !d_knots || !d_x_coef || !d_y_coef || !d_max_s || !d_start || !d_goal ||
                       !d_n_points || !d_offsets || !d_ref || !d_x0 || !d_end_heading || !d_ok))) {
        pqp_set_err("pqp_segment_reference_device: bad argument");
        return PQP_ERR_ARG;
    }
    if (batch > h->max_batch || capacity > h->max_total) {
        pqp_set_err("batch / capacity exceed what the handle was created for (max_batch, max_total_points)");
        return PQP_ERR_CAPACITY;
    }
    EnvState *e;
    int rc = env_get(h, &e);
    if (rc != PQP_OK) return rc;
    PQP_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
    if (batch == 0) {                     // an empty batch still gets offsets[0] = 0 when the array is given
        if (d_offsets) PQP_CUDA(cudaMemsetAsync(d_offsets, 0, sizeof(int32_t), st));
        return PQP_OK;
    }
    if (!e->d_seg) PQP_CUDA(cudaMalloc(&e->d_seg, (size_t)h->max_batch * sizeof(int32_t)));
    SegmentArgs a;
    a.f = pqp::SegmentFlags{delta_s_smaller, delta_s_larger, search_delta_s, dynamic_segmentation ? 1 : 0, max_n_points};
    a.batch = batch; a.capacity = capacity;
    a.koff = d_knot_offsets; a.knots = d_knots; a.xc = d_x_coef; a.yc = d_y_coef;
    a.max_s = d_max_s; a.start = d_start; a.goal = d_goal; a.count = e->d_seg;
    a.n_points = d_n_points; a.offsets = d_offsets; a.ok = d_ok; a.ref = d_ref; a.x0 = d_x0; a.end_heading = d_end_heading;
    const int grid = (batch + kSegmentThreads - 1) / kSegmentThreads;
    pqp_segment_count_kernel<<<grid, kSegmentThreads, 0, st>>>(a);
    PQP_CUDA(cudaGetLastError());
    pqp_segment_scan_kernel<<<1, 32, 0, st>>>(a);
    PQP_CUDA(cudaGetLastError());
    pqp_segment_write_kernel<<<grid, kSegmentThreads, 0, st>>>(a);
    PQP_CUDA(cudaGetLastError());
    return PQP_OK;
}

int pqp_update_bounds_batch(pqp_handle *h, int mode, int batch, const int32_t *n_points, const pqp_state *ref,
                            const int32_t *n_knots, const double *knots, const double *x_coef, const double *y_coef,
                            pqp_station_bounds *out_bounds, int32_t *out_n_valid, pqp_stats *stats) {
    if (!h || batch < 0 || (batch > 0 && (!n_points || !ref || !out_bounds || !out_n_valid)) ||
        (mode != PQP_BOUNDS_IMPROVED && mode != PQP_BOUNDS_SIMPLE)) {
        pqp_set_err("pqp_update_bounds_batch: bad argument");
        return PQP_ERR_ARG;
    }
    if (stats) memset(stats, 0, sizeof(*stats));
    EnvState *e;
    int rc = need_map(h, &e);
    if (rc != PQP_OK || batch == 0) return rc;
    PQP_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = h->stream;
    long long total = 0;
    int max_n = 0;
    int64_t h2d = 0;
    PQP_CUDA(cudaEventRecord(e->ev[0], st));
    rc = upload_paths(h, e, batch, n_points, ref, mode, n_knots, knots, x_coef, y_coef, &total, &max_n, &h2d, st);
    if (rc != PQP_OK) return rc;
    PQP_CUDA(cudaEventRecord(e->ev[1], st));
    rc = launch_bounds_kernel(h, e, mode, batch, max_n, handle_paths(h, e), nullptr, kSet0, h->d_bounds, st);
    if (rc != PQP_OK) return rc;
    PQP_CUDA(cudaEventRecord(e->ev[2], st));
    PQP_CUDA(cudaMemcpyAsync(out_bounds, h->d_bounds, (size_t)total * sizeof(pqp_station_bounds), cudaMemcpyDeviceToHost, st));
    PQP_CUDA(cudaMemcpyAsync(out_n_valid, e->d_nvalid, (size_t)batch * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    PQP_CUDA(cudaEventRecord(e->ev[3], st));
    PQP_CUDA(cudaStreamSynchronize(st));
    if (stats) {
        PQP_CUDA(cudaEventElapsedTime(&stats->h2d_ms, e->ev[0], e->ev[1]));
        PQP_CUDA(cudaEventElapsedTime(&stats->kernel_ms, e->ev[1], e->ev[2]));
        PQP_CUDA(cudaEventElapsedTime(&stats->d2h_ms, e->ev[2], e->ev[3]));
        stats->h2d_bytes = h2d;
        stats->d2h_bytes = (int64_t)((size_t)total * sizeof(pqp_station_bounds) + (size_t)batch * sizeof(int32_t));
        stats->kernel_launches = max_n > 0 ? 1 : 0;
    }
    return PQP_OK;
}

// ReferencePathImpl::updateLimits, reference_path_impl.cpp:221-233.  Products and differences are rounded one by one
// (no contraction into fused multiply-adds) so that host, device and the reference's own sequence agree bit for bit.
static __host__ __device__ inline void limits_of(double mu, double rate, double v, double a, double *mk, double *mkp) {
#ifdef __CUDA_ARCH__
    const double ay2 = __dsub_rn(__dmul_rn(mu * 9.8, mu * 9.8), __dmul_rn(a, a));
    const double v2 = __dmul_rn(v, v);
#else
    volatile double t1 = (mu * 9.8) * (mu * 9.8), t2 = a * a;
    const double ay2 = t1 - t2;
    volatile double v2v = v * v;
    const double v2 = v2v;
#endif
    const double ay = sqrt(ay2);
    *mk = (v > 0.0001) ? ay / v2 : 1.7976931348623157e308;
    *mkp = (v > 0.0001) ? rate / v : 1.7976931348623157e308;
}

__global__ void pqp_limits_kernel(double mu, double rate, double kmax, int from_spline, int n, const pqp_state *ref,
                                  double *max_k, double *max_kp) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (from_spline) { max_k[i] = kmax; max_kp[i] = 1.7976931348623157e308; return; }
    limits_of(mu, rate, ref[i].v, ref[i].a, max_k + i, max_kp + i);
}

// The same limits with a parameter set per path (plan chain with a set index): grid (ceil(maxN/128), batch), thread =
// station of path blockIdx.y, looking its row up once.  A path whose set is out of range is skipped (it is not solved).
struct LimitsArgs {
    ParamTable<kSetRows> prm;
    const int32_t *n_points, *offsets;
    const pqp_state *ref;
    double *max_k, *max_kp;
    int first_path;
};
__global__ void __launch_bounds__(128)
pqp_limits_sets_kernel(const __grid_constant__ LimitsArgs a) {
    const int b = a.first_path + blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n_points[b]) return;
    const ParamRow *pr = pqp::param_of(a.prm, b);
    if (!pr) return;
    const int s = a.offsets[b] + i;
    limits_of(pr->mu, pr->rate, a.ref[s].v, a.ref[s].a, a.max_k + s, a.max_kp + s);
}

static int launch_limits_sets(pqp_handle *h, int batch, int max_n, const int32_t *d_n, const int32_t *d_off,
                              const pqp_state *d_ref, SetIndex set, double *d_max_k, double *d_max_kp, cudaStream_t st) {
    LimitsArgs a;
    a.prm = param_table<kSetRows>(h, set.index, set.n_sets);
    a.n_points = d_n; a.offsets = d_off; a.ref = d_ref; a.max_k = d_max_k; a.max_kp = d_max_kp;
    for (int first = 0; max_n > 0 && first < batch; first += 65535) {
        a.first_path = first;
        pqp_limits_sets_kernel<<<dim3((unsigned)((max_n + 127) / 128), (unsigned)std::min(65535, batch - first)), 128, 0, st>>>(a);
        PQP_CUDA(cudaGetLastError());
    }
    return PQP_OK;
}

int pqp_update_limits(const pqp_params *params, int from_spline, int n, const pqp_state *ref, double *max_k, double *max_kp) {
    if (!params || n < 0 || (n > 0 && (!ref || !max_k || !max_kp))) { pqp_set_err("pqp_update_limits: bad argument"); return PQP_ERR_ARG; }
    const double kmax = tan(params->max_steering_angle) / params->wheel_base;
    for (int i = 0; i < n; ++i) {
        if (from_spline) { max_k[i] = kmax; max_kp[i] = 1.7976931348623157e308; }
        else limits_of(params->mu, params->max_curvature_rate, ref[i].v, ref[i].a, max_k + i, max_kp + i);
    }
    return PQP_OK;
}

int pqp_update_limits_device(pqp_handle *h, int from_spline, int n, const pqp_state *d_ref, double *d_max_k, double *d_max_kp,
                             void *stream) {
    if (!h || n < 0 || (n > 0 && (!d_ref || !d_max_k || !d_max_kp))) { pqp_set_err("pqp_update_limits_device: bad argument"); return PQP_ERR_ARG; }
    if (n == 0) return PQP_OK;
    PQP_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
    const double kmax = tan(h->params.max_steering_angle) / h->params.wheel_base;
    pqp_limits_kernel<<<(n + 255) / 256, 256, 0, st>>>(h->params.mu, h->params.max_curvature_rate, kmax, from_spline, n, d_ref,
                                                       d_max_k, d_max_kp);
    PQP_CUDA(cudaGetLastError());
    return PQP_OK;
}

int pqp_check_states(pqp_handle *h, int n, const pqp_state *states, int32_t *ok) {
    if (!h || n < 0 || (n > 0 && (!states || !ok))) { pqp_set_err("pqp_check_states: bad argument"); return PQP_ERR_ARG; }
    EnvState *e;
    int rc = need_map(h, &e);
    if (rc != PQP_OK || n == 0) return rc;
    PQP_CUDA(cudaSetDevice(h->device));
    rc = grow(&e->d_tmp, &e->tmp_cap, (size_t)n * (sizeof(pqp_state) + sizeof(int32_t)));
    if (rc != PQP_OK) return rc;
    pqp_state *d_s = (pqp_state *)e->d_tmp;
    int32_t *d_ok = (int32_t *)(d_s + n);
    cudaStream_t st = h->stream;
    PQP_CUDA(cudaMemcpyAsync(d_s, states, (size_t)n * sizeof(pqp_state), cudaMemcpyHostToDevice, st));
    const CarCircles car = pqp::make_car_circles(h->params);
    pqp_check_states_kernel<<<(n + 127) / 128, 128, 0, st>>>(e->d_maps, car, n, d_s, d_ok);
    PQP_CUDA(cudaGetLastError());
    PQP_CUDA(cudaMemcpyAsync(ok, d_ok, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    PQP_CUDA(cudaStreamSynchronize(st));
    return PQP_OK;
}

int pqp_finish_raw_batch(pqp_handle *h, int batch, const int32_t *n_points, pqp_state *paths, int collision_check,
                         int32_t *out_n_kept, int32_t *out_ok, pqp_stats *stats) {
    if (!h || batch < 0 || (batch > 0 && (!n_points || !paths || !out_n_kept || !out_ok))) {
        pqp_set_err("pqp_finish_raw_batch: bad argument");
        return PQP_ERR_ARG;
    }
    if (stats) memset(stats, 0, sizeof(*stats));
    EnvState *e;
    int rc = collision_check ? need_map(h, &e) : env_get(h, &e);
    if (rc != PQP_OK || batch == 0) return rc;
    PQP_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = h->stream;
    long long total = 0;
    int max_n = 0;
    int64_t h2d = 0;
    PQP_CUDA(cudaEventRecord(e->ev[0], st));
    // the solved paths travel through d_ref and are copied device-side into d_out (the tail's buffer)
    rc = upload_paths(h, e, batch, n_points, paths, PQP_BOUNDS_SIMPLE, nullptr, nullptr, nullptr, nullptr, &total, &max_n, &h2d, st);
    if (rc != PQP_OK) return rc;
    PQP_CUDA(cudaMemcpyAsync(h->d_out, h->d_ref, (size_t)total * sizeof(pqp_state), cudaMemcpyDeviceToDevice, st));
    PQP_CUDA(cudaEventRecord(e->ev[1], st));
    rc = launch_finish_raw(h, e, batch, h->d_n, h->d_off, nullptr, nullptr, kSet0, h->d_out, collision_check, e->d_nkept,
                           e->d_ok, st);
    if (rc != PQP_OK) return rc;
    PQP_CUDA(cudaEventRecord(e->ev[2], st));
    PQP_CUDA(cudaMemcpyAsync(paths, h->d_out, (size_t)total * sizeof(pqp_state), cudaMemcpyDeviceToHost, st));
    PQP_CUDA(cudaMemcpyAsync(out_n_kept, e->d_nkept, (size_t)batch * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    PQP_CUDA(cudaMemcpyAsync(out_ok, e->d_ok, (size_t)batch * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    PQP_CUDA(cudaEventRecord(e->ev[3], st));
    PQP_CUDA(cudaStreamSynchronize(st));
    if (stats) {
        PQP_CUDA(cudaEventElapsedTime(&stats->h2d_ms, e->ev[0], e->ev[1]));
        PQP_CUDA(cudaEventElapsedTime(&stats->kernel_ms, e->ev[1], e->ev[2]));
        PQP_CUDA(cudaEventElapsedTime(&stats->d2h_ms, e->ev[2], e->ev[3]));
        stats->h2d_bytes = h2d;
        stats->d2h_bytes = (int64_t)((size_t)total * sizeof(pqp_state) + (size_t)batch * 2 * sizeof(int32_t));
        stats->kernel_launches = 1;
    }
    return PQP_OK;
}

}  // extern "C"

template <int R>
static int launch_densify_impl(pqp_handle *h, EnvState *e, int batch, const int32_t *d_n, const int32_t *d_off,
                               const int32_t *d_status, const int32_t *d_map_index, SetIndex set, const pqp_state *d_paths,
                               double spacing, int collision_check, int max_out, pqp_state *d_out, int32_t *d_n_out,
                               int32_t *d_ok, cudaStream_t st) {
    DensifyArgs<R> a;
    a.maps = map_table(e, d_map_index); a.prm = param_table<R>(h, set.index, set.n_sets);
    a.n_points = d_n; a.offsets = d_off; a.status = d_status; a.paths = d_paths;
    a.ws = e->d_spl; a.spacing = spacing; a.collision_check = collision_check ? 1 : 0; a.max_out = max_out;
    a.out = d_out; a.n_out = d_n_out; a.ok = d_ok;
    pqp_densify_kernel<R><<<batch, 128, 0, st>>>(a);
    PQP_CUDA(cudaGetLastError());
    return PQP_OK;
}

static int launch_densify(pqp_handle *h, EnvState *e, int batch, const int32_t *d_n, const int32_t *d_off,
                          const int32_t *d_status, const int32_t *d_map_index, SetIndex set, const pqp_state *d_paths,
                          double spacing, int collision_check, int max_out, pqp_state *d_out, int32_t *d_n_out,
                          int32_t *d_ok, cudaStream_t st) {
    return set.index ? launch_densify_impl<kSetRows>(h, e, batch, d_n, d_off, d_status, d_map_index, set, d_paths, spacing,
                                                     collision_check, max_out, d_out, d_n_out, d_ok, st)
                     : launch_densify_impl<1>(h, e, batch, d_n, d_off, d_status, d_map_index, kSet0, d_paths, spacing,
                                              collision_check, max_out, d_out, d_n_out, d_ok, st);
}

extern "C" {

int pqp_densify_batch(pqp_handle *h, int batch, const int32_t *n_points, const pqp_state *paths, double output_spacing,
                      int collision_check, int max_out, pqp_state *out_states, int32_t *out_n, int32_t *out_ok,
                      pqp_stats *stats) {
    if (!h || batch < 0 || max_out < 1 || !(output_spacing > 0.0) ||
        (batch > 0 && (!n_points || !paths || !out_states || !out_n || !out_ok))) {
        pqp_set_err("pqp_densify_batch: bad argument");
        return PQP_ERR_ARG;
    }
    if (stats) memset(stats, 0, sizeof(*stats));
    EnvState *e;
    int rc = collision_check ? need_map(h, &e) : env_get(h, &e);
    if (rc != PQP_OK || batch == 0) return rc;
    PQP_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = h->stream;
    long long total = 0;
    int max_n = 0;
    int64_t h2d = 0;
    PQP_CUDA(cudaEventRecord(e->ev[0], st));
    rc = upload_paths(h, e, batch, n_points, paths, PQP_BOUNDS_SIMPLE, nullptr, nullptr, nullptr, nullptr, &total, &max_n, &h2d, st);
    if (rc != PQP_OK) return rc;
    PQP_CUDA(cudaEventRecord(e->ev[1], st));
    rc = grow(&e->d_dense, &e->dense_cap, (size_t)batch * (size_t)max_out * sizeof(pqp_state));
    if (rc != PQP_OK) return rc;
    rc = launch_densify(h, e, batch, h->d_n, h->d_off, nullptr, nullptr, kSet0, h->d_ref, output_spacing, collision_check,
                        max_out, e->d_dense, e->d_nkept, e->d_ok, st);
    if (rc != PQP_OK) return rc;
    PQP_CUDA(cudaEventRecord(e->ev[2], st));
    PQP_CUDA(cudaMemcpyAsync(out_states, e->d_dense, (size_t)batch * max_out * sizeof(pqp_state), cudaMemcpyDeviceToHost, st));
    PQP_CUDA(cudaMemcpyAsync(out_n, e->d_nkept, (size_t)batch * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    PQP_CUDA(cudaMemcpyAsync(out_ok, e->d_ok, (size_t)batch * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    PQP_CUDA(cudaEventRecord(e->ev[3], st));
    PQP_CUDA(cudaStreamSynchronize(st));
    if (stats) {
        PQP_CUDA(cudaEventElapsedTime(&stats->h2d_ms, e->ev[0], e->ev[1]));
        PQP_CUDA(cudaEventElapsedTime(&stats->kernel_ms, e->ev[1], e->ev[2]));
        PQP_CUDA(cudaEventElapsedTime(&stats->d2h_ms, e->ev[2], e->ev[3]));
        stats->h2d_bytes = h2d;
        stats->d2h_bytes = (int64_t)((size_t)batch * max_out * sizeof(pqp_state) + (size_t)batch * 2 * sizeof(int32_t));
        stats->kernel_launches = 1;
    }
    return PQP_OK;
}

// ---- the plan chain: one body on device pointers, two front ends ---------------------------------------------
// pqp_plan_batch_maps uploads host buffers into the handle's, runs the body and downloads; pqp_plan_batch_device_maps
// runs the body on the caller's device arrays.  pqp_plan_batch and pqp_plan_batch_device are the same with no index.
struct ChainIO {
    int bounds_mode, output_mode, batch;
    int max_n;                      // >= every n_points[b]: sizes the bounds grid
    size_t total;
    PathsView paths;
    const int32_t *map_index;       // [batch] map of every path (bounds and collision check), NULL: map 0
    SetIndex set;                   // parameter set of every path (device index, NULL: set 0) and the sets it may name
    const int32_t *h_set;           // host copy of set.index (host class plan), else NULL
    // formulations: form_mask = the ones a path may name (1 << PQP_FORM_*), max_n_form[f] the longest path of formulation
    // f the device dispatch takes, and the per-path array of the _forms entries: on the host (host class plan) or on the
    // device (device dispatch).  A single-formulation call has a one-bit mask and no array.
    int form_mask = 0;
    int max_n_form[3] = {};
    const int32_t *h_form = nullptr, *d_form = nullptr;
    const double *x0, *end_heading;
    double spacing;
    int collision_check, max_out;
    pqp_state *qp_states;           // [total] QP output; RAW: also the final states (cut, s re-accumulated in place)
    pqp_state *dense;               // DENSIFY: [batch][max_out]
    int32_t *out_n, *out_ok, *status, *iters;
    pqp_station_bounds *bounds;     // [total]
};

// bounds -> (KPC: limits) -> QP on the unblocked prefix -> tail.  The one branch is how the QP step picks kernel
// classes: with `h_ref` (the host copy of the reference states, offsets in h->h_off) the prefix lengths come back to
// the host, one 4-byte-per-path copy and a stream synchronisation; without it the device dispatch picks the same
// classes with no host round trip.  `timed`: e->ev[1..4] mark the stages.
static int run_chain(pqp_handle *h, EnvState *e, const ChainIO &c, const pqp_state *h_ref, bool timed, cudaStream_t st,
                     int *qp_launches) {
    PQP_CUDA(cudaMemsetAsync(c.qp_states, 0, c.total * sizeof(pqp_state), st));   // stations past a cut read as zeros
    if (timed) PQP_CUDA(cudaEventRecord(e->ev[1], st));
    // (1) bounds; n_valid = unblocked prefix of every path
    int rc = launch_bounds_kernel(h, e, c.bounds_mode, c.batch, c.max_n, c.paths, c.map_index, c.set, c.bounds, st);
    if (rc != PQP_OK) return rc;
    if (timed) PQP_CUDA(cudaEventRecord(e->ev[2], st));
    // (2) QP on the unblocked prefix, every path on the kernel class of its own (length, keep_control_steps), exactly
    // as pqp_solve_batch would choose it
    pqp::BatchView bv;
    bv.batch = c.batch; bv.n_points = e->d_nvalid; bv.offsets = c.paths.offsets; bv.ref = c.paths.ref; bv.bounds = c.bounds;
    bv.x0 = c.x0; bv.end_heading = c.end_heading; bv.out_states = c.qp_states; bv.out_frenet = nullptr;
    bv.status = c.status; bv.iters = c.iters; bv.workspace = h->d_ws; bv.debug = nullptr;
    if (pqp::form_in_mask(PQP_FORM_KPC, c.form_mask)) {
        // updateLimits (reference_path_impl.cpp:203-235) between updateBounds and the QP, as solveWithoutSmoothing
        // does (path_optimizer.cpp:100-105): limits from the v, a fields of the reference states.  With per-path
        // formulations every path gets them; only the "KPC" paths read them.
        if (!h->d_max_k) {
            PQP_CUDA(cudaMalloc(&h->d_max_k, (size_t)h->max_total * sizeof(double)));
            PQP_CUDA(cudaMalloc(&h->d_max_kp, (size_t)h->max_total * sizeof(double)));
        }
        if (c.set.index)
            rc = launch_limits_sets(h, c.batch, c.max_n, c.paths.n_points, c.paths.offsets, c.paths.ref, c.set, h->d_max_k,
                                    h->d_max_kp, st);
        else
            rc = pqp_update_limits_device(h, 0, (int)c.total, c.paths.ref, h->d_max_k, h->d_max_kp, st);
        if (rc != PQP_OK) return rc;
        bv.max_k = h->d_max_k; bv.max_kp = h->d_max_kp;
    }
    if (h_ref) {
        std::vector<int32_t> nv((size_t)c.batch);
        PQP_CUDA(cudaMemcpyAsync(nv.data(), e->d_nvalid, (size_t)c.batch * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        PQP_CUDA(cudaStreamSynchronize(st));
        rc = pqp_launch_kp_classes(h, bv, c.batch, nv.data(), h->h_off, h_ref, nullptr, st, qp_launches,
                                   pqp::mask_form(c.form_mask), c.h_set, c.h_form);
    } else {
        rc = pqp_launch_dispatch(h, bv, c.form_mask, c.d_form, c.batch, (int)c.total, c.max_n_form, 0, 0, st, qp_launches,
                                 c.set.index, c.set.n_sets);
    }
    if (rc != PQP_OK) return rc;
    if (timed) PQP_CUDA(cudaEventRecord(e->ev[3], st));
    // (3) tail
    if (c.output_mode == PQP_OUTPUT_RAW) {
        rc = launch_finish_raw(h, e, c.batch, e->d_nvalid, c.paths.offsets, c.status, c.map_index, c.set, c.qp_states,
                               c.collision_check, c.out_n, c.out_ok, st);
    } else {
        rc = launch_densify(h, e, c.batch, e->d_nvalid, c.paths.offsets, c.status, c.map_index, c.set, c.qp_states,
                            c.spacing, c.collision_check, c.max_out, c.dense, c.out_n, c.out_ok, st);
    }
    if (rc != PQP_OK) return rc;
    if (timed) PQP_CUDA(cudaEventRecord(e->ev[4], st));
    return PQP_OK;
}

int pqp_plan_batch_maps(pqp_handle *h, int formulation, int bounds_mode, int output_mode, int batch,
                        const int32_t *n_points, const pqp_state *ref, const int32_t *map_index,
                        const int32_t *n_knots, const double *knots, const double *x_coef, const double *y_coef,
                        const double *x0, const double *end_heading, double output_spacing, int collision_check,
                        int max_out, pqp_state *out_states, int32_t *out_n, int32_t *out_ok, int32_t *status,
                        int32_t *iters, pqp_station_bounds *out_bounds, pqp_stats *stats) {
    return pqp_plan_batch_sets(h, formulation, bounds_mode, output_mode, batch, n_points, ref, map_index, nullptr, n_knots,
                               knots, x_coef, y_coef, x0, end_heading, output_spacing, collision_check, max_out,
                               out_states, out_n, out_ok, status, iters, out_bounds, stats);
}

}  // extern "C"

// The body of pqp_plan_batch_sets (forms NULL) and pqp_plan_batch_forms (forms [batch] on the host); arguments checked
// by the callers.
static int plan_batch_host(pqp_handle *h, int formulation, const int32_t *forms, int bounds_mode, int output_mode,
                           int batch, const int32_t *n_points, const pqp_state *ref, const int32_t *map_index,
                           const int32_t *param_index, const int32_t *n_knots, const double *knots,
                           const double *x_coef, const double *y_coef, const double *x0, const double *end_heading,
                           double output_spacing, int collision_check, int max_out, pqp_state *out_states,
                           int32_t *out_n, int32_t *out_ok, int32_t *status, int32_t *iters,
                           pqp_station_bounds *out_bounds, pqp_stats *stats) {
    if (stats) memset(stats, 0, sizeof(*stats));
    EnvState *e;
    int rc = need_map(h, &e);
    if (rc != PQP_OK || batch == 0) return rc;
    PQP_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = h->stream;
    long long total = 0;
    int max_n = 0;
    int64_t h2d = 0;
    PQP_CUDA(cudaEventRecord(e->ev[0], st));
    rc = upload_paths(h, e, batch, n_points, ref, bounds_mode, n_knots, knots, x_coef, y_coef, &total, &max_n, &h2d, st);
    if (rc != PQP_OK) return rc;
    const size_t B = (size_t)batch, T = (size_t)total;
    PQP_CUDA(cudaMemcpyAsync(h->d_x0, x0, B * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
    PQP_CUDA(cudaMemcpyAsync(h->d_end, end_heading, B * sizeof(double), cudaMemcpyHostToDevice, st));
    h2d += (int64_t)(B * 4 * sizeof(double));
    if (map_index) {
        PQP_CUDA(cudaMemcpyAsync(e->d_mapidx, map_index, B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        h2d += (int64_t)(B * sizeof(int32_t));
    }
    if (param_index) {
        PQP_CUDA(cudaMemcpyAsync(e->d_setidx, param_index, B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        h2d += (int64_t)(B * sizeof(int32_t));
    }
    if (output_mode == PQP_OUTPUT_DENSIFY) {
        rc = grow(&e->d_dense, &e->dense_cap, B * (size_t)max_out * sizeof(pqp_state));
        if (rc != PQP_OK) return rc;
    }
    ChainIO c;
    c.bounds_mode = bounds_mode; c.output_mode = output_mode; c.batch = batch;
    c.max_n = max_n; c.total = T; c.paths = handle_paths(h, e); c.map_index = map_index ? e->d_mapidx : nullptr;
    c.set = param_index ? SetIndex{e->d_setidx, (int)h->sets.size()} : kSet0;
    c.h_set = param_index;
    c.h_form = forms;
    c.form_mask = forms ? 0 : 1 << formulation;
    for (int b = 0; forms && b < batch; ++b)
        if (pqp::form_in_mask(forms[b], 7)) c.form_mask |= 1 << forms[b];
    c.x0 = h->d_x0; c.end_heading = h->d_end;
    c.spacing = output_spacing; c.collision_check = collision_check; c.max_out = max_out;
    c.qp_states = h->d_out; c.dense = e->d_dense; c.out_n = e->d_nkept; c.out_ok = e->d_ok;
    c.status = h->d_status; c.iters = h->d_iters; c.bounds = h->d_bounds;
    int qp_launches = 0;
    rc = run_chain(h, e, c, ref, true, st, &qp_launches);
    if (rc != PQP_OK) return rc;
    int64_t d2h = 0;
    if (output_mode == PQP_OUTPUT_RAW) {
        PQP_CUDA(cudaMemcpyAsync(out_states, h->d_out, T * sizeof(pqp_state), cudaMemcpyDeviceToHost, st));
        d2h += (int64_t)(T * sizeof(pqp_state));
    } else {
        PQP_CUDA(cudaMemcpyAsync(out_states, e->d_dense, B * max_out * sizeof(pqp_state), cudaMemcpyDeviceToHost, st));
        d2h += (int64_t)(B * max_out * sizeof(pqp_state));
    }
    PQP_CUDA(cudaMemcpyAsync(out_n, e->d_nkept, B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    PQP_CUDA(cudaMemcpyAsync(out_ok, e->d_ok, B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    d2h += (int64_t)(B * 2 * sizeof(int32_t));
    std::vector<int32_t> st_local, it_local;
    int32_t *st_dst = status, *it_dst = iters;
    if (!st_dst && stats) { st_local.resize(B); st_dst = st_local.data(); }
    if (!it_dst && stats) { it_local.resize(B); it_dst = it_local.data(); }
    if (st_dst) { PQP_CUDA(cudaMemcpyAsync(st_dst, h->d_status, B * sizeof(int32_t), cudaMemcpyDeviceToHost, st)); d2h += (int64_t)(B * sizeof(int32_t)); }
    if (it_dst) { PQP_CUDA(cudaMemcpyAsync(it_dst, h->d_iters, B * sizeof(int32_t), cudaMemcpyDeviceToHost, st)); d2h += (int64_t)(B * sizeof(int32_t)); }
    if (out_bounds) {
        PQP_CUDA(cudaMemcpyAsync(out_bounds, h->d_bounds, T * sizeof(pqp_station_bounds), cudaMemcpyDeviceToHost, st));
        d2h += (int64_t)(T * sizeof(pqp_station_bounds));
    }
    PQP_CUDA(cudaEventRecord(e->ev[5], st));
    PQP_CUDA(cudaStreamSynchronize(st));
    if (stats) {
        float t_b = 0, t_q = 0, t_t = 0;
        PQP_CUDA(cudaEventElapsedTime(&stats->h2d_ms, e->ev[0], e->ev[1]));
        PQP_CUDA(cudaEventElapsedTime(&t_b, e->ev[1], e->ev[2]));
        PQP_CUDA(cudaEventElapsedTime(&t_q, e->ev[2], e->ev[3]));
        PQP_CUDA(cudaEventElapsedTime(&t_t, e->ev[3], e->ev[4]));
        PQP_CUDA(cudaEventElapsedTime(&stats->d2h_ms, e->ev[4], e->ev[5]));
        stats->kernel_ms = t_b + t_q + t_t;
        stats->h2d_bytes = h2d;
        stats->d2h_bytes = d2h;
        stats->kernel_launches = 2 + qp_launches;
        for (size_t b = 0; b < B; ++b) {
            stats->total_iters += it_dst[b];
            stats->max_iters = std::max(stats->max_iters, it_dst[b]);
            stats->n_solved += (st_dst[b] == PQP_SOLVED);
        }
    }
    return PQP_OK;
}

static bool plan_args_ok(int bounds_mode, int output_mode, double output_spacing, int max_out) {
    return (bounds_mode == PQP_BOUNDS_IMPROVED || bounds_mode == PQP_BOUNDS_SIMPLE) &&
           (output_mode == PQP_OUTPUT_RAW || output_mode == PQP_OUTPUT_DENSIFY) &&
           (output_mode != PQP_OUTPUT_DENSIFY || (max_out >= 1 && output_spacing > 0.0));
}

extern "C" {

int pqp_plan_batch_sets(pqp_handle *h, int formulation, int bounds_mode, int output_mode, int batch,
                        const int32_t *n_points, const pqp_state *ref, const int32_t *map_index,
                        const int32_t *param_index, const int32_t *n_knots, const double *knots, const double *x_coef,
                        const double *y_coef, const double *x0, const double *end_heading, double output_spacing,
                        int collision_check, int max_out, pqp_state *out_states, int32_t *out_n, int32_t *out_ok,
                        int32_t *status, int32_t *iters, pqp_station_bounds *out_bounds, pqp_stats *stats) {
    if (!h || batch < 0 || (batch > 0 && (!n_points || !ref || !x0 || !end_heading || !out_states || !out_n || !out_ok)) ||
        !plan_args_ok(bounds_mode, output_mode, output_spacing, max_out)) {
        pqp_set_err("pqp_plan_batch(_maps, _sets): bad argument");
        return PQP_ERR_ARG;
    }
    if (formulation != PQP_FORM_KP && formulation != PQP_FORM_KPC && formulation != PQP_FORM_K) {
        pqp_set_err("pqp_plan_batch(_maps, _sets): unknown formulation");
        return PQP_ERR_ARG;
    }
    return plan_batch_host(h, formulation, nullptr, bounds_mode, output_mode, batch, n_points, ref, map_index,
                           param_index, n_knots, knots, x_coef, y_coef, x0, end_heading, output_spacing,
                           collision_check, max_out, out_states, out_n, out_ok, status, iters, out_bounds, stats);
}

int pqp_plan_batch_forms(pqp_handle *h, int bounds_mode, int output_mode, int batch, const int32_t *n_points,
                         const pqp_state *ref, const int32_t *map_index, const int32_t *param_index,
                         const int32_t *formulation, const int32_t *n_knots, const double *knots,
                         const double *x_coef, const double *y_coef, const double *x0, const double *end_heading,
                         double output_spacing, int collision_check, int max_out, pqp_state *out_states,
                         int32_t *out_n, int32_t *out_ok, int32_t *status, int32_t *iters,
                         pqp_station_bounds *out_bounds, pqp_stats *stats) {
    if (!h || batch < 0 ||
        (batch > 0 && (!n_points || !ref || !formulation || !x0 || !end_heading || !out_states || !out_n || !out_ok)) ||
        !plan_args_ok(bounds_mode, output_mode, output_spacing, max_out)) {
        pqp_set_err("pqp_plan_batch_forms: bad argument");
        return PQP_ERR_ARG;
    }
    return plan_batch_host(h, PQP_FORM_KP, formulation, bounds_mode, output_mode, batch, n_points, ref, map_index,
                           param_index, n_knots, knots, x_coef, y_coef, x0, end_heading, output_spacing,
                           collision_check, max_out, out_states, out_n, out_ok, status, iters, out_bounds, stats);
}

int pqp_plan_batch(pqp_handle *h, int formulation, int bounds_mode, int output_mode, int batch, const int32_t *n_points,
                   const pqp_state *ref, const int32_t *n_knots, const double *knots, const double *x_coef,
                   const double *y_coef, const double *x0, const double *end_heading, double output_spacing,
                   int collision_check, int max_out, pqp_state *out_states, int32_t *out_n, int32_t *out_ok,
                   int32_t *status, int32_t *iters, pqp_station_bounds *out_bounds, pqp_stats *stats) {
    return pqp_plan_batch_maps(h, formulation, bounds_mode, output_mode, batch, n_points, ref, nullptr, n_knots, knots,
                               x_coef, y_coef, x0, end_heading, output_spacing, collision_check, max_out, out_states,
                               out_n, out_ok, status, iters, out_bounds, stats);
}

int pqp_plan_batch_device_maps(pqp_handle *h, int formulation, int bounds_mode, int output_mode, int batch,
                               int total_points, int max_n_points, const int32_t *d_n_points, const int32_t *d_offsets,
                               const pqp_state *d_ref, const int32_t *d_map_index, const int32_t *d_knot_offsets,
                               const double *d_knots, const double *d_x_coef, const double *d_y_coef,
                               const double *d_x0, const double *d_end_heading, double output_spacing,
                               int collision_check, int max_out, pqp_state *d_out_states, int32_t *d_out_n,
                               int32_t *d_out_ok, int32_t *d_status, int32_t *d_iters,
                               pqp_station_bounds *d_out_bounds, void *stream, pqp_stats *stats) {
    return pqp_plan_batch_device_sets(h, formulation, bounds_mode, output_mode, batch, total_points, max_n_points, 0,
                                      d_n_points, d_offsets, d_ref, d_map_index, nullptr, d_knot_offsets, d_knots,
                                      d_x_coef, d_y_coef, d_x0, d_end_heading, output_spacing, collision_check, max_out,
                                      d_out_states, d_out_n, d_out_ok, d_status, d_iters, d_out_bounds, stream, stats);
}

}  // extern "C"

// The body of pqp_plan_batch_device_sets (a one-bit form_mask, d_form NULL) and pqp_plan_batch_device_forms (d_form
// [batch] on the device, form_mask nonzero); arguments checked by the callers.
static int plan_batch_device(pqp_handle *h, int form_mask, const int32_t *d_form, int bounds_mode,
                             int output_mode, int batch, int total_points, int max_n_points, int n_param_sets,
                             const int32_t *d_n_points, const int32_t *d_offsets, const pqp_state *d_ref,
                             const int32_t *d_map_index, const int32_t *d_param_index, const int32_t *d_knot_offsets,
                             const double *d_knots, const double *d_x_coef, const double *d_y_coef,
                             const double *d_x0, const double *d_end_heading, double output_spacing,
                             int collision_check, int max_out, pqp_state *d_out_states, int32_t *d_out_n,
                             int32_t *d_out_ok, int32_t *d_status, int32_t *d_iters,
                             pqp_station_bounds *d_out_bounds, void *stream, pqp_stats *stats) {
    if (stats) memset(stats, 0, sizeof(*stats));
    EnvState *e;
    int rc = need_map(h, &e);
    if (rc != PQP_OK || batch == 0) return rc;
    if (batch > h->max_batch || total_points > h->max_total) {
        pqp_set_err("batch / total_points exceed what the handle was created for (workspace size)");
        return PQP_ERR_CAPACITY;
    }
    PQP_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
    ChainIO c;
    c.bounds_mode = bounds_mode; c.output_mode = output_mode; c.batch = batch;
    // every formulation bounded by max_n_points (0: the longest path any of its classes takes; a longer one reports
    // PQP_INVALID_PROBLEM); the bounds grid covers the longest bound of the mask
    c.form_mask = form_mask; c.d_form = d_form; c.max_n = 0;
    for (int f : {PQP_FORM_KP, PQP_FORM_K, PQP_FORM_KPC}) {
        c.max_n_form[f] = max_n_points > 0 ? max_n_points : h->cls_ncols[f] - 2;
        if (pqp::form_in_mask(f, form_mask)) c.max_n = std::max(c.max_n, c.max_n_form[f]);
    }
    c.total = (size_t)total_points;
    c.paths = PathsView{d_n_points, d_offsets, d_ref, d_knot_offsets, d_knots, d_x_coef, d_y_coef};
    c.map_index = d_map_index;
    const int n_sets = (int)h->sets.size();
    c.set = d_param_index ? SetIndex{d_param_index, n_param_sets > 0 ? std::min(n_param_sets, n_sets) : n_sets} : kSet0;
    c.h_set = nullptr;
    c.x0 = d_x0; c.end_heading = d_end_heading;
    c.spacing = output_spacing; c.collision_check = collision_check; c.max_out = max_out;
    c.qp_states = output_mode == PQP_OUTPUT_RAW ? d_out_states : h->d_out;
    c.dense = d_out_states; c.out_n = d_out_n; c.out_ok = d_out_ok;
    c.status = d_status; c.iters = d_iters ? d_iters : h->d_iters; c.bounds = d_out_bounds ? d_out_bounds : h->d_bounds;
    if (stats) PQP_CUDA(cudaEventRecord(e->ev[0], st));
    int qp_launches = 0;
    rc = run_chain(h, e, c, nullptr, stats != nullptr, st, &qp_launches);
    if (rc != PQP_OK) return rc;
    if (stats) {
        float t_b = 0, t_q = 0, t_t = 0;
        PQP_CUDA(cudaEventSynchronize(e->ev[4]));
        PQP_CUDA(cudaEventElapsedTime(&t_b, e->ev[1], e->ev[2]));
        PQP_CUDA(cudaEventElapsedTime(&t_q, e->ev[2], e->ev[3]));
        PQP_CUDA(cudaEventElapsedTime(&t_t, e->ev[3], e->ev[4]));
        stats->kernel_ms = t_b + t_q + t_t;
        stats->kernel_launches = 2 + qp_launches;
    }
    return PQP_OK;
}

static bool plan_device_args_ok(int bounds_mode, int output_mode, int batch, const int32_t *d_knot_offsets,
                                const double *d_knots, const double *d_x_coef, const double *d_y_coef,
                                double output_spacing, int max_out) {
    return plan_args_ok(bounds_mode, output_mode, output_spacing, max_out) &&
           !(bounds_mode == PQP_BOUNDS_IMPROVED && batch > 0 && (!d_knot_offsets || !d_knots || !d_x_coef || !d_y_coef));
}

extern "C" {

int pqp_plan_batch_device_sets(pqp_handle *h, int formulation, int bounds_mode, int output_mode, int batch,
                               int total_points, int max_n_points, int n_param_sets, const int32_t *d_n_points,
                               const int32_t *d_offsets, const pqp_state *d_ref, const int32_t *d_map_index,
                               const int32_t *d_param_index, const int32_t *d_knot_offsets, const double *d_knots,
                               const double *d_x_coef, const double *d_y_coef, const double *d_x0,
                               const double *d_end_heading, double output_spacing, int collision_check, int max_out,
                               pqp_state *d_out_states, int32_t *d_out_n, int32_t *d_out_ok, int32_t *d_status,
                               int32_t *d_iters, pqp_station_bounds *d_out_bounds, void *stream, pqp_stats *stats) {
    if (!h || batch < 0 || total_points < 0 || n_param_sets < 0 ||
        (batch > 0 && (!d_n_points || !d_offsets || !d_ref || !d_x0 || !d_end_heading || !d_out_states || !d_out_n ||
                       !d_out_ok || !d_status)) ||
        !plan_device_args_ok(bounds_mode, output_mode, batch, d_knot_offsets, d_knots, d_x_coef, d_y_coef,
                             output_spacing, max_out)) {
        pqp_set_err("pqp_plan_batch_device(_maps, _sets): bad argument");
        return PQP_ERR_ARG;
    }
    if (formulation != PQP_FORM_KP && formulation != PQP_FORM_KPC && formulation != PQP_FORM_K) {
        pqp_set_err("pqp_plan_batch_device(_maps, _sets): unknown formulation");
        return PQP_ERR_ARG;
    }
    return plan_batch_device(h, 1 << formulation, nullptr, bounds_mode, output_mode, batch, total_points, max_n_points,
                             n_param_sets, d_n_points, d_offsets, d_ref, d_map_index, d_param_index, d_knot_offsets,
                             d_knots, d_x_coef, d_y_coef, d_x0, d_end_heading, output_spacing, collision_check, max_out,
                             d_out_states, d_out_n, d_out_ok, d_status, d_iters, d_out_bounds, stream, stats);
}

int pqp_plan_batch_device_forms(pqp_handle *h, int bounds_mode, int output_mode, int batch, int total_points,
                                int max_n_points, int n_param_sets, int form_mask, const int32_t *d_n_points,
                                const int32_t *d_offsets, const pqp_state *d_ref, const int32_t *d_map_index,
                                const int32_t *d_param_index, const int32_t *d_formulation,
                                const int32_t *d_knot_offsets, const double *d_knots, const double *d_x_coef,
                                const double *d_y_coef, const double *d_x0, const double *d_end_heading,
                                double output_spacing, int collision_check, int max_out, pqp_state *d_out_states,
                                int32_t *d_out_n, int32_t *d_out_ok, int32_t *d_status, int32_t *d_iters,
                                pqp_station_bounds *d_out_bounds, void *stream, pqp_stats *stats) {
    if (!h || batch < 0 || total_points < 0 || n_param_sets < 0 || form_mask < 0 || form_mask > 7 ||
        (batch > 0 && (!d_n_points || !d_offsets || !d_ref || !d_formulation || !d_x0 || !d_end_heading ||
                       !d_out_states || !d_out_n || !d_out_ok || !d_status)) ||
        !plan_device_args_ok(bounds_mode, output_mode, batch, d_knot_offsets, d_knots, d_x_coef, d_y_coef,
                             output_spacing, max_out)) {
        pqp_set_err("pqp_plan_batch_device_forms: bad argument");
        return PQP_ERR_ARG;
    }
    return plan_batch_device(h, form_mask ? form_mask : 7, d_formulation, bounds_mode, output_mode, batch,
                             total_points, max_n_points, n_param_sets, d_n_points, d_offsets, d_ref, d_map_index,
                             d_param_index, d_knot_offsets, d_knots, d_x_coef, d_y_coef, d_x0, d_end_heading,
                             output_spacing, collision_check, max_out, d_out_states, d_out_n, d_out_ok, d_status,
                             d_iters, d_out_bounds, stream, stats);
}

int pqp_plan_batch_device(pqp_handle *h, int formulation, int bounds_mode, int output_mode, int batch, int total_points,
                          int max_n_points, const int32_t *d_n_points, const int32_t *d_offsets, const pqp_state *d_ref,
                          const int32_t *d_knot_offsets, const double *d_knots, const double *d_x_coef,
                          const double *d_y_coef, const double *d_x0, const double *d_end_heading, double output_spacing,
                          int collision_check, int max_out, pqp_state *d_out_states, int32_t *d_out_n, int32_t *d_out_ok,
                          int32_t *d_status, int32_t *d_iters, pqp_station_bounds *d_out_bounds, void *stream,
                          pqp_stats *stats) {
    return pqp_plan_batch_device_maps(h, formulation, bounds_mode, output_mode, batch, total_points, max_n_points,
                                      d_n_points, d_offsets, d_ref, nullptr, d_knot_offsets, d_knots, d_x_coef,
                                      d_y_coef, d_x0, d_end_heading, output_spacing, collision_check, max_out,
                                      d_out_states, d_out_n, d_out_ok, d_status, d_iters, d_out_bounds, stream, stats);
}

}  // extern "C"
