// pqp_capi.cu -- extern "C" boundary of libpqp.so (declared in include/pqp.h) and the kernel
// launchers.  Host orchestration only: all numerics run in the sm_90a kernels; there is no CPU
// fallback (pqp_create fails when no CUDA device / kernel image is usable).
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <new>
#include <vector>

#include "pqp_dispatch.h"
#include "pqp_kernels.h"
#include "pqp_kp_core3.cuh"
#include "pqp_gen_core.cuh"
#include "pqp_forms.h"
#include "pqp_handle.h"
#include <thread>

thread_local char pqp_g_err[512] = "";

namespace {

#define set_err pqp_set_err
#define g_err pqp_g_err

// Shape classes, in order of preference (the records come from the kernels' own translation units, pqp_kernels.h).
// keep_control_steps <= 4 (station spacing >= 0.24 m) and up to 408 stations map onto one of the thread-per-station
// (Kp3) instantiations; anything else runs on the one-warp generic kernel (last).
typedef PqpVariant Variant;
constexpr int kNumKp = 9;          // "KP" classes: thread-per-station kernels, then the one-warp kernel (index kNumKp - 1)
constexpr int kNumKpc = 12;        // + the "KPC" thread-per-station classes [kNumKp, kNumKpc)
constexpr int kNumVariants = 15;   // + the "K" thread-per-station classes [kNumKpc, kNumVariants) (pqp_kk_core.cuh)
struct VariantTable {
    Variant v[kNumVariants];
    VariantTable() {
        int k = 0;
        pqp_variant_k3_17_6_4_17(&v[k++]); pqp_variant_k3_23_7_4_17(&v[k++]);
        pqp_variant_k3_17_6_8_34(&v[k++]); pqp_variant_k3_23_7_8_34(&v[k++]); pqp_variant_k3_27_7_8_34(&v[k++]);
        pqp_variant_k3_27_7_10_34(&v[k++]); pqp_variant_k3_37_7_12_34(&v[k++]); pqp_variant_k3_37_7_13_34(&v[k++]);
        pqp_variant_k1_generic(&v[k++]);
        pqp_variant_k3c_13_7_8_34(&v[k++]); pqp_variant_k3c_23_7_4_17(&v[k++]); pqp_variant_k3c_23_7_8_34(&v[k++]);
        pqp_variant_kk_4(&v[k++]); pqp_variant_kk_8(&v[k++]); pqp_variant_kk_13(&v[k++]);
    }
};
const Variant *variants() {
    static const VariantTable t;
    return t.v;
}
#define kVariants (variants())
constexpr int kMaxChunks = PQP_MAX_CHUNKS;   // host-buffer entry point: pipelined chunks per call

// PQP_SKIP_VARIANTS=<bitmask> (diagnostics only): leave shape classes out of the selection, e.g. to time a
// fallback kernel on a batch the preferred class would take.
unsigned skip_mask() {
    static const unsigned m = [] { const char *e = getenv("PQP_SKIP_VARIANTS"); return e ? (unsigned)strtoul(e, nullptr, 0) : 0u; }();
    return m;
}

// classes of a formulation: [v0, v1) of the table
void form_range(int form, int *v0, int *v1) {
    *v0 = form == PQP_FORM_KPC ? kNumKp : form == PQP_FORM_K ? kNumKpc : 0;
    *v1 = form == PQP_FORM_KPC ? kNumKpc : form == PQP_FORM_K ? kNumVariants : kNumKp;
}

int pick_variant(int n, int keep, int form = PQP_FORM_KP) {
    int v0, v1;
    form_range(form, &v0, &v1);
    for (int v = v0; v < v1; ++v)
        if (!((skip_mask() >> v) & 1u) && kVariants[v].fits(n, keep)) return v;
    return -1;
}

// Kernel class and shared-memory need of ONE path of n stations at keep_control_steps = keep, exactly as every entry
// point that sees the lengths on the host selects it: the first class that takes (n, keep); when that class needs more
// shared memory than the device offers, the one-warp kernel if the path fits there; else the smallest launch of the
// one-warp kernel, which reports PQP_INVALID_PROBLEM for the path.  Returns false in that last case.
// "KPC" has thread-per-station classes only (up to 256 stations, more than the host-assembled generic kernel can hold in
// one SM): a longer path is launched on the last class with the smallest shared-memory size, where the kernel's own shape
// check reports PQP_INVALID_PROBLEM for it.  Returns false in that case.
bool class_for(const pqp_handle *h, int n, int keep, int *v_out, size_t *need_out, int form = PQP_FORM_KP) {
    if (form == PQP_FORM_KPC || form == PQP_FORM_K) {
        const int fk = form == PQP_FORM_KPC ? 4 : 1;
        const int pv = n >= 2 ? pick_variant(n, fk, form) : -1;
        if (pv >= 0 && kVariants[pv].smem(n, fk) <= (size_t)h->smem_optin) {
            *v_out = pv;
            *need_out = kVariants[pv].smem(n, fk);
            return true;
        }
        int v0, v1;
        form_range(form, &v0, &v1);
        *v_out = v1 - 1;
        *need_out = kVariants[v1 - 1].smem(2, fk);
        return false;
    }
    int v = kNumKp - 1;
    if (n >= 2) {
        const int pv = pick_variant(n, keep);
        if (pv >= 0) v = pv;
    }
    const int ke = std::min(std::max(keep, 1), 10), ne = std::max(n, 2);
    size_t need = kVariants[v].smem(ne, ke);
    bool ok = n >= 2 && keep >= 1 && keep <= 10;
    if (need > (size_t)h->smem_optin) {
        v = kNumKp - 1;
        need = (keep <= 10) ? kVariants[v].smem(ne, ke) : (size_t)h->smem_optin + 1;
        if (need > (size_t)h->smem_optin) { need = kVariants[v].smem(2, 1); ok = false; }
    }
    *v_out = v;
    *need_out = need;
    return ok;
}

// The class table of one formulation (pqp_dispatch.h), filled by class_for itself: entry [keep - 1][n] for keep 1..10
// and one row for keep > 10, n = 0 .. one station past the longest path any class takes (a column every longer path
// shares: class_for gives all of them the same invalid slot).  Returns the number of columns.
constexpr int kTableScanN = 4096;   // (pqp_max_points_keep scans as far)
int class_table(const pqp_handle *h, int form, std::vector<int8_t> *tab) {
    int longest = 0, v;
    size_t need;
    for (int keep = 1; keep <= 10; ++keep)
        for (int n = 2; n <= kTableScanN; ++n)
            if (class_for(h, n, keep, &v, &need, form)) longest = std::max(longest, n);
    const int ncols = longest + 2;
    tab->assign((size_t)pqp::kTableKeepRows * ncols, 0);
    for (int r = 0; r < pqp::kTableKeepRows; ++r)
        for (int n = 0; n < ncols; ++n) {
            class_for(h, n, r + 1, &v, &need, form);
            (*tab)[(size_t)r * ncols + n] = (int8_t)v;
        }
    return ncols;
}

// One class for a whole device-resident batch of which the host only knows bounds: it must take EVERY (n, keep) with
// 2 <= n <= nmax, k_lo <= keep <= k_hi (neither fits() nor the shared-memory need is monotone in n: the separator and
// interior counts change with it), and is launched with the largest shared-memory need over that range.
bool device_class(pqp_handle *h, int nmax, int k_lo, int k_hi, int *v_out, size_t *smem_out, int form = PQP_FORM_KP) {
    if (form == PQP_FORM_KPC) k_lo = k_hi = 4;
    if (form == PQP_FORM_K) k_lo = k_hi = 1;
    if (h->dc_nmax == nmax && h->dc_klo == k_lo && h->dc_khi == k_hi && h->dc_skip == (int)skip_mask() && h->dc_form == form) {
        *v_out = h->dc_v; *smem_out = h->dc_smem;
        return h->dc_v >= 0;
    }
    int v = -1;
    size_t smem = 0;
    int c0, c1;
    form_range(form, &c0, &c1);
    for (int cand = c0; cand < c1 && v < 0; ++cand) {
        if ((skip_mask() >> cand) & 1u) continue;
        bool all = true;
        size_t need = 0;
        for (int k = k_lo; k <= k_hi && all; ++k)
            for (int n = 2; n <= nmax && all; ++n) {
                if (!kVariants[cand].fits(n, k)) all = false;
                else need = std::max(need, kVariants[cand].smem(n, k));
            }
        if (all && need <= (size_t)h->smem_optin) { v = cand; smem = need; }
    }
    h->dc_nmax = nmax; h->dc_klo = k_lo; h->dc_khi = k_hi; h->dc_skip = (int)skip_mask(); h->dc_v = v; h->dc_smem = smem;
    h->dc_form = form;
    *v_out = v; *smem_out = smem;
    return v >= 0;
}

}  // namespace


// ---- launch order from the inputs ------------------------------------------------------------------------------
// A launch of a few paths per resident CTA slot ends with a tail set by the paths that happen to start last.  Paths that
// start far from the corridor centre relative to its width tend to need more ADMM iterations (correlation 0.3-0.4 on the
// BASELINE corridors: weak, but enough to keep the long ones out of the last wave), so small batches are launched in the
// order of  stations x (1 + min(|e_y0| / w, 2)),  largest first.  Results do not depend on the order.
constexpr int kAutoOrderMax = 2048;    // beyond ~7 paths per slot the tail is a few per cent: index order
PQP_HD double order_key(int n, double ey0, double lb, double ub) {
    const double w = 0.5 * (ub - lb);
    double sc = fabs(ey0) / (w > 1e-3 ? w : 1e-3);
    if (!(sc == sc)) sc = 0.0;
    if (sc > 2.0) sc = 2.0;
    return (double)n * (1.0 + sc);
}
__global__ void __launch_bounds__(1024)
pqp_order_kernel(const int32_t *__restrict__ n_points, const int32_t *__restrict__ offsets, const pqp_station_bounds *__restrict__ bounds,
                 const double *__restrict__ x0, int batch, int32_t *__restrict__ order) {
    __shared__ double key[kAutoOrderMax];
    for (int b = threadIdx.x; b < batch; b += blockDim.x) {
        const int n = n_points[b];
        double k = 0.0;
        if (n >= 1) {
            const pqp_station_bounds bb = bounds[offsets[b]];
            k = order_key(n, x0[3 * (size_t)b], bb.c0_lb, bb.c0_ub);
        }
        key[b] = k;
    }
    __syncthreads();
    for (int b = threadIdx.x; b < batch; b += blockDim.x) {
        const double kb = key[b];
        int rank = 0;
        for (int j = 0; j < batch; ++j) {
            const double kj = key[j];
            rank += (kj > kb) || (kj == kb && j < b);
        }
        order[rank] = b;
    }
}
bool auto_order_enabled() {
    static const bool on = [] { const char *e = getenv("PQP_NO_AUTO_ORDER"); return !(e && *e == '1'); }();
    return on;
}

extern "C" {
static int launch_variant(pqp_handle *h, int v, const pqp::DevParams *prm, const pqp::BatchView &bv, int count,
                          const int32_t *d_order, size_t smem_bytes, cudaStream_t st);
}

// What a kernel writes into the stations of a path it cannot take (with PQP_INVALID_PROBLEM and 0 iterations): NaN
// states, v = a = 0, NaN Frenet states.  Stations i0, i0 + step, ... of the n at `off`.
__device__ __forceinline__ void write_invalid(pqp_state *out_states, double *out_frenet, int off, int n, int i0,
                                              int step) {
    const double qnan = nan("");
    for (int i = i0; i < n; i += step) {
        pqp_state &o = out_states[off + i];
        o.x = o.y = o.z = o.k = o.s = qnan;
        o.v = o.a = 0.0;
        if (out_frenet) {
            double *f = out_frenet + 3 * (size_t)(off + i);
            f[0] = f[1] = f[2] = qnan;
        }
    }
}

// Paths a host plan does not launch because their parameter set is out of range: one CTA per order entry writes what a
// kernel writes for a path it cannot take (PQP_INVALID_PROBLEM, 0 iterations, NaN states).
__global__ void __launch_bounds__(128)
pqp_reject_kernel(const __grid_constant__ pqp::BatchView bv, const int32_t *__restrict__ order) {
    const int b = order[blockIdx.x];
    if (threadIdx.x == 0) {
        bv.status[b] = PQP_INVALID_PROBLEM;
        if (bv.iters) bv.iters[b] = 0;
    }
    write_invalid(bv.out_states, bv.out_frenet, bv.offsets[b], bv.n_points[b], threadIdx.x, blockDim.x);
}

// One launch per (set, class) segment g = set * kNumVariants + v with count[g] > 0: count[g] CTAs over the order entries
// d_order + start[g], with smem[g] bytes and set `set`'s parameters.  A mixed batch has several: they go out on the
// handle's class lanes (forked from and joined back into `st`), the class of the longest paths first (and inside a class
// the sets in order), so that the CTAs of the next segment fill the SMs the tail of the previous one leaves idle instead
// of waiting for its last path.  n_reject > 0: the order entries d_order + reject_start name paths to reject.
static int launch_class_set(pqp_handle *h, const pqp::BatchView &bv, int n_sets, const int *count, const int *start,
                            const size_t *smem, const int32_t *d_order, cudaStream_t st, int *launches,
                            int n_reject = 0, int reject_start = 0) {
    int n_cls = n_reject > 0;
    for (int g = 0; g < n_sets * kNumVariants; ++g) n_cls += count[g] > 0;
    const bool fork = n_cls > 1;
    if (fork) PQP_CUDA(cudaEventRecord(h->ev_fork, st));
    int lane = 0, rc = PQP_OK;
    for (int v = kNumVariants - 1; v >= 0 && rc == PQP_OK; --v)
        for (int s = 0; s < n_sets && rc == PQP_OK; ++s) {
            const int g = s * kNumVariants + v;
            if (!count[g]) continue;
            cudaStream_t cs = st;
            if (fork) {
                cs = h->cls_stream[lane % PQP_CLASS_LANES];
                if (lane < PQP_CLASS_LANES) PQP_CUDA(cudaStreamWaitEvent(cs, h->ev_fork, 0));
                ++lane;
            }
            rc = launch_variant(h, v, &h->dsets[s], bv, count[g], d_order + start[g], smem[g], cs);
            if (rc == PQP_OK && launches) ++*launches;
        }
    if (rc == PQP_OK && n_reject > 0) {
        cudaStream_t cs = st;
        if (fork) {
            cs = h->cls_stream[lane % PQP_CLASS_LANES];
            if (lane < PQP_CLASS_LANES) PQP_CUDA(cudaStreamWaitEvent(cs, h->ev_fork, 0));
            ++lane;
        }
        pqp_reject_kernel<<<n_reject, 128, 0, cs>>>(bv, d_order + reject_start);
        if (cudaGetLastError() != cudaSuccess) { set_err("pqp_reject_kernel launch failed"); rc = PQP_ERR_CUDA; }
        else if (launches) ++*launches;
    }
    if (fork)   // join every lane that was used, also after a failed launch: `st` must not run ahead of them
        for (int k = 0; k < std::min(lane, PQP_CLASS_LANES); ++k) {
            PQP_CUDA(cudaEventRecord(h->ev_cls[k], h->cls_stream[k]));
            PQP_CUDA(cudaStreamWaitEvent(st, h->ev_cls[k], 0));
        }
    return rc;
}

// The host class plan of the paths [b0, b1): every path's segment g = set * kNumVariants + class (class_for on its
// length, keep and formulation; `set` / `forms` NULL: set 0 / `form` for every path), or segment G = n_sets *
// kNumVariants when its set lies outside [0, n_sets) or its formulation is none (rejected, not launched).  Fills
// count[0, G], start[0, G + 1] (start[0] = b0), smem[0, G] and h->h_order[b0, b1): the segments in turn, each stably
// sorted longest EXPECTED WORK first with a hint (pqp_set_order_hint: stations x expected iterations), else by `before`.
template <class Before>
static void plan_classes(pqp_handle *h, int batch, int b0, int b1, int n_sets, const int32_t *n, const int32_t *keep,
                         int form, const int32_t *forms, const int32_t *set, Before before, int *count, int *start,
                         size_t *smem) {
    const int G = n_sets * kNumVariants;
    std::vector<int> seg((size_t)(b1 - b0));
    std::fill(count, count + G + 1, 0);
    std::fill(smem, smem + G + 1, 0);
    for (int b = b0; b < b1; ++b) {
        const int s = set ? set[b] : 0;
        const int f = forms ? forms[b] : form;
        int &g = seg[b - b0];
        if (s < 0 || s >= n_sets || (forms && !pqp::form_in_mask(f, 7))) { g = G; count[G]++; continue; }
        int v;
        size_t need;
        class_for(h, n[b], keep[b], &v, &need, f);
        g = s * kNumVariants + v;
        smem[g] = std::max(smem[g], need);
        count[g]++;
    }
    start[0] = b0;
    for (int g = 0; g <= G; ++g) start[g + 1] = start[g] + count[g];
    std::vector<int> fill(start, start + G + 1);
    for (int b = b0; b < b1; ++b) h->h_order[fill[seg[b - b0]]++] = b;
    const bool hinted = h->order_hint.size() == (size_t)batch;
    const int32_t *hint = h->order_hint.data();
    for (int g = 0; g < G; ++g)
        std::stable_sort(h->h_order + start[g], h->h_order + start[g + 1], [&](int a, int b) {
            if (hinted) return (long long)n[a] * hint[a] > (long long)n[b] * hint[b];
            return before(a, b);
        });
}

int pqp_launch_kp_classes(pqp_handle *h, const pqp::BatchView &bv, int batch, const int32_t *n, const int32_t *off,
                          const pqp_state *ref, const int32_t *keep_in, cudaStream_t st, int *launches, int form,
                          const int32_t *set, const int32_t *forms) {
    static_assert(kNumVariants <= PQP_MAX_VARIANTS, "class plan arrays");
    // keep_control_steps per path
    std::vector<int32_t> keepv((size_t)batch);
    for (int b = 0; b < batch; ++b) {
        const int f = forms ? forms[b] : form;
        keepv[b] = f == PQP_FORM_KPC ? 4 : f == PQP_FORM_K ? 1 : keep_in ? keep_in[b] : (n[b] >= 2 ? pqp_keep_control_steps(PQP_FORM_KP, ref + off[b], n[b]) : 1);
    }
    const int n_sets = set ? (int)h->dsets.size() : 1;
    const int G = n_sets * kNumVariants;   // segment G: the rejected paths
    // The plan (segment per path, longest-first order inside a segment) only depends on (n, keep, set, formulation): a
    // caller that solves batches of the same shape back to back reuses it, and the order array already on the device
    // with it.
    pqp_handle::ClassPlan &pl = h->plan;
    const bool same = pl.valid && pl.form == form && pl.skip == (int)skip_mask() && pl.n.size() == (size_t)batch &&
                      std::equal(pl.n.begin(), pl.n.end(), n) && pl.keep == keepv && pl.n_sets == n_sets &&
                      (set ? pl.set.size() == (size_t)batch && std::equal(pl.set.begin(), pl.set.end(), set) : pl.set.empty()) &&
                      (forms ? pl.forms.size() == (size_t)batch && std::equal(pl.forms.begin(), pl.forms.end(), forms) : pl.forms.empty());
    if (!same) {
        // the pinned order array may still be the source of an earlier asynchronous upload
        PQP_CUDA(cudaStreamSynchronize(st));
        if (pl.stream && pl.stream != st) PQP_CUDA(cudaStreamSynchronize(pl.stream));
        pl.valid = false;
        pl.count.resize((size_t)G + 1);
        pl.start.resize((size_t)G + 2);
        pl.smem.resize((size_t)G + 1);
        auto longest = [&](int a, int b) { return n[a] > n[b]; };
        plan_classes(h, batch, 0, batch, n_sets, n, keepv.data(), form, forms, set, longest, pl.count.data(),
                     pl.start.data(), pl.smem.data());
        PQP_CUDA(cudaMemcpyAsync(h->d_order, h->h_order, (size_t)batch * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        pl.n.assign(n, n + batch);
        pl.keep = keepv;
        if (set) pl.set.assign(set, set + batch);
        else pl.set.clear();
        if (forms) pl.forms.assign(forms, forms + batch);
        else pl.forms.clear();
        pl.n_sets = n_sets;
        pl.skip = (int)skip_mask();
        pl.form = form;
        pl.stream = st;
        pl.valid = true;
    }
    return launch_class_set(h, bv, n_sets, pl.count.data(), pl.start.data(), pl.smem.data(), h->d_order, st, launches,
                            pl.count[G], pl.start[G]);
}

// ---- class selection on the device -------------------------------------------------------------------------------
// One CTA sorts the batch: keep_control_steps and class of every path (pqp_dispatch.h), a histogram over (class,
// length), its exclusive prefix, then a scatter into the per-class order segments, longest path first (paths of one
// length in any order: results do not depend on it).  A path outside the caller's bounds gets no entry; it is answered
// here exactly as a kernel answers a path it cannot take: PQP_INVALID_PROBLEM, 0 iterations, NaN states.
//
// The host launches every class the bounds can reach without knowing how many paths it got, so a segment has unused
// entries.  They name path `batch`, which the launches see with 0 stations (n_view[batch] = 0) and status / iterations
// slots of its own: every solve kernel turns such a path away before touching anything else (status -100 into that
// slot).  The kernels themselves are unchanged: a `prob < 0` exit in their entries moved ptxas' register allocation
// and spills in 11 of the 16 solve kernels, which sit at their register limits.
constexpr int kDispatchThreads = 1024;
struct DispatchArgs {
    pqp::FormTables t;         // class table, ncols and length bound of every formulation
    const int32_t *form_of;    // [batch] formulation of every path, NULL: `form` for every path
    int form, form_mask;       // the call's single formulation (mask_form(form_mask)) and the formulations launched
    int v0, nv, ncols;         // order layout: the classes [v0, v0 + nv) the mask spans, `ncols` length buckets each
    int min_keep, max_keep, batch;
    const int32_t *n_points, *offsets;
    const pqp_state *ref;
    pqp_state *out_states;
    double *out_frenet;
    int32_t *status, *iters;   // [batch + 1] what the launches write into (copied to the caller's afterwards)
    int32_t *n_view;           // [batch + 1] station counts the launches read: n_points, then 0
    int32_t *key;              // [batch] histogram bucket of every path, -1: outside the bounds
    int32_t *order;            // [n_sets][nv][batch] order segments, pre-filled with `batch`
    const int32_t *set;        // [batch] parameter set of every path, NULL: set 0
    int n_sets;                // sets launched: a path whose set lies outside [0, n_sets) is answered here; 1 without `set`
    int32_t *hist;             // [n_sets * nv * ncols + n_sets * nv] histogram and bases in global memory, NULL: shared
};

__global__ void pqp_fill_kernel(int32_t *p, size_t n, int32_t value) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = value;
}

__global__ void __launch_bounds__(kDispatchThreads)
pqp_dispatch_kernel(const __grid_constant__ DispatchArgs a) {
    // [n_sets * nv * ncols] paths per (set, class, longest-first length bucket), then [n_sets * nv] bases: in shared
    // memory for one set, in global memory (a.hist) for several
    extern __shared__ int32_t hist_s[];
    __shared__ int32_t warp_sum[kDispatchThreads / 32];
    int32_t *hist = a.hist ? a.hist : hist_s;
    const int nsv = a.n_sets * a.nv, nb = nsv * a.ncols, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int i = tid; i < nb; i += kDispatchThreads) hist[i] = 0;
    if (tid == 0) a.n_view[a.batch] = 0;
    __syncthreads();
    for (int b = tid; b < a.batch; b += kDispatchThreads) {
        const int n = a.n_points[b], off = a.offsets[b];
        a.n_view[b] = n;
        const int s = a.set ? a.set[b] : 0;
        const int f = a.form_of ? a.form_of[b] : a.form;
        const bool ok = pqp::form_in_mask(f, a.form_mask) && s >= 0 && s < a.n_sets;
        const int keep = ok ? pqp::keep_control_steps(f, a.ref + off, n) : 0;
        const int key = pqp::dispatch_key_forms(a.t, a.form_mask, f, s, a.n_sets, n, keep, a.min_keep, a.max_keep, a.nv,
                                                a.ncols, a.v0);
        if (key >= 0) {
            atomicAdd(&hist[key], 1);
        } else {   // not launched: answered as a kernel answers a path it cannot take
            a.status[b] = PQP_INVALID_PROBLEM;
            a.iters[b] = 0;
            write_invalid(a.out_states, a.out_frenet, off, n, 0, 1);
        }
        a.key[b] = key;
    }
    __syncthreads();
    // exclusive prefix of the histogram: every thread owns a run of consecutive buckets
    int32_t *base = hist + nb;
    const int per = (nb + kDispatchThreads - 1) / kDispatchThreads, lo = min(tid * per, nb), hi = min(lo + per, nb);
    int sum = 0;
    for (int i = lo; i < hi; ++i) sum += hist[i];
    int incl = sum;
    for (int d = 1; d < 32; d <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += y;
    }
    if (lane == 31) warp_sum[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        const int w = warp_sum[lane];
        int wi = w;
        for (int d = 1; d < 32; d <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, wi, d);
            if (lane >= d) wi += y;
        }
        warp_sum[lane] = wi - w;
    }
    __syncthreads();
    int run = warp_sum[wid] + incl - sum;
    for (int i = lo; i < hi; ++i) {
        const int c = hist[i];
        hist[i] = run;
        run += c;
    }
    __syncthreads();
    // scatter into the order segments (nsv of them, `batch` entries each)
    for (int r = tid; r < nsv; r += kDispatchThreads) base[r] = hist[r * a.ncols];
    __syncthreads();
    for (int b = tid; b < a.batch; b += kDispatchThreads) {
        const int key = a.key[b];
        if (key < 0) continue;
        const int r = key / a.ncols;
        a.order[(size_t)r * a.batch + (atomicAdd(&hist[key], 1) - base[r])] = b;
    }
}

namespace {
size_t dispatch_smem(int nv, int ncols) { return ((size_t)nv * ncols + nv) * sizeof(int32_t); }

int max_ncols(const pqp_handle *h) { return std::max({h->cls_ncols[0], h->cls_ncols[1], h->cls_ncols[2]}); }

// Which classes of `form` the stated bounds reach, the shortest path each of them can get and the shared memory it
// needs: every (n, keep) inside the bounds, as class_for maps it.  Adds to `d` (min_n starts at INT32_MAX).
void reach_classes(const pqp_handle *h, pqp_handle::DispatchLaunches &d, int form, int max_n, int min_keep, int max_keep) {
    const int ncols = h->cls_ncols[form];
    const int col_hi = max_n > 0 ? std::min(max_n, ncols - 1) : ncols - 1;
    int r_lo = 0, r_hi = pqp::kTableKeepRows - 1;
    if (form == PQP_FORM_KP) {
        if (min_keep > 0) r_lo = std::min(min_keep, pqp::kTableKeepRows) - 1;
        if (max_keep > 0) r_hi = std::min(max_keep, pqp::kTableKeepRows) - 1;
    } else {
        r_lo = r_hi = pqp::keep_control_steps(form, nullptr, 0) - 1;
    }
    for (int r = r_lo; r <= r_hi; ++r)
        for (int n = 0; n <= col_hi; ++n) {
            int v;
            size_t need;
            class_for(h, n, r + 1, &v, &need, form);
            d.reach[v] = true;
            d.smem[v] = std::max(d.smem[v], need);
            d.min_n[v] = std::min(d.min_n[v], n);
        }
}

// The classes the bounds reach over the formulations of `form_mask`, formulation f bounded by max_n[f].  Classes belong
// to one formulation each, so every class gets exactly what its formulation's bounds give it alone.  Cached per (mask,
// bounds) in PQP_DISPATCH_SLOTS slots, so that a caller alternating between masks or bounds keeps each of them.
const pqp_handle::DispatchLaunches &dispatch_launches(pqp_handle *h, int form_mask, const int max_n[3], int min_keep,
                                                      int max_keep) {
    for (const pqp_handle::DispatchLaunches &d : h->disp)
        if (d.valid && d.form_mask == form_mask && std::equal(max_n, max_n + 3, d.max_n) && d.min_keep == min_keep &&
            d.max_keep == max_keep)
            return d;
    pqp_handle::DispatchLaunches &d = h->disp[h->disp_next];
    h->disp_next = (h->disp_next + 1) % PQP_DISPATCH_SLOTS;
    d = pqp_handle::DispatchLaunches();
    for (int v = 0; v < kNumVariants; ++v) d.min_n[v] = INT32_MAX;
    for (int f : {PQP_FORM_KP, PQP_FORM_K, PQP_FORM_KPC})
        if (pqp::form_in_mask(f, form_mask)) reach_classes(h, d, f, max_n[f], min_keep, max_keep);
    d.form_mask = form_mask; std::copy(max_n, max_n + 3, d.max_n); d.min_keep = min_keep; d.max_keep = max_keep;
    d.valid = true;
    return d;
}

// Room in the sort scratch for n_sets parameter sets (pqp_handle::d_disp_order / d_disp_hist).
int dispatch_scratch(pqp_handle *h, int n_sets) {
    if (n_sets <= h->disp_cap) return PQP_OK;
    int cap = 1;
    while (cap < n_sets) cap *= 2;
    int32_t *o = nullptr, *hs = nullptr;
    PQP_CUDA(cudaMalloc(&o, (size_t)cap * kNumVariants * h->max_batch * sizeof(int32_t)));
    if (cudaMalloc(&hs, (size_t)cap * kNumVariants * (max_ncols(h) + 1) * sizeof(int32_t)) != cudaSuccess) {
        cudaFree(o);
        set_err("pqp_launch_dispatch: cudaMalloc of the sort scratch failed");
        return PQP_ERR_CUDA;
    }
    if (h->d_disp_order) { h->retired.push_back(h->d_disp_order); h->retired.push_back(h->d_disp_hist); }
    h->d_disp_order = o; h->d_disp_hist = hs; h->disp_cap = cap;
    return PQP_OK;
}
}  // namespace

int pqp_launch_dispatch(pqp_handle *h, const pqp::BatchView &bv, int form_mask, const int32_t *d_form, int batch,
                        int total, const int max_n[3], int min_keep, int max_keep, cudaStream_t st, int *launches,
                        const int32_t *d_set, int n_param_sets) {
    // Layout: the order segments and the histogram span the classes [v_lo, v_hi) of the mask's formulations, with the
    // largest ncols among them as the stride.  For one formulation that is its own classes and table width.
    int v_lo = kNumVariants, v_hi = 0, ncols = 0;
    DispatchArgs a;
    for (int f : {PQP_FORM_KP, PQP_FORM_K, PQP_FORM_KPC}) {
        a.t.table[f] = h->d_cls_table + h->cls_off[f];
        a.t.ncols[f] = h->cls_ncols[f];
        a.t.max_n[f] = pqp::form_in_mask(f, form_mask) ? max_n[f] : 0;   // (the reach cache's key as well)
        if (!pqp::form_in_mask(f, form_mask)) continue;
        int v0, v1;
        form_range(f, &v0, &v1);
        v_lo = std::min(v_lo, v0);
        v_hi = std::max(v_hi, v1);
        ncols = std::max(ncols, h->cls_ncols[f]);
    }
    const int nv = v_hi - v_lo;
    const pqp_handle::DispatchLaunches &d = dispatch_launches(h, form_mask, a.t.max_n, min_keep, max_keep);
    // with a set index: every set below n_param_sets (0: all of them), the histogram in global scratch
    int n_sets = 1;
    if (d_set) {
        n_sets = (int)h->dsets.size();
        if (n_param_sets > 0) n_sets = std::min(n_sets, n_param_sets);
    }
    const int rs = dispatch_scratch(h, n_sets);
    if (rs != PQP_OK) return rs;
    int32_t *order = h->d_disp_order, *hist = d_set ? h->d_disp_hist : nullptr;
    const size_t n_order = (size_t)n_sets * nv * batch;
    pqp_fill_kernel<<<(unsigned)std::min<size_t>((n_order + 255) / 256, 1024), 256, 0, st>>>(order, n_order, batch);
    PQP_CUDA(cudaGetLastError());
    a.form_of = d_form; a.form = pqp::mask_form(form_mask); a.form_mask = form_mask;
    a.v0 = v_lo; a.nv = nv; a.ncols = ncols;
    a.min_keep = min_keep; a.max_keep = max_keep; a.batch = batch;
    a.n_points = bv.n_points; a.offsets = bv.offsets; a.ref = bv.ref;
    a.out_states = bv.out_states; a.out_frenet = bv.out_frenet; a.status = h->d_disp_status; a.iters = h->d_disp_iters;
    a.n_view = h->d_disp_n; a.key = h->d_disp_key; a.order = order;
    a.set = d_set; a.n_sets = n_sets; a.hist = hist;
    pqp_dispatch_kernel<<<1, kDispatchThreads, hist ? 0 : dispatch_smem(nv, ncols), st>>>(a);
    PQP_CUDA(cudaGetLastError());
    if (launches) *launches += 2;
    pqp::BatchView dv = bv;
    dv.n_points = h->d_disp_n; dv.status = h->d_disp_status; dv.iters = h->d_disp_iters;
    // Grid per (set, class): `batch` CTAs, or fewer when the class's shortest path says so (its paths hold at least min_n
    // stations each, `total` in all); the CTAs past the segment's last path find the sentinel path and return.
    std::vector<int> count((size_t)n_sets * kNumVariants, 0), start((size_t)n_sets * kNumVariants, 0);
    std::vector<size_t> smem((size_t)n_sets * kNumVariants, 0);
    for (int s = 0; s < n_sets; ++s)
        for (int v = v_lo; v < v_hi; ++v) {
            if (!d.reach[v]) continue;
            const int g = s * kNumVariants + v;
            count[g] = d.min_n[v] >= 1 ? (int)std::min<long long>(batch, (long long)total / d.min_n[v]) : batch;
            start[g] = (s * nv + v - v_lo) * batch;
            smem[g] = d.smem[v];
        }
    const int rc = launch_class_set(h, dv, n_sets, count.data(), start.data(), smem.data(), order, st, launches);
    if (rc != PQP_OK) return rc;
    PQP_CUDA(cudaMemcpyAsync(bv.status, h->d_disp_status, (size_t)batch * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    if (bv.iters)
        PQP_CUDA(cudaMemcpyAsync(bv.iters, h->d_disp_iters, (size_t)batch * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    return PQP_OK;
}

// OSQP 0.6's validate_settings on the settings pqp_params carries (pqp.h): false, with the rule in pqp_last_error(),
// where osqp_setup would refuse them.  Every test is written so that a NaN fails it.
static bool settings_ok(const pqp_params &p, const char *entry) {
    const char *bad = !(p.rho > 0) ? "rho > 0"
                      : !(p.sigma > 0) ? "sigma > 0"
                      : !(p.alpha > 0 && p.alpha < 2) ? "0 < alpha < 2"
                      : !(p.max_iter > 0) ? "max_iter > 0"
                      : !(p.eps_abs >= 0 && p.eps_rel >= 0) ? "eps_abs >= 0 and eps_rel >= 0"
                      : (p.eps_abs == 0 && p.eps_rel == 0) ? "eps_abs and eps_rel not both 0"
                      : !(p.eps_prim_inf > 0 && p.eps_dual_inf > 0) ? "eps_prim_inf > 0 and eps_dual_inf > 0"
                      : !(p.scaling >= 0 && p.check_termination >= 0) ? "scaling >= 0 and check_termination >= 0"
                      : !(p.adaptive_rho == 0 || p.adaptive_rho == 1) ? "adaptive_rho 0 or 1"
                      : !(p.adaptive_rho_interval >= 0) ? "adaptive_rho_interval >= 0"
                      : !(p.adaptive_rho_tolerance >= 1) ? "adaptive_rho_tolerance >= 1"
                      : nullptr;
    if (bad) set_err("%s: OSQP refuses these settings (needs %s)", entry, bad);
    return !bad;
}

// The formulation checks of the single-formulation device entries.
static int device_form_ok(int formulation, const double *d_max_k, const double *d_max_kp) {
    if (formulation == PQP_FORM_KPC && (!d_max_k || !d_max_kp)) {
        set_err("KPC needs d_max_k and d_max_kp (pqp_update_limits_device)");
        return PQP_ERR_ARG;
    }
    if (formulation != PQP_FORM_KP && formulation != PQP_FORM_KPC && formulation != PQP_FORM_K) {
        set_err("unknown formulation");
        return PQP_ERR_ARG;
    }
    return PQP_OK;
}

// The BatchView and stream of a device entry's arguments (`stream` NULL: the handle's), once the batch fits the handle.
static int device_batch(pqp_handle *h, int batch, int total_points, const int32_t *d_n_points, const int32_t *d_offsets,
                        const pqp_state *d_ref, const pqp_station_bounds *d_bounds, const double *d_x0,
                        const double *d_end_heading, const double *d_max_k, const double *d_max_kp,
                        pqp_state *d_out_states, double *d_out_frenet, int32_t *d_status, int32_t *d_iters, void *stream,
                        pqp::BatchView *bv, cudaStream_t *st) {
    if (batch > h->max_batch || total_points > h->max_total) {
        set_err("batch / total_points exceed what the handle was created for (workspace size)");
        return PQP_ERR_CAPACITY;
    }
    PQP_CUDA(cudaSetDevice(h->device));
    *st = stream ? (cudaStream_t)stream : h->stream;
    bv->batch = batch; bv->n_points = d_n_points; bv->offsets = d_offsets; bv->ref = d_ref; bv->bounds = d_bounds;
    bv->x0 = d_x0; bv->end_heading = d_end_heading; bv->out_states = d_out_states; bv->out_frenet = d_out_frenet;
    bv->status = d_status; bv->iters = d_iters; bv->workspace = h->d_ws; bv->debug = nullptr;
    bv->max_k = d_max_k; bv->max_kp = d_max_kp;
    return PQP_OK;
}

// The stats of a device entry: kernel_ms from h->ev[0], recorded on `st` before its launches, to their end (waited for).
static int device_stats(pqp_handle *h, cudaStream_t st, int launches, pqp_stats *stats) {
    memset(stats, 0, sizeof(*stats));
    PQP_CUDA(cudaEventRecord(h->ev[1], st));
    PQP_CUDA(cudaEventSynchronize(h->ev[1]));
    PQP_CUDA(cudaEventElapsedTime(&stats->kernel_ms, h->ev[0], h->ev[1]));
    stats->kernel_launches = launches;
    return PQP_OK;
}

extern "C" {

const char *pqp_last_error(void) { return g_err; }

const char *pqp_version(void) { return "pqp abi 1 / sm_90a / fp64 ADMM, one CTA per path (thread per station)"; }

int pqp_params_update_config(pqp_params *p) {
    if (!p) return PQP_ERR_ARG;
    // updateConfig(), planning_flags.cpp:8-14
    p->circle_radius = sqrt(pow(p->car_length / 8, 2) + pow(p->car_width / 2, 2)) + p->safety_margin;
    p->d1 = -3.0 / 8.0 * p->car_length + p->rear_axle_to_center;
    p->d2 = -1.0 / 8.0 * p->car_length + p->rear_axle_to_center;
    p->d3 = 1.0 / 8.0 * p->car_length + p->rear_axle_to_center;
    p->d4 = 3.0 / 8.0 * p->car_length + p->rear_axle_to_center;
    return PQP_OK;
}

int pqp_params_default(pqp_params *p) {
    if (!p) return PQP_ERR_ARG;
    memset(p, 0, sizeof(*p));
    // planning_flags.cpp:18-43
    p->car_width = 2.0;
    p->car_length = 4.9;
    p->safety_margin = 0.0;
    p->wheel_base = 2.85;
    p->rear_axle_to_center = 1.45;
    p->max_steering_angle = 30.0 * M_PI / 180.0;
    p->mu = 0.4;
    p->max_curvature_rate = 0.1;
    // planning_flags.cpp:102-119
    p->K_curvature_weight = 50;
    p->K_curvature_rate_weight = 200;
    p->K_deviation_weight = 0;
    p->KP_curvature_weight = 10;
    p->KP_curvature_rate_weight = 200;
    p->KP_deviation_weight = 0;
    p->KP_slack_weight = 3;
    p->expected_safety_margin = 1.3;
    p->constraint_end_heading = 1;
    // OSQP 0.6.x defaults (the reference only touches verbosity / warm start, solver.cpp:48-49)
    p->rho = 0.1;
    p->sigma = 1e-6;
    p->alpha = 1.6;
    p->eps_abs = 1e-3;
    p->eps_rel = 1e-3;
    p->eps_prim_inf = 1e-4;
    p->eps_dual_inf = 1e-4;
    p->max_iter = 4000;
    p->scaling = 10;
    p->check_termination = 25;
    p->adaptive_rho = 1;
    p->adaptive_rho_interval = 25;
    p->adaptive_rho_tolerance = 5;
    return pqp_params_update_config(p);
}

int pqp_keep_control_steps(int formulation, const pqp_state *ref, int n_points) {
    return pqp::keep_control_steps(formulation, ref, n_points);   // (pqp_dispatch.h: the device dispatch evaluates the same)
}

int pqp_problem_size(int formulation, int n, int keep, int *n_var, int *n_con) {
    if (n < 2 || keep < 1 || !n_var || !n_con) return PQP_ERR_ARG;
    const int ch = (n + keep - 2) / keep;
    switch (formulation) {
    case PQP_FORM_KP: *n_var = 5 * n + ch; *n_con = 11 * n + ch + 2; return PQP_OK;       // :18-23
    case PQP_FORM_K: *n_var = 4 * n - 1; *n_con = 11 * n - 1; return PQP_OK;              // :18-19
    case PQP_FORM_KPC: *n_var = 6 * n + ch; *n_con = 12 * n + 3 * ch + 2; return PQP_OK;  // :18-24
    default: return PQP_ERR_ARG;
    }
}

extern "C" int pqp_comm_destroy(pqp_handle *h);   // pqp_multi.cu

void pqp_destroy(pqp_handle *h) {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->nccl_comm) pqp_comm_destroy(h);
    cudaFree(h->d_n); cudaFree(h->d_off); cudaFree(h->d_order); cudaFree(h->d_order_auto); cudaFree(h->d_status); cudaFree(h->d_iters);
    cudaFree(h->d_ref); cudaFree(h->d_out); cudaFree(h->d_bounds);
    cudaFree(h->d_x0); cudaFree(h->d_end); cudaFree(h->d_frenet); cudaFree(h->d_ws);
    cudaFree(h->d_max_k); cudaFree(h->d_max_kp);
    cudaFree(h->d_cls_table); cudaFree(h->d_disp_order); cudaFree(h->d_disp_hist); cudaFree(h->d_disp_key);
    cudaFree(h->d_disp_n); cudaFree(h->d_disp_status); cudaFree(h->d_disp_iters);
    for (void *p : h->retired) cudaFree(p);
    cudaFreeHost(h->h_off); cudaFreeHost(h->h_order);
    cudaFree(h->d_gen); cudaFreeHost(h->h_gen);
    if (h->env && h->env_free) h->env_free(h->env);
    for (auto &e : h->ev) if (e) cudaEventDestroy(e);
    for (auto &e : h->ev_chunk) if (e) cudaEventDestroy(e);
    for (auto &e : h->ev_cls) if (e) cudaEventDestroy(e);
    if (h->ev_fork) cudaEventDestroy(h->ev_fork);
    for (auto &q : h->cls_stream) if (q) cudaStreamDestroy(q);
    if (h->stream) cudaStreamDestroy(h->stream);
    if (h->stream2) cudaStreamDestroy(h->stream2);
    delete h;
}

int pqp_set_param_sets(pqp_handle *h, int n_sets, const pqp_params *sets) {
    if (!h || !sets || n_sets < 1 || n_sets > PQP_MAX_PARAM_SETS) {
        set_err("pqp_set_param_sets: bad argument (needs a handle and 1..PQP_MAX_PARAM_SETS sets)");
        return PQP_ERR_ARG;
    }
    for (int s = 0; s < n_sets; ++s)
        if (!settings_ok(sets[s], "pqp_set_param_sets")) return PQP_ERR_ARG;
    h->sets.assign(sets, sets + n_sets);
    h->dsets.resize((size_t)n_sets);
    for (int s = 0; s < n_sets; ++s) h->dsets[s] = pqp::dev_params_from(sets[s]);
    h->params = h->sets[0];
    h->dprm = h->dsets[0];
    h->dprm_gen[0] = h->dprm_gen[1] = h->dprm;
    return PQP_OK;
}

int pqp_set_params(pqp_handle *h, const pqp_params *params) { return pqp_set_param_sets(h, 1, params); }

int pqp_create(pqp_handle **out, const pqp_params *params, int device, int max_batch, int max_total_points) {
    if (!out || !params || max_batch < 1 || max_total_points < 2) {
        set_err("pqp_create: bad argument");
        return PQP_ERR_ARG;
    }
    *out = nullptr;
    if (!settings_ok(*params, "pqp_create")) return PQP_ERR_ARG;
    int ndev = 0;
    PQP_CUDA(cudaGetDeviceCount(&ndev));
    if (device < 0 || device >= ndev) {
        set_err("pqp_create: no such CUDA device");
        return PQP_ERR_CUDA;
    }
    PQP_CUDA(cudaSetDevice(device));
    pqp_handle *h = new (std::nothrow) pqp_handle;
    if (!h) return PQP_ERR_ARG;
    h->device = device;
    h->max_batch = max_batch;
    h->max_total = max_total_points;
    pqp_set_params(h, params);
    int rc = PQP_OK;
    auto fail = [&](int code) { pqp_destroy(h); return code; };
#define PQP_TRY(call)                                                      \
    do {                                                                   \
        cudaError_t e_ = (call);                                           \
        if (e_ != cudaSuccess) {                                           \
            set_err("%s failed: %s", #call, cudaGetErrorString(e_));       \
            return fail(PQP_ERR_CUDA);                                     \
        }                                                                  \
    } while (0)
    PQP_TRY(cudaDeviceGetAttribute(&h->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
    PQP_TRY(cudaDeviceGetAttribute(&h->num_sms, cudaDevAttrMultiProcessorCount, device));
    pqp_k1_set_smem_cap(h->smem_optin);
    // fails with cudaErrorNoKernelImageForDevice / InvalidDeviceFunction on anything but sm_90
    for (int v = 0; v < kNumVariants; ++v)
        PQP_TRY(cudaFuncSetAttribute(kVariants[v].fn, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem_optin));
    PQP_TRY(cudaFuncSetAttribute(pqp_gen_kernel_fn(), cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem_optin));
    PQP_TRY(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    PQP_TRY(cudaStreamCreateWithFlags(&h->stream2, cudaStreamNonBlocking));
    for (auto &e : h->ev_chunk) PQP_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    for (auto &q : h->cls_stream) PQP_TRY(cudaStreamCreateWithFlags(&q, cudaStreamNonBlocking));
    for (auto &e : h->ev_cls) PQP_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    PQP_TRY(cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
    for (auto &e : h->ev) PQP_TRY(cudaEventCreate(&e));
    const size_t B = (size_t)max_batch, T = (size_t)max_total_points;
    PQP_TRY(cudaMalloc(&h->d_n, B * sizeof(int32_t)));
    PQP_TRY(cudaMalloc(&h->d_off, (B + 1) * sizeof(int32_t)));
    PQP_TRY(cudaMalloc(&h->d_order, B * sizeof(int32_t)));
    PQP_TRY(cudaMalloc(&h->d_order_auto, (size_t)std::min(max_batch, kAutoOrderMax) * sizeof(int32_t)));
    PQP_TRY(cudaMalloc(&h->d_status, B * sizeof(int32_t)));
    PQP_TRY(cudaMalloc(&h->d_iters, B * sizeof(int32_t)));
    PQP_TRY(cudaMalloc(&h->d_ref, T * sizeof(pqp_state)));
    PQP_TRY(cudaMalloc(&h->d_out, T * sizeof(pqp_state)));
    PQP_TRY(cudaMalloc(&h->d_bounds, T * sizeof(pqp_station_bounds)));
    PQP_TRY(cudaMalloc(&h->d_x0, B * 3 * sizeof(double)));
    PQP_TRY(cudaMalloc(&h->d_end, B * sizeof(double)));
    PQP_TRY(cudaMalloc(&h->d_frenet, T * 3 * sizeof(double)));
    PQP_TRY(cudaMemset(h->d_frenet, 0, T * 3 * sizeof(double)));   // (padded rows of a multi-GPU gather read as zeros)
    PQP_TRY(cudaMalloc(&h->d_ws, pqp::kp2_ws_doubles(T, B) * sizeof(double)));
    PQP_TRY(cudaMallocHost(&h->h_off, (B + 1) * sizeof(int32_t)));
    PQP_TRY(cudaMallocHost(&h->h_order, B * sizeof(int32_t)));
    // class tables of the device dispatch, uploaded once; its sort scratch for one parameter set
    {
        std::vector<int8_t> all, tab;
        for (int form : {PQP_FORM_KP, PQP_FORM_K, PQP_FORM_KPC}) {
            h->cls_ncols[form] = class_table(h, form, &tab);
            h->cls_off[form] = (int)all.size();
            all.insert(all.end(), tab.begin(), tab.end());
        }
        PQP_TRY(cudaMalloc(&h->d_cls_table, all.size()));
        PQP_TRY(cudaMemcpy(h->d_cls_table, all.data(), all.size(), cudaMemcpyHostToDevice));
        PQP_TRY(cudaFuncSetAttribute(pqp_dispatch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)dispatch_smem(kNumVariants, max_ncols(h))));
        if (dispatch_scratch(h, 1) != PQP_OK) return fail(PQP_ERR_CUDA);
        PQP_TRY(cudaMalloc(&h->d_disp_key, B * sizeof(int32_t)));
        PQP_TRY(cudaMalloc(&h->d_disp_n, (B + 1) * sizeof(int32_t)));
        PQP_TRY(cudaMalloc(&h->d_disp_status, (B + 1) * sizeof(int32_t)));
        PQP_TRY(cudaMalloc(&h->d_disp_iters, (B + 1) * sizeof(int32_t)));
    }
#undef PQP_TRY
    (void)rc;
    *out = h;
    return PQP_OK;
}

const char *pqp_class_name(int variant) {
    return (variant >= 0 && variant < kNumVariants) ? kVariants[variant].name : "";
}

int pqp_class_info(int n_points, int keep, int smem_optin, int *variant, int *threads, int64_t *smem_bytes) {
    pqp_handle fake;
    fake.smem_optin = smem_optin > 0 ? smem_optin : 232448;
    int v;
    size_t need;
    const bool ok = class_for(&fake, n_points, keep, &v, &need);
    if (variant) *variant = v;
    if (threads) *threads = kVariants[v].threads;
    if (smem_bytes) *smem_bytes = (int64_t)need;
    return ok ? PQP_OK : PQP_ERR_UNSUPPORTED;
}

int pqp_class_info_kpc(int n_points, int smem_optin, int *variant, int *threads, int64_t *smem_bytes) {
    pqp_handle fake;
    fake.smem_optin = smem_optin > 0 ? smem_optin : 232448;
    int v;
    size_t need;
    const bool ok = class_for(&fake, n_points, 4, &v, &need, PQP_FORM_KPC);
    if (variant) *variant = v;
    if (threads) *threads = ok ? kVariants[v].threads : 0;
    if (smem_bytes) *smem_bytes = (int64_t)need;
    return ok ? PQP_OK : PQP_ERR_UNSUPPORTED;
}

int pqp_set_order_hint(pqp_handle *h, int batch, const int32_t *expected_iters) {
    if (!h || batch < 0) return PQP_ERR_ARG;
    if (!expected_iters || batch == 0) h->order_hint.clear();
    else h->order_hint.assign(expected_iters, expected_iters + batch);
    h->plan.valid = false;     // the cached class plan carries the launch order
    return PQP_OK;
}

int pqp_class_info_form(int formulation, int n_points, int keep, int smem_optin, int *variant, int *threads, int64_t *smem_bytes) {
    if (formulation != PQP_FORM_KP && formulation != PQP_FORM_KPC && formulation != PQP_FORM_K) return PQP_ERR_ARG;
    pqp_handle fake;
    fake.smem_optin = smem_optin > 0 ? smem_optin : 232448;
    int v;
    size_t need;
    const bool ok = class_for(&fake, n_points, keep, &v, &need, formulation);
    if (variant) *variant = v;
    if (threads) *threads = ok ? kVariants[v].threads : 0;
    if (smem_bytes) *smem_bytes = (int64_t)need;
    return ok ? PQP_OK : PQP_ERR_UNSUPPORTED;
}

int pqp_device_class_info(int max_n_points, int min_keep, int max_keep, int smem_optin, int *variant, int *threads,
                          int64_t *smem_bytes) {
    pqp_handle fake;
    fake.smem_optin = smem_optin > 0 ? smem_optin : 232448;
    int v = -1;
    size_t need = 0;
    const bool ok = device_class(&fake, max_n_points, min_keep, max_keep, &v, &need);
    if (variant) *variant = v;
    if (threads) *threads = ok ? kVariants[v].threads : 0;
    if (smem_bytes) *smem_bytes = (int64_t)need;
    if (!ok) return PQP_ERR_UNSUPPORTED;
    // every (n, keep) inside the bounds must pass the checks the kernel itself makes
    for (int k = min_keep; k <= max_keep; ++k)
        for (int n = 2; n <= max_n_points; ++n)
            if (!kVariants[v].fits(n, k) || kVariants[v].smem(n, k) > need) return PQP_ERR_ARG;
    return PQP_OK;
}

int pqp_max_points_keep(pqp_handle *h, int formulation, int keep) {
    if (!h || (formulation != PQP_FORM_KP && formulation != PQP_FORM_KPC && formulation != PQP_FORM_K) || keep < 1 || keep > 10) return 0;
    // mirrors the per-path selection of pqp_solve_batch (class_for): preferred class, else the one-warp kernel (KP only)
    int best = 0;
    for (int n = 2; n <= 4096; ++n) {
        int v;
        size_t need;
        if (class_for(h, n, keep, &v, &need, formulation)) best = n;
        else break;
    }
    return best;
}

int pqp_max_points(pqp_handle *h, int formulation) {
    int best = 0;
    for (int keep = 1; keep <= 10; ++keep) {
        const int m = pqp_max_points_keep(h, formulation, keep);
        best = (keep == 1) ? m : std::min(best, m);
    }
    return best;
}

static int launch_variant(pqp_handle *h, int v, const pqp::DevParams *prm, const pqp::BatchView &bv, int count,
                          const int32_t *d_order, size_t smem_bytes, cudaStream_t st) {
    if (smem_bytes > (size_t)h->smem_optin) {
        set_err("path too long for one SM's shared memory");
        return PQP_ERR_UNSUPPORTED;
    }
    // PQP_FORCE_SMEM=<bytes> (diagnostics only): launch with at least that much dynamic shared memory, e.g. to hold a
    // two-CTA-per-SM class at one CTA per SM.  The kernel still lays out what the path needs.
    static const size_t force = [] { const char *e = getenv("PQP_FORCE_SMEM"); return e ? (size_t)strtoul(e, nullptr, 0) : (size_t)0; }();
    if (force > smem_bytes) smem_bytes = std::min(force, (size_t)h->smem_optin);
    int smem_doubles = (int)(smem_bytes / sizeof(double));
    void *args[] = {(void *)prm, (void *)&bv, (void *)&d_order, (void *)&smem_doubles};
    PQP_CUDA(cudaLaunchKernel(kVariants[v].fn, dim3(count), dim3(kVariants[v].threads), args, smem_bytes, st));
    return PQP_OK;
}

int pqp_solve_batch_device(pqp_handle *h, int formulation, int batch, int total_points,
                           int max_n_points, int min_keep, int max_keep, const int32_t *d_n_points, const int32_t *d_offsets, const pqp_state *d_ref,
                           const pqp_station_bounds *d_bounds, const double *d_x0, const double *d_end_heading,
                           const double *d_max_k, const double *d_max_kp, pqp_state *d_out_states,
                           double *d_out_frenet, int32_t *d_status, int32_t *d_iters, void *stream,
                           pqp_stats *stats) {
    if (!h || batch < 0 || !d_n_points || !d_offsets || !d_ref || !d_bounds || !d_x0 || !d_end_heading ||
        !d_out_states || !d_status) {
        set_err("pqp_solve_batch_device: bad argument");
        return PQP_ERR_ARG;
    }
    int rc = device_form_ok(formulation, d_max_k, d_max_kp);
    if (rc != PQP_OK) return rc;
    if (batch == 0) return PQP_OK;
    pqp::BatchView bv;
    cudaStream_t st;
    rc = device_batch(h, batch, total_points, d_n_points, d_offsets, d_ref, d_bounds, d_x0, d_end_heading, d_max_k,
                      d_max_kp, d_out_states, d_out_frenet, d_status, d_iters, stream, &bv, &st);
    if (rc != PQP_OK) return rc;
    // The host does not see n_points / keep here: the kernel shape class and the shared memory are
    // chosen from the caller's bounds; a path that does not fit reports PQP_INVALID_PROBLEM.
    const int nmax = max_n_points >= 2 ? max_n_points : std::min(h->max_total, 400);
    const int k_hi = (max_keep >= 1) ? std::min(max_keep, 10) : 4;
    const int k_lo = (min_keep >= 1) ? std::min(min_keep, k_hi) : 1;
    int v = -1;
    size_t smem = 0;
    if (!device_class(h, nmax, k_lo, k_hi, &v, &smem, formulation)) {
        set_err("no single kernel shape class takes every (n_points <= max_n_points, min_keep..max_keep): "
                "tighten the bounds or use pqp_solve_batch_device_classes");
        return PQP_ERR_UNSUPPORTED;
    }
    if (stats) PQP_CUDA(cudaEventRecord(h->ev[0], st));
    // small batches: launch order from the inputs (see pqp_order_kernel); the host sees none of them here
    const int32_t *order = nullptr;
    const bool ordered = auto_order_enabled() && batch > h->num_sms && batch <= kAutoOrderMax;
    if (ordered) {
        pqp_order_kernel<<<1, 1024, 0, st>>>(d_n_points, d_offsets, d_bounds, d_x0, batch, h->d_order_auto);
        PQP_CUDA(cudaGetLastError());
        order = h->d_order_auto;
    }
    rc = launch_variant(h, v, &h->dprm, bv, batch, order, smem, st);
    if (rc != PQP_OK) return rc;
    return stats ? device_stats(h, st, ordered ? 2 : 1, stats) : PQP_OK;
}

int pqp_solve_batch_device_classes(pqp_handle *h, int formulation, int batch, int total_points,
                                   const int32_t *h_n_points, const int32_t *h_keep,
                                   const int32_t *d_n_points, const int32_t *d_offsets, const pqp_state *d_ref,
                                   const pqp_station_bounds *d_bounds, const double *d_x0, const double *d_end_heading,
                                   const double *d_max_k, const double *d_max_kp, pqp_state *d_out_states,
                                   double *d_out_frenet, int32_t *d_status, int32_t *d_iters, void *stream,
                                   pqp_stats *stats) {
    if (!h || batch < 0 || !h_n_points || (!h_keep && formulation == PQP_FORM_KP) || !d_n_points || !d_offsets || !d_ref ||
        !d_bounds || !d_x0 || !d_end_heading || !d_out_states || !d_status) {
        set_err("pqp_solve_batch_device_classes: bad argument");
        return PQP_ERR_ARG;
    }
    int rc = device_form_ok(formulation, d_max_k, d_max_kp);
    if (rc != PQP_OK) return rc;
    if (batch == 0) return PQP_OK;
    pqp::BatchView bv;
    cudaStream_t st;
    rc = device_batch(h, batch, total_points, d_n_points, d_offsets, d_ref, d_bounds, d_x0, d_end_heading, d_max_k,
                      d_max_kp, d_out_states, d_out_frenet, d_status, d_iters, stream, &bv, &st);
    if (rc != PQP_OK) return rc;
    if (stats) PQP_CUDA(cudaEventRecord(h->ev[0], st));
    int launches = 0;
    rc = pqp_launch_kp_classes(h, bv, batch, h_n_points, nullptr, nullptr, h_keep, st, &launches, formulation);
    if (rc != PQP_OK) return rc;
    return stats ? device_stats(h, st, launches, stats) : PQP_OK;
}

int pqp_solve_batch_device_dispatch(pqp_handle *h, int formulation, int batch, int total_points,
                                    int max_n_points, int min_keep, int max_keep, const int32_t *d_n_points,
                                    const int32_t *d_offsets, const pqp_state *d_ref, const pqp_station_bounds *d_bounds,
                                    const double *d_x0, const double *d_end_heading, const double *d_max_k,
                                    const double *d_max_kp, pqp_state *d_out_states, double *d_out_frenet,
                                    int32_t *d_status, int32_t *d_iters, void *stream, pqp_stats *stats) {
    return pqp_solve_batch_device_dispatch_sets(h, formulation, batch, total_points, max_n_points, min_keep, max_keep, 0,
                                                d_n_points, d_offsets, d_ref, d_bounds, d_x0, d_end_heading, d_max_k,
                                                d_max_kp, nullptr, d_out_states, d_out_frenet, d_status, d_iters, stream,
                                                stats);
}

int pqp_solve_batch_device_dispatch_sets(pqp_handle *h, int formulation, int batch, int total_points,
                                         int max_n_points, int min_keep, int max_keep, int n_param_sets,
                                         const int32_t *d_n_points, const int32_t *d_offsets, const pqp_state *d_ref,
                                         const pqp_station_bounds *d_bounds, const double *d_x0,
                                         const double *d_end_heading, const double *d_max_k, const double *d_max_kp,
                                         const int32_t *d_param_index, pqp_state *d_out_states, double *d_out_frenet,
                                         int32_t *d_status, int32_t *d_iters, void *stream, pqp_stats *stats) {
    if (!h || batch < 0 || n_param_sets < 0 || !d_n_points || !d_offsets || !d_ref || !d_bounds || !d_x0 ||
        !d_end_heading || !d_out_states || !d_status) {
        set_err("pqp_solve_batch_device_dispatch(_sets): bad argument");
        return PQP_ERR_ARG;
    }
    int rc = device_form_ok(formulation, d_max_k, d_max_kp);
    if (rc != PQP_OK) return rc;
    if (batch == 0) return PQP_OK;
    pqp::BatchView bv;
    cudaStream_t st;
    rc = device_batch(h, batch, total_points, d_n_points, d_offsets, d_ref, d_bounds, d_x0, d_end_heading, d_max_k,
                      d_max_kp, d_out_states, d_out_frenet, d_status, d_iters, stream, &bv, &st);
    if (rc != PQP_OK) return rc;
    if (stats) PQP_CUDA(cudaEventRecord(h->ev[0], st));
    int launches = 0;
    const int max_n[3] = {max_n_points, max_n_points, max_n_points};
    rc = pqp_launch_dispatch(h, bv, 1 << formulation, nullptr, batch, total_points, max_n, min_keep, max_keep, st,
                             &launches, d_param_index, n_param_sets);
    if (rc != PQP_OK) return rc;
    return stats ? device_stats(h, st, launches, stats) : PQP_OK;
}

int pqp_solve_batch_device_dispatch_forms(pqp_handle *h, int batch, int total_points, int max_n_points, int min_keep,
                                          int max_keep, int n_param_sets, int form_mask, const int32_t *d_n_points,
                                          const int32_t *d_offsets, const pqp_state *d_ref,
                                          const pqp_station_bounds *d_bounds, const double *d_x0,
                                          const double *d_end_heading, const double *d_max_k, const double *d_max_kp,
                                          const int32_t *d_param_index, const int32_t *d_formulation,
                                          pqp_state *d_out_states, double *d_out_frenet, int32_t *d_status,
                                          int32_t *d_iters, void *stream, pqp_stats *stats) {
    if (!h || batch < 0 || n_param_sets < 0 || form_mask < 0 || form_mask > 7 || !d_n_points || !d_offsets || !d_ref ||
        !d_bounds || !d_x0 || !d_end_heading || !d_formulation || !d_out_states || !d_status) {
        set_err("pqp_solve_batch_device_dispatch_forms: bad argument");
        return PQP_ERR_ARG;
    }
    const int mask = form_mask ? form_mask : 7;
    if (pqp::form_in_mask(PQP_FORM_KPC, mask) && (!d_max_k || !d_max_kp)) {
        set_err("a form_mask with \"KPC\" needs d_max_k and d_max_kp (pqp_update_limits_device)");
        return PQP_ERR_ARG;
    }
    if (batch == 0) return PQP_OK;
    pqp::BatchView bv;
    cudaStream_t st;
    int rc = device_batch(h, batch, total_points, d_n_points, d_offsets, d_ref, d_bounds, d_x0, d_end_heading, d_max_k,
                          d_max_kp, d_out_states, d_out_frenet, d_status, d_iters, stream, &bv, &st);
    if (rc != PQP_OK) return rc;
    if (stats) PQP_CUDA(cudaEventRecord(h->ev[0], st));
    int launches = 0;
    const int max_n[3] = {max_n_points, max_n_points, max_n_points};
    rc = pqp_launch_dispatch(h, bv, mask, d_formulation, batch, total_points, max_n, min_keep, max_keep, st, &launches,
                             d_param_index, n_param_sets);
    if (rc != PQP_OK) return rc;
    return stats ? device_stats(h, st, launches, stats) : PQP_OK;
}

int pqp_class_table(int formulation, int smem_optin, int8_t *table, int capacity, int *ncols) {
    if ((formulation != PQP_FORM_KP && formulation != PQP_FORM_KPC && formulation != PQP_FORM_K) || !ncols) return PQP_ERR_ARG;
    pqp_handle fake;
    fake.smem_optin = smem_optin > 0 ? smem_optin : 232448;
    std::vector<int8_t> tab;
    *ncols = class_table(&fake, formulation, &tab);
    if (!table) return PQP_OK;
    if (capacity < (int)tab.size()) return PQP_ERR_CAPACITY;
    memcpy(table, tab.data(), tab.size());
    return PQP_OK;
}

// ---- "K" / "KPC": host assembles sparse band-ordered QPs, the generic kernel solves them ----------
static int solve_batch_generic(pqp_handle *h, int formulation, int batch, const int32_t *n_points, const pqp_state *ref,
                               const pqp_station_bounds *bounds, const double *x0, const double *end_heading,
                               const double *max_k, const double *max_kp, pqp_state *out_states, double *out_frenet,
                               int32_t *status, int32_t *iters, pqp_stats *stats) {
    if (formulation == PQP_FORM_KPC && (!max_k || !max_kp)) {
        set_err("KPC needs max_k and max_kp (ReferencePath::getMaxKList / getMaxKpList)");
        return PQP_ERR_ARG;
    }
    std::vector<int64_t> off((size_t)batch + 1, 0);
    for (int b = 0; b < batch; ++b) {
        if (n_points[b] < 0) { set_err("negative n_points"); return PQP_ERR_ARG; }
        off[b + 1] = off[b] + n_points[b];
    }
    if (off[batch] > h->max_total || batch > h->max_batch) { set_err("batch exceeds the handle's capacity"); return PQP_ERR_CAPACITY; }
    std::vector<pqp::GenProblem> gp((size_t)batch);
    std::vector<char> okv((size_t)batch, 0);
    {
        unsigned nt = std::min(16u, std::max(1u, std::thread::hardware_concurrency()));
        nt = std::min<unsigned>(nt, (unsigned)batch);
        std::vector<std::thread> th;
        for (unsigned t = 0; t < nt; ++t)
            th.emplace_back([&, t]() {
                for (int b = (int)t; b < batch; b += (int)nt) {
                    const int64_t o = off[b];
                    const int n = n_points[b];
                    bool ok = false;
                    if (formulation == PQP_FORM_K)
                        ok = pqp::assemble_k(h->params, n, ref + o, bounds + o, x0 + 3 * (size_t)b, end_heading[b], gp[b]);
                    else
                        ok = pqp::assemble_kpc(h->params, n, ref + o, bounds + o, x0 + 3 * (size_t)b, end_heading[b],
                                               max_k + o, max_kp + o, gp[b]);
                    okv[b] = ok ? 1 : 0;
                }
            });
        for (auto &t : th) t.join();
    }
    // layout of the staging blob
    size_t sn = 0, sm = 0, sz = 0;
    size_t smem = 0;
    for (int b = 0; b < batch; ++b) {
        if (!okv[b]) { gp[b] = pqp::GenProblem(); gp[b].N = n_points[b]; gp[b].out_idx.assign(3 * (size_t)n_points[b], 0); }
        sn += gp[b].n; sm += gp[b].m; sz += gp[b].csc_row.size();
        if (okv[b]) smem = std::max(smem, pqp::gen_smem_doubles(gp[b].n, gp[b].m, gp[b].bw) * sizeof(double));
    }
    if (smem > (size_t)h->smem_optin) {
        // paths too long for one SM: they report PQP_INVALID_PROBLEM (the kernel checks the capacity)
        smem = (size_t)h->smem_optin;
    }
    if (smem == 0) smem = 1024;
    const size_t T = (size_t)off[batch], B = (size_t)batch;
    auto al = [](size_t x) { return (x + 15) & ~(size_t)15; };
    size_t o_meta = 0, o_Acol = al(o_meta + B * pqp::kGenMeta * 4), o_Aval = al(o_Acol + sm * 16), o_l = al(o_Aval + sm * 32),
           o_u = al(o_l + sm * 8), o_Pd = al(o_u + sm * 8), o_Poi = al(o_Pd + sn * 8), o_Pov = al(o_Poi + sn * 8),
           o_cp = al(o_Pov + sn * 16), o_cr = al(o_cp + (sn + B) * 4), o_cv = al(o_cr + sz * 4), o_sep = al(o_cv + sz * 8),
           o_oi = al(o_sep + B * 128), o_end = al(o_oi + T * 12);
    if (o_end > h->gen_cap) {
        cudaFree(h->d_gen); cudaFreeHost(h->h_gen);
        h->d_gen = nullptr; h->h_gen = nullptr; h->gen_cap = 0;
        PQP_CUDA(cudaMalloc(&h->d_gen, o_end));
        PQP_CUDA(cudaMallocHost(&h->h_gen, o_end));
        h->gen_cap = o_end;
    }
    char *H = h->h_gen;
    int32_t *meta = (int32_t *)(H + o_meta);
    size_t an = 0, am = 0, az = 0;
    for (int b = 0; b < batch; ++b) {
        const pqp::GenProblem &g = gp[b];
        int32_t *mb = meta + (size_t)pqp::kGenMeta * b;
        memset(mb, 0, pqp::kGenMeta * 4);
        mb[0] = g.n; mb[1] = g.m; mb[2] = g.n_den; mb[3] = g.bw; mb[4] = g.M; mb[5] = n_points[b];
        mb[6] = (int32_t)off[b]; mb[7] = (int32_t)an; mb[8] = (int32_t)am; mb[9] = (int32_t)az; mb[10] = (int32_t)(an + b);
        memcpy(H + o_Acol + am * 16, g.A_col.data(), g.A_col.size() * 4);
        memcpy(H + o_Aval + am * 32, g.A_val.data(), g.A_val.size() * 8);
        memcpy(H + o_l + am * 8, g.l.data(), g.l.size() * 8);
        memcpy(H + o_u + am * 8, g.u.data(), g.u.size() * 8);
        memcpy(H + o_Pd + an * 8, g.Pd.data(), g.Pd.size() * 8);
        memcpy(H + o_Poi + an * 8, g.Po_idx.data(), g.Po_idx.size() * 4);
        memcpy(H + o_Pov + an * 16, g.Po_val.data(), g.Po_val.size() * 8);
        if (g.n > 0) memcpy(H + o_cp + (an + b) * 4, g.csc_ptr.data(), g.csc_ptr.size() * 4);
        else *(int32_t *)(H + o_cp + (an + b) * 4) = 0;
        memcpy(H + o_cr + az * 4, g.csc_row.data(), g.csc_row.size() * 4);
        memcpy(H + o_cv + az * 8, g.csc_val.data(), g.csc_val.size() * 8);
        memcpy(H + o_sep + (size_t)b * 128, g.sep, 128);
        memcpy(H + o_oi + (size_t)off[b] * 12, g.out_idx.data(), g.out_idx.size() * 4);
        an += g.n; am += g.m; az += g.csc_row.size();
    }
    PQP_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = h->stream;
    PQP_CUDA(cudaEventRecord(h->ev[0], st));
    PQP_CUDA(cudaMemcpyAsync(h->d_gen, H, o_end, cudaMemcpyHostToDevice, st));
    PQP_CUDA(cudaMemcpyAsync(h->d_ref, ref, T * sizeof(pqp_state), cudaMemcpyHostToDevice, st));
    PQP_CUDA(cudaEventRecord(h->ev[1], st));
    char *D = h->d_gen;
    pqp::GenView gv;
    gv.batch = batch; gv.meta = (const int32_t *)(D + o_meta);
    gv.A_col = (const int32_t *)(D + o_Acol); gv.A_val = (const double *)(D + o_Aval);
    gv.l = (const double *)(D + o_l); gv.u = (const double *)(D + o_u); gv.Pd = (const double *)(D + o_Pd);
    gv.Po_idx = (const int32_t *)(D + o_Poi); gv.Po_val = (const double *)(D + o_Pov);
    gv.csc_ptr = (const int32_t *)(D + o_cp); gv.csc_row = (const int32_t *)(D + o_cr); gv.csc_val = (const double *)(D + o_cv);
    gv.sep = (const int32_t *)(D + o_sep); gv.out_idx = (const int32_t *)(D + o_oi);
    gv.ref = h->d_ref; gv.out_states = h->d_out; gv.out_frenet = out_frenet ? h->d_frenet : nullptr;
    gv.status = h->d_status; gv.iters = h->d_iters;
    {
        int smem_doubles = (int)(smem / sizeof(double));
        void *args[] = {(void *)&h->dprm_gen[formulation == PQP_FORM_K ? 0 : 1], (void *)&gv, (void *)&smem_doubles};
        PQP_CUDA(cudaLaunchKernel(pqp_gen_kernel_fn(), dim3(batch), dim3(32), args, smem, st));
    }
    PQP_CUDA(cudaEventRecord(h->ev[2], st));
    PQP_CUDA(cudaMemcpyAsync(out_states, h->d_out, T * sizeof(pqp_state), cudaMemcpyDeviceToHost, st));
    if (out_frenet) PQP_CUDA(cudaMemcpyAsync(out_frenet, h->d_frenet, T * 3 * sizeof(double), cudaMemcpyDeviceToHost, st));
    PQP_CUDA(cudaMemcpyAsync(status, h->d_status, B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    std::vector<int32_t> iters_local;
    int32_t *it_dst = iters;
    if (!it_dst && stats) { iters_local.resize(B); it_dst = iters_local.data(); }
    if (it_dst) PQP_CUDA(cudaMemcpyAsync(it_dst, h->d_iters, B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    PQP_CUDA(cudaEventRecord(h->ev[3], st));
    PQP_CUDA(cudaStreamSynchronize(st));
    if (stats) {
        PQP_CUDA(cudaEventElapsedTime(&stats->h2d_ms, h->ev[0], h->ev[1]));
        PQP_CUDA(cudaEventElapsedTime(&stats->kernel_ms, h->ev[1], h->ev[2]));
        PQP_CUDA(cudaEventElapsedTime(&stats->d2h_ms, h->ev[2], h->ev[3]));
        stats->h2d_bytes = (int64_t)(o_end + T * sizeof(pqp_state));
        stats->d2h_bytes = (int64_t)(T * sizeof(pqp_state) + (out_frenet ? T * 3 * sizeof(double) : 0) + B * 8);
        stats->kernel_launches = 1;
        for (size_t b = 0; b < B; ++b) {
            stats->total_iters += it_dst[b];
            stats->max_iters = std::max(stats->max_iters, it_dst[b]);
            stats->n_solved += (status[b] == PQP_SOLVED);
        }
    }
    return PQP_OK;
}

}  // extern "C"

// PQP_GENERIC_KPC=1 / PQP_GENERIC_K=1 (diagnostics): route "KPC" / "K" through the host-assembled generic kernel
// (round 1's path for them) instead of their thread-per-station classes
static bool generic_form(int formulation) {
    static const bool generic_kpc = [] { const char *e = getenv("PQP_GENERIC_KPC"); return e && *e == '1'; }();
    static const bool generic_k = [] { const char *e = getenv("PQP_GENERIC_K"); return e && *e == '1'; }();
    return (formulation == PQP_FORM_KPC && generic_kpc) || (formulation == PQP_FORM_K && generic_k);
}
static int solve_batch_classes(pqp_handle *h, int formulation, const int32_t *forms, int batch, const int32_t *n_points,
                               const pqp_state *ref, const pqp_station_bounds *bounds, const double *x0,
                               const double *end_heading, const double *max_k, const double *max_kp,
                               const int32_t *param_index, pqp_state *out_states, double *out_frenet, int32_t *status,
                               int32_t *iters, pqp_stats *stats);

extern "C" {

int pqp_solve_batch(pqp_handle *h, int formulation, int batch, const int32_t *n_points, const pqp_state *ref,
                    const pqp_station_bounds *bounds, const double *x0, const double *end_heading,
                    const double *max_k, const double *max_kp, pqp_state *out_states, double *out_frenet,
                    int32_t *status, int32_t *iters, pqp_stats *stats) {
    return pqp_solve_batch_sets(h, formulation, batch, n_points, ref, bounds, x0, end_heading, max_k, max_kp, nullptr,
                                out_states, out_frenet, status, iters, stats);
}

int pqp_solve_batch_sets(pqp_handle *h, int formulation, int batch, const int32_t *n_points, const pqp_state *ref,
                         const pqp_station_bounds *bounds, const double *x0, const double *end_heading,
                         const double *max_k, const double *max_kp, const int32_t *param_index, pqp_state *out_states,
                         double *out_frenet, int32_t *status, int32_t *iters, pqp_stats *stats) {
    if (!h || batch < 0 || (batch > 0 && (!n_points || !ref || !bounds || !x0 || !end_heading || !out_states || !status))) {
        set_err("pqp_solve_batch(_sets): bad argument");
        return PQP_ERR_ARG;
    }
    if (formulation != PQP_FORM_KP && formulation != PQP_FORM_K && formulation != PQP_FORM_KPC) {
        set_err("unknown formulation");
        return PQP_ERR_ARG;
    }
    if (stats) memset(stats, 0, sizeof(*stats));
    if (batch == 0) return PQP_OK;
    if (formulation == PQP_FORM_KPC && (!max_k || !max_kp)) {
        set_err("KPC needs max_k and max_kp (ReferencePath::getMaxKList / getMaxKpList; pqp_update_limits)");
        return PQP_ERR_ARG;
    }
    if (generic_form(formulation)) {
        if (param_index) {
            set_err("the host-assembled diagnostic path (PQP_GENERIC_K / PQP_GENERIC_KPC) takes no parameter-set index");
            return PQP_ERR_UNSUPPORTED;
        }
        return solve_batch_generic(h, formulation, batch, n_points, ref, bounds, x0, end_heading, max_k, max_kp, out_states,
                                   out_frenet, status, iters, stats);
    }
    return solve_batch_classes(h, formulation, nullptr, batch, n_points, ref, bounds, x0, end_heading, max_k, max_kp,
                               param_index, out_states, out_frenet, status, iters, stats);
}

int pqp_solve_batch_forms(pqp_handle *h, int batch, const int32_t *n_points, const pqp_state *ref,
                          const pqp_station_bounds *bounds, const double *x0, const double *end_heading,
                          const double *max_k, const double *max_kp, const int32_t *param_index,
                          const int32_t *formulation, pqp_state *out_states, double *out_frenet, int32_t *status,
                          int32_t *iters, pqp_stats *stats) {
    if (!h || batch < 0 ||
        (batch > 0 && (!n_points || !ref || !bounds || !x0 || !end_heading || !formulation || !out_states || !status))) {
        set_err("pqp_solve_batch_forms: bad argument");
        return PQP_ERR_ARG;
    }
    if (stats) memset(stats, 0, sizeof(*stats));
    bool any_kpc = false, any_generic = false;
    for (int b = 0; b < batch; ++b) {
        any_kpc |= formulation[b] == PQP_FORM_KPC;
        any_generic |= pqp::form_in_mask(formulation[b], 7) && generic_form(formulation[b]);
    }
    if (any_kpc && (!max_k || !max_kp)) {
        set_err("a \"KPC\" path needs max_k and max_kp (ReferencePath::getMaxKList / getMaxKpList; pqp_update_limits)");
        return PQP_ERR_ARG;
    }
    if (any_generic) {
        set_err("the host-assembled diagnostic path (PQP_GENERIC_K / PQP_GENERIC_KPC) takes no per-path formulation");
        return PQP_ERR_UNSUPPORTED;
    }
    if (batch == 0) return PQP_OK;
    if (h->defer_sync) {
        set_err("pqp_solve_batch_forms: no per-path formulation on a multi-device handle");
        return PQP_ERR_UNSUPPORTED;
    }
    return solve_batch_classes(h, PQP_FORM_KP, formulation, batch, n_points, ref, bounds, x0, end_heading, max_k, max_kp,
                               param_index, out_states, out_frenet, status, iters, stats);
}

}  // extern "C"

// The host-buffer solve on the kernel classes: pqp_solve_batch_sets (forms NULL: `formulation` for every path) and
// pqp_solve_batch_forms (forms [batch]: every path's own; one that is not a PQP_FORM_* is rejected like an out-of-range
// set index).  Arguments checked by the callers.
static int solve_batch_classes(pqp_handle *h, int formulation, const int32_t *forms, int batch, const int32_t *n_points,
                               const pqp_state *ref, const pqp_station_bounds *bounds, const double *x0,
                               const double *end_heading, const double *max_k, const double *max_kp,
                               const int32_t *param_index, pqp_state *out_states, double *out_frenet, int32_t *status,
                               int32_t *iters, pqp_stats *stats) {
    bool kpc_classes = formulation == PQP_FORM_KPC;
    for (int b = 0; forms && b < batch; ++b) kpc_classes |= forms[b] == PQP_FORM_KPC;
    if (batch > h->max_batch) {
        set_err("batch exceeds the handle's max_batch");
        return PQP_ERR_CAPACITY;
    }
    if (param_index && h->defer_sync) {
        set_err("pqp_solve_batch_sets: no parameter-set index on a multi-device handle");
        return PQP_ERR_UNSUPPORTED;
    }
    // offsets and keep_control_steps per path; launch segment set * kNumVariants + shape class, segment G = the paths
    // whose set index or formulation is out of range (rejected, not launched)
    const int n_sets = param_index ? (int)h->dsets.size() : 1;
    const int G = n_sets * kNumVariants;
    long long total = 0;
    h->h_off[0] = 0;
    std::vector<int32_t> keep((size_t)batch);
    for (int b = 0; b < batch; ++b) {
        const int n = n_points[b];
        if (n < 0) { set_err("negative n_points"); return PQP_ERR_ARG; }
        total += n;
        if (total > h->max_total) { set_err("station count exceeds the handle's max_total_points"); return PQP_ERR_CAPACITY; }
        h->h_off[b + 1] = (int32_t)total;
        keep[b] = (n >= 2) ? pqp_keep_control_steps(forms ? forms[b] : formulation, ref + h->h_off[b], n) : 1;
    }
    // The batch is cut into contiguous chunks of paths that are pipelined over two streams: the
    // upload of chunk k+1 and the download of chunk k-1 overlap the kernels of chunk k (whose CTAs
    // also fill the SMs the previous chunk's tail leaves idle).  Small batches stay in one chunk.
    const int n_chunks = std::max(1, std::min(kMaxChunks, batch / 192));
    int cb[kMaxChunks + 1];
    cb[0] = 0;
    for (int k = 1; k <= n_chunks; ++k) {
        // equal station counts per chunk
        const long long target = total * k / n_chunks;
        int b = cb[k - 1];
        while (b < batch && h->h_off[b] < target) ++b;
        cb[k] = (k == n_chunks) ? batch : std::max(b, cb[k - 1]);
    }
    h->plan.valid = false;   // (this call rewrites the order array the class plan of the device entry points refers to)
    // per chunk: per-segment order (written into the pinned order array at the chunk's range), the rejected paths last;
    // small batches by the input-derived key, as pqp_order_kernel does on the device
    const bool keyed = batch <= kAutoOrderMax && auto_order_enabled();
    std::vector<double> okey(keyed ? (size_t)batch : 0);
    for (int b = 0; keyed && b < batch; ++b) {
        const int n = n_points[b];
        okey[b] = n >= 1 ? order_key(n, x0[3 * (size_t)b], bounds[h->h_off[b]].c0_lb, bounds[h->h_off[b]].c0_ub) : 0.0;
    }
    auto before = [&](int a, int b) { return keyed ? okey[a] > okey[b] : n_points[a] > n_points[b]; };
    std::vector<int> count_cv((size_t)n_chunks * (G + 1)), start_cv((size_t)n_chunks * (G + 2));
    std::vector<size_t> smem_cv((size_t)n_chunks * (G + 1));
    for (int k = 0; k < n_chunks; ++k)
        plan_classes(h, batch, cb[k], cb[k + 1], n_sets, n_points, keep.data(), formulation, forms, param_index, before,
                     count_cv.data() + (size_t)k * (G + 1), start_cv.data() + (size_t)k * (G + 2),
                     smem_cv.data() + (size_t)k * (G + 1));
    PQP_CUDA(cudaSetDevice(h->device));
    const size_t B = (size_t)batch, T = (size_t)total;
    pqp::BatchView bv;
    bv.batch = batch; bv.n_points = h->d_n; bv.offsets = h->d_off; bv.ref = h->d_ref; bv.bounds = h->d_bounds;
    bv.x0 = h->d_x0; bv.end_heading = h->d_end; bv.out_states = h->d_out;
    bv.out_frenet = (out_frenet || h->force_frenet) ? h->d_frenet : nullptr;
    bv.status = h->d_status; bv.iters = h->d_iters;
    bv.workspace = h->d_ws;
    bv.debug = nullptr;
    if (kpc_classes) {
        if (!h->d_max_k) {
            PQP_CUDA(cudaMalloc(&h->d_max_k, (size_t)h->max_total * sizeof(double)));
            PQP_CUDA(cudaMalloc(&h->d_max_kp, (size_t)h->max_total * sizeof(double)));
        }
        bv.max_k = h->d_max_k; bv.max_kp = h->d_max_kp;
    }
#ifdef PQP_PHASE_TIMING
    static long long *d_dbg = nullptr;
    if (!d_dbg) cudaMalloc(&d_dbg, sizeof(long long) * 64 * 65536);
    cudaMemsetAsync(d_dbg, 0, sizeof(long long) * 16 * (size_t)batch, h->stream);
    cudaStreamSynchronize(h->stream);
    bv.debug = d_dbg;
#endif
    std::vector<int32_t> iters_local;
    int32_t *it_dst = iters;
    if (!it_dst && stats) { iters_local.resize(B); it_dst = iters_local.data(); }
    cudaStream_t sts[2] = {h->stream, h->stream2};
    int launches = 0;
    bool ev1_done = false;
    // Once copies into the caller's buffers are in flight, no error return may leave them running: both lanes are
    // drained first (PQP_CUDA_DRAIN = PQP_CUDA with that drain).
    auto drain = [&]() {
        cudaStreamSynchronize(sts[0]); cudaStreamSynchronize(sts[1]);
        for (auto &q : h->cls_stream) cudaStreamSynchronize(q);
    };
#define PQP_CUDA_DRAIN(call)                                                 \
    do {                                                                     \
        cudaError_t e_ = (call);                                             \
        if (e_ != cudaSuccess) {                                             \
            pqp_set_err("%s failed: %s", #call, cudaGetErrorString(e_));     \
            drain();                                                         \
            return PQP_ERR_CUDA;                                             \
        }                                                                    \
    } while (0)
    // ev[0] start | ev[1] first kernel may start | ev[2] last kernel done | ev[3] all done
    PQP_CUDA(cudaEventRecord(h->ev[0], sts[0]));
    PQP_CUDA(cudaStreamWaitEvent(sts[1], h->ev[0], 0));
    // the offsets array is indexed by absolute path id and read by every chunk's kernel
    PQP_CUDA(cudaMemcpyAsync(h->d_off, h->h_off, (B + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, sts[0]));
    PQP_CUDA(cudaMemcpyAsync(h->d_order, h->h_order, B * sizeof(int32_t), cudaMemcpyHostToDevice, sts[0]));
    PQP_CUDA(cudaEventRecord(h->ev_chunk[0], sts[0]));
    PQP_CUDA(cudaStreamWaitEvent(sts[1], h->ev_chunk[0], 0));
    for (int k = 0; k < n_chunks; ++k) {
        cudaStream_t st = sts[k & 1];
        const int pb = cb[k], pe = cb[k + 1];
        if (pe == pb) continue;
        const size_t o0 = (size_t)h->h_off[pb], nT = (size_t)h->h_off[pe] - o0, nB = (size_t)(pe - pb);
        PQP_CUDA_DRAIN(cudaMemcpyAsync(h->d_n + pb, n_points + pb, nB * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        PQP_CUDA_DRAIN(cudaMemcpyAsync(h->d_ref + o0, ref + o0, nT * sizeof(pqp_state), cudaMemcpyHostToDevice, st));
        PQP_CUDA_DRAIN(cudaMemcpyAsync(h->d_bounds + o0, bounds + o0, nT * sizeof(pqp_station_bounds), cudaMemcpyHostToDevice, st));
        PQP_CUDA_DRAIN(cudaMemcpyAsync(h->d_x0 + 3 * (size_t)pb, x0 + 3 * (size_t)pb, nB * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
        PQP_CUDA_DRAIN(cudaMemcpyAsync(h->d_end + pb, end_heading + pb, nB * sizeof(double), cudaMemcpyHostToDevice, st));
        if (kpc_classes) {
            PQP_CUDA_DRAIN(cudaMemcpyAsync(h->d_max_k + o0, max_k + o0, nT * sizeof(double), cudaMemcpyHostToDevice, st));
            PQP_CUDA_DRAIN(cudaMemcpyAsync(h->d_max_kp + o0, max_kp + o0, nT * sizeof(double), cudaMemcpyHostToDevice, st));
        }
        if (!ev1_done) { PQP_CUDA_DRAIN(cudaEventRecord(h->ev[1], st)); ev1_done = true; }
        // One launch per segment of the chunk (and one for its rejected paths); a mixed-length chunk has several: they go
        // out on the class lanes (forked after the chunk's upload, joined before its download), longest class first, so
        // that they overlap instead of each waiting for the tail of the one before.
        const int *count_k = count_cv.data() + (size_t)k * (G + 1), *start_k = start_cv.data() + (size_t)k * (G + 2);
        const int rc = launch_class_set(h, bv, n_sets, count_k, start_k, smem_cv.data() + (size_t)k * (G + 1), h->d_order,
                                        st, &launches, count_k[G], start_k[G]);
        if (rc != PQP_OK) { drain(); return rc; }
        PQP_CUDA_DRAIN(cudaEventRecord(h->ev_chunk[1 + k], st));   // this chunk's kernels done
        PQP_CUDA_DRAIN(cudaMemcpyAsync(out_states + o0, h->d_out + o0, nT * sizeof(pqp_state), cudaMemcpyDeviceToHost, st));
        if (out_frenet)
            PQP_CUDA_DRAIN(cudaMemcpyAsync(out_frenet + 3 * o0, h->d_frenet + 3 * o0, nT * 3 * sizeof(double), cudaMemcpyDeviceToHost, st));
        PQP_CUDA_DRAIN(cudaMemcpyAsync(status + pb, h->d_status + pb, nB * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        if (it_dst) PQP_CUDA_DRAIN(cudaMemcpyAsync(it_dst + pb, h->d_iters + pb, nB * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    }
    if (!ev1_done) PQP_CUDA_DRAIN(cudaEventRecord(h->ev[1], sts[0]));   // (every chunk was empty)
    // join: stream 0 waits for every chunk's kernels (ev[2]) and then for stream 1's copies (ev[3])
    for (int k = 0; k < n_chunks; ++k)
        if (cb[k + 1] > cb[k] && (k & 1)) PQP_CUDA_DRAIN(cudaStreamWaitEvent(sts[0], h->ev_chunk[1 + k], 0));
    PQP_CUDA_DRAIN(cudaEventRecord(h->ev[2], sts[0]));
    PQP_CUDA_DRAIN(cudaEventRecord(h->ev_chunk[kMaxChunks + 1], sts[1]));
    PQP_CUDA_DRAIN(cudaStreamWaitEvent(sts[0], h->ev_chunk[kMaxChunks + 1], 0));
    PQP_CUDA_DRAIN(cudaEventRecord(h->ev[3], sts[0]));
    if (h->defer_sync) {   // pqp_multi_solve_batch: every device is enqueued first, the caller synchronises (and has passed `iters`)
        h->deferred_launches = launches;
        return PQP_OK;
    }
    PQP_CUDA(cudaStreamSynchronize(sts[0]));
#undef PQP_CUDA_DRAIN
#ifdef PQP_PHASE_TIMING
    {
        std::vector<long long> dbg(16 * (size_t)batch);
        cudaMemcpy(dbg.data(), bv.debug, dbg.size() * sizeof(long long), cudaMemcpyDeviceToHost);
        const char *names[6] = {"a1 publish", "a2 rhs", "b1 sep rhs", "b2 Sinv g || y", "b3 x-tilde", "c update"};
        for (int wsel = 0; wsel < 2; ++wsel) {
            double tot[6] = {0}, its = 0;
            for (int b = 0; b < batch; ++b) {
                for (int k = 0; k < 6; ++k) tot[k] += (double)dbg[(2 * (size_t)b + wsel) * 8 + k];
                its += (double)dbg[(2 * (size_t)b + wsel) * 8 + 6];
            }
            fprintf(stderr, "[phase cycles per iteration, warp %d]", wsel);
            double sum = 0;
            for (int k = 0; k < 6; ++k) { fprintf(stderr, " %s=%.0f", names[k], tot[k] / its); sum += tot[k] / its; }
            fprintf(stderr, " | total=%.0f (%.0f iterations)\n", sum, its / batch);
        }
        {
            std::vector<long long> g(4 * (size_t)batch);
            cudaMemcpy(g.data(), bv.debug + 16 * 65536, g.size() * sizeof(long long), cudaMemcpyDeviceToHost);
            double sc = 0, rf = 0, ck = 0, tot = 0, loop = 0, nref = 0;
            long long nref_max = 0;
            for (int b = 0; b < batch; ++b) {
                sc += (double)g[4 * (size_t)b]; rf += (double)g[4 * (size_t)b + 1]; ck += (double)g[4 * (size_t)b + 2];
                nref += (double)g[4 * (size_t)b + 3];
                nref_max = std::max(nref_max, g[4 * (size_t)b + 3]);
                tot += (double)dbg[(2 * (size_t)b) * 8 + 7];
                for (int k = 0; k < 6; ++k) loop += (double)dbg[(2 * (size_t)b) * 8 + k];
            }
            std::vector<long long> g2(8 * (size_t)batch);
            cudaMemcpy(g2.data(), bv.debug + 20 * 65536, g2.size() * sizeof(long long), cudaMemcpyDeviceToHost);
            double rt[8] = {0};
            for (int b = 0; b < batch; ++b) for (int k = 0; k < 8; ++k) rt[k] += (double)g2[8 * (size_t)b + k] / batch;
            fprintf(stderr, "[refactor cycles per path, all refactorisations] weights=%.0f assembly=%.0f interior LDL=%.0f spikes=%.0f schur=%.0f block LDL=%.0f dense Sinv=%.0f dense interiors=%.0f\n",
                    rt[0], rt[1], rt[2], rt[3], rt[4], rt[5], rt[6], rt[7]);
            fprintf(stderr, "[cycles per path] kernel=%.0f  iterations(a..c)=%.0f  scaling=%.0f  refactor(all)=%.0f  check blocks(all, without their refactors)=%.0f\n",
                    tot / batch, loop / batch, sc / batch, rf / batch, ck / batch);
            fprintf(stderr, "[refactorisations per path] mean=%.2f max=%lld\n", nref / batch, nref_max);
            std::vector<long long> g3(32 * (size_t)batch);
            cudaMemcpy(g3.data(), bv.debug + 32 * 65536, g3.size() * sizeof(long long), cudaMemcpyDeviceToHost);
            for (int w = 0; w < 4; ++w) {
                double ckp[6] = {0};
                for (int b = 0; b < batch; ++b) for (int k = 0; k < 6; ++k) ckp[k] += (double)g3[32 * (size_t)b + 8 * w + k] / batch;
                fprintf(stderr, "[check-block cycles per path, all checks, warp %d] loads+publish x=%.0f primal=%.0f barrier=%.0f dual=%.0f certificate=%.0f reduction=%.0f\n",
                        w, ckp[0], ckp[1], ckp[2], ckp[3], ckp[4], ckp[5]);
            }
        }
    }
#endif
    if (stats) {
        // Consecutive, non-overlapping spans of the pipelined call: head (before the first kernel
        // can start) | middle (first kernel start -> last kernel end; later chunks' copies overlap
        // it) | tail (remaining downloads).  Their sum is the whole device-side time of the call.
        PQP_CUDA(cudaEventElapsedTime(&stats->h2d_ms, h->ev[0], h->ev[1]));
        PQP_CUDA(cudaEventElapsedTime(&stats->kernel_ms, h->ev[1], h->ev[2]));
        PQP_CUDA(cudaEventElapsedTime(&stats->d2h_ms, h->ev[2], h->ev[3]));
        stats->h2d_bytes = (int64_t)(B * sizeof(int32_t) * 3 + sizeof(int32_t) + T * (sizeof(pqp_state) + sizeof(pqp_station_bounds)) + B * 4 * sizeof(double) +
                                     (kpc_classes ? T * 2 * sizeof(double) : 0));
        stats->d2h_bytes = (int64_t)(T * sizeof(pqp_state) + (out_frenet ? T * 3 * sizeof(double) : 0) + B * sizeof(int32_t) * 2);
        stats->kernel_launches = launches;
        for (size_t b = 0; b < B; ++b) {
            stats->total_iters += it_dst[b];
            stats->max_iters = std::max(stats->max_iters, it_dst[b]);
            stats->n_solved += (status[b] == PQP_SOLVED);
        }
    }
    return PQP_OK;
}

