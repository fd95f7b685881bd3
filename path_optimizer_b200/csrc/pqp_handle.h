// pqp_handle.h -- the opaque handle behind include/pqp.h, shared by the translation units of
// libpqp.so (pqp_capi.cu: the QP; pqp_env.cu: bounds / collision check / densify / plan chain).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <vector>

#include "../../include/pqp.h"
#include "pqp_device.cuh"

#define PQP_MAX_CHUNKS 4
#define PQP_CLASS_LANES 4
#define PQP_MAX_VARIANTS 24
#define PQP_DISPATCH_SLOTS 4

struct pqp_handle {
    int device = 0;
    int max_batch = 0, max_total = 0;
    int smem_optin = 0;
    int num_sms = 0;
    pqp_params params;               // set 0
    pqp::DevParams dprm;
    pqp::DevParams dprm_gen[2];
    // the parameter sets (pqp_set_param_sets); params / dprm above are set 0
    std::vector<pqp_params> sets;
    std::vector<pqp::DevParams> dsets;
    cudaStream_t stream = nullptr;
    cudaStream_t stream2 = nullptr;                 // second lane of the host-buffer pipeline
    cudaEvent_t ev_chunk[PQP_MAX_CHUNKS + 2] = {};  // [0] shared arrays uploaded, [1+k] chunk k kernels done, [last] lane 2 drained
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    cudaStream_t cls_stream[PQP_CLASS_LANES] = {};  // lanes for the per-class launches of a mixed-length batch
    cudaEvent_t ev_fork = nullptr, ev_cls[PQP_CLASS_LANES] = {};
    // pqp_multi_solve_batch enqueues the host-buffer call on every device before synchronising any
    bool defer_sync = false;
    bool force_frenet = false;       // keep the Frenet states on the device even when the caller passes no host buffer
    int deferred_launches = 0;
    // NCCL communicator bound to this handle's device (pqp_multi.cu; void*: nccl.h stays out of this header)
    void *nccl_comm = nullptr;
    // cached choice of pqp_solve_batch_device for (max_n_points, min_keep, max_keep)
    int dc_nmax = -1, dc_klo = -1, dc_khi = -1, dc_skip = -1, dc_v = -1, dc_form = 0;
    size_t dc_smem = 0;
    // class plan of the last pqp_launch_kp_classes call (reused while the batch shape stays the same)
    // launch segment g = set * (classes) + class; the entries past the last segment name the paths whose set index is
    // out of range (count[last] of them)
    struct ClassPlan {
        bool valid = false;
        int skip = 0, form = 0, n_sets = 1;
        cudaStream_t stream = nullptr;
        std::vector<int32_t> n, keep, set;   // (set: empty without a set index)
        std::vector<int32_t> forms;          // formulation of every path (empty without a per-path formulation)
        std::vector<int> count, start;
        std::vector<size_t> smem;
    } plan;
    // pqp_set_order_hint: expected ADMM iterations per path (e.g. the previous planning cycle's counts); launch order
    // inside a class becomes longest-expected-first
    std::vector<int32_t> order_hint;
    // device dispatch (pqp_launch_dispatch): the class table of every formulation (pqp_dispatch.h; rows x
    // cls_ncols[form] entries at d_cls_table + cls_off[form]), one sort key per path, and the station counts, status and
    // iterations the dispatched launches see: max_batch + 1 entries, the last one a path of 0 stations for unused order
    // entries
    int8_t *d_cls_table = nullptr;
    int cls_ncols[3] = {}, cls_off[3] = {};
    int32_t *d_disp_key = nullptr;
    int32_t *d_disp_n = nullptr, *d_disp_status = nullptr, *d_disp_iters = nullptr;
    // the dispatch's sort scratch, for disp_cap parameter sets: per-(set, class) order segments (disp_cap x every class
    // x max_batch) and the (set, class, length) histogram, in global memory with a set index (disp_cap x every class x
    // (largest ncols + 1)).  pqp_create allocates it for one set; it grows on
    // demand and an outgrown pair stays allocated until pqp_destroy: a graph captured before the growth still reads it.
    int32_t *d_disp_order = nullptr, *d_disp_hist = nullptr;
    int disp_cap = 0;
    std::vector<void *> retired;
    // launches the dispatch makes for (form_mask, max_n per formulation, min_keep, max_keep as passed), for the last
    // PQP_DISPATCH_SLOTS such bounds
    struct DispatchLaunches {
        bool valid = false;
        int form_mask = 0, min_keep = 0, max_keep = 0;
        int max_n[3] = {};
        bool reach[PQP_MAX_VARIANTS] = {};
        int min_n[PQP_MAX_VARIANTS] = {};
        size_t smem[PQP_MAX_VARIANTS] = {};
    } disp[PQP_DISPATCH_SLOTS];
    int disp_next = 0;
    // device buffers for the host-pointer entry point
    int32_t *d_n = nullptr, *d_off = nullptr, *d_order = nullptr, *d_status = nullptr, *d_iters = nullptr;
    int32_t *d_order_auto = nullptr;   // launch order computed on the device (pqp_solve_batch_device, small batches)
    pqp_state *d_ref = nullptr, *d_out = nullptr;
    pqp_station_bounds *d_bounds = nullptr;
    double *d_x0 = nullptr, *d_end = nullptr, *d_frenet = nullptr, *d_ws = nullptr;
    double *d_max_k = nullptr, *d_max_kp = nullptr;   // KPC limits of the host-buffer / plan entry points (allocated on first use)
    // pinned host scratch for the small per-batch arrays
    int32_t *h_off = nullptr, *h_order = nullptr;
    // generic-kernel staging (grow-only): one device blob + one pinned host blob
    char *d_gen = nullptr, *h_gen = nullptr;
    size_t gen_cap = 0;
    // state of the stages either side of the QP (pqp_env.cu): map, scratch buffers
    void *env = nullptr;
    void (*env_free)(void *) = nullptr;
};

// Internal (pqp_capi.cu): launch the KP solve kernels for paths whose station counts n[b] are known on the host,
// each path on the kernel class picked for (n[b], its keep_control_steps), longest first inside a class.  The
// device-side counts (BatchView::n_points) must equal n.  keep[b] = keep_control_steps per path, or NULL to derive
// them from the host copy `ref` of the reference states.  Used by pqp_plan_batch after the bounds stage and by
// pqp_solve_batch_device_classes.
// `set` [batch]: parameter set of every path (host), NULL: set 0.  A path whose set lies outside the handle's sets is not
// launched: a small kernel reports it PQP_INVALID_PROBLEM (0 iterations, NaN states).
// `forms` [batch]: formulation of every path (host), NULL: `form` for every path.  With it each path takes the class of
// its own formulation (bv.max_k / max_kp set when any path is "KPC"); a path whose formulation is not one of
// PQP_FORM_* is not launched and reports PQP_INVALID_PROBLEM.
int pqp_launch_kp_classes(pqp_handle *h, const pqp::BatchView &bv, int batch, const int32_t *n, const int32_t *off,
                          const pqp_state *ref, const int32_t *keep, cudaStream_t st, int *launches, int form = 0 /* PQP_FORM_KP; 2 = KPC (bv.max_k / max_kp set) */,
                          const int32_t *set = nullptr, const int32_t *forms = nullptr);

// Internal (pqp_capi.cu): the same launches when the station counts exist on the device only.  A dispatch kernel reads
// them, derives keep_control_steps from the device-side reference states, looks every path up in the class table of its
// formulation and sorts the paths into per-(set, class) order segments (longest first); every (set, class) pair the
// bounds can reach is launched over its segment.  No host synchronisation, and no allocation after a call with the same
// or a smaller set count.
// `form_mask` (1 << PQP_FORM_*, nonzero): the formulations launched.  `d_form` [batch] (device) names every path's
// formulation; NULL: every path is the one formulation of a one-bit mask.  max_n[f] bounds the paths of formulation f
// (0: unknown); min_keep / max_keep (0: unknown) apply to "KP".  bv.max_k / max_kp must be set when the mask holds "KPC".
// `total` = offsets[batch] bounds the grid of each class.
// `d_set` [batch] (device): parameter set of every path, NULL: set 0; with it every set below n_sets = min(n_param_sets,
// the handle's count) (n_param_sets 0: the handle's count) is launched.
// A path whose formulation lies outside the mask, or whose set or length lies outside the bounds, reports
// PQP_INVALID_PROBLEM.
int pqp_launch_dispatch(pqp_handle *h, const pqp::BatchView &bv, int form_mask, const int32_t *d_form, int batch,
                        int total, const int max_n[3], int min_keep, int max_keep, cudaStream_t st, int *launches,
                        const int32_t *d_set = nullptr, int n_param_sets = 0);

// thread-local error text returned by pqp_last_error()
extern thread_local char pqp_g_err[512];
inline void pqp_set_err(const char *fmt, const char *a = "", const char *b = "") {
    snprintf(pqp_g_err, sizeof(pqp_g_err), fmt, a, b);
}

#define PQP_CUDA(call)                                                       \
    do {                                                                     \
        cudaError_t e_ = (call);                                             \
        if (e_ != cudaSuccess) {                                             \
            pqp_set_err("%s failed: %s", #call, cudaGetErrorString(e_));     \
            return PQP_ERR_CUDA;                                             \
        }                                                                    \
    } while (0)
