// one kernel per translation unit: see pqp_kernels.h
#include "pqp_kernels.h"
#include "pqp_kp_core.cuh"

// One warp (= one CTA) per path.  Shared memory holds the whole ADMM state and the KKT factor.
__global__ void __launch_bounds__(32)
pqp_kp_solve_kernel(const __grid_constant__ pqp::DevParams prm, const __grid_constant__ pqp::BatchView bv,
                    const int32_t *__restrict__ order, int smem_doubles) {
    extern __shared__ double pqp_smem[];
    int prob = blockIdx.x;
    if (order) prob = order[prob];
    pqp::Warp w;
    pqp::kp_solve_path(w, prm, bv, prob, pqp_smem, (size_t)smem_doubles);
}

// Shared memory for a path: with the scalings on chip when that fits the 227 KB a CTA can opt into, else with the
// scalings in the global workspace (the kernel makes the same choice from the size it is launched with).  The choice is
// per path: a launch carries the largest need of the paths it may get, never more than the opt-in, so a path whose
// on-chip layout fits the opt-in finds at least that much and one whose layout does not finds less.  A launch sized
// for more paths (the device dispatch) cannot move a path's scalings.
static size_t g_cap = 232448;   // opt-in shared memory per block of the device in use (H100: 227 KB); pqp_create passes the real value
void pqp_k1_set_smem_cap(int bytes) { if (bytes > 0) g_cap = (size_t)bytes; }
static size_t g_smem(int n, int keep) {
    const pqp::KpDims d = pqp::kp_dims(n, keep);
    const size_t full = pqp::kp_smem_doubles(d) * sizeof(double);
    return full <= g_cap ? full : pqp::kp_smem_doubles(d, true) * sizeof(double);
}
static bool g_fits(int, int keep) { return keep <= 10; }
void pqp_variant_k1_generic(PqpVariant *out) {
    *out = PqpVariant{0, pqp::kMaxBand, 32, (const void *)pqp_kp_solve_kernel, g_smem, g_fits, "pqp_kp_solve_kernel"};
}
