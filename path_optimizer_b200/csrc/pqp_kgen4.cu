// one kernel per translation unit: see pqp_kernels.h
#include "pqp_kernels.h"
#include "pqp_gen_core.cuh"

// Generic banded-QP kernel with 4-unknown separators and a linear cost term: the TENSION2 smoothing QP of
// pqp_smooth_reference_device (pqp_env.cu), one warp per path.  q: [sum n] in band order.
__global__ void __launch_bounds__(32)
pqp_gen4_solve_kernel(const __grid_constant__ pqp::DevParams prm, const __grid_constant__ pqp::GenView gv, int smem_doubles,
                      const double *q) {
    extern __shared__ double pqp_smem[];
    pqp::Warp w;
    pqp::gen_solve_qp<4, true>(w, prm, gv, blockIdx.x, pqp_smem, (size_t)smem_doubles, q);
}

const void *pqp_gen4_kernel_fn() { return (const void *)pqp_gen4_solve_kernel; }
