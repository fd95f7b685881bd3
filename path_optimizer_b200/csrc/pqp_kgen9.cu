// one kernel per translation unit: see pqp_kernels.h
#include "pqp_kernels.h"
#include "pqp_gen_core.cuh"

// Generic banded-QP kernel with 9-unknown separators (three stations) and six P partners per unknown: the TENSION
// smoothing QP of pqp_smooth_reference_tension_device (pqp_env.cu), one warp per path.  q = 0.
__global__ void __launch_bounds__(32)
pqp_gen9_solve_kernel(const __grid_constant__ pqp::DevParams prm, const __grid_constant__ pqp::GenView gv, int smem_doubles) {
    extern __shared__ double pqp_smem[];
    pqp::Warp w;
    pqp::gen_solve_qp<9, false, 6>(w, prm, gv, blockIdx.x, pqp_smem, (size_t)smem_doubles);
}

const void *pqp_gen9_kernel_fn() { return (const void *)pqp_gen9_solve_kernel; }
