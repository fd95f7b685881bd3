// pqp_kernels.h -- one record per compiled solve kernel ("shape class").  Every kernel lives in its own
// translation unit (pqp_k*.cu): at the 255-register limit ptxas' allocation for one kernel changes with whatever
// else is compiled next to it (the same source has run several times slower after unrelated instantiations were added
// to the same file), so the kernels are compiled in isolation and only these records cross the boundary.
#pragma once
#include <stddef.h>

struct PqpVariant {
    int imax, bw, threads;
    const void *fn;                      // __global__ entry, for cudaLaunchKernel / cudaFuncSetAttribute
    size_t (*smem)(int n, int keep);     // dynamic shared memory (bytes) for a path of n stations
    bool (*fits)(int n, int keep);
    const char *name;                    // kernel name as profilers print it
};

#define PQP_DECLARE_VARIANT(name) void pqp_variant_##name(PqpVariant *out);
// thread-per-station kernels Kp3<IMAX, BW, NW, MMAX>
PQP_DECLARE_VARIANT(k3_17_6_4_17)
PQP_DECLARE_VARIANT(k3_23_7_4_17)
PQP_DECLARE_VARIANT(k3_17_6_8_34)
PQP_DECLARE_VARIANT(k3_23_7_8_34)
PQP_DECLARE_VARIANT(k3_27_7_8_34)
PQP_DECLARE_VARIANT(k3_27_7_10_34)
PQP_DECLARE_VARIANT(k3_37_7_12_34)
PQP_DECLARE_VARIANT(k3_37_7_13_34)
// thread-per-station kernels of the "KPC" formulation Kp3<IMAX, BW, NW, MMAX, KPC>
PQP_DECLARE_VARIANT(k3c_13_7_8_34)
PQP_DECLARE_VARIANT(k3c_23_7_4_17)
PQP_DECLARE_VARIANT(k3c_23_7_8_34)
// thread-per-station block-cyclic-reduction kernels of the "K" formulation Kk<NW> (pqp_kk_core.cuh)
PQP_DECLARE_VARIANT(kk_4)
PQP_DECLARE_VARIANT(kk_8)
PQP_DECLARE_VARIANT(kk_13)
// one-warp generic KP kernel (any keep <= 10) and the generic banded-QP kernel of "K" / "KPC"
PQP_DECLARE_VARIANT(k1_generic)
const void *pqp_gen_kernel_fn();
const void *pqp_gen4_kernel_fn();    // the same core with 4-unknown separators and a linear cost (pqp_kgen4.cu)
const void *pqp_gen9_kernel_fn();    // the same core with 9-unknown separators and six P partners (pqp_kgen9.cu)
void pqp_k1_set_smem_cap(int bytes);   // device's opt-in shared memory per block (decides where the one-warp kernel keeps its scalings)
