// edt_emu.cpp -- TEST HARNESS: the distance transform of pqp_set_maps_occupancy(_device) on the CPU, compiled with plain
// g++ (-DPQP_HOST_EMU) into a library of its own (tests/emu/edt_emu.py).  It runs the per-thread functions of
// csrc/pqp_edt_core.cuh over the same scratch layout the kernels use: edt_column for every column, then edt_row for
// every row.  Never linked into libpqp.so.
#define PQP_HOST_EMU 1
#include <vector>

#include "../../path_optimizer_b200/csrc/pqp_edt_core.cuh"

extern "C" {

// occ [rows][cols] (0 = obstacle) -> out [rows][cols] float
void edt_emu(const uint8_t *occ, int rows, int cols, double resolution, float *out) {
    const size_t R = (size_t)rows, n = R * (size_t)cols;
    std::vector<int32_t> scratch(3 * n);
    int32_t *g = scratch.data(), *s = g + n, *t = s + n;
    for (int j = 0; j < cols; ++j) pqp::edt_column(occ, rows, cols, j, g + (size_t)j * R, 1);
    for (int i = 0; i < rows; ++i)
        pqp::edt_row(g + i, R, cols, s + i, t + i, R, (float)resolution, out + (size_t)i * cols);
}

}  // extern "C"
