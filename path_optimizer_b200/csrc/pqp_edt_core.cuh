// pqp_edt_core.cuh -- per-thread functions of the exact Euclidean distance transform that builds a distance layer from
// an occupancy grid on the device (pqp_set_maps_occupancy, pqp_set_maps_occupancy_device).  Like pqp_env_core.cuh
// they are straight per-thread code, so the test-only host build (-DPQP_HOST_EMU, tests/emu/edt_emu.cpp) calls the
// same source in a loop.
//
// Reference behaviour being replaced: the benchmark's and demo's map recipe
//   cv::distanceTransform(binary, dist, CV_DIST_L2, CV_DIST_MASK_PRECISE); dist *= resolution
// (src/test/path_optimizer_benchmark.cpp:28-43, src/test/demo.cpp:103-110), binary = 0 at obstacles.
//
// Algorithm: the separable exact transform of Meijster, Roerdink and Hesselink (2000).
//   1. column pass: g(i, j) = rows from (i, j) to the nearest obstacle in column j (kEdtNone when the column has none),
//      a down and an up sweep;
//   2. row pass: d2(i, j) = min over columns u with an obstacle of (j - u)^2 + g(i, u)^2, the lower envelope of those
//      parabolas, with integer separators, so d2 is the exact squared distance in cells.
// Everything is 64-bit integer arithmetic: with rows, cols < 2^31 every f and separator numerator is below
// rows^2 + cols^2 < 2^63.  The cell value is (float)sqrt((double)d2) * (float)resolution, rounded step by step, which is
// what ndimage.distance_transform_edt(occ != 0).astype(float32) * float32(resolution) gives; obstacle cells are 0.
// A grid with no obstacle gets cv::distanceTransform's 2^64 (times the resolution) everywhere.
//
// Scratch layout of one map (int32, 3 * rows * cols): g column-major (g[j * rows + i]), then the envelope's sites s and
// their starting columns t, entry q of row i at [q * rows + i].  The row pass runs one thread per row, so consecutive
// threads read consecutive words.
#pragma once
#include <math.h>
#include <stdint.h>

#include "pqp_env_core.cuh"

namespace pqp {

constexpr int32_t kEdtNone = 0x7fffffff;            // g of a column with no obstacle
constexpr float kEdtEmpty = 18446744073709551616.0f; // 2^64: cv::distanceTransform's value on a grid with no obstacle

PQP_HD float edt_mul(float a, float b) {
#if defined(__CUDA_ARCH__) && !defined(PQP_HOST_EMU)
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}

PQP_HD float edt_cell(int64_t d2, float res) {
#if defined(__CUDA_ARCH__) && !defined(PQP_HOST_EMU)
    return edt_mul(__double2float_rn(__dsqrt_rn((double)d2)), res);
#else
    return edt_mul((float)sqrt((double)d2), res);
#endif
}

// Column pass of column j: occupancy `occ` [rows][cols] row-major (0 = obstacle), g[i * gstride] for row i.
PQP_HD void edt_column(const uint8_t *occ, int rows, int cols, int j, int32_t *g, size_t gstride) {
    int32_t d = kEdtNone;
    for (int i = 0; i < rows; ++i) {
        if (occ[(size_t)i * cols + j] == 0) d = 0;
        else if (d != kEdtNone) ++d;
        g[(size_t)i * gstride] = d;
    }
    d = kEdtNone;
    for (int i = rows - 1; i >= 0; --i) {
        const int32_t gi = g[(size_t)i * gstride];
        if (gi == 0) d = 0;
        else if (d != kEdtNone) ++d;
        if (d < gi) g[(size_t)i * gstride] = d;
    }
}

PQP_HD int64_t edt_floor_div(int64_t n, int64_t d) {   // d > 0
    const int64_t q = n / d;
    return (n % d != 0 && n < 0) ? q - 1 : q;
}

// Row pass of one row: g(u) = g[u * gstride] for column u, envelope entries s[q * sstride], t[q * sstride], output
// out[j] for j < cols.
PQP_HD void edt_row(const int32_t *g, size_t gstride, int cols, int32_t *s, int32_t *t, size_t sstride, float res,
                    float *out) {
    int q = -1;
    int64_t gq2 = 0;   // g(s[q])^2
    for (int u = 0; u < cols; ++u) {
        const int32_t gu = g[(size_t)u * gstride];
        if (gu == kEdtNone) continue;
        const int64_t gu2 = (int64_t)gu * gu;
        // drop the sites that column u beats at the first column they own
        while (q >= 0) {
            const int64_t tq = t[(size_t)q * sstride], sq = s[(size_t)q * sstride];
            if ((tq - sq) * (tq - sq) + gq2 <= (tq - u) * (tq - u) + gu2) break;
            if (--q >= 0) {
                const int64_t gp = g[(size_t)s[(size_t)q * sstride] * gstride];
                gq2 = gp * gp;
            }
        }
        if (q < 0) {
            q = 0;
            s[0] = u;
            t[0] = 0;
            gq2 = gu2;
        } else {
            // the last column where s[q] is no worse than u
            const int64_t sq = s[(size_t)q * sstride];
            const int64_t w = 1 + edt_floor_div((int64_t)u * u - sq * sq + gu2 - gq2, 2 * ((int64_t)u - sq));
            if (w < cols) {
                ++q;
                s[(size_t)q * sstride] = u;
                t[(size_t)q * sstride] = (int32_t)w;
                gq2 = gu2;
            }
        }
    }
    if (q < 0) {   // no obstacle in any column: the grid has none
        const float v = edt_mul(kEdtEmpty, res);
        for (int j = 0; j < cols; ++j) out[j] = v;
        return;
    }
    int64_t sq = s[(size_t)q * sstride], tq = t[(size_t)q * sstride];
    int64_t gs = g[(size_t)sq * gstride];
    for (int j = cols - 1; j >= 0; --j) {
        out[j] = edt_cell((j - sq) * (j - sq) + gs * gs, res);
        if (j == tq && q > 0) {
            --q;
            sq = s[(size_t)q * sstride];
            tq = t[(size_t)q * sstride];
            gs = g[(size_t)sq * gstride];
        }
    }
}

}  // namespace pqp
