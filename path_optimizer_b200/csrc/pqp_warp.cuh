// pqp_warp.cuh -- the warp abstraction the solver core is written against.
//
// Product build (nvcc, sm_90a): `Warp` maps 1:1 onto hardware intrinsics (__shfl_sync,
// __syncwarp); everything inlines away.
//
// Test-only build (-DPQP_HOST_EMU, plain g++): `Warp` is backed by 32 host threads and a barrier so
// the very same warp-synchronous source can be exercised on a machine without a GPU
// (tests/emu/).  That build is a TEST HARNESS: it is never linked into libpqp.so and the product
// has no CPU path.
#pragma once

#ifdef PQP_HOST_EMU
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#define PQP_DEV inline
namespace pqp {
struct EmuShared {            // one per emulated warp
    pthread_barrier_t bar;
    double slot_d[32];
    int slot_i[32];
};
struct EmuCta {               // one per emulated CTA
    pthread_barrier_t bar;
    int nthreads;
};
struct Warp {
    int lane_;
    EmuShared *sh;
    int lane() const { return lane_; }
    void sync() const { pthread_barrier_wait(&sh->bar); }
    double shfl(double v, int src) const {
        sh->slot_d[lane_] = v;
        pthread_barrier_wait(&sh->bar);
        double r = sh->slot_d[src & 31];
        pthread_barrier_wait(&sh->bar);
        return r;
    }
    int shfl(int v, int src) const {
        sh->slot_i[lane_] = v;
        pthread_barrier_wait(&sh->bar);
        int r = sh->slot_i[src & 31];
        pthread_barrier_wait(&sh->bar);
        return r;
    }
    double max(double v) const {
        sh->slot_d[lane_] = v;
        pthread_barrier_wait(&sh->bar);
        double r = sh->slot_d[0];
        for (int k = 1; k < 32; ++k) r = fmax(r, sh->slot_d[k]);
        pthread_barrier_wait(&sh->bar);
        return r;
    }
    double sum(double v) const {
        sh->slot_d[lane_] = v;
        pthread_barrier_wait(&sh->bar);
        // same xor-butterfly association order as the device version
        double t[32];
        for (int k = 0; k < 32; ++k) t[k] = sh->slot_d[k];
        for (int o = 16; o > 0; o >>= 1) {
            double u[32];
            for (int k = 0; k < 32; ++k) u[k] = t[k] + t[k ^ o];
            for (int k = 0; k < 32; ++k) t[k] = u[k];
        }
        pthread_barrier_wait(&sh->bar);
        return t[lane_];
    }
    int any(int v) const {
        sh->slot_i[lane_] = v;
        pthread_barrier_wait(&sh->bar);
        int r = 0;
        for (int k = 0; k < 32; ++k) r |= sh->slot_i[k];
        pthread_barrier_wait(&sh->bar);
        return r;
    }
};
struct CtaSync {
    EmuCta *cta;
    void sync() const { pthread_barrier_wait(&cta->bar); }
};
}  // namespace pqp
#else
#include <cuda_runtime.h>
#define PQP_DEV __device__ __forceinline__
namespace pqp {
struct Warp {
    PQP_DEV int lane() const { return threadIdx.x & 31; }
    PQP_DEV void sync() const { __syncwarp(); }
    PQP_DEV double shfl(double v, int src) const { return __shfl_sync(0xffffffffu, v, src); }
    PQP_DEV int shfl(int v, int src) const { return __shfl_sync(0xffffffffu, v, src); }
    PQP_DEV double max(double v) const {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
        return v;
    }
    PQP_DEV double sum(double v) const {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        return v;
    }
    PQP_DEV int any(int v) const { return __any_sync(0xffffffffu, v); }
};
struct CtaSync {
    PQP_DEV void sync() const { __syncthreads(); }
};
}  // namespace pqp
#endif

namespace pqp {
// A CTA of NW warps working on ONE path.  Block-wide reductions go through a small shared scratch
// (NW doubles) in a fixed order, so results are deterministic and identical on every thread.
struct Cta {
    Warp w;
    CtaSync cs;
    int wid, nw;
    double *scratch;   // >= 16 * nw doubles of shared memory (128 reserved, nw <= 8)
    PQP_DEV int lane() const { return w.lane(); }
    PQP_DEV int tid() const { return wid * 32 + w.lane(); }
    PQP_DEV int nthreads() const { return nw * 32; }
    PQP_DEV void sync() const {
        if (nw == 1) w.sync();
        else cs.sync();
    }
    PQP_DEV double max(double v) const {
        v = w.max(v);
        if (nw == 1) return v;
        if (w.lane() == 0) scratch[wid] = v;
        cs.sync();
        double r = scratch[0];
        for (int k = 1; k < nw; ++k) r = fmax(r, scratch[k]);
        cs.sync();
        return r;
    }
    PQP_DEV double sum(double v) const {
        v = w.sum(v);
        if (nw == 1) return v;
        if (w.lane() == 0) scratch[wid] = v;
        cs.sync();
        double r = scratch[0];
        for (int k = 1; k < nw; ++k) r += scratch[k];
        cs.sync();
        return r;
    }
    // n (<= 16) max-reductions at once: one shared-memory exchange and two barriers in total
    PQP_DEV void max_n(double *v, int n) const {
        for (int k = 0; k < n; ++k) v[k] = w.max(v[k]);
        if (nw == 1) return;
        if (w.lane() == 0)
            for (int k = 0; k < n; ++k) scratch[wid * 16 + k] = v[k];
        cs.sync();
        for (int k = 0; k < n; ++k) {
            double r = scratch[k];
            for (int q = 1; q < nw; ++q) r = fmax(r, scratch[q * 16 + k]);
            v[k] = r;
        }
        cs.sync();
    }
    PQP_DEV int any(int v) const {
        v = w.any(v);
        if (nw == 1) return v;
        if (w.lane() == 0) scratch[wid] = v ? 1.0 : 0.0;
        cs.sync();
        int r = 0;
        for (int k = 0; k < nw; ++k) r |= (scratch[k] != 0.0);
        cs.sync();
        return r;
    }
};
}  // namespace pqp
