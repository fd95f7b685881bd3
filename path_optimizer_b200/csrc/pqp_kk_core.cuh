// pqp_kk_core.cuh -- thread-per-station solver for the "K" formulation (SolverKAsInput).
//
// Reference being replaced: src/solver/solver_k_as_input.cpp:14-207 (setHessianMatrix, setDynamicMatrix,
// setConstraintMatrix, getOptimizedPath) + the OSQP solve behind src/solver/solver.cpp:46-77.
//
// The QP (N stations): unknowns e_phi_i, e_y_i (state), delta_i (steering, i < N-1), e_i (corridor slack of the second
// circle); n = 4N-1, m = 11N-1.  Thread i owns station i: its 11 rows
//     0  -e_phi_i + e_phi_{i-1} + q_{i-1} e_y_{i-1} + c_{i-1} delta_{i-1}  = b0      (dynamics, :89-121,156-167)
//     1  -e_y_i   + ds_{i-1} e_phi_{i-1} + e_y_{i-1}                        = b1
//     2  e_phi_i   free (end-heading window at the last station, :172-178)            (identity rows, :124-126,169-187)
//     3  e_y_i     free
//     4  delta_i   in +-max_steering_angle          (i < N-1)
//     5  e_i       in [0, margin]
//     6..8  d1|d3|d4 e_phi_i + e_y_i in the clearance of circles 0|2|3                (:129-137,189-199)
//     9  d2 e_phi_i + e_y_i - e_i <= ub1 - margin,  10  d2 e_phi_i + e_y_i + e_i >= lb1 + margin   (:141-147,200-207)
// and its 4 columns stay in registers for the whole solve.  OSQP's recurrence (Ruiz scaling, rho classes, ADMM,
// termination, primal-infeasibility certificate, adaptive rho) is the one of pqp_gen_core.cuh -- same unscaled-weighted
// form v = z + w, W = rho_row E^2 -- with the sparse gathers replaced by these stencils.
//
// Reduced KKT  c P + sigma D^-2 + A' W A : the slack e_i couples to (e_phi_i, e_y_i) only through rows 9 / 10, which have
// equal weight (same rho class, bit-identical Ruiz factors) and opposite sign on e_i: the coupling cancels exactly and
// e_i is a scalar division.  What remains is block tridiagonal by station with 3 x 3 blocks (e_phi, e_y, delta; the
// curvature-rate term of P couples delta_i to delta_{i+1}).  It is factored and solved by block CYCLIC REDUCTION: at
// level l the stations with index = 2^l (mod 2^(l+1)) are eliminated, each by its own thread, which keeps
// A_j^-1, G_L = A_j^-1 C_{j,j-s}, G_R = A_j^-1 C_{j,j+s} (24 doubles) in registers.  One solve is ceil(log2 N) levels
// down (each eliminated station pushes G' r to its two neighbours) and as many up (x_j = A_j^-1 r_j - G_L x_a - G_R x_b),
// one barrier per level, no serial chain longer than a 3 x 3 product (thirteen-warp class, up to 416 stations).  The four- and
// eight-warp classes (up to 256 stations) use a SPIKE form with dense inverses instead: see factor_spike / solve_spike.
#pragma once
#include "pqp_kp_core.cuh"

#ifndef PQP_KK_G_SMEM
#define PQP_KK_G_SMEM 0     // 1: G_L / G_R are read from their shared-memory rows in every solve instead of living in registers (slower: more shared-memory traffic on the solve's critical path)
#endif

namespace pqp {

template <int NW>
struct Kk {
    static constexpr int kT = NW * 32;            // threads = max stations
    static constexpr int kP = kT + 2;             // pitch of the exchange rows: entry 0 = "station -1", entry N+1 = "station N" (zeros)
    static constexpr int kCtaScratch = (NW <= 8) ? 128 : 256;
    // shared memory (doubles): 3 x-rows + 2 dual rows + 2 weight rows + 1 delta-scale row (pitch kP); 6 push rows, 9 coupling
    // rows, 18 G rows, 11 parked-dual rows, 11 E rows, 2 output rows, 1 row of pushes that cross a warp boundary (pitch kT)
    static constexpr int kXRows = 8, kTRows = 6 + 9 + 18 + 11 + 11 + 2 + 1;
    // The four- and eight-warp classes (N <= 256) solve the reduced KKT in SPIKE form instead (see factor_spike):
    // separators every L stations (at most kMS of them), dense interior inverses, a dense inverse of the separator system.
    static constexpr bool kSpike = (NW <= 8);
    static constexpr int kMS = (NW <= 4) ? 26 : 32;   // most separators
    static constexpr int kIM = (NW <= 4) ? 12 : 21;   // most interior unknowns of a chunk (L <= 5 / L <= 8)
    static constexpr int kNB = kIM / 3;              // most interior stations of a chunk
    static constexpr int kKP = kIM + 1 + (kIM & 1);   // row pitch of an interior inverse (odd)
    static constexpr int kKC = kIM * kKP + 3 - ((kIM * kKP) & 1);   // chunk stride (odd: chunks start on different banks)
    static constexpr int kCF = kNB * 18;              // block factor of a chunk: D_k^-1 | L_k per interior station
    static constexpr int kSpRows = 7;              // rhs (3), y (3), separator rhs (1); the Schur scratch of a factorisation overlays them
    static constexpr int kSpScratch = 15 * kT + kMS * kCF + kMS * 27;   // doubles a factorisation needs in the (later) separator-inverse region
    struct SpDims { int L, M, pitch; size_t reg; };
    PQP_HD static SpDims sp_dims(int N) {
        SpDims d;
        d.L = (N + kMS - 1) / kMS;
        if (d.L < 2) d.L = 2;
        d.M = (N - 1) / d.L + 1;
        int pch = 3 * d.M;
        pch += (pch & 1);
        if ((pch & 3) == 0) pch += 2;              // even (128-bit loads), = 2 mod 4 (rows of neighbouring threads on different banks)
        d.pitch = pch;
        d.reg = (size_t)pch * 3 * d.M;
        if (d.reg < (size_t)kSpScratch) d.reg = kSpScratch;
        return d;
    }
    PQP_HD static size_t smem_doubles(int N) {
        if (kSpike) {
            const SpDims d = sp_dims(N < 2 ? 2 : N);
            return (size_t)kXRows * kP + (size_t)kSpRows * kT + (size_t)((d.M * kKC + 1) & ~1) + d.reg;
        }
        return (size_t)kXRows * kP + (size_t)kTRows * kT;
    }
    PQP_HD static bool fits(int N, int /*keep*/) { return N >= 2 && N <= kT; }

    struct Sm {
        double *b;
        int M;                                                                // (SPIKE form: separators)
        PQP_DEV double *xr(int c) const { return b + c * kP + 1; }            // c: 0 e_phi, 1 e_y, 2 delta; index i in [-1, N]
        PQP_DEV double *gr(int c) const { return b + (3 + c) * kP + 1; }      // dual-like values of rows 0 / 1
        PQP_DEV double *wr(int c) const { return b + (5 + c) * kP + 1; }      // W (or E) of rows 0 / 1
        PQP_DEV double *dr() const { return b + 7 * kP + 1; }                 // D of delta (Ruiz sweeps)
        PQP_DEV double *t(int k) const { return b + kXRows * kP + k * kT; }
        PQP_DEV double *push(int k) const { return t(k); }                    // 0..2 to the left neighbour, 3..5 to the right
        PQP_DEV double *cpl(int k) const { return t(6 + k); }                 // current coupling to the right neighbour (factor)
        PQP_DEV double *gl(int k) const { return t(15 + k); }                 // G_L, G_R of the level being eliminated (factor)
        PQP_DEV double *gR(int k) const { return t(24 + k); }
        PQP_DEV double *wold(int k) const { return t(33 + k); }
        PQP_DEV double *E(int k) const { return t(44 + k); }
        PQP_DEV double *ox() const { return t(kSpike ? 0 : 55); }
        PQP_DEV double *oy() const { return t(kSpike ? 1 : 56); }
        // SPIKE form
        PQP_DEV double *rr(int c) const { return t(c); }                      // rhs per station
        PQP_DEV double *yy(int c) const { return t(3 + c); }                  // K_I^-1 r_I per station
        PQP_DEV double *gg() const { return t(6); }                           // separator rhs [3M], zero up to the pitch
        PQP_DEV double *sch() const { return t(0); }                          // Schur blocks [M][27] while a factorisation runs
        PQP_DEV double *kinv() const { return t(kSpRows); }                   // [M][kKC]
        PQP_DEV double *sinv() const { return t(kSpRows) + (size_t)((M * kKC + 1) & ~1); } // [3M][pitch]; factor scratch before it is written
        PQP_DEV double *bp() const { return t(57); }                          // [level < 5][warp][3]
    };

    // two consecutive doubles from a 16-byte aligned shared-memory address
    PQP_DEV static void ld2(const double *q, double &a, double &b) {
#ifdef PQP_HOST_EMU
        a = q[0]; b = q[1];
#else
        const double2 t = *reinterpret_cast<const double2 *>(q);
        a = t.x; b = t.y;
#endif
    }
    // 3 x 3 helpers (row-major)
    PQP_DEV static void mm(const double *a, const double *b, double *o) {          // o = a b
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int cc = 0; cc < 3; ++cc) o[r * 3 + cc] = a[r * 3] * b[cc] + a[r * 3 + 1] * b[3 + cc] + a[r * 3 + 2] * b[6 + cc];
    }
    PQP_DEV static void mtm(const double *a, const double *b, double *o) {         // o = a' b
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int cc = 0; cc < 3; ++cc) o[r * 3 + cc] = a[r] * b[cc] + a[3 + r] * b[3 + cc] + a[6 + r] * b[6 + cc];
    }

    PQP_DEV static void solve_path(const Cta &c, const DevParams &pm, const BatchView &bv, int prob, double *smem,
                                   size_t smem_cap) {
        const int tid = c.tid();
        const int N = bv.n_points[prob];
        const int off = bv.offsets[prob];
        const pqp_state *ref = bv.ref + off;
        const pqp_station_bounds *bnd = bv.bounds + off;
        pqp_state *out = bv.out_states + off;
        const double qnan = nan("");
        if (!fits(N, 1) || smem_doubles(N) > smem_cap || (kSpike && !bv.workspace)) {
            if (tid == 0) {
                bv.status[prob] = PQP_INVALID_PROBLEM;
                if (bv.iters) bv.iters[prob] = 0;
            }
            for (int i = tid; i < N; i += kT) {
                out[i].x = out[i].y = out[i].z = out[i].k = out[i].s = qnan;
                out[i].v = out[i].a = 0.0;
                if (bv.out_frenet) {
                    double *f = bv.out_frenet + 3 * (size_t)(off + i);
                    f[0] = f[1] = f[2] = qnan;
                }
            }
            return;
        }
        const SpDims sd = sp_dims(N);
        Sm s{smem, sd.M};
        // scalings E and the parked duals of the last check: shared memory, or (SPIKE form: no room) the path's slice of
        // the global workspace -- both only touched at termination checks
        double *const ews = kSpike ? kp_ws_base(bv.workspace, off, prob) : nullptr;
        auto Ek = [&](int k) -> double * { return kSpike ? ews + (size_t)k * N : s.E(k); };
        auto Wk = [&](int k) -> double * { return kSpike ? ews + (size_t)(11 + k) * N : s.wold(k); };
        const int i = tid;
        const bool live = i < N, first = (i == 0), last = (i == N - 1);
        const bool hasd = live && !last;                 // delta_i exists
        int Lv = 0;
        while ((1 << Lv) < N) ++Lv;
        int lev = Lv;                                    // level at which this station is eliminated (station 0: never)
        if (i > 0) { lev = 0; while (!((i >> lev) & 1)) ++lev; }

        // ---- per-station data ------------------------------------------------------------------------
        // transition i-1 -> i (rows 0 / 1 of this station) and i -> i+1 (the same rows of the next station, seen from my columns)
        double pa = 0, qp = 0, cp = 0, dsp = 0, pb = 0, na = 0, qn = 0, cn = 0, dsn = 0, nb = 0;
        double lo[11], hi[11];
#pragma unroll
        for (int k = 0; k < 11; ++k) { lo[k] = -kOsqpInfty; hi[k] = kOsqpInfty; }
        double Pdd = 0.0;                                // diagonal of R for delta_i
        const double w_cr = pm.k_w_cr;
        const bool dprev = hasd && i >= 1, dnext = hasd && (i + 1 <= N - 2);   // partners of delta_i in R
        int invalid = 0;
        if (live) {
            if (!first) {
                const double rk = ref[i - 1].k, rs = ref[i].s - ref[i - 1].s;
                const double rd = atan(rk * pm.wheel_base);
                pa = 1.0; pb = 1.0;
                qp = -rs * pow(rk, 2);
                dsp = rs;
                cp = rs / pm.wheel_base / pow(cos(rd), 2);
                lo[0] = hi[0] = rs * rd / pm.wheel_base / pow(cos(rd), 2);
                lo[1] = hi[1] = 0.0;
            } else {
                lo[0] = hi[0] = -bv.x0[3 * (size_t)prob + 1];     // x0 << err[1], err[0]  (:156-159)
                lo[1] = hi[1] = -bv.x0[3 * (size_t)prob];
            }
            if (!last) {
                const double rk = ref[i].k, rs = ref[i + 1].s - ref[i].s;
                const double rd = atan(rk * pm.wheel_base);
                na = 1.0; nb = 1.0;
                qn = -rs * pow(rk, 2);
                dsn = rs;
                cn = rs / pm.wheel_base / pow(cos(rd), 2);
                lo[4] = -pm.max_steer; hi[4] = pm.max_steer;
                const int nc = N - 1;
                Pdd = (i == 0 || i == nc - 1) ? (pm.k_w_c + w_cr) : (w_cr * 2 + pm.k_w_c);
            }
            if (last && pm.constraint_end_heading) {
                const double pi = 3.14159265358979323846;
                const double end_psi = constraint_angle(bv.end_heading[prob] - ref[N - 1].z);
                if (end_psi < 70 * pi / 180) {
                    lo[2] = end_psi - 5 * pi / 180;
                    hi[2] = end_psi + 5 * pi / 180;
                }
            }
            lo[5] = 0.0; hi[5] = pm.margin;
            const pqp_station_bounds bb = bnd[i];
            lo[6] = bb.c0_lb; hi[6] = bb.c0_ub;
            lo[7] = bb.c2_lb; hi[7] = bb.c2_ub;
            lo[8] = bb.c3_lb; hi[8] = bb.c3_ub;
            hi[9] = bb.c1_ub - pm.margin;
            lo[10] = bb.c1_lb + pm.margin;
#pragma unroll
            for (int k = 0; k < 11; ++k)
                if (!(lo[k] <= hi[k])) invalid = 1;
            if (!(ref[i].s - ref[i].s == 0.0)) invalid = 1;   // a NaN or infinite s is refused (pqp.h)
        }
        const double cf[5] = {pm.d1, pm.d3, pm.d4, pm.d2, pm.d2};     // e_phi coefficient of rows 6..10
        // zero entries either side of the exchange rows
        if (tid == 0) {
            for (int r = 0; r < kXRows; ++r) { smem[r * kP] = 0.0; smem[r * kP + N + 1] = 0.0; }
        }
        invalid = c.any(invalid);

        // A x for my rows: own (xf, xy, xd, xe), previous station's (e_phi, e_y, delta) from the exchange rows
        auto rows_of = [&](double xf, double xy, double xd, double xe, double *ax) {
            const double pf = s.xr(0)[i - 1], py = s.xr(1)[i - 1], pd = s.xr(2)[i - 1];
            ax[0] = ((pa * pf + qp * py) - xf) + cp * pd;
            ax[1] = (dsp * pf + pb * py) - xy;
            ax[2] = xf; ax[3] = xy; ax[4] = xd; ax[5] = xe;
#pragma unroll
            for (int k = 0; k < 3; ++k) ax[6 + k] = cf[k] * xf + xy;
            ax[9] = (cf[3] * xf + xy) - xe;
            ax[10] = (cf[4] * xf + xy) + xe;
        };
        // A' g for my columns: my rows' g, rows 0 / 1 of the next station from the exchange rows
        auto cols_of = [&](const double *g, double *aty) {
            const double g0n = s.gr(0)[i + 1], g1n = s.gr(1)[i + 1];
            aty[0] = ((((((-g[0] + na * g0n) + dsn * g1n) + g[2]) + cf[0] * g[6]) + cf[1] * g[7]) + cf[2] * g[8]) + cf[3] * g[9] + cf[4] * g[10];
            aty[1] = ((((((-g[1] + qn * g0n) + nb * g1n) + g[3]) + g[6]) + g[7]) + g[8]) + g[9] + g[10];
            aty[2] = cn * g0n + g[4];
            aty[3] = (g[5] - g[9]) + g[10];
        };

        int status = PQP_UNSOLVED, iter = 0;
        double x[4] = {0, 0, 0, 0};                      // e_phi, e_y, delta, e
        double v[11], W[11];
#pragma unroll
        for (int k = 0; k < 11; ++k) { v[k] = 0.0; W[k] = 0.0; }
        double cost_c = 1.0;
        if (invalid) {
            status = PQP_INVALID_PROBLEM;
        } else {
            // ================= Ruiz equilibration + cost scaling (OSQP scale_data) =================
            double D[4] = {1, 1, 1, 1}, E[11];
#pragma unroll
            for (int k = 0; k < 11; ++k) E[k] = 1.0;
            const double Pd[4] = {0.0, pm.k_w_pq, Pdd, pm.w_s};
            for (int sweep = 0; sweep < pm.scaling; ++sweep) {
                if (live) {
                    s.xr(0)[i] = D[0]; s.xr(1)[i] = D[1]; s.xr(2)[i] = hasd ? D[2] : 0.0;
                    s.wr(0)[i] = E[0]; s.wr(1)[i] = E[1];
                }
                c.sync();
                double fD[4] = {1, 1, 1, 1}, fE[11];
#pragma unroll
                for (int k = 0; k < 11; ++k) fE[k] = 1.0;
                if (live) {
                    const double E0n = s.wr(0)[i + 1], E1n = s.wr(1)[i + 1];
                    const double Dfp = s.xr(0)[i - 1], Dyp = s.xr(1)[i - 1], Ddp = s.xr(2)[i - 1], Ddn = s.xr(2)[i + 1];
                    double an[4];
                    an[0] = fmax(fmax(E[0], E[2]), fmax(na * E0n, fabs(dsn) * E1n));
                    an[1] = fmax(fmax(E[1], E[3]), fmax(fabs(qn) * E0n, nb * E1n));
#pragma unroll
                    for (int k = 0; k < 5; ++k) { an[0] = fmax(an[0], fabs(cf[k]) * E[6 + k]); an[1] = fmax(an[1], E[6 + k]); }
                    an[2] = fmax(E[4], fabs(cn) * E0n);
                    an[3] = fmax(E[5], fmax(E[9], E[10]));
                    double pn[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) pn[q] = cost_c * fabs(Pd[q]) * D[q] * D[q];
                    if (dprev) pn[2] = fmax(pn[2], cost_c * fabs(w_cr) * D[2] * Ddp);
                    if (dnext) pn[2] = fmax(pn[2], cost_c * fabs(w_cr) * D[2] * Ddn);
#pragma unroll
                    for (int q = 0; q < 4; ++q) fD[q] = 1.0 / sqrt(limit_scaling(fmax(pn[q], an[q] * D[q])));
                    double rn[11];
                    rn[0] = fmax(fmax(D[0], pa * Dfp), fmax(fabs(qp) * Dyp, fabs(cp) * Ddp));
                    rn[1] = fmax(D[1], fmax(fabs(dsp) * Dfp, pb * Dyp));
                    rn[2] = D[0]; rn[3] = D[1]; rn[4] = D[2]; rn[5] = D[3];
#pragma unroll
                    for (int k = 0; k < 3; ++k) rn[6 + k] = fmax(fabs(cf[k]) * D[0], D[1]);
                    rn[9] = rn[10] = fmax(fmax(fabs(cf[3]) * D[0], D[1]), D[3]);
#pragma unroll
                    for (int k = 0; k < 11; ++k) fE[k] = 1.0 / sqrt(limit_scaling(rn[k] * E[k]));
                }
                c.sync();
#pragma unroll
                for (int q = 0; q < 4; ++q) D[q] *= fD[q];
#pragma unroll
                for (int k = 0; k < 11; ++k) E[k] *= fE[k];
                if (hasd) s.dr()[i] = D[2];
                else if (live) s.dr()[i] = 0.0;
                c.sync();
                double part = 0.0;
                if (live) {
                    const double Ddp = s.dr()[i - 1], Ddn = s.dr()[i + 1];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        if (q == 2 && !hasd) continue;
                        double nrm = cost_c * fabs(Pd[q]) * D[q] * D[q];
                        if (q == 2 && dprev) nrm = fmax(nrm, cost_c * fabs(w_cr) * D[2] * Ddp);
                        if (q == 2 && dnext) nrm = fmax(nrm, cost_c * fabs(w_cr) * D[2] * Ddn);
                        part += nrm;
                    }
                }
                const double mean = c.sum(part) / (double)(4 * N - 1);
                double ct = fmax(mean, 1.0);
                ct = limit_scaling(ct);
                cost_c = cost_c * (1.0 / ct);
            }
            double sg[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) sg[q] = pm.sigma / (D[q] * D[q]);
            double rho = fmin(fmax(pm.rho, kRhoMin), kRhoMax);
#pragma unroll
            for (int k = 0; k < 11; ++k) {
                W[k] = rho_bar(E[k] * lo[k], E[k] * hi[k], rho) * E[k] * E[k];
                if (live) Ek(k)[tid] = E[k];
            }
            if (!live || last) W[4] = 0.0;               // no delta at the last station: the row does not exist
            if (!live) {
#pragma unroll
                for (int k = 0; k < 11; ++k) W[k] = 0.0;
            }

            // ---- factorisation state: A_j^-1 (symmetric, 6), G_L, G_R of my elimination level; 1 / pivot of the slack
            double Ai[6] = {1, 0, 0, 1, 0, 1}, GL[9], GR[9], inv_e = 1.0;
#pragma unroll
            for (int k = 0; k < 9; ++k) GL[k] = GR[k] = 0.0;

            // my diagonal block A = K[i, i] and the coupling C = K[i, i+1] of the reduced KKT (block tridiagonal by station)
            auto blocks = [&](double *A, double *C) {
                if (live) { s.wr(0)[i] = W[0]; s.wr(1)[i] = W[1]; }
                c.sync();
#pragma unroll
                for (int k = 0; k < 9; ++k) { A[k] = 0.0; C[k] = 0.0; }
                A[0] = A[4] = A[8] = 1.0;
                if (live) {
                    const double W0n = s.wr(0)[i + 1], W1n = s.wr(1)[i + 1];   // 0 beyond the last station
                    double sw = 0.0, swd = 0.0, swdd = 0.0;                      // sums over rows 6..10 of W, W d, W d^2
#pragma unroll
                    for (int k = 0; k < 5; ++k) { sw += W[6 + k]; swd += W[6 + k] * cf[k]; swdd += W[6 + k] * cf[k] * cf[k]; }
                    const double u0[3] = {na, qn, cn}, u1[3] = {dsn, nb, 0.0};   // rows 0 / 1 of the next station on my columns
                    A[0] = cost_c * Pd[0] + sg[0] + W[0] + W[2] + swdd + W0n * u0[0] * u0[0] + W1n * u1[0] * u1[0];
                    A[1] = swd + W0n * u0[0] * u0[1] + W1n * u1[0] * u1[1];
                    A[2] = W0n * u0[0] * u0[2];
                    A[4] = cost_c * Pd[1] + sg[1] + W[1] + W[3] + sw + W0n * u0[1] * u0[1] + W1n * u1[1] * u1[1];
                    A[5] = W0n * u0[1] * u0[2];
                    A[8] = hasd ? (cost_c * Pd[2] + sg[2] + W[4] + W0n * u0[2] * u0[2]) : 1.0;
                    A[3] = A[1]; A[6] = A[2]; A[7] = A[5];
                    if (!last) {       // K[i, i+1]: rows 0 / 1 of the next station carry -1 on its e_phi / e_y; R couples the deltas
#pragma unroll
                        for (int r = 0; r < 3; ++r) { C[r * 3] = -(W0n * u0[r]); C[r * 3 + 1] = -(W1n * u1[r]); }
                        if (dnext) C[8] = cost_c * (-w_cr);
                    }
                    inv_e = 1.0 / (cost_c * Pd[3] + sg[3] + W[5] + W[9] + W[10]);
                }
            };

            // ---- block cyclic reduction (classes of more than four warps) ----
            auto factor_cr = [&]() -> int {
                int ok = 1;
                double A[9], C[9];
                blocks(A, C);
                if (live) {
#pragma unroll
                    for (int k = 0; k < 9; ++k) s.cpl(k)[i] = C[k];
                }
                c.sync();
                for (int l = 0; l < Lv; ++l) {
                    const int st = 1 << l;
                    if (live && lev == l) {
                        if (!(A[0] > 0.0)) ok = 0;
                        double inv[9], Ca[9], Ct[9];
                        inv3_spd(A, inv);
                        Ai[0] = inv[0]; Ai[1] = inv[1]; Ai[2] = inv[2]; Ai[3] = inv[4]; Ai[4] = inv[5]; Ai[5] = inv[8];
#pragma unroll
                        for (int k = 0; k < 9; ++k) Ca[k] = s.cpl(k)[i - st];       // K[a, j]
#pragma unroll
                        for (int r = 0; r < 3; ++r)
#pragma unroll
                            for (int cc = 0; cc < 3; ++cc) Ct[r * 3 + cc] = Ca[cc * 3 + r];   // K[j, a]
                        mm(inv, Ct, GL);
                        if (i + st < N) mm(inv, C, GR);
#pragma unroll
                        for (int k = 0; k < 9; ++k) { s.gl(k)[i] = GL[k]; s.gR(k)[i] = GR[k]; }
                    }
                    c.sync();
                    if (live && lev > l) {
                        double Cn[9];
#pragma unroll
                        for (int k = 0; k < 9; ++k) Cn[k] = 0.0;
                        if (i + st < N) {               // right neighbour j = i + st is eliminated
                            double G[9], Pm[9];
#pragma unroll
                            for (int k = 0; k < 9; ++k) G[k] = s.gl(k)[i + st];
                            mm(C, G, Pm);
#pragma unroll
                            for (int k = 0; k < 9; ++k) A[k] -= Pm[k];
                            if (i + 2 * st < N) {
#pragma unroll
                                for (int k = 0; k < 9; ++k) G[k] = s.gR(k)[i + st];
                                mm(C, G, Pm);
#pragma unroll
                                for (int k = 0; k < 9; ++k) Cn[k] = -Pm[k];
                            }
                        }
                        if (i >= st && i > 0) {         // left neighbour j' = i - st is eliminated: K[i, j'] = cpl(j')'
                            double Cj[9], G[9], Pm[9];
#pragma unroll
                            for (int k = 0; k < 9; ++k) { Cj[k] = s.cpl(k)[i - st]; G[k] = s.gR(k)[i - st]; }
                            mtm(Cj, G, Pm);
#pragma unroll
                            for (int k = 0; k < 9; ++k) A[k] -= Pm[k];
                        }
                        // keep the block symmetric (upper part is authoritative)
                        A[3] = A[1]; A[6] = A[2]; A[7] = A[5];
                        // (only survivors write their coupling row; this level's readers of it were the eliminated
                        // stations, before the barrier above)
#pragma unroll
                        for (int k = 0; k < 9; ++k) { C[k] = Cn[k]; s.cpl(k)[i] = Cn[k]; }
                    }
                    c.sync();
                }
                if (tid == 0) {
                    if (!(A[0] > 0.0)) ok = 0;
                    double inv[9];
                    inv3_spd(A, inv);
                    Ai[0] = inv[0]; Ai[1] = inv[1]; Ai[2] = inv[2]; Ai[3] = inv[4]; Ai[4] = inv[5]; Ai[5] = inv[8];
                }
                return !c.any(!ok);
            };

            // K x = r for the (e_phi, e_y, delta) blocks; r in / x out in registers, x also left in the exchange rows.
            // Levels 0..4 (strides < 32) stay inside a warp: pushes and x travel by shuffles, no barrier; the one push per
            // level that crosses into the next warp (lane 32 - st -> lane 0 of the next warp) is parked in shared memory
            // and collected after the first barrier, and x of the next warp's lane 0 is read from its exchange row.
            // Levels >= 5 (the stations 32 w) go through shared memory, one barrier per level.
            const int lane = c.lane(), wid = c.wid;
            constexpr int kLoc = 5;
            const int Ll = Lv < kLoc ? Lv : kLoc;
            auto solve_cr = [&](double *r) {
#pragma unroll
                for (int l = 0; l < kLoc; ++l) {
                    if (l < Ll) {
                        const int st = 1 << l;
                        const bool el = live && lev == l;
                        double pl[3] = {0.0, 0.0, 0.0}, pr[3] = {0.0, 0.0, 0.0};
                        if (el) {
#if PQP_KK_G_SMEM
                            double GL[9], GR[9];
#pragma unroll
                            for (int k = 0; k < 9; ++k) { GL[k] = s.gl(k)[i]; GR[k] = s.gR(k)[i]; }
#endif
#pragma unroll
                            for (int cc = 0; cc < 3; ++cc) {
                                pl[cc] = GL[cc] * r[0] + GL[3 + cc] * r[1] + GL[6 + cc] * r[2];
                                pr[cc] = GR[cc] * r[0] + GR[3 + cc] * r[1] + GR[6 + cc] * r[2];
                            }
                            if (lane + st == 32) {
#pragma unroll
                                for (int cc = 0; cc < 3; ++cc) s.bp()[(l * NW + wid) * 3 + cc] = pr[cc];
                            }
                        }
                        double fl[3], fr[3];
#pragma unroll
                        for (int cc = 0; cc < 3; ++cc) {
                            fl[cc] = c.w.shfl(pl[cc], lane + st);      // what the station st to my right pushes left
                            fr[cc] = c.w.shfl(pr[cc], lane - st);      // what the station st to my left pushes right
                        }
                        if (live && lev > l) {
#pragma unroll
                            for (int cc = 0; cc < 3; ++cc) r[cc] -= fl[cc];
                            if (lane > 0) {
#pragma unroll
                                for (int cc = 0; cc < 3; ++cc) r[cc] -= fr[cc];
                            }
                        }
                    }
                }
                if (Lv > kLoc) {
                    c.sync();
                    if (live && lane == 0 && wid > 0) {
#pragma unroll
                        for (int l = 0; l < kLoc; ++l)
#pragma unroll
                            for (int cc = 0; cc < 3; ++cc) r[cc] -= s.bp()[(l * NW + wid - 1) * 3 + cc];
                    }
                    for (int l = kLoc; l < Lv; ++l) {
                        const int st = 1 << l;
                        if (live && lev == l) {
#if PQP_KK_G_SMEM
                            double GL[9], GR[9];
#pragma unroll
                            for (int k = 0; k < 9; ++k) { GL[k] = s.gl(k)[i]; GR[k] = s.gR(k)[i]; }
#endif
#pragma unroll
                            for (int cc = 0; cc < 3; ++cc) {
                                s.push(cc)[i] = GL[cc] * r[0] + GL[3 + cc] * r[1] + GL[6 + cc] * r[2];
                                s.push(3 + cc)[i] = GR[cc] * r[0] + GR[3 + cc] * r[1] + GR[6 + cc] * r[2];
                            }
                        }
                        c.sync();
                        if (live && lev > l) {
                            if (i + st < N) {
#pragma unroll
                                for (int cc = 0; cc < 3; ++cc) r[cc] -= s.push(cc)[i + st];
                            }
                            if (i > 0) {
#pragma unroll
                                for (int cc = 0; cc < 3; ++cc) r[cc] -= s.push(3 + cc)[i - st];
                            }
                        }
                    }
                }
                // up: the stations 32 w (and station 0) through shared memory ...
                for (int l = Lv; l >= kLoc || l == Lv; --l) {
                    if (live && lev == l) {
                        double t0 = Ai[0] * r[0] + Ai[1] * r[1] + Ai[2] * r[2];
                        double t1 = Ai[1] * r[0] + Ai[3] * r[1] + Ai[4] * r[2];
                        double t2 = Ai[2] * r[0] + Ai[4] * r[1] + Ai[5] * r[2];
                        if (l < Lv) {
                            const int st = 1 << l;
#if PQP_KK_G_SMEM
                            double GL[9], GR[9];
#pragma unroll
                            for (int k = 0; k < 9; ++k) { GL[k] = s.gl(k)[i]; GR[k] = s.gR(k)[i]; }
#endif
                            const double a0 = s.xr(0)[i - st], a1 = s.xr(1)[i - st], a2 = s.xr(2)[i - st];
                            t0 -= GL[0] * a0 + GL[1] * a1 + GL[2] * a2;
                            t1 -= GL[3] * a0 + GL[4] * a1 + GL[5] * a2;
                            t2 -= GL[6] * a0 + GL[7] * a1 + GL[8] * a2;
                            if (i + st < N) {
                                const double b0 = s.xr(0)[i + st], b1 = s.xr(1)[i + st], b2 = s.xr(2)[i + st];
                                t0 -= GR[0] * b0 + GR[1] * b1 + GR[2] * b2;
                                t1 -= GR[3] * b0 + GR[4] * b1 + GR[5] * b2;
                                t2 -= GR[6] * b0 + GR[7] * b1 + GR[8] * b2;
                            }
                        }
                        r[0] = t0; r[1] = t1; r[2] = t2;
                        s.xr(0)[i] = t0; s.xr(1)[i] = t1; s.xr(2)[i] = t2;
                    }
                    if (Lv > kLoc) c.sync();
                    if (l == 0) break;
                }
                // ... then down the warp-local levels with shuffles
#pragma unroll
                for (int l = kLoc - 1; l >= 0; --l) {
                    if (l < Ll) {
                        const int st = 1 << l;
                        double xa[3], xb[3];
#pragma unroll
                        for (int cc = 0; cc < 3; ++cc) {
                            xa[cc] = c.w.shfl(r[cc], lane - st);
                            xb[cc] = c.w.shfl(r[cc], lane + st);
                        }
                        if (live && lev == l) {
                            if (lane + st == 32) {      // right neighbour = lane 0 of the next warp
#pragma unroll
                                for (int cc = 0; cc < 3; ++cc) xb[cc] = (i + st < N) ? s.xr(cc)[i + st] : 0.0;
                            }
#if PQP_KK_G_SMEM
                            double GL[9], GR[9];
#pragma unroll
                            for (int k = 0; k < 9; ++k) { GL[k] = s.gl(k)[i]; GR[k] = s.gR(k)[i]; }
#endif
                            double t0 = Ai[0] * r[0] + Ai[1] * r[1] + Ai[2] * r[2];
                            double t1 = Ai[1] * r[0] + Ai[3] * r[1] + Ai[4] * r[2];
                            double t2 = Ai[2] * r[0] + Ai[4] * r[1] + Ai[5] * r[2];
                            t0 -= GL[0] * xa[0] + GL[1] * xa[1] + GL[2] * xa[2];
                            t1 -= GL[3] * xa[0] + GL[4] * xa[1] + GL[5] * xa[2];
                            t2 -= GL[6] * xa[0] + GL[7] * xa[1] + GL[8] * xa[2];
                            if (i + st < N) {
                                t0 -= GR[0] * xb[0] + GR[1] * xb[1] + GR[2] * xb[2];
                                t1 -= GR[3] * xb[0] + GR[4] * xb[1] + GR[5] * xb[2];
                                t2 -= GR[6] * xb[0] + GR[7] * xb[1] + GR[8] * xb[2];
                            }
                            r[0] = t0; r[1] = t1; r[2] = t2;
                        }
                    }
                }
                // (the stations 32 w published their x on the way up: the warp before them may still be reading it)
                if (live && !(Lv > kLoc && lane == 0)) { s.xr(0)[i] = r[0]; s.xr(1)[i] = r[1]; s.xr(2)[i] = r[2]; }
                c.sync();
            };


            // ---- SPIKE form (four- and eight-warp classes) -----------------------------------------------------------------
            // Separator p = station p L (3 unknowns), chunk p = the L - 1 stations after it (I <= 12 unknowns, block
            // tridiagonal K_I).  Per factorisation: the first interior thread of a chunk factors K_I = L D L' (3 x 3
            // blocks); every interior thread then solves its three unit vectors = its three rows of K_I^-1 (kept dense in
            // shared memory) and its rows of the spikes T_l = K_I^-1 E_l, T_r = K_I^-1 E_r (kept in registers); the
            // separator threads form the block-tridiagonal Schur complement, thread 0 factors it, and 3 M threads
            // solve one unit vector each: its inverse is kept dense.  Per iteration:
            //     y = K_I^-1 r_I  (interior threads, dense rows)        g = r_S - E' y  (separator threads)
            //     x_S = S^-1 g    (3 M threads, dense rows)             x_I = y - T_l x_p - T_r x_{p+1}
            // five barriers, no chain longer than one dense row.
            const int L = sd.L, M = sd.M, pitch = sd.pitch;
            const int p = i / L, jj = i - p * L;                               // chunk, position in it (0 = separator)
            int nI = N - 1 - p * L;                                            // interior stations of my chunk
            if (nI > L - 1) nI = L - 1;
            if (nI < 0) nI = 0;
            const int I3 = 3 * nI;
            const bool isSep = live && jj == 0, isInt = live && jj >= 1;
            auto factor_spike = [&]() -> int {
                int ok = 1;
                double A[9], C[9];
                blocks(A, C);
                double *const reg = s.sinv();
                double *const acs = reg, *const cfs = reg + 15 * kT, *const pub = reg + 15 * kT + kMS * kCF;
                if (live) {
                    acs[0 * kT + i] = A[0]; acs[1 * kT + i] = A[1]; acs[2 * kT + i] = A[2];
                    acs[3 * kT + i] = A[4]; acs[4 * kT + i] = A[5]; acs[5 * kT + i] = A[8];
#pragma unroll
                    for (int k = 0; k < 9; ++k) acs[(6 + k) * kT + i] = C[k];
                }
                c.sync();
                auto ldA = [&](int st_, double *o) {
                    o[0] = acs[0 * kT + st_]; o[1] = o[3] = acs[1 * kT + st_]; o[2] = o[6] = acs[2 * kT + st_];
                    o[4] = acs[3 * kT + st_]; o[5] = o[7] = acs[4 * kT + st_]; o[8] = acs[5 * kT + st_];
                };
                auto ldC = [&](int st_, double *o) {
#pragma unroll
                    for (int k = 0; k < 9; ++k) o[k] = acs[(6 + k) * kT + st_];
                };
                double *const cf_ = cfs + p * kCF;          // block k (station p L + k): D_k^-1 at [(k-1) 18], L_k at [(k-1) 18 + 9]
                if (isInt && jj == 1) {
                    double Dm[9], Di[9], Cp[9], Lk[9], Tm[9];
                    ldA(i, Dm);
#pragma unroll
                    for (int k = 1; k <= kNB; ++k) {
                        if (k <= nI) {
                            if (!(Dm[0] > 0.0)) ok = 0;
                            inv3_spd(Dm, Di);
#pragma unroll
                            for (int q = 0; q < 9; ++q) cf_[(k - 1) * 18 + q] = Di[q];
                            if (k < nI) {
                                ldC(i + k - 1, Cp);                    // K[s_k, s_k+1]
                                mtm(Cp, Di, Lk);                       // L_{k+1} = K[s_k+1, s_k] D_k^-1
#pragma unroll
                                for (int q = 0; q < 9; ++q) cf_[k * 18 + 9 + q] = Lk[q];
                                ldA(i + k, Dm);
                                mm(Lk, Cp, Tm);
#pragma unroll
                                for (int q = 0; q < 9; ++q) Dm[q] -= Tm[q];
                                Dm[3] = Dm[1]; Dm[6] = Dm[2]; Dm[7] = Dm[5];
                            }
                        }
                    }
                }
                c.sync();
                if (isInt) {
                    const int m = jj;
                    double Cl[9], Cr[9];
                    ldC(p * L, Cl);                                    // K[separator p, s_1]
                    const bool hasr = (p * L + nI + 1 < N);            // separator p + 1 exists
#pragma unroll
                    for (int q = 0; q < 9; ++q) Cr[q] = 0.0;
                    if (hasr) ldC(p * L + nI, Cr);                     // K[s_nI, separator p + 1]
                    double *const kv = s.kinv() + (size_t)p * kKC + 3 * (m - 1) * kKP;
#pragma unroll
                    for (int cu = 0; cu < 3; ++cu) {
                        double xk[kNB][3], w[3] = {cu == 0 ? 1.0 : 0.0, cu == 1 ? 1.0 : 0.0, cu == 2 ? 1.0 : 0.0};
#pragma unroll
                        for (int k = 1; k <= kNB; ++k) {
                            xk[k - 1][0] = xk[k - 1][1] = xk[k - 1][2] = 0.0;
                            if (k >= m && k <= nI) {
                                const double *Dk = cf_ + (k - 1) * 18;
                                if (k > m) {
                                    const double *Lk = Dk + 9;
                                    const double w0 = -(Lk[0] * w[0] + Lk[1] * w[1] + Lk[2] * w[2]);
                                    const double w1 = -(Lk[3] * w[0] + Lk[4] * w[1] + Lk[5] * w[2]);
                                    const double w2 = -(Lk[6] * w[0] + Lk[7] * w[1] + Lk[8] * w[2]);
                                    w[0] = w0; w[1] = w1; w[2] = w2;
                                }
#pragma unroll
                                for (int q = 0; q < 3; ++q) xk[k - 1][q] = Dk[q * 3] * w[0] + Dk[q * 3 + 1] * w[1] + Dk[q * 3 + 2] * w[2];
                            }
                        }
#pragma unroll
                        for (int k = kNB - 1; k >= 1; --k) {
                            if (k < nI) {                              // x_k -= L_{k+1}' x_{k+1}
                                const double *Ln = cf_ + k * 18 + 9;
#pragma unroll
                                for (int q = 0; q < 3; ++q)
                                    xk[k - 1][q] -= Ln[q] * xk[k][0] + Ln[3 + q] * xk[k][1] + Ln[6 + q] * xk[k][2];
                            }
                        }
#pragma unroll
                        for (int k = 1; k <= kNB; ++k) {
                            if (k <= nI) {
#pragma unroll
                                for (int q = 0; q < 3; ++q) kv[cu * kKP + 3 * (k - 1) + q] = xk[k - 1][q];
                            }
                        }
                        // my rows of the spikes: T_l = K_I^-1[:, first] K[s_1, sep p], T_r = K_I^-1[:, last] K[s_nI, sep p+1]
                        double xl[3] = {xk[0][0], xk[0][1], xk[0][2]}, xr_[3] = {0.0, 0.0, 0.0};
#pragma unroll
                        for (int k = 1; k <= kNB; ++k)
                            if (k == nI) { xr_[0] = xk[k - 1][0]; xr_[1] = xk[k - 1][1]; xr_[2] = xk[k - 1][2]; }
#pragma unroll
                        for (int q = 0; q < 3; ++q) {
                            GL[cu * 3 + q] = xl[0] * Cl[q * 3] + xl[1] * Cl[q * 3 + 1] + xl[2] * Cl[q * 3 + 2];
                            GR[cu * 3 + q] = xr_[0] * Cr[q] + xr_[1] * Cr[3 + q] + xr_[2] * Cr[6 + q];
                        }
                    }
                    // the pieces the Schur complement needs: rows 0..2 of T_l and T_r (first interior station), the last
                    // three rows of T_r (last interior station)
                    double *const pb = pub + p * 27;
                    if (m == 1) {
#pragma unroll
                        for (int q = 0; q < 9; ++q) { pb[q] = GL[q]; pb[9 + q] = GR[q]; }
                    }
                    if (m == nI) {
#pragma unroll
                        for (int q = 0; q < 9; ++q) pb[18 + q] = GR[q];
                    }
                }
                c.sync();
                double *const sc = s.sch();
                if (isSep) {
                    double S[9], Of[9], Co[9], Cpv[9], Tm[9], Pb[9];
                    ldA(i, S);
                    ldC(i, Co);
#pragma unroll
                    for (int q = 0; q < 9; ++q) { Of[q] = 0.0; Cpv[q] = 0.0; }
                    if (nI >= 1) {
#pragma unroll
                        for (int q = 0; q < 9; ++q) Pb[q] = pub[p * 27 + q];
                        mm(Co, Pb, Tm);
#pragma unroll
                        for (int q = 0; q < 9; ++q) S[q] -= Tm[q];
                        if (p + 1 < M) {
#pragma unroll
                            for (int q = 0; q < 9; ++q) Pb[q] = pub[p * 27 + 9 + q];
                            mm(Co, Pb, Tm);
#pragma unroll
                            for (int q = 0; q < 9; ++q) Of[q] = -Tm[q];
                        }
                    }
                    if (p >= 1) {
                        ldC(i - 1, Cpv);                               // K[last interior station of chunk p - 1, separator p]
#pragma unroll
                        for (int q = 0; q < 9; ++q) Pb[q] = pub[(p - 1) * 27 + 18 + q];
                        mtm(Cpv, Pb, Tm);
#pragma unroll
                        for (int q = 0; q < 9; ++q) S[q] -= Tm[q];
                    }
                    S[3] = S[1]; S[6] = S[2]; S[7] = S[5];
#pragma unroll
                    for (int q = 0; q < 9; ++q) { GL[q] = Co[q]; GR[q] = Cpv[q]; }
#pragma unroll
                    for (int q = 0; q < 9; ++q) { sc[p * 27 + q] = S[q]; sc[p * 27 + 9 + q] = Of[q]; }
                }
                c.sync();
                if (tid == 0) {                                        // block L D L' of the separator system
                    double Dg[9], Di[9], Of[9], Lb[9], Tm[9];
#pragma unroll
                    for (int q = 0; q < 9; ++q) Dg[q] = sc[q];
                    for (int q_ = 0; q_ < M; ++q_) {
                        if (!(Dg[0] > 0.0)) ok = 0;
                        inv3_spd(Dg, Di);
#pragma unroll
                        for (int q = 0; q < 9; ++q) sc[q_ * 27 + q] = Di[q];
                        if (q_ + 1 < M) {
#pragma unroll
                            for (int q = 0; q < 9; ++q) Of[q] = sc[q_ * 27 + 9 + q];
                            mtm(Of, Di, Lb);                           // L_{q+1} = S[q+1, q] D_q^-1
#pragma unroll
                            for (int q = 0; q < 9; ++q) { sc[(q_ + 1) * 27 + 18 + q] = Lb[q]; Dg[q] = sc[(q_ + 1) * 27 + q]; }
                            mm(Lb, Of, Tm);
#pragma unroll
                            for (int q = 0; q < 9; ++q) Dg[q] -= Tm[q];
                            Dg[3] = Dg[1]; Dg[6] = Dg[2]; Dg[7] = Dg[5];
                        }
                    }
                }
                c.sync();
                if (tid < 3 * M) {                                     // row tid of the dense inverse: one unit vector
                    double *const sv = reg + (size_t)tid * pitch;
                    const int bt = tid / 3, ct = tid - 3 * bt;
                    double w[3] = {ct == 0 ? 1.0 : 0.0, ct == 1 ? 1.0 : 0.0, ct == 2 ? 1.0 : 0.0};
                    for (int q_ = 0; q_ < bt; ++q_) { sv[3 * q_] = 0.0; sv[3 * q_ + 1] = 0.0; sv[3 * q_ + 2] = 0.0; }
                    for (int q_ = bt; q_ < M; ++q_) {
                        const double *Dk = sc + q_ * 27;
                        if (q_ > bt) {
                            const double *Lk = Dk + 18;
                            const double w0 = -(Lk[0] * w[0] + Lk[1] * w[1] + Lk[2] * w[2]);
                            const double w1 = -(Lk[3] * w[0] + Lk[4] * w[1] + Lk[5] * w[2]);
                            const double w2 = -(Lk[6] * w[0] + Lk[7] * w[1] + Lk[8] * w[2]);
                            w[0] = w0; w[1] = w1; w[2] = w2;
                        }
#pragma unroll
                        for (int q = 0; q < 3; ++q) sv[3 * q_ + q] = Dk[q * 3] * w[0] + Dk[q * 3 + 1] * w[1] + Dk[q * 3 + 2] * w[2];
                    }
                    for (int q_ = M - 2; q_ >= 0; --q_) {
                        const double *Ln = sc + (q_ + 1) * 27 + 18;
                        const double x0 = sv[3 * q_ + 3], x1 = sv[3 * q_ + 4], x2 = sv[3 * q_ + 5];
#pragma unroll
                        for (int q = 0; q < 3; ++q) sv[3 * q_ + q] -= Ln[q] * x0 + Ln[3 + q] * x1 + Ln[6 + q] * x2;
                    }
                    for (int k = 3 * M; k < pitch; ++k) sv[k] = 0.0;
                }
                c.sync();
                // (the Schur scratch lay over the rhs rows: leave the separator rhs row finite up to the pitch)
                for (int k = tid; k < kT; k += kT) s.gg()[k] = 0.0;
                return !c.any(!ok);
            };
            auto solve_spike = [&](double *r) {
                if (live) { s.rr(0)[i] = r[0]; s.rr(1)[i] = r[1]; s.rr(2)[i] = r[2]; }
                c.sync();
                double y[3] = {0.0, 0.0, 0.0};
                if (isInt) {
                    const double *kv = s.kinv() + (size_t)p * kKC + 3 * (jj - 1) * kKP;
                    const int s1 = p * L + 1;
#pragma unroll
                    for (int k = 0; k < kNB; ++k) {
                        if (k < nI) {
                            const double r0 = s.rr(0)[s1 + k], r1 = s.rr(1)[s1 + k], r2 = s.rr(2)[s1 + k];
#pragma unroll
                            for (int q = 0; q < 3; ++q)
                                y[q] += kv[q * kKP + 3 * k] * r0 + kv[q * kKP + 3 * k + 1] * r1 + kv[q * kKP + 3 * k + 2] * r2;
                        }
                    }
                    s.yy(0)[i] = y[0]; s.yy(1)[i] = y[1]; s.yy(2)[i] = y[2];
                }
                c.sync();
                if (isSep) {
                    double g0 = r[0], g1 = r[1], g2 = r[2];
                    if (nI >= 1) {                                     // - K[sep, s_1] y_{s_1}
                        const double a0 = s.yy(0)[i + 1], a1 = s.yy(1)[i + 1], a2 = s.yy(2)[i + 1];
                        g0 -= GL[0] * a0 + GL[1] * a1 + GL[2] * a2;
                        g1 -= GL[3] * a0 + GL[4] * a1 + GL[5] * a2;
                        g2 -= GL[6] * a0 + GL[7] * a1 + GL[8] * a2;
                    }
                    if (p >= 1) {                                      // - K[sep, last interior station of chunk p - 1] y
                        const double a0 = s.yy(0)[i - 1], a1 = s.yy(1)[i - 1], a2 = s.yy(2)[i - 1];
                        g0 -= GR[0] * a0 + GR[3] * a1 + GR[6] * a2;
                        g1 -= GR[1] * a0 + GR[4] * a1 + GR[7] * a2;
                        g2 -= GR[2] * a0 + GR[5] * a1 + GR[8] * a2;
                    }
                    s.gg()[3 * p] = g0; s.gg()[3 * p + 1] = g1; s.gg()[3 * p + 2] = g2;
                }
                c.sync();
                if (tid < 3 * M) {
                    const double *sv = s.sinv() + (size_t)tid * pitch, *gv = s.gg();
                    double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
                    int k = 0;
                    for (; k + 4 <= pitch; k += 4) {
                        double s0, s1_, s2, s3, h0, h1, h2, h3;
                        ld2(sv + k, s0, s1_); ld2(sv + k + 2, s2, s3);
                        ld2(gv + k, h0, h1); ld2(gv + k + 2, h2, h3);
                        a0 += s0 * h0; a1 += s1_ * h1; a2 += s2 * h2; a3 += s3 * h3;
                    }
                    for (; k < pitch; k += 2) {
                        double s0, s1_, h0, h1;
                        ld2(sv + k, s0, s1_); ld2(gv + k, h0, h1);
                        a0 += s0 * h0; a1 += s1_ * h1;
                    }
                    const int bt = tid / 3;
                    s.xr(tid - 3 * bt)[bt * L] = (a0 + a1) + (a2 + a3);
                }
                c.sync();
                if (isSep) {
                    r[0] = s.xr(0)[i]; r[1] = s.xr(1)[i]; r[2] = s.xr(2)[i];
                } else if (isInt) {
                    const int sp_ = p * L, sn = (p + 1) * L;
                    const double a0 = s.xr(0)[sp_], a1 = s.xr(1)[sp_], a2 = s.xr(2)[sp_];
                    double t0 = y[0] - (GL[0] * a0 + GL[1] * a1 + GL[2] * a2);
                    double t1 = y[1] - (GL[3] * a0 + GL[4] * a1 + GL[5] * a2);
                    double t2 = y[2] - (GL[6] * a0 + GL[7] * a1 + GL[8] * a2);
                    if (sn < N) {
                        const double b0 = s.xr(0)[sn], b1 = s.xr(1)[sn], b2 = s.xr(2)[sn];
                        t0 -= GR[0] * b0 + GR[1] * b1 + GR[2] * b2;
                        t1 -= GR[3] * b0 + GR[4] * b1 + GR[5] * b2;
                        t2 -= GR[6] * b0 + GR[7] * b1 + GR[8] * b2;
                    }
                    r[0] = t0; r[1] = t1; r[2] = t2;
                    s.xr(0)[i] = t0; s.xr(1)[i] = t1; s.xr(2)[i] = t2;
                }
                c.sync();
            };
            auto factor = [&]() -> int {
                if constexpr (kSpike) return factor_spike();
                else return factor_cr();
            };
            auto kkt_solve = [&](double *r) {
                if constexpr (kSpike) solve_spike(r);
                else solve_cr(r);
            };

            // a +-OSQP_INFTY bound on the open side of one row of the c1 slack pair (rows 9, 10) makes that row free
            // (RHO_MIN) while its partner keeps the inequality rho; the slack's pivot assumes equal weights: refused
            // (PQP_INVALID_PROBLEM, 0 iterations; see pqp.h)
            const bool split = live && rho_bar(E[9] * lo[9], E[9] * hi[9], 1.0) != rho_bar(E[10] * lo[10], E[10] * hi[10], 1.0);
            if (c.any(split)) status = PQP_INVALID_PROBLEM;
            else if (!factor()) status = PQP_NON_CVX;
            const double alpha = pm.alpha;
            Residuals res{};
            iter = 0;
            // (iter % interval == 0 without a division per iteration: the next multiple is tracked)
            const int ct = pm.check_termination, ai = (pm.adaptive_rho ? pm.adaptive_rho_interval : 0);
            int next_chk = ct, next_ad = ai;
            while (status == PQP_UNSOLVED && iter < pm.max_iter) {
                ++iter;
                const bool can_check = ct > 0 && iter == next_chk;
                const bool can_adapt = ai > 0 && iter == next_ad;
                if (can_check) next_chk += ct;
                if (can_adapt) next_ad += ai;
                const bool chk = can_check || iter == pm.max_iter;
                double z[11];
                if (iter == 1) {
                    // OSQP's first iteration from x = z = y = 0 ends at the cold start (x = 0, v = 0: z = clamp(0),
                    // y = -rho clamp(0)).  Its check and rho adaptation still run below, on w_old = y_0 / rho = 0.
                    if (chk && live) {
#pragma unroll
                        for (int k = 0; k < 11; ++k) Wk(k)[tid] = 0.0;
                    }
                } else {
                    // rhs = sigma x + A' W (2 clamp(v) - v)
                    double g[11];
#pragma unroll
                    for (int k = 0; k < 11; ++k) {
                        z[k] = clamp2(v[k], lo[k], hi[k]);
                        g[k] = W[k] * (2.0 * z[k] - v[k]);
                    }
                    if (live) { s.gr(0)[i] = g[0]; s.gr(1)[i] = g[1]; }
                    c.sync();
                    double r[4] = {0, 0, 0, 0}, xt[4] = {0, 0, 0, 0};
                    if (live) {
                        cols_of(g, r);
#pragma unroll
                        for (int q = 0; q < 4; ++q) r[q] += sg[q] * x[q];
                        if (!hasd) r[2] = 0.0;
                    }
                    xt[3] = r[3] * inv_e;
                    kkt_solve(r);
                    xt[0] = r[0]; xt[1] = r[1]; xt[2] = r[2];
                    if (live) {
                        double ax[11];
                        rows_of(xt[0], xt[1], xt[2], xt[3], ax);
#pragma unroll
                        for (int k = 0; k < 11; ++k) {
                            if (chk) Wk(k)[tid] = v[k] - z[k];
                            v[k] = v[k] + alpha * (ax[k] - z[k]);
                        }
                        if (last) v[4] = 0.0;
#pragma unroll
                        for (int q = 0; q < 4; ++q) x[q] = alpha * xt[q] + (1.0 - alpha) * x[q];
                    }
                }
                if (can_check || can_adapt || iter == pm.max_iter) {
                    c.sync();                        // everybody is done with the x-tilde rows
                    const double cinv = 1.0 / cost_c;
                    double yv[11];
#pragma unroll
                    for (int k = 0; k < 11; ++k) {
                        z[k] = clamp2(v[k], lo[k], hi[k]);
                        yv[k] = W[k] * (v[k] - z[k]) * cinv;
                    }
                    if (live) {
                        s.xr(0)[i] = x[0]; s.xr(1)[i] = x[1]; s.xr(2)[i] = x[2];
                        s.gr(0)[i] = yv[0]; s.gr(1)[i] = yv[1];
                    }
                    c.sync();
                    double red[12];
#pragma unroll
                    for (int k = 0; k < 12; ++k) red[k] = 0.0;
                    if (live) {
                        double ax[11];
                        rows_of(x[0], x[1], x[2], x[3], ax);
#pragma unroll
                        for (int k = 0; k < 11; ++k) {
                            if (k == 4 && last) continue;
                            const double rr = ax[k] - z[k], e = Ek(k)[tid];
                            red[0] = fmax(red[0], fabs(rr)); red[1] = fmax(red[1], fabs(z[k])); red[2] = fmax(red[2], fabs(ax[k]));
                            red[3] = fmax(red[3], e * fabs(rr)); red[4] = fmax(red[4], e * fabs(z[k])); red[5] = fmax(red[5], e * fabs(ax[k]));
                        }
                        double aty[4], px[4];
                        cols_of(yv, aty);
                        px[0] = Pd[0] * x[0]; px[1] = Pd[1] * x[1]; px[3] = Pd[3] * x[3];
                        px[2] = Pd[2] * x[2];
                        if (dprev) px[2] += (-w_cr) * s.xr(2)[i - 1];
                        if (dnext) px[2] += (-w_cr) * s.xr(2)[i + 1];
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            if (q == 2 && !hasd) continue;
                            const double rr = px[q] + aty[q], cd = cost_c * D[q];
                            red[6] = fmax(red[6], fabs(rr)); red[7] = fmax(red[7], fabs(px[q])); red[8] = fmax(red[8], fabs(aty[q]));
                            red[9] = fmax(red[9], cd * fabs(rr)); red[10] = fmax(red[10], cd * fabs(px[q])); red[11] = fmax(red[11], cd * fabs(aty[q]));
                        }
                    }
                    c.max_n(red, 12);
                    const double pr = red[0], nz = red[1], nax = red[2], prs = red[3], nzs = red[4], naxs = red[5];
                    const double dr = red[6], npx = red[7], naty = red[8], drs = red[9], npxs = red[10], natys = red[11];
                    if (chk) {
                        // primal-infeasibility certificate (OSQP is_primal_infeasible), see pqp_gen_core.cuh
                        double gq[11], c_nrm = 0, c_lhs = 0, c_cert = 0;
#pragma unroll
                        for (int k = 0; k < 11; ++k) {
                            gq[k] = 0.0;
                            if (!live || (k == 4 && last)) continue;
                            const double e = Ek(k)[tid];
                            double gg = W[k] * ((v[k] - z[k]) - Wk(k)[tid]);
                            const bool u_inf = e * hi[k] > kOsqpInfty * kMinScaling;
                            const bool l_inf = e * lo[k] < -kOsqpInfty * kMinScaling;
                            if (u_inf) gg = l_inf ? 0.0 : fmin(gg, 0.0);
                            else if (l_inf) gg = fmax(gg, 0.0);
                            gq[k] = gg;
                            c_nrm = fmax(c_nrm, fabs(gg));
                            c_lhs += hi[k] * fmax(gg, 0.0) + lo[k] * fmin(gg, 0.0);
                        }
                        if (live) { s.gr(0)[i] = gq[0]; s.gr(1)[i] = gq[1]; }
                        c.sync();
                        if (live) {
                            double aty[4];
                            cols_of(gq, aty);
#pragma unroll
                            for (int q = 0; q < 4; ++q) {
                                if (q == 2 && !hasd) continue;
                                c_cert = fmax(c_cert, fabs(aty[q]));
                            }
                        }
                        double r2[2] = {c_nrm, c_cert};
                        c.max_n(r2, 2);
                        res.inf_nrm = r2[0]; res.inf_cert = r2[1];
                        res.inf_lhs = c.sum(c_lhs);
                    }
                    res.pri_res = pr; res.dua_res = dr; res.pri_nrm = fmax(nz, nax); res.dua_nrm = fmax(npx, naty);
                    if (can_check || iter == pm.max_iter) status = termination_verdict(pm, res);
                    if (status == PQP_UNSOLVED && can_adapt) {
                        const double rho_new = rho_estimate(rho, prs, drs, fmax(nzs, naxs), fmax(npxs, natys));
                        if (rho_changed(pm, rho_new, rho)) {
                            if (live) {
#pragma unroll
                                for (int k = 0; k < 11; ++k) {
                                    if (k == 4 && last) continue;
                                    const double e = Ek(k)[tid];
                                    const double El = e * lo[k], Eu = e * hi[k];
                                    const double ro = rho_bar(El, Eu, rho), rn = rho_bar(El, Eu, rho_new);
                                    const double zz = clamp2(v[k], lo[k], hi[k]);
                                    v[k] = zz + (v[k] - zz) * (ro / rn);
                                    W[k] = rn * e * e;
                                }
                            }
                            rho = rho_new;
                            if (!factor()) status = PQP_NON_CVX;
                        }
                    }
                }
            }
            if (status == PQP_UNSOLVED) status = max_iter_verdict(pm, res);
        }
        // ---- epilogue: getOptimizedPath (solver_k_as_input.cpp:22-44)
        const bool has_sol = has_solution(status);
        c.sync();
        if (live) s.xr(2)[i] = x[2];
        c.sync();
        if (live) {
            double ey = qnan, ephi = qnan, kk = qnan, tx, ty;
            if (has_sol) { ey = x[1]; ephi = x[0]; kk = last ? s.xr(2)[i - 1] : x[2]; }
            optimized_station(ref[i], ey, ephi, kk, out[i], tx, ty);
            s.ox()[i] = tx; s.oy()[i] = ty;
            store_frenet(bv.out_frenet, off + i, ey, ephi, kk);
        }
        c.sync();
        if (tid == 0) {
            double acc = 0.0;
            for (int k = 0; k < N; ++k) {
                if (k > 0) {
                    const double dx = s.ox()[k] - s.ox()[k - 1], dy = s.oy()[k] - s.oy()[k - 1];
                    acc += sqrt(dx * dx + dy * dy);
                }
                out[k].s = acc;
            }
            bv.status[prob] = status;
            if (bv.iters) bv.iters[prob] = iter;
        }
    }
};

}  // namespace pqp
