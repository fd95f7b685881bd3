// pqp_kp_core3.cuh -- thread-per-station "KP" solver: the production kernel for N <= 32*NW stations.
//
// Same mathematics as pqp_kp_core.cuh / pqp_kp_core2.cuh (read their headers first).  A CTA of NW
// warps solves one path; what changes is WHERE things live and HOW the reduced KKT is applied:
//   * thread t owns station t: its 11 row values v, 9 row weights W, 8 bounds, transition
//     coefficients, proximal terms and its slice (e_y, e_phi, kappa, s) of the iterate stay in
//     REGISTERS for the whole solve (thread j < ch additionally owns held control u_j);
//   * shared memory only holds what is exchanged: the rhs / x-tilde vector, the dynamics-row values a
//     neighbouring station needs, and the factorisation;
//   * reduced KKT, per (re)factorisation: lane p of warp 0 factors the interior after separator p
//     (banded LDL'), 6M threads build the spikes T_p = K_I^-1 K[I, S_p | S_p+1], and the M x M
//     block-tridiagonal Schur complement over the separators is inverted DENSELY (3M threads, one
//     unit vector each).  Per ADMM iteration:
//         g   = r_S - T' r_I                (3M threads, no dependency chain)
//         y   = K_I^-1 r_I                  (warp 0, one banded solve per lane)   } concurrently
//         x_S = Sinv g                      (3M threads of warps 1.., dense dot)  }
//         x_I = y - T x_S                   (station threads)
//     so the only serial chain left in an iteration is ONE interior substitution.
//
// Reference being replaced: src/solver/solver_kp_as_input.cpp:26-203 + the OSQP solve at
// src/solver/solver.cpp:66-74.
#pragma once
#include <type_traits>
#include "pqp_kp_core2.cuh"

namespace pqp {

struct Kp3Dims {
    int N, keep, ch, h, L, M, I, CS, nv, bw, nS;
};

// separators every L stations with at most mmax of them (the dense separator inverse is (3M)^2)
PQP_HD Kp3Dims kp3_dims_raw(int N, int keep, int mmax = 17) {
    const KpDims a = kp_dims(N, keep);
    Kp3Dims d;
    d.N = N; d.keep = keep; d.ch = a.ch; d.h = a.h; d.bw = a.bw;
    int L = keep * ((N - 1) / (mmax * keep) + 1);   // smallest multiple of keep with (N-1)/L < mmax
    if (L < 2) L = 2;
    d.L = L;
    d.M = (N - 1) / L + 1;
    d.I = 3 * (L - 1) + L / keep;
    d.CS = d.I + 3;
    d.nv = d.M * d.CS;
    d.nS = 3 * d.M;
    return d;
}

// MMAX = most separators a path may have: 17 (two CTAs of four warps per SM) or 34 for the eight-warp form, which
// keeps the interiors of a 200-station path at 17 unknowns instead of 37 (the interior solves are the serial part).
// FORM = 0: "KP" (SolverKpAsInput); FORM = 2: "KPC" (SolverKpAsInputConstrained, solver_kp_as_input_constrained.cpp:13-221):
// the same banded reduced KKT -- its extra slacks (curvature slack per station, curvature-rate slack per held control)
// couple to kappa / u through soft-row PAIRS of equal weight and opposite sign and therefore decouple exactly, like the
// corridor slack -- with another row set per station: three hard circles (d1, d2, d4), one soft pair (d3), a soft
// pair instead of the curvature box, keep_control_steps fixed at 4, the end offset row free.
template <int IMAX, int BW, int NW, int MMAX = 17, int FORM = 0>
struct Kp3 {
    static constexpr bool kKPC = (FORM == 2);
    static constexpr int kWE = kKPC ? 10 : 9;    // row scalings E kept per station in the workspace
    static constexpr int kWD = kKPC ? 5 : 4;     // column scalings D per station
    static constexpr int kWR = kKPC ? 12 : 11;   // parked dual rows per station
    static constexpr int kUbF = kKPC ? 11 : 4;   // shared-memory fields per held control
    static constexpr int kT = NW * 32;     // threads = max stations
    using K2 = Kp2<IMAX, BW, NW * 100 + MMAX + 1000 * FORM>;   // reuses the unrolled interior factor / solve (own copies per kernel)
    // Small interiors keep a DENSE inverse (row-major, [interior][row][kRow]) in place of the band
    // factor once a refactorisation is done: y = K_I^-1 r_I then is a mat-vec spread over every thread
    // of the CTA instead of M serial banded substitutions on warp 0 (the longest phase of an iteration).
    // Two-level separator system (every 34-separator class): the odd separators of the block-tridiagonal Schur system
    // are eliminated in closed form (3x3 blocks), only the even ones keep a dense inverse (<= 51 x 51 instead of
    // 102 x 102: a quarter of the shared memory and of the separator product's work).
    static constexpr bool kTwoLevel = (MMAX > 17);
    static constexpr bool kDense = (IMAX <= 17);   // (17-unknown interiors: 2 x 95 KB at 17 separators, 181 KB at 34 -- one CTA per SM either way)
    static constexpr int kSolveT = (MMAX + 31) / 32 * 32;   // threads that run the banded interior solves (non-dense form)
    static constexpr int kRow = IMAX + 1;                // row pitch of a dense inverse (even: 128-bit loads stay aligned, 4*lane word offsets)
    static constexpr int kFacSlots = kDense ? IMAX * kRow : IMAX * (BW + 1);
    static_assert(!kDense || IMAX * kRow >= IMAX * (BW + 1) + kRed2 + 27 + 12, "refactorisation scratch must fit behind the band factor");
    // Long-path classes (more than eight warps: up to 416 stations, 37-unknown interiors) need every byte of the
    // 227 KB a CTA can opt into: their refactorisation scratch is overlaid on the rhs / y vectors (free while a
    // refactorisation runs; both are zeroed again at its end so that the padded entries stay finite).
    static constexpr bool kScratchOnVec = !kDense && (NW > 8) && kTwoLevel && (2 * ((IMAX + 3) | 1) >= kRed2 + 27 + 12);
    static_assert(!(kKPC && kScratchOnVec), "the long-path classes have no room for the KPC control state");
    // exchange rows of kT doubles: 0..5, ds, separator rhs; the long-path classes park the separator rhs in row 5
    // (only the Ruiz sweeps and diagnostic builds use that row otherwise)
    static constexpr int kExRows = kScratchOnVec ? 7 : 8;
    static constexpr int kCtaScratch = (NW <= 8) ? 128 : 256;   // doubles reserved ahead of the layout for the CTA reductions (16 per warp)
#ifdef PQP_PHASE_TIMING
    static constexpr bool kPhTime = !kScratchOnVec;   // (diagnostic builds: which classes record phase times)
#endif
    // The 100-station class (config 2's kernel) runs a leaner ADMM iteration: four CTA barriers instead of six (the row
    // warps of (b2) do not wait for the separator rhs, x-tilde is published without a barrier of its own) and a smaller
    // inner loop (direct barriers, a rolled held-control loop, no integer division).  Same floating-point operations in
    // the same order, so the same bits; every other class compiles exactly as before.
    static constexpr bool kLean = IMAX == 17 && BW == 6 && NW == 4 && MMAX == 17 && FORM == 0;

    PQP_HD static Kp3Dims dims(int N, int keep) {
        Kp3Dims d = kp3_dims_raw(N, keep, MMAX);
        d.CS = (IMAX + 3) | 1;
        d.nv = d.M * d.CS;
        return d;
    }
    PQP_HD static bool fits(int N, int keep) {
        if (N < 2 || N > kT || keep < 1 || keep > 10) return false;
        const Kp3Dims d = kp3_dims_raw(N, keep, MMAX);
        if (kScratchOnVec && 2 * ((d.ch + 1) & ~1) > kT - 64) return false;   // (held-control state in the row tails, see Smem)
        return d.I <= IMAX && d.bw <= BW && d.M <= MMAX && 6 * d.M <= kT && kSolveT + 3 * d.M <= kT;
    }

    // ---- shared memory (doubles) ---------------------------------------------------------------
    struct Smem {
        double *base;
        int nv, M, nS, ch;
        PQP_DEV double *tr() const { return base; }                       // rhs, then x-tilde  [nv]
        PQP_DEV double *yv() const { return base + nv; }                  // K_I^-1 r_I         [nv]
        PQP_DEV double *ex(int k) const { return base + 2 * nv + k * kT; }  // 6 exchange rows of kT
        PQP_DEV double *dsS() const { return ex(6); }                     // ds per station     [kT]
        PQP_DEV double *gS() const { return ex(kScratchOnVec ? 5 : 7); }     // separator rhs      [nS <= kT]
        // 100-station class: per thread, i / L and tid / M as ints in exchange row 4 (in that class only the Ruiz sweeps
        // use the row), read back in every iteration instead of two integer divisions
        PQP_DEV int *ixS() const { return reinterpret_cast<int *>(ex(4)); }
        // State only a few threads touch lives in shared memory instead of in (everybody's) registers: the two end rows of
        // the last station (v, W, window: 6 doubles) and the held controls' (v, W, x, sigma), ch each.  It has a region of
        // its own after the exchange rows -- except in the long-path classes, which have no byte to spare: there it sits
        // in the unused tails of the separator rows 3 (x_S: 3M <= 102 entries used), 4 (<= 51 used) and 5 (<= 102 used).
        PQP_DEV int chp() const { return (ch + 1) & ~1; }
        PQP_DEV double *endr() const { return kScratchOnVec ? ex(4) + 56 : ex(kExRows); }   // vEY vEH WEY WEH lEH uEH . .
        PQP_DEV double *ubs(int f) const {                                                 // f: 0 v, 1 W, 2 x, 3 sigma (, 4.. KPC)
            if (!kScratchOnVec) return ex(kExRows) + 8 + f * chp();
            return f == 0 ? ex(4) + 64 : f == 3 ? ex(4) + 64 + chp() : f == 1 ? ex(3) + 104 : ex(5) + 104;
        }
        PQP_HD static int aux_doubles(int ch_) { return kScratchOnVec ? 0 : 8 + kUbF * ((ch_ + 1) & ~1); }
        PQP_DEV double *fac() const { return ex(kExRows) + aux_doubles(ch); }   // [IMAX*(BW+1)*M]; kDense: then K_I^-1 [M][IMAX][kRow]
        PQP_DEV double *T() const { return fac() + kFacSlots * M; }       // spikes T[c][pos], c < 6: [6*nv]
        PQP_DEV int nSd() const { return kTwoLevel ? 3 * ((M + 1) / 2) : nS; }   // order of the dense separator inverse
        PQP_DEV double *Sinv() const { return T() + 6 * nv; }             // [nSd*nSd]
        // refactorisation scratch [kRed2*M] + blocks [27*M] + couplings [12*M].  With dense interiors it lives in the
        // part of the fac / kinv region the band factor does not use (free until the dense inverses are written, which
        // is the last step of a refactorisation): two CTAs then need < 196 KB and the SM keeps 60 KB of L1 for the spills.
        PQP_DEV double *red() const { return kDense ? fac() + IMAX * (BW + 1) * M : (kScratchOnVec ? base : Sinv() + nSd() * nSd()); }
        PQP_DEV double *blk() const { return red() + kRed2 * M; }         // A|C|Off per chunk [27*M]
        PQP_DEV double *cpl() const { return blk() + 27 * M; }            // coupling coefs [12*M]
        // two-level form: per separator E = Dg^-1 (odd) | PL | PR (even) | Off copy [36*M]; reduced system [kRed2*ceil(M/2)]
        PQP_DEV double *lv() const { return (kDense || kScratchOnVec) ? Sinv() + nSd() * nSd() : cpl() + 12 * M; }
        PQP_DEV double *red2() const { return lv() + 36 * M; }
    };
    PQP_HD static size_t smem_doubles(const Kp3Dims &d) {
        return 2 * (size_t)d.nv + (size_t)kExRows * kT + (size_t)Smem::aux_doubles(d.ch) + (size_t)kFacSlots * d.M + 6 * (size_t)d.nv +
               (kTwoLevel ? (size_t)9 * ((d.M + 1) / 2) * ((d.M + 1) / 2) : (size_t)d.nS * d.nS) +
               ((kDense || kScratchOnVec) ? 0 : (size_t)(kRed2 + 27 + 12) * d.M) +
               (kTwoLevel ? (size_t)36 * d.M + (size_t)kRed2 * ((d.M + 1) / 2) : 0);
    }

#define PQP_F(k, dd) fcol[((k) * (BW + 1) + (dd)) * Mst]

    // per-thread station state ------------------------------------------------------------------
    struct St {
        // row state and data
        double vD0, vD1, vD2, vKB, vSB, vH1, vH3, vS4m, vS4p, vS2m, vS2p;
        double WD0, WD1, WD2, WKB, WSB, WH1, WH3, WS4, WS2;
        double lH1, uH1, lH3, uH3, uS4m, lS4p, uS2m, lS2p;
        double b0, b1, b2;          // bounds of the dynamics (equality) rows
        double ds, q10;             // transition i -> i+1
        double dst, qt;             // transition i-1 -> i
        double sga, sgb, sgc, sgs, ksinv;
        double xa, xb, xc, xs;      // iterate
        // KPC only: soft curvature-limit pair (kappa + sk >= -mk, kappa - sk <= mk), the box of its slack sk, the third
        // hard circle row (d4); the KP names H3 / S4 then stand for the d2 hard row and the d3 soft pair
        double vKL, vKU, WK, mk, vSK, WSK, uSK, xk, sgk, kkinv, vH4, WH4, lH4, uH4;
        int pos, posp, posup;       // padded index of a_i, a_{i-1}, u of transition i-1
        bool live, first, last, sep;
    };
    struct Ub {                     // held control j (thread j < ch)
        int pos, t0, t1;            // padded index, first / last transition of the block (v, W, x, sigma: shared memory)
        bool live;
    };

    // Dense interior inverses over the band factor (see the call site).  Out of line: what it needs in registers stays out
    // of the solve's own allocation.
    PQP_NOINLINE static void dense_build(const Cta &c, double *fac, int M, int tid) {
        const int Mst = M;
        c.sync();   // the separator-system phases before it are done with the scratch behind the band factor
        const int bandEnd = IMAX * (BW + 1) * M;
        const int nStaged = (bandEnd + kRow - 1) / kRow;        // <= kT for every dense class
        static_assert(!kDense || (IMAX * (BW + 1) * MMAX + kRow - 1) / kRow <= kT, "one staged row per thread");
        for (int r = nStaged + tid; r < IMAX * M; r += kT) {
            const int p = r / IMAX, j = r - p * IMAX;
            double *kv = fac + (size_t)r * kRow;
            K2::local_solve_unit_mem(j, kv, fac + p, Mst);
            kv[IMAX] = 0.0;
        }
        double xc[IMAX];
        const bool staged = tid < nStaged && tid < IMAX * M;
        if (staged) K2::local_solve_unit(tid % IMAX, xc, fac + tid / IMAX, Mst);
        c.sync();
        if (staged) {
            double *kv = fac + (size_t)tid * kRow;
#pragma unroll
            for (int k = 0; k < IMAX; ++k) kv[k] = xc[k];
            kv[IMAX] = 0.0;
        }
    }

    // ---- the whole per-path solve ----------------------------------------------------------------
    // Is the constant of the dynamics rows of transition r[0] -> r[1] NaN as the reference computes it (see the call
    // site)?  Out of line: the division's registers stay out of the solve's own allocation.
    PQP_NOINLINE static int dyn_const_nan(const pqp_state *r) {
        const double ds = r[1].s - r[0].s, rkp = (r[1].k - r[0].k) / ds;
        return !(ds * (rkp - rkp) == 0.0);
    }

    PQP_DEV static void solve_path(const Cta &c, const DevParams &pm, const BatchView &bv, int prob, double *smem,
                                   size_t smem_cap) {
        const int lane = c.lane(), tid = c.tid(), wid = c.wid;
#ifdef PQP_PHASE_TIMING
        const long long ph_kernel_t0 = clock64();
        long long ph_refactor = 0, ph_check = 0, ph_scale = 0, ph_nref = 0;
        long long rt_acc[8] = {0, 0, 0, 0, 0, 0, 0, 0}, rt_t = 0;
        long long ck_acc[6] = {0, 0, 0, 0, 0, 0}, ck_t = 0;   // check block (d), per warp: see PQP_CK
#endif
        const int N = bv.n_points[prob];
        const int off = bv.offsets[prob];
        const pqp_state *ref = bv.ref + off;
        const pqp_station_bounds *bnd = bv.bounds + off;
        pqp_state *out = bv.out_states + off;
        int keep = 1;
        if constexpr (kKPC) {
            keep = 4;               // solver_kp_as_input_constrained.cpp:17
        } else {
            double interval = 0.0;  // solver.cpp:21-27 (std::max: a NaN interval is skipped), solver_kp_as_input.cpp:17
            for (int i = 1; i < N && i < 10; ++i) {
                const double dd = ref[i].s - ref[i - 1].s;
                interval = interval < dd ? dd : interval;
            }
            const double q = 1.2 / interval;
            keep = (q < 2147483647.0) ? (int)q : 2147483647;
            if (!(q == q)) keep = 0;
            if (keep < 1) keep = 1;
        }
        const double qnan = nan("");
        const bool shape_ok = fits(N, keep);
        const Kp3Dims d = dims(shape_ok ? N : 2, shape_ok ? keep : 1);
        if (!shape_ok || smem_doubles(d) > smem_cap || !bv.workspace || (kKPC && (!bv.max_k || !bv.max_kp))) {
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
        Smem s;
        s.base = smem; s.nv = d.nv; s.M = d.M; s.nS = d.nS; s.ch = d.ch;
        const int M = d.M, L = d.L, ch = d.ch, nS = d.nS, Mst = d.M;
        const int Mr = kTwoLevel ? (M + 1) / 2 : M, nSr = 3 * Mr;   // order of the dense separator inverse (reduced system)
        double *ws = kp_ws_base(bv.workspace, off, prob);  // E[9] per station, [9N..] EUB, EEnd; then D
        double *wold = kp_ws_wold(ws, N);                  // w = v - clamp(v) of the previous iterate (infeasibility check)
        const KpDims ka = kp_dims(N, keep);
        // workspace layout of the scalings: E per station [kWE], E of the control rows, the two end rows, D per station, D per control
        const size_t oEU = (size_t)kWE * N, oEnd = oEU + (size_t)(kKPC ? 2 : 1) * ch, oD = oEnd + 2, oDu = oD + (size_t)kWD * N;
        // per-form row coefficients: hard rows H1, H3 (, H4), soft pairs S4 (, S2); bounds of the end-offset row
        const double cH1 = pm.d1, cH3 = kKPC ? pm.d2 : pm.d3, cS4 = kKPC ? pm.d3 : pm.d4, cS2 = pm.d2, cH4 = pm.d4;
        const double lEY = kKPC ? -kOsqpInfty : -1.0, uEY = kKPC ? kOsqpInfty : 1.0;   // :204-205: end e_y is not constrained in KPC
        // ---- station / control ownership and padded positions
        St st;
        const int i = tid;
        st.live = i < N;
        st.first = (i == 0);
        st.last = (i == N - 1);
        st.sep = st.live && (i % L == 0);
        st.pos = st.posp = st.posup = 0;
        if (st.live) {
            const int p = i / L;
            st.pos = p * d.CS + (kp_gx(ka, i) - kp_gx(ka, p * L));
            if (i > 0) {
                const int t = i - 1, pt = t / L;
                st.posp = pt * d.CS + (kp_gx(ka, t) - kp_gx(ka, pt * L));
                const int j = t / keep;
                int home = j * keep + d.h;
                if (home > N - 1) home = N - 1;
                const int pu = home / L;
                st.posup = pu * d.CS + (kp_gu(ka, j) - kp_gx(ka, pu * L));
            }
        }
        Ub ub;
        ub.live = tid < ch;
        ub.pos = 0; ub.t0 = 0; ub.t1 = -1;
        if (ub.live) {
            const int j = tid;
            int home = j * keep + d.h;
            if (home > N - 1) home = N - 1;
            const int pu = home / L;
            ub.pos = pu * d.CS + (kp_gu(ka, j) - kp_gx(ka, pu * L));
            ub.t0 = j * keep;
            ub.t1 = j * keep + keep - 1;
            if (ub.t1 > N - 2) ub.t1 = N - 2;
        }
        // partition threads (the first M): interior after separator p
        int lo = 3, cnt = 0;
        const bool solver = (MMAX <= 32) ? (wid == 0 && lane < M) : (tid < M);
        const int sid = (MMAX <= 32) ? lane : tid;      // interior owned by a solver thread
        if (solver) {
            const int g0 = kp_gx(ka, sid * L);
            const int g1 = (sid + 1 < M) ? kp_gx(ka, (sid + 1) * L) : ka.nred;
            lo = sid * d.CS + 3;
            cnt = g1 - g0 - 3;
        }
        // end-heading window, solver_kp_as_input.cpp:193-201
        double lEH0 = -kOsqpInfty, uEH0 = kOsqpInfty;
        if (pm.constraint_end_heading) {
            const double pi = 3.14159265358979323846;
            const double end_psi = constraint_angle(bv.end_heading[prob] - ref[N - 1].z);
            if (end_psi < 70 * pi / 180) {
                lEH0 = end_psi - 5 * pi / 180;
                uEH0 = end_psi + 5 * pi / 180;
            }
        }
        // ---- per-station coefficients (setConstraintMatrix :84-98, :143-151, :166-187)
        int invalid = (cnt > IMAX);
        // The reference's constant of the dynamics rows, ds (c - a ref - b ref_kp) with ref_kp = dk / ds (:86-97), is NaN
        // -- and osqp_setup refuses the path -- exactly when its kappa row ds (ref_kp - ref_kp) is: a zero-length
        // interval, a non-finite s or kappa.  A pass of its own, so that nothing of it stays live in the block below.
        if (tid + 1 < N && dyn_const_nan(ref + tid)) invalid = 1;
        st.ds = st.q10 = st.dst = st.qt = 0.0;
        st.b0 = st.b1 = st.b2 = 0.0;
        st.lH1 = st.lH3 = -1.0; st.uH1 = st.uH3 = 1.0;
        st.uS4m = st.uS2m = 0.0; st.lS4p = st.lS2p = 0.0;
        st.vKL = st.vKU = st.WK = st.mk = st.vSK = st.WSK = st.uSK = st.xk = st.sgk = st.kkinv = 0.0;
        st.vH4 = st.WH4 = 0.0; st.lH4 = -1.0; st.uH4 = 1.0;
        if (st.live) {
            const double kap = ref[i].k;
            if (!st.last) {
                st.ds = ref[i + 1].s - ref[i].s;
                st.q10 = -(kap * kap) * st.ds;
            }
            if (st.first) {
                st.b0 = -bv.x0[3 * (size_t)prob];
                st.b1 = -bv.x0[3 * (size_t)prob + 1];
                st.b2 = -bv.x0[3 * (size_t)prob + 2];
            } else {
                const double kp_ = ref[i - 1].k;
                st.dst = ref[i].s - ref[i - 1].s;
                st.qt = -(kp_ * kp_) * st.dst;
                st.b1 = st.dst * kp_;
            }
            const pqp_station_bounds bb = bnd[i];
            st.lH1 = bb.c0_lb; st.uH1 = bb.c0_ub;
            if constexpr (kKPC) {   // solver_kp_as_input_constrained.cpp:185-200: hard c0, c1, c3; soft c2
                st.lH3 = bb.c1_lb; st.uH3 = bb.c1_ub;
                st.lH4 = bb.c3_lb; st.uH4 = bb.c3_ub;
                st.uS4m = bb.c2_ub - pm.margin; st.lS4p = bb.c2_lb + pm.margin;
                st.uS2m = 0.0; st.lS2p = 0.0;
                st.mk = bv.max_k[off + i];                               // :160-172
                st.uSK = fmax(pm.kmax - st.mk, 0.0);
                if (!(bb.c3_lb <= bb.c3_ub) || !(-st.mk <= kOsqpInfty) || !(-kOsqpInfty <= st.mk) || !(0.0 <= st.uSK)) invalid = 1;
            } else {
                st.lH3 = bb.c2_lb; st.uH3 = bb.c2_ub;
                st.uS4m = bb.c3_ub - pm.margin; st.lS4p = bb.c3_lb + pm.margin;
                st.uS2m = bb.c1_ub - pm.margin; st.lS2p = bb.c1_lb + pm.margin;
            }
            if (!(st.lH1 <= st.uH1) || !(st.lH3 <= st.uH3)) invalid = 1;
            if (!(-kOsqpInfty <= st.uS4m) || !(st.lS4p <= kOsqpInfty) || !(-kOsqpInfty <= st.uS2m) ||
                !(st.lS2p <= kOsqpInfty))
                invalid = 1;
            s.dsS()[i] = st.ds;
        }
        if (!(0.0 <= pm.margin) || !(-pm.kmax <= pm.kmax) || !(lEH0 <= uEH0)) invalid = 1;
        invalid = c.any(invalid);

        int status = PQP_UNSOLVED;
        int iter = 0;
        // end rows (only the thread of station N-1 touches them) and held controls (threads j < ch): in shared memory
        double *const er = s.endr();
        double *const uS0 = s.ubs(0), *const uS1 = s.ubs(1), *const uS2 = s.ubs(2), *const uS3 = s.ubs(3);
        // KPC: the control has a soft rate-limit pair (u + p >= -mkp, u - p <= mkp) and the box of its slack p >= 0:
        // field 0 v(KPL) 1 W(KP pair) 2 x(u) 3 sigma(u) | 4 v(KPU) 5 v(box p) 6 W(box p) 7 x(p) 8 sigma(p) 9 1 / pivot(p) 10 mkp
        double *const uSx = s.ubs(4);   // fields 4.. at uSx[(f - 4) * s.chp() + tid]
        const int uCp = s.chp();
#define PQP_UBF(f) uSx[((f) - 4) * uCp + tid]
#define vEY er[0]
#define vEH er[1]
#define WEY er[2]
#define WEH er[3]
#define lEH er[4]
#define uEH er[5]
#define PQP_UBV uS0[tid]
#define PQP_UBW uS1[tid]
#define PQP_UBX uS2[tid]
#define PQP_UBSG uS3[tid]
        st.xa = st.xb = st.xc = st.xs = 0.0;
        double cost_c = 1.0;
        if (invalid) {
            status = PQP_INVALID_PROBLEM;
        } else {
#ifdef PQP_PHASE_TIMING
            const long long ph_scale_t0 = clock64();
#endif
            // ================= Ruiz equilibration + cost scaling (OSQP scale_data) =================
            double Da = 1, Db = 1, Dc = 1, Dsv = 1, Du = 1, Dt = 1;
            double e0 = 1, e1 = 1, e2 = 1, eKB = 1, eSB = 1, eH1 = 1, eH3 = 1, eS4 = 1, eS2 = 1, eUB = 1, eEY = 1, eEH = 1;
            double Dk = 1, Dp = 1, eSK = 1, eH4 = 1, eSKP = 1;   // KPC: sk, p columns; sk box, d4 hard row, p box  (eKB = the kappa pair, eUB = the rate pair)
            const double ad1 = fabs(pm.d1), ad2 = fabs(pm.d2), ad3 = fabs(pm.d3), ad4 = fabs(pm.d4);
            if constexpr (kKPC) {
                const double aH1 = fabs(cH1), aH3 = fabs(cH3), aH4 = fabs(cH4), aS4 = fabs(cS4);
                const double wk_ = 500.0, wp_ = 25000.0 * keep;   // w_k_slack, w_kp_slack * keep_control_steps_ (:52-53,63)
                for (int sweep = 0; sweep < pm.scaling; ++sweep) {
                    if (st.live) {
                        s.ex(0)[i] = Da; s.ex(1)[i] = Db; s.ex(2)[i] = Dc;
                        s.ex(3)[i] = e0; s.ex(4)[i] = e1; s.ex(5)[i] = e2;
                    }
                    if (ub.live) s.tr()[tid] = Du;
                    c.sync();
                    double fDa = 1, fDb = 1, fDc = 1, fDs = 1, fDu = 1, fDk = 1, fDp = 1;
                    double f0 = 1, f1 = 1, f2 = 1, fK = 1, fSB = 1, fSK = 1, fH1 = 1, fH3 = 1, fH4 = 1, fS4 = 1, fKP = 1, fSKP = 1, fEY = 1, fEH = 1;
                    if (st.live) {
                        double Aa = fmax(fmax(e0, eH1), fmax(eH3, fmax(eH4, eS4)));
                        double Ab = fmax(fmax(e1, eH1 * aH1), fmax(eH3 * aH3, fmax(eH4 * aH4, eS4 * aS4)));
                        double Ac = fmax(e2, eKB);
                        if (!st.last) {
                            const double e0n = s.ex(3)[i + 1], e1n = s.ex(4)[i + 1], e2n = s.ex(5)[i + 1];
                            const double aq = fabs(st.q10);
                            Aa = fmax(Aa, fmax(e0n, e1n * aq));
                            Ab = fmax(Ab, fmax(e0n * st.ds, e1n));
                            Ac = fmax(Ac, fmax(e1n * st.ds, e2n));
                        } else {
                            Aa = fmax(Aa, eEY);
                            Ab = fmax(Ab, eEH);
                        }
                        const double As = fmax(eSB, eS4);
                        const double Ak = fmax(eSK, eKB);
                        fDa = 1.0 / sqrt(limit_scaling(fmax(cost_c * pm.w_pq * Da * Da, Aa * Da)));
                        fDb = 1.0 / sqrt(limit_scaling(Ab * Db));
                        fDc = 1.0 / sqrt(limit_scaling(fmax(cost_c * pm.w_c * Dc * Dc, Ac * Dc)));
                        fDs = 1.0 / sqrt(limit_scaling(fmax(cost_c * pm.w_s * Dsv * Dsv, As * Dsv)));
                        fDk = 1.0 / sqrt(limit_scaling(fmax(cost_c * wk_ * Dk * Dk, Ak * Dk)));
                        double r0, r1, r2;
                        if (st.first) {
                            r0 = e0 * Da; r1 = e1 * Db; r2 = e2 * Dc;
                        } else {
                            const double Dat = s.ex(0)[i - 1], Dbt = s.ex(1)[i - 1], Dct = s.ex(2)[i - 1];
                            const double Dut = s.tr()[(i - 1) / keep];
                            const double aqt = fabs(st.qt);
                            r0 = e0 * fmax(Da, fmax(Dat, st.dst * Dbt));
                            r1 = e1 * fmax(fmax(Db, aqt * Dat), fmax(Dbt, st.dst * Dct));
                            r2 = e2 * fmax(Dc, fmax(Dct, st.dst * Dut));
                        }
                        f0 = 1.0 / sqrt(limit_scaling(r0));
                        f1 = 1.0 / sqrt(limit_scaling(r1));
                        f2 = 1.0 / sqrt(limit_scaling(r2));
                        fK = 1.0 / sqrt(limit_scaling(eKB * fmax(Dc, Dk)));
                        fSB = 1.0 / sqrt(limit_scaling(eSB * Dsv));
                        fSK = 1.0 / sqrt(limit_scaling(eSK * Dk));
                        fH1 = 1.0 / sqrt(limit_scaling(eH1 * fmax(Da, aH1 * Db)));
                        fH3 = 1.0 / sqrt(limit_scaling(eH3 * fmax(Da, aH3 * Db)));
                        fH4 = 1.0 / sqrt(limit_scaling(eH4 * fmax(Da, aH4 * Db)));
                        fS4 = 1.0 / sqrt(limit_scaling(eS4 * fmax(Da, fmax(aS4 * Db, Dsv))));
                        if (st.last) {
                            fEY = 1.0 / sqrt(limit_scaling(eEY * Da));
                            fEH = 1.0 / sqrt(limit_scaling(eEH * Db));
                        }
                    }
                    if (ub.live) {
                        double Au = eUB;
                        for (int t = ub.t0; t <= ub.t1; ++t) Au = fmax(Au, s.ex(5)[t + 1] * s.dsS()[t]);
                        fDu = 1.0 / sqrt(limit_scaling(fmax(cost_c * (keep * pm.w_cr) * Du * Du, Au * Du)));
                        fDp = 1.0 / sqrt(limit_scaling(fmax(cost_c * wp_ * Dp * Dp, fmax(eSKP, eUB) * Dp)));
                        fKP = 1.0 / sqrt(limit_scaling(eUB * fmax(Du, Dp)));
                        fSKP = 1.0 / sqrt(limit_scaling(eSKP * Dp));
                    }
                    Da *= fDa; Db *= fDb; Dc *= fDc; Dsv *= fDs; Du *= fDu; Dk *= fDk; Dp *= fDp;
                    e0 *= f0; e1 *= f1; e2 *= f2; eKB *= fK; eSB *= fSB; eSK *= fSK; eH1 *= fH1; eH3 *= fH3; eH4 *= fH4; eS4 *= fS4;
                    eUB *= fKP; eSKP *= fSKP; eEY *= fEY; eEH *= fEH;
                    double part = 0.0;   // (the N - ch unused slack variables of the reference have zero cost and no row: D = 1, nothing here)
                    if (st.live)
                        part += cost_c * pm.w_pq * Da * Da + cost_c * pm.w_c * Dc * Dc + cost_c * pm.w_s * Dsv * Dsv +
                                cost_c * wk_ * Dk * Dk;
                    if (ub.live) part += cost_c * (keep * pm.w_cr) * Du * Du + cost_c * wp_ * Dp * Dp;
                    const double mean = c.sum(part) / (double)(6 * N + ch);   // (contains CTA barriers)
                    double ct = fmax(mean, 1.0);
                    ct = limit_scaling(ct);
                    cost_c = cost_c * (1.0 / ct);
                }
            } else
            for (int sweep = 0; sweep < pm.scaling; ++sweep) {
                // publish what neighbours need: D of this station, E of its dynamics rows, Du
                if (st.live) {
                    s.ex(0)[i] = Da; s.ex(1)[i] = Db; s.ex(2)[i] = Dc;
                    s.ex(3)[i] = e0; s.ex(4)[i] = e1; s.ex(5)[i] = e2;
                }
                if (ub.live) s.tr()[tid] = Du;       // Du per control (tr is free during scaling; ch <= kT <= nv)
                c.sync();
                double fDa = 1, fDb = 1, fDc = 1, fDs = 1, fDu = 1;
                double f0 = 1, f1 = 1, f2 = 1, fKB = 1, fSB = 1, fH1 = 1, fH3 = 1, fS4 = 1, fS2 = 1, fUB = 1, fEY = 1, fEH = 1;
                if (st.live) {
                    double Aa = fmax(fmax(e0, eH1), fmax(eH3, fmax(eS4, eS2)));
                    double Ab = fmax(fmax(e1, eH1 * ad1), fmax(eH3 * ad3, fmax(eS4 * ad4, eS2 * ad2)));
                    double Ac = fmax(e2, eKB);
                    if (!st.last) {
                        const double e0n = s.ex(3)[i + 1], e1n = s.ex(4)[i + 1], e2n = s.ex(5)[i + 1];
                        const double aq = fabs(st.q10);
                        Aa = fmax(Aa, fmax(e0n, e1n * aq));
                        Ab = fmax(Ab, fmax(e0n * st.ds, e1n));
                        Ac = fmax(Ac, fmax(e1n * st.ds, e2n));
                    } else {
                        Aa = fmax(Aa, eEY);
                        Ab = fmax(Ab, eEH);
                    }
                    const double As = fmax(eSB, fmax(eS4, eS2));
                    fDa = 1.0 / sqrt(limit_scaling(fmax(cost_c * pm.w_pq * Da * Da, Aa * Da)));
                    fDb = 1.0 / sqrt(limit_scaling(Ab * Db));
                    fDc = 1.0 / sqrt(limit_scaling(fmax(cost_c * pm.w_c * Dc * Dc, Ac * Dc)));
                    fDs = 1.0 / sqrt(limit_scaling(fmax(cost_c * pm.w_s * Dsv * Dsv, As * Dsv)));
                    double r0, r1, r2;
                    if (st.first) {
                        r0 = e0 * Da; r1 = e1 * Db; r2 = e2 * Dc;
                    } else {
                        const double Dat = s.ex(0)[i - 1], Dbt = s.ex(1)[i - 1], Dct = s.ex(2)[i - 1];
                        const double Dut = s.tr()[(i - 1) / keep];
                        const double aqt = fabs(st.qt);
                        r0 = e0 * fmax(Da, fmax(Dat, st.dst * Dbt));
                        r1 = e1 * fmax(fmax(Db, aqt * Dat), fmax(Dbt, st.dst * Dct));
                        r2 = e2 * fmax(Dc, fmax(Dct, st.dst * Dut));
                    }
                    f0 = 1.0 / sqrt(limit_scaling(r0));
                    f1 = 1.0 / sqrt(limit_scaling(r1));
                    f2 = 1.0 / sqrt(limit_scaling(r2));
                    fKB = 1.0 / sqrt(limit_scaling(eKB * Dc));
                    fSB = 1.0 / sqrt(limit_scaling(eSB * Dsv));
                    fH1 = 1.0 / sqrt(limit_scaling(eH1 * fmax(Da, ad1 * Db)));
                    fH3 = 1.0 / sqrt(limit_scaling(eH3 * fmax(Da, ad3 * Db)));
                    fS4 = 1.0 / sqrt(limit_scaling(eS4 * fmax(Da, fmax(ad4 * Db, Dsv))));
                    fS2 = 1.0 / sqrt(limit_scaling(eS2 * fmax(Da, fmax(ad2 * Db, Dsv))));
                    if (st.last) {
                        fEY = 1.0 / sqrt(limit_scaling(eEY * Da));
                        fEH = 1.0 / sqrt(limit_scaling(eEH * Db));
                    }
                }
                if (ub.live) {
                    double Au = eUB;
                    for (int t = ub.t0; t <= ub.t1; ++t) Au = fmax(Au, s.ex(5)[t + 1] * s.dsS()[t]);
                    fDu = 1.0 / sqrt(limit_scaling(fmax(cost_c * (keep * pm.w_cr) * Du * Du, Au * Du)));
                    fUB = 1.0 / sqrt(limit_scaling(eUB * Du));
                }
                const double fDt = 1.0 / sqrt(limit_scaling(cost_c * pm.w_s * Dt * Dt));
                Da *= fDa; Db *= fDb; Dc *= fDc; Dsv *= fDs; Du *= fDu; Dt *= fDt;
                e0 *= f0; e1 *= f1; e2 *= f2; eKB *= fKB; eSB *= fSB; eH1 *= fH1; eH3 *= fH3; eS4 *= fS4; eS2 *= fS2;
                eUB *= fUB; eEY *= fEY; eEH *= fEH;
                double part = 0.0;
                if (st.live)
                    part += cost_c * pm.w_pq * Da * Da + cost_c * pm.w_c * Dc * Dc + cost_c * pm.w_s * Dsv * Dsv +
                            cost_c * pm.w_s * Dt * Dt;
                if (ub.live) part += cost_c * (keep * pm.w_cr) * Du * Du;
                const double mean = c.sum(part) / (double)(5 * N + ch);   // (contains CTA barriers)
                double ct = fmax(mean, 1.0);
                ct = limit_scaling(ct);
                cost_c = cost_c * (1.0 / ct);
            }
            // publish E, D to the workspace (read back at residual checks / refactorisations)
            if (st.live) {
                double *w9 = ws + (size_t)kWE * i;
                w9[0] = e0; w9[1] = e1; w9[2] = e2; w9[3] = eKB; w9[4] = eSB; w9[5] = eH1; w9[6] = eH3; w9[7] = eS4;
                w9[8] = kKPC ? eH4 : eS2;
                double *wD = ws + oD + (size_t)kWD * i;
                wD[0] = Da; wD[1] = Db; wD[2] = Dc; wD[3] = Dsv;
                if constexpr (kKPC) { w9[9] = eSK; wD[4] = Dk; st.sgk = pm.sigma / (Dk * Dk); }
                st.sga = pm.sigma / (Da * Da); st.sgb = pm.sigma / (Db * Db);
                st.sgc = pm.sigma / (Dc * Dc); st.sgs = pm.sigma / (Dsv * Dsv);
                if (st.last) { ws[oEnd] = eEY; ws[oEnd + 1] = eEH; }
            }
            if (ub.live) {
                ws[oEU + tid] = eUB;
                ws[oDu + tid] = Du;
                PQP_UBSG = pm.sigma / (Du * Du);
                if constexpr (kKPC) {
                    ws[oEU + ch + tid] = eSKP;
                    ws[oDu + ch + tid] = Dp;
                    PQP_UBF(8) = pm.sigma / (Dp * Dp);
                    PQP_UBF(10) = bv.max_kp[off + tid];   // :173-182 (entry j of the path's list for control j)
                }
            }
            // (the shared-memory state of the end rows and the held controls is set up only now: in the long-path classes it
            // sits in the tails of exchange rows the Ruiz sweeps have just used)
            if (tid == 0) { er[0] = 0.0; er[1] = 0.0; er[2] = 0.0; er[3] = 0.0; er[4] = lEH0; er[5] = uEH0; }
            if (ub.live) {
                PQP_UBX = 0.0; PQP_UBV = 0.0; PQP_UBW = 0.0;
                if constexpr (kKPC) { PQP_UBF(4) = 0.0; PQP_UBF(5) = 0.0; PQP_UBF(6) = 0.0; PQP_UBF(7) = 0.0; PQP_UBF(9) = 0.0; }
            }
            // cold start: OSQP's first iteration from zero leaves x = 0, v = 0 (see pqp_kp_core.cuh)
            st.vD0 = st.vD1 = st.vD2 = st.vKB = st.vSB = st.vH1 = st.vH3 = 0.0;
            st.vS4m = st.vS4p = st.vS2m = st.vS2p = 0.0;
            for (int g = tid; g < d.nv; g += kT) { s.tr()[g] = 0.0; s.yv()[g] = 0.0; }
            double rho = fmin(fmax(pm.rho, kRhoMin), kRhoMax);
            c.sync();

            // ================= (re)factorisation =====================================================
#ifdef PQP_PHASE_TIMING
#define PQP_RT(k) if (tid == 0) { const long long now_ = clock64(); rt_acc[k] += now_ - rt_t; rt_t = now_; }
#else
#define PQP_RT(k)
#endif
            auto refactor = [&]() -> int {
#ifdef PQP_PHASE_TIMING
                if (tid == 0) rt_t = clock64();
#endif
                // ---- row weights W = rho_row E^2 from the workspace E
                if (st.live) {
                    const double *w9 = ws + (size_t)kWE * i;
                    st.WD0 = kp_w_eq(w9[0], rho); st.WD1 = kp_w_eq(w9[1], rho); st.WD2 = kp_w_eq(w9[2], rho);
                    st.WSB = kp_w_box(w9[4], 0.0, pm.margin, rho);
                    st.WH1 = kp_w_box(w9[5], st.lH1, st.uH1, rho);
                    st.WH3 = kp_w_box(w9[6], st.lH3, st.uH3, rho);
                    st.WS4 = kp_w_box(w9[7], -kOsqpInfty, st.uS4m, rho);
                    if constexpr (kKPC) {
                        st.WK = kp_w_box(w9[3], -st.mk, kOsqpInfty, rho);      // both rows of the pair fall in the same rho class
                        st.WH4 = kp_w_box(w9[8], st.lH4, st.uH4, rho);
                        st.WSK = kp_w_box(w9[9], 0.0, st.uSK, rho);
                    } else {
                        st.WKB = kp_w_box(w9[3], -pm.kmax, pm.kmax, rho);
                        st.WS2 = kp_w_box(w9[8], -kOsqpInfty, st.uS2m, rho);
                    }
                    if (st.last) {
                        WEY = kp_w_box(ws[oEnd], lEY, uEY, rho);
                        WEH = kp_w_box(ws[oEnd + 1], lEH, uEH, rho);
                    }
                    if constexpr (kKPC) {
                        st.ksinv = 1.0 / (cost_c * pm.w_s + st.sgs + st.WSB + 2.0 * st.WS4);
                        st.kkinv = 1.0 / (cost_c * 500.0 + st.sgk + st.WSK + 2.0 * st.WK);
                    } else {
                        st.ksinv = 1.0 / (cost_c * pm.w_s + st.sgs + st.WSB + 2.0 * st.WS4 + 2.0 * st.WS2);
                    }
                    s.ex(0)[i] = st.WD0; s.ex(1)[i] = st.WD1; s.ex(2)[i] = st.WD2;   // neighbours need these
                }
                if (ub.live) {
                    if constexpr (kKPC) {
                        const double mkp = PQP_UBF(10);
                        PQP_UBW = kp_w_box(ws[oEU + tid], -mkp, kOsqpInfty, rho);
                        PQP_UBF(6) = kp_w_box(ws[oEU + ch + tid], 0.0, kOsqpInfty, rho);
                        PQP_UBF(9) = 1.0 / (cost_c * (25000.0 * keep) + PQP_UBF(8) + PQP_UBF(6) + 2.0 * PQP_UBW);
                    } else {
                        PQP_UBW = kp_w_box(ws[oEU + tid], -kOsqpInfty, kOsqpInfty, rho);
                    }
                }
                // zero the factor storage (identity on padded rows)
                for (int k = tid; k < IMAX * (BW + 1) * M; k += kT) {
                    const int p = k % M, kd = k / M, dd = kd % (BW + 1), kk = kd / (BW + 1);
                    int cp = 0;
                    {   // interior size of chunk p
                        const int g0 = kp_gx(ka, p * L);
                        const int g1 = (p + 1 < M) ? kp_gx(ka, (p + 1) * L) : ka.nred;
                        cp = g1 - g0 - 3;
                    }
                    s.fac()[k] = (dd == 0 && kk >= cp) ? 1.0 : 0.0;
                }
                c.sync();
                PQP_RT(0)
                // ---- assembly: every station / control thread writes its own band rows
                double N0 = 0, N1 = 0, N2 = 0;
                if (st.live && !st.last) { N0 = s.ex(0)[i + 1]; N1 = s.ex(1)[i + 1]; N2 = s.ex(2)[i + 1]; }
                const double d1 = pm.d1, d2 = pm.d2, d3 = pm.d3, d4 = pm.d4;
                double da = 0, db = 0, dc = 0, kba = 0, kca = 0, kcb = 0;
                if (st.live) {
                    if constexpr (kKPC) {
                        da = cost_c * pm.w_pq + st.sga + st.WD0 + N0 + N1 * st.q10 * st.q10 + st.WH1 + st.WH3 + st.WH4 + 2.0 * st.WS4;
                        db = st.sgb + st.WD1 + N0 * st.ds * st.ds + N1 + st.WH1 * cH1 * cH1 + st.WH3 * cH3 * cH3 +
                             st.WH4 * cH4 * cH4 + 2.0 * st.WS4 * cS4 * cS4;
                        dc = cost_c * pm.w_c + st.sgc + st.WD2 + N1 * st.ds * st.ds + N2 + 2.0 * st.WK;
                        kba = N0 * st.ds + N1 * st.q10 + st.WH1 * cH1 + st.WH3 * cH3 + st.WH4 * cH4 + 2.0 * st.WS4 * cS4;
                    } else {
                    da = cost_c * pm.w_pq + st.sga + st.WD0 + N0 + N1 * st.q10 * st.q10 + st.WH1 + st.WH3 + 2.0 * st.WS4 + 2.0 * st.WS2;
                    db = st.sgb + st.WD1 + N0 * st.ds * st.ds + N1 + st.WH1 * d1 * d1 + st.WH3 * d3 * d3 +
                         2.0 * st.WS4 * d4 * d4 + 2.0 * st.WS2 * d2 * d2;
                    dc = cost_c * pm.w_c + st.sgc + st.WD2 + N1 * st.ds * st.ds + N2 + st.WKB;
                    kba = N0 * st.ds + N1 * st.q10 + st.WH1 * d1 + st.WH3 * d3 + 2.0 * st.WS4 * d4 + 2.0 * st.WS2 * d2;
                    }
                    if (st.last) { da += WEY; db += WEH; }
                    kca = N1 * st.q10 * st.ds;
                    kcb = N1 * st.ds;
                    if (!st.sep) {
                        const int p = i / L;
                        double *fcol = s.fac() + p;
                        const int k0 = st.pos - (p * d.CS + 3);
                        PQP_F(k0, 0) = da; PQP_F(k0 + 1, 0) = db; PQP_F(k0 + 2, 0) = dc;
                        PQP_F(k0 + 1, 1) = kba; PQP_F(k0 + 2, 2) = kca; PQP_F(k0 + 2, 1) = kcb;
                        if ((i - 1) % L != 0) {   // previous station is interior as well
                            const int o = st.pos - st.posp;
                            PQP_F(k0, o) = -st.WD0;
                            PQP_F(k0, o - 1) = -st.WD0 * st.dst;
                            PQP_F(k0 + 1, o + 1) = -st.WD1 * st.qt;
                            PQP_F(k0 + 1, o) = -st.WD1;
                            PQP_F(k0 + 1, o - 1) = -st.WD1 * st.dst;
                            PQP_F(k0 + 2, o) = -st.WD2;
                        }
                    }
                }
                if (ub.live) {
                    const int p = ub.pos / d.CS;
                    double *fcol = s.fac() + p;
                    const int ku = ub.pos - (p * d.CS + 3);
                    double du = cost_c * (keep * pm.w_cr) + PQP_UBSG + (kKPC ? 2.0 : 1.0) * PQP_UBW;
                    int ii1 = tid * keep + keep;
                    if (ii1 > N - 1) ii1 = N - 1;
                    for (int ii = tid * keep; ii <= ii1; ++ii) {
                        double val = 0.0;
                        if (ii >= 1 && (ii - 1) / keep == tid) {
                            const double wv = s.ex(2)[ii], dst = s.dsS()[ii - 1];
                            val -= wv * dst;
                            du += wv * dst * dst;
                        }
                        if (ii <= N - 2 && ii / keep == tid) val += s.ex(2)[ii + 1] * s.dsS()[ii];
                        if (ii % L == 0) continue;   // c of a separator station: handled through the spikes
                        const int pi = ii / L;
                        const int kc = pi * d.CS + (kp_gx(ka, ii) - kp_gx(ka, pi * L)) + 2 - (p * d.CS + 3);
                        if (kc < ku) PQP_F(ku, ku - kc) = val;
                        else PQP_F(kc, kc - ku) = val;
                    }
                    PQP_F(ku, 0) = du;
                }
                c.sync();
                PQP_RT(1)
                // ---- interior LDL' (warp 0, lane p) and coupling coefficients per chunk:
                //      cpl[p] = left  (transition e -> e+1):  N0 N1 N2 ds q
                //               right (transition e2-1 -> e2): W0 W1 W2 ds q ; + flags
                int ok = 1;
                if (solver) ok = K2::local_factor(s.fac() + sid, Mst);
                if (st.live && i >= 1) {
                    if ((i - 1) % L == 0) {          // first interior station of chunk p: owns the LEFT coupling
                        double *cp = s.cpl() + 12 * ((i - 1) / L);
                        cp[0] = st.WD0; cp[1] = st.WD1; cp[2] = st.WD2; cp[3] = st.dst; cp[4] = st.qt;
                    }
                    if (st.sep) {                   // separator p: owns the RIGHT coupling of chunk p-1
                        double *cp = s.cpl() + 12 * (i / L - 1);
                        cp[5] = st.WD0; cp[6] = st.WD1; cp[7] = st.WD2; cp[8] = st.dst; cp[9] = st.qt;
                    }
                }
                c.sync();
                PQP_RT(2)
                // ---- spikes: thread (p, col) solves K_I t = K[I, s_col]  (col 0..2 left, 3..5 right separator)
                const int sp_p = tid / 6, sp_c = tid % 6;
                bool sp_act = tid < 6 * M;
                int ka1 = 0, kul = 0, kat = 0, kur = 0;
                bool has_int = false, has_right = false;
                double lN0 = 0, lN1 = 0, lN2 = 0, lds = 0, lq = 0, rW0 = 0, rW1 = 0, rW2 = 0, rds = 0, rq = 0;
                double *tcol = s.T() + sp_c * s.nv + sp_p * d.CS + 3;   // spike column: element k at tcol[k]
                if (sp_act) {
                    const int e = sp_p * L, e2 = e + L;
                    const int g0 = kp_gx(ka, e);
                    const int g1 = (sp_p + 1 < M) ? kp_gx(ka, e2) : ka.nred;
                    const int cn = g1 - g0 - 3;
                    has_int = cn > 0 && e < N - 1;
                    has_right = sp_p + 1 < M;
                    const double *cp = s.cpl() + 12 * sp_p;
                    const int lo_p = sp_p * d.CS + 3;
                    if (has_int) {
                        lN0 = cp[0]; lN1 = cp[1]; lN2 = cp[2]; lds = cp[3]; lq = cp[4];
                        ka1 = (kp_gx(ka, e + 1) - g0) - 3;
                        int home = (e / keep) * keep + d.h;
                        if (home > N - 1) home = N - 1;
                        kul = (home / L) * d.CS + (kp_gu(ka, e / keep) - kp_gx(ka, (home / L) * L)) - lo_p;
                    }
                    if (has_right) {
                        rW0 = cp[5]; rW1 = cp[6]; rW2 = cp[7]; rds = cp[8]; rq = cp[9];
                        kat = (kp_gx(ka, e2 - 1) - g0) - 3;
                        const int j = (e2 - 1) / keep;
                        int home = j * keep + d.h;
                        if (home > N - 1) home = N - 1;
                        kur = (home / L) * d.CS + (kp_gu(ka, j) - kp_gx(ka, (home / L) * L)) - lo_p;
                    }
#pragma unroll
                    for (int k = 0; k < IMAX; ++k) tcol[k] = 0.0;
                    const bool colok = (sp_c < 3) ? has_int : has_right;
                    if (colok) {
#define PQP_TC(k) tcol[(k)]
                        if (sp_c == 0) { PQP_TC(ka1) += -lN0; PQP_TC(ka1 + 1) += -lN1 * lq; }
                        else if (sp_c == 1) { PQP_TC(ka1) += -lN0 * lds; PQP_TC(ka1 + 1) += -lN1; }
                        else if (sp_c == 2) { PQP_TC(ka1 + 1) += -lN1 * lds; PQP_TC(ka1 + 2) += -lN2; PQP_TC(kul) += lN2 * lds; }
                        else if (sp_c == 3) { PQP_TC(kat) += -rW0; PQP_TC(kat + 1) += -rW0 * rds; }
                        else if (sp_c == 4) { PQP_TC(kat) += -rW1 * rq; PQP_TC(kat + 1) += -rW1; PQP_TC(kat + 2) += -rW1 * rds; }
                        else { PQP_TC(kat + 2) += -rW2; PQP_TC(kur) += -rW2 * rds; }
#undef PQP_TC
                        K2::local_solve_mem(tcol, s.fac() + sp_p, Mst);   // in place in shared memory
                    }
                }
                c.sync();
                PQP_RT(3)
                // ---- Schur blocks: A_p = K[S_p,I] T_left, Off_p = -(K[S_q,I] T_left)', C_p = K[S_q,I] T_right
                if (sp_act) {
                    double tl0 = 0, tl1 = 0, tl2 = 0, tr0 = 0, tr1 = 0, tr2 = 0;
                    const bool colok = (sp_c < 3) ? has_int : has_right;
                    if (colok) {
#define PQP_TC(k) tcol[(k)]
                        if (has_int) {
                            const double wa = PQP_TC(ka1), wb = PQP_TC(ka1 + 1), wc = PQP_TC(ka1 + 2), wu = PQP_TC(kul);
                            tl0 = -lN0 * wa - lN1 * lq * wb;
                            tl1 = -lN0 * lds * wa - lN1 * wb;
                            tl2 = -lN1 * lds * wb - lN2 * wc + lN2 * lds * wu;
                        }
                        if (has_right) {
                            const double wa = PQP_TC(kat), wb = PQP_TC(kat + 1), wc = PQP_TC(kat + 2), wu = PQP_TC(kur);
                            tr0 = -rW0 * wa - rW0 * rds * wb;
                            tr1 = -rW1 * rq * wa - rW1 * wb - rW1 * rds * wc;
                            tr2 = -rW2 * wc - rW2 * rds * wu;
                        }
#undef PQP_TC
                    }
                    double *B = s.blk() + 27 * sp_p;   // A[9] | C[9] | Off[9]
                    if (sp_c < 3) {
                        B[0 * 3 + sp_c] = tl0; B[1 * 3 + sp_c] = tl1; B[2 * 3 + sp_c] = tl2;                 // A[r][col]
                        B[18 + sp_c * 3 + 0] = -tr0; B[18 + sp_c * 3 + 1] = -tr1; B[18 + sp_c * 3 + 2] = -tr2;  // Off[col][r]
                    } else {
                        const int cc = sp_c - 3;
                        B[9 + 0 * 3 + cc] = tr0; B[9 + 1 * 3 + cc] = tr1; B[9 + 2 * 3 + cc] = tr2;          // C[r][col]
                    }
                }
                c.sync();
                // ---- Dg_p = K[S_p,S_p] - A_p - C_{p-1}  (separator station threads), Off_p -> red
                if (st.sep) {
                    const int p = i / L;
                    const double *B = s.blk() + 27 * p;
                    double *R = s.red() + kRed2 * p;
                    double Dg[9];
#pragma unroll
                    for (int k = 0; k < 9; ++k) {
                        Dg[k] = -B[k];
                        if (p > 0) Dg[k] -= B[k - 27 + 9];
                    }
                    Dg[0] += da; Dg[4] += db; Dg[8] += dc;
                    Dg[1] += kba; Dg[3] += kba; Dg[2] += kca; Dg[6] += kca; Dg[5] += kcb; Dg[7] += kcb;
#pragma unroll
                    for (int k = 0; k < 9; ++k) { R[k] = Dg[k]; R[9 + k] = B[18 + k]; }
                    if constexpr (kTwoLevel) {
#pragma unroll
                        for (int k = 0; k < 9; ++k) s.lv()[36 * p + 27 + k] = B[18 + k];   // Off_p = S[p, p+1]
                    }
                }
                c.sync();
                if constexpr (kTwoLevel) {
                    // ---- level 1: odd separators are eliminated.  E_p = Dg_p^-1 (p odd); for even p
                    //      PL_p = Off_{p-1}' E_{p-1},  PR_p = Off_p E_{p+1},
                    //      Dg'_p = Dg_p - PL_p Off_{p-1} - PR_p Off_p',   Off'_p = -PR_p Off_{p+1}   (couples p and p+2)
                    if (tid < M && (tid & 1)) {
                        const double *R = s.red() + kRed2 * tid;
                        double Dg[9], E[9];
#pragma unroll
                        for (int k = 0; k < 9; ++k) Dg[k] = R[k];
                        if (!(Dg[0] > 0.0)) ok = 0;
                        inv3_spd(Dg, E);
#pragma unroll
                        for (int k = 0; k < 9; ++k) s.lv()[36 * tid + k] = E[k];
                    }
                    c.sync();
                    if (tid < M && !(tid & 1)) {
                        const int pe = tid;
                        const double *R = s.red() + kRed2 * pe;
                        double *R2 = s.red2() + kRed2 * (pe >> 1);
                        double *lvp = s.lv() + 36 * pe;
                        double Dg[9], PL[9], PR[9], On[9];
#pragma unroll
                        for (int k = 0; k < 9; ++k) { Dg[k] = R[k]; PL[k] = 0.0; PR[k] = 0.0; On[k] = 0.0; }
                        if (pe > 0) {
                            const double *Om = s.lv() + 36 * (pe - 1) + 27, *Em = s.lv() + 36 * (pe - 1);
                            for (int r = 0; r < 3; ++r)
                                for (int cc = 0; cc < 3; ++cc) {
                                    double a = 0.0;
                                    for (int k = 0; k < 3; ++k) a += Om[k * 3 + r] * Em[k * 3 + cc];
                                    PL[r * 3 + cc] = a;
                                }
                            for (int r = 0; r < 3; ++r)
                                for (int cc = 0; cc < 3; ++cc) {
                                    double a = 0.0;
                                    for (int k = 0; k < 3; ++k) a += PL[r * 3 + k] * Om[k * 3 + cc];
                                    Dg[r * 3 + cc] -= a;
                                }
                        }
                        if (pe + 1 < M) {
                            const double *Op = s.lv() + 36 * pe + 27, *Ep = s.lv() + 36 * (pe + 1);
                            for (int r = 0; r < 3; ++r)
                                for (int cc = 0; cc < 3; ++cc) {
                                    double a = 0.0;
                                    for (int k = 0; k < 3; ++k) a += Op[r * 3 + k] * Ep[k * 3 + cc];
                                    PR[r * 3 + cc] = a;
                                }
                            for (int r = 0; r < 3; ++r)
                                for (int cc = 0; cc < 3; ++cc) {
                                    double a = 0.0;
                                    for (int k = 0; k < 3; ++k) a += PR[r * 3 + k] * Op[cc * 3 + k];
                                    Dg[r * 3 + cc] -= a;
                                }
                            if (pe + 2 < M) {
                                const double *Oq = s.lv() + 36 * (pe + 1) + 27;
                                for (int r = 0; r < 3; ++r)
                                    for (int cc = 0; cc < 3; ++cc) {
                                        double a = 0.0;
                                        for (int k = 0; k < 3; ++k) a += PR[r * 3 + k] * Oq[k * 3 + cc];
                                        On[r * 3 + cc] = -a;
                                    }
                            }
                        }
#pragma unroll
                        for (int k = 0; k < 9; ++k) { R2[k] = Dg[k]; R2[9 + k] = On[k]; lvp[9 + k] = PL[k]; lvp[18 + k] = PR[k]; }
                    }
                    c.sync();
                }
                double *const redp = kTwoLevel ? s.red2() : s.red();
                const int Mx = kTwoLevel ? (M + 1) / 2 : M, nSx = 3 * Mx;
                PQP_RT(4)
                // ---- block LDL' of the separator system (one thread), as in pqp_kp_core2.cuh:
                //      red[p] = Sinv_p | H_p = Sinv_p Off_p | G_p = Off_{p-1}' Sinv_{p-1}
                if (tid == 0) {
                    double Sch[9], Sinv[9];
                    for (int k = 0; k < 9; ++k) Sch[k] = redp[k];
                    for (int p = 0; p < Mx; ++p) {
                        double *Rp = redp + kRed2 * p;
                        if (!(Sch[0] > 0.0)) ok = 0;
                        inv3_spd(Sch, Sinv);
                        if (p + 1 < Mx) {
                            double *Rn = Rp + kRed2;
                            double Off[9];
                            for (int k = 0; k < 9; ++k) Off[k] = Rp[9 + k];
                            for (int r = 0; r < 3; ++r)
                                for (int cc = 0; cc < 3; ++cc) {
                                    double a = 0.0, hh = 0.0;
                                    for (int k = 0; k < 3; ++k) {
                                        a += Off[k * 3 + r] * Sinv[k * 3 + cc];
                                        hh += Sinv[r * 3 + k] * Off[k * 3 + cc];
                                    }
                                    Rn[18 + r * 3 + cc] = a;
                                    Rp[9 + r * 3 + cc] = hh;
                                }
                            for (int r = 0; r < 3; ++r)
                                for (int cc = 0; cc < 3; ++cc) {
                                    double a = Rn[r * 3 + cc];
                                    for (int k = 0; k < 3; ++k) a -= Rn[18 + r * 3 + k] * Off[k * 3 + cc];
                                    Sch[r * 3 + cc] = a;
                                }
                        }
                        for (int k = 0; k < 9; ++k) Rp[k] = Sinv[k];
                    }
                }
                c.sync();
                PQP_RT(5)
                // ---- dense inverse of the separator system: thread t solves for unit vector e_t and
                //      stores column t (= row t, the matrix is symmetric) as Sinv[k*nS + t]
                if (tid < nSx) {
                    const int pt = tid / 3, rt = tid % 3;
                    double *col = s.Sinv() + tid;
                    // forward: g'_p = g_p - G_p g'_{p-1}; g is e_t  -> zero before block pt
                    double g0 = 0, g1 = 0, g2 = 0;
                    for (int p = 0; p < Mx; ++p) {
                        const double *Rp = redp + kRed2 * p;
                        double n0 = (p == pt && rt == 0) ? 1.0 : 0.0, n1 = (p == pt && rt == 1) ? 1.0 : 0.0,
                               n2 = (p == pt && rt == 2) ? 1.0 : 0.0;
                        if (p > pt) {
                            n0 -= Rp[18] * g0 + Rp[19] * g1 + Rp[20] * g2;
                            n1 -= Rp[21] * g0 + Rp[22] * g1 + Rp[23] * g2;
                            n2 -= Rp[24] * g0 + Rp[25] * g1 + Rp[26] * g2;
                        }
                        g0 = n0; g1 = n1; g2 = n2;
                        // g^ = Sinv_p g' parked in the output column
                        col[(3 * p) * nSx] = Rp[0] * g0 + Rp[1] * g1 + Rp[2] * g2;
                        col[(3 * p + 1) * nSx] = Rp[3] * g0 + Rp[4] * g1 + Rp[5] * g2;
                        col[(3 * p + 2) * nSx] = Rp[6] * g0 + Rp[7] * g1 + Rp[8] * g2;
                    }
                    double x0 = col[(3 * (Mx - 1)) * nSx], x1 = col[(3 * (Mx - 1) + 1) * nSx], x2 = col[(3 * (Mx - 1) + 2) * nSx];
                    for (int p = Mx - 2; p >= 0; --p) {
                        const double *Rp = redp + kRed2 * p;
                        const double y0 = col[(3 * p) * nSx] - (Rp[9] * x0 + Rp[10] * x1 + Rp[11] * x2);
                        const double y1 = col[(3 * p + 1) * nSx] - (Rp[12] * x0 + Rp[13] * x1 + Rp[14] * x2);
                        const double y2 = col[(3 * p + 2) * nSx] - (Rp[15] * x0 + Rp[16] * x1 + Rp[17] * x2);
                        col[(3 * p) * nSx] = y0; col[(3 * p + 1) * nSx] = y1; col[(3 * p + 2) * nSx] = y2;
                        x0 = y0; x1 = y1; x2 = y2;
                    }
                }
                PQP_RT(6)
                if constexpr (kDense) {
                    // ---- dense interior inverses, row-major over the band factor: row r = p * IMAX + j of the
                    //      region is column j of K_p^-1 (symmetric: = row j).  Rows whose slots lie BEHIND the band factor
                    //      (the refactorisation scratch there is dead by now) are solved in place in shared memory; the
                    //      first kStaged rows overlap the factor every thread is still reading: one per thread, solved
                    //      in registers and written once everybody is done.
                    dense_build(c, s.fac(), M, tid);
                }
                PQP_RT(7)
                if constexpr (kScratchOnVec) {
                    c.sync();   // every reader of the scratch is done: give the two vectors back, padded entries zero
                    for (int g = tid; g < d.nv; g += kT) { s.tr()[g] = 0.0; s.yv()[g] = 0.0; }
                }
                return !c.any(!ok);   // (contains CTA barriers)
            };

            // A bound of +-OSQP_INFTY on the open side of a slack-pair row (S4, KP also S2) makes that row free: OSQP gives
            // it RHO_MIN while its partner keeps the inequality rho.  Unequal weights couple the slack to (a, b), which this
            // solve relies on not happening: such a path is refused (PQP_INVALID_PROBLEM, 0 iterations; see pqp.h).
            bool split = false;
            if (st.live) {
                const double *w9 = ws + (size_t)kWE * i;
                split = kp_w_box(w9[7], -kOsqpInfty, st.uS4m, 1.0) != kp_w_box(w9[7], st.lS4p, kOsqpInfty, 1.0);
                if constexpr (!kKPC)
                    split = split || kp_w_box(w9[8], -kOsqpInfty, st.uS2m, 1.0) != kp_w_box(w9[8], st.lS2p, kOsqpInfty, 1.0);
            }
            if (c.any(split)) status = PQP_INVALID_PROBLEM;
#ifdef PQP_PHASE_TIMING
            ph_scale = clock64() - ph_scale_t0;
            {
                const long long t0_ = clock64();
                if (status == PQP_UNSOLVED) { ++ph_nref; if (!refactor()) status = PQP_NON_CVX; }
                ph_refactor += clock64() - t0_;
            }
#else
            if (status == PQP_UNSOLVED && !refactor()) status = PQP_NON_CVX;
#endif
            const double d1 = pm.d1, d2 = pm.d2, d3 = pm.d3, d4 = pm.d4;
            // An iteration that ends in a termination check needs delta_y = W (w_new - w_old) (OSQP
            // update_y / is_primal_infeasible): w = v - clamp(v) is parked in the workspace at the END
            // of the iteration before it, which keeps the hot part of the loop free of this code.
            auto is_check = [&](int k) { return (pm.check_termination && (k % pm.check_termination == 0)) || k == pm.max_iter; };
            // OSQP's first iteration from x = z = y = 0 ends at the cold start (x = 0, v = 0: z = clamp(0),
            // y = -rho clamp(0)).  When it is an event (check, adaptation or the last iteration), it runs as a step
            // with alpha = 0, which leaves that iterate as it is, followed by (d) on w_old = y_0 / rho = 0.
            const bool first_event = is_check(1) || (pm.adaptive_rho && pm.adaptive_rho_interval == 1);
            // (the plain form reads the constant: the inner loop sees no variable alpha)
            const double alpha_pm = pm.alpha;
            double alpha_ev = first_event ? 0.0 : alpha_pm;
            auto park_w = [&]() {
                if constexpr (kKPC) {
                    if (st.live) {
                        double *wo = wold + i;
                        wo[0] = st.vD0 - st.b0; wo[N] = st.vD1 - st.b1; wo[2 * N] = st.vD2 - st.b2;
                        wo[3 * N] = st.vKL - fmax(st.vKL, -st.mk);
                        wo[4 * N] = st.vKU - fmin(st.vKU, st.mk);
                        wo[5 * N] = st.vSB - clamp2(st.vSB, 0.0, pm.margin);
                        wo[6 * N] = st.vSK - clamp2(st.vSK, 0.0, st.uSK);
                        wo[7 * N] = st.vH1 - clamp2(st.vH1, st.lH1, st.uH1);
                        wo[8 * N] = st.vH3 - clamp2(st.vH3, st.lH3, st.uH3);
                        wo[9 * N] = st.vH4 - clamp2(st.vH4, st.lH4, st.uH4);
                        wo[10 * N] = st.vS4m - fmin(st.vS4m, st.uS4m);
                        wo[11 * N] = st.vS4p - fmax(st.vS4p, st.lS4p);
                        if (st.last) {
                            wold[kWR * N] = vEY - clamp2(vEY, lEY, uEY);
                            wold[kWR * N + 1] = vEH - clamp2(vEH, lEH, uEH);
                        }
                    }
                    if (ub.live) {
                        double *wc = wold + kWR * N + 2 + tid;
                        const double mkp = PQP_UBF(10);
                        wc[0] = PQP_UBV - fmax(PQP_UBV, -mkp);
                        wc[ch] = PQP_UBF(4) - fmin(PQP_UBF(4), mkp);
                        wc[2 * ch] = PQP_UBF(5) - fmax(PQP_UBF(5), 0.0);
                    }
                } else
                if (st.live) {
                    double *wo = wold + i;
                    wo[0] = st.vD0 - st.b0; wo[N] = st.vD1 - st.b1; wo[2 * N] = st.vD2 - st.b2;
                    wo[3 * N] = st.vKB - clamp2(st.vKB, -pm.kmax, pm.kmax);
                    wo[4 * N] = st.vSB - clamp2(st.vSB, 0.0, pm.margin);
                    wo[5 * N] = st.vH1 - clamp2(st.vH1, st.lH1, st.uH1);
                    wo[6 * N] = st.vH3 - clamp2(st.vH3, st.lH3, st.uH3);
                    wo[7 * N] = st.vS4m - fmin(st.vS4m, st.uS4m);
                    wo[8 * N] = st.vS4p - fmax(st.vS4p, st.lS4p);
                    wo[9 * N] = st.vS2m - fmin(st.vS2m, st.uS2m);
                    wo[10 * N] = st.vS2p - fmax(st.vS2p, st.lS2p);
                    if (st.last) {
                        wold[kWR * N] = vEY - clamp2(vEY, -1.0, 1.0);
                        wold[kWR * N + 1] = vEH - clamp2(vEH, lEH, uEH);
                    }
                }
            };
            // One ADMM iteration.  Instantiated twice: the plain form runs in the tight inner loop between
            // two "events" (termination check / rho adaptation / last iteration), the checked form runs
            // the event iteration itself -- the rarely executed residual, certificate and refactorisation
            // code then does not take part in the register allocation of the hot loop.
            // y = K_I^-1 r_I for the dense interiors: row tasks q = (p, k) in [q0, q1) strided over the warps that own
            // no separator row.  (Spreading them over the b1 phase as well, or splitting b1 over lane pairs, shortens the
            // per-CTA critical path but measured SLOWER: with two CTAs per SM the idle warps of one CTA are the issue
            // slots of the other, so what counts is the instruction total, not the balance inside one CTA.)
            auto dense_rows = [&](int qfirst, int q1, int stride) {
                if constexpr (kDense) {
                    int q = qfirst;
                    for (; q < q1; q += stride) {
                        const int p = q / IMAX, k = q - p * IMAX;
                        const double *kv = s.fac() + (size_t)q * kRow;
                        const double *rI = s.tr() + p * d.CS + 3;
                        double a0 = 0.0, a1 = 0.0;
#pragma unroll
                        for (int j = 0; j < IMAX; ++j) {
                            if (j & 1) a1 += kv[j] * rI[j];
                            else a0 += kv[j] * rI[j];
                        }
                        s.yv()[p * d.CS + 3 + k] = a0 + a1;
                    }
                }
            };
            const int yQ = IMAX * M;
            // Phase (b2) of the dense form.  The separator product x_S = Sinv g runs on the first nSr threads, the row tasks
            // of y = K_I^-1 r_I on the WARPS after them: a warp that held both kinds of thread would run the two pieces of
            // work one after the other and become the slowest of the phase.  (Handing the last, partly filled round of row
            // tasks to the product warps, or two row tasks per loop trip, were slower.)
            const int yT0 = (nSr + 31) & ~31, yNw = kT - yT0;
#ifdef PQP_PHASE_TIMING
            // clock64() at the phase boundaries, accumulated per warp-0 / warp-1 lead thread in shared scratch
            // (diagnostic builds only): slots 0..5 = a1, a2, b1, b2, b3, c ; 6 = iterations.  Not in the long-path
            // classes: they give exchange row 5 to the separator rhs.
            double *ph_acc = s.ex(5) + 8 * (wid & 1);   // (row 5 is free once the scaling is done)
            if (kPhTime && (tid & 31) == 0 && wid < 2) for (int k = 0; k < 8; ++k) ph_acc[k] = 0.0;
            long long ph_t = 0;
#define PQP_PH(k) if (kPhTime && (tid & 31) == 0 && wid < 2) { const long long now_ = clock64(); ph_acc[k] += (double)(now_ - ph_t); ph_t = now_; }
#define PQP_PH_START if (kPhTime && (tid & 31) == 0 && wid < 2) { ph_t = clock64(); ph_acc[6] += 1.0; }
#else
#define PQP_PH(k)
#define PQP_PH_START
#endif
            // CTA barrier of the iteration.  The 100-station class calls __syncthreads() directly: c.sync() also serves
            // one-warp CTAs and tests for them at run time, which puts a branch and a warp sync beside every barrier.
#define PQP_BAR() do { if constexpr (kLean) c.cs.sync(); else c.sync(); } while (0)
            auto step = [&](auto with_check) {
                const double alpha = decltype(with_check)::value ? alpha_ev : alpha_pm;
                PQP_PH_START
                // ---- (a) g = W (2 clamp(v) - v) per row; rhs = sigma x + A' g
                const double gD0 = st.WD0 * (2.0 * st.b0 - st.vD0);
                const double gD1 = st.WD1 * (2.0 * st.b1 - st.vD1);
                const double gD2 = st.WD2 * (2.0 * st.b2 - st.vD2);
                if (st.live) { s.ex(0)[i] = gD0; s.ex(1)[i] = gD1; s.ex(2)[i] = gD2; }
                PQP_BAR();
                PQP_PH(0)
                double tsl = 0.0;   // x-tilde of the slack (decouples exactly)
                double tskp = 0.0;  // KPC: x-tilde of the rate slack of this thread's held control
                // z = clamp(v) of the station-local rows is needed twice per iteration (here and in the update (c)):
                // computed once, carried across the solve phases
                double zKB = 0, zSB = 0, zH1 = 0, zH3 = 0, z4m = 0, z4p = 0, z2m = 0, z2p = 0;
                double zKU = 0, zSK = 0, zH4 = 0, tsk = 0.0;   // KPC (zKB then holds the kappa-pair's lower row, z2m / z2p are unused)
                if constexpr (kKPC) {
                  if (st.live) {
                    zKB = fmax(st.vKL, -st.mk);
                    zKU = fmin(st.vKU, st.mk);
                    zSB = clamp2(st.vSB, 0.0, pm.margin);
                    zSK = clamp2(st.vSK, 0.0, st.uSK);
                    zH1 = clamp2(st.vH1, st.lH1, st.uH1);
                    zH3 = clamp2(st.vH3, st.lH3, st.uH3);
                    zH4 = clamp2(st.vH4, st.lH4, st.uH4);
                    z4m = fmin(st.vS4m, st.uS4m);
                    z4p = fmax(st.vS4p, st.lS4p);
                    const double gKL = st.WK * (2.0 * zKB - st.vKL);
                    const double gKU = st.WK * (2.0 * zKU - st.vKU);
                    const double gSB = st.WSB * (2.0 * zSB - st.vSB);
                    const double gSK = st.WSK * (2.0 * zSK - st.vSK);
                    const double gH1 = st.WH1 * (2.0 * zH1 - st.vH1);
                    const double gH3 = st.WH3 * (2.0 * zH3 - st.vH3);
                    const double gH4 = st.WH4 * (2.0 * zH4 - st.vH4);
                    const double g4m = st.WS4 * (2.0 * z4m - st.vS4m);
                    const double g4p = st.WS4 * (2.0 * z4p - st.vS4p);
                    const double s4 = g4m + g4p;
                    double ra = -gD0 + gH1 + gH3 + gH4 + s4;
                    double rb = -gD1 + cH1 * gH1 + cH3 * gH3 + cH4 * gH4 + cS4 * s4;
                    double rc = -gD2 + gKL + gKU;
                    const double rs = gSB - g4m + g4p;
                    const double rk = gSK + gKL - gKU;
                    if (!st.last) {
                        const double n0 = s.ex(0)[i + 1], n1 = s.ex(1)[i + 1], n2 = s.ex(2)[i + 1];
                        ra += n0 + st.q10 * n1;
                        rb += st.ds * n0 + n1;
                        rc += st.ds * n1 + n2;
                    } else {
                        ra += WEY * (2.0 * clamp2(vEY, lEY, uEY) - vEY);
                        rb += WEH * (2.0 * clamp2(vEH, lEH, uEH) - vEH);
                    }
                    s.tr()[st.pos] = st.sga * st.xa + ra;
                    s.tr()[st.pos + 1] = st.sgb * st.xb + rb;
                    s.tr()[st.pos + 2] = st.sgc * st.xc + rc;
                    tsl = (st.sgs * st.xs + rs) * st.ksinv;
                    tsk = (st.sgk * st.xk + rk) * st.kkinv;
                  }
                  if (ub.live) {   // rate pair (u + p >= -mkp, u - p <= mkp), p >= 0: p decouples like the other slacks
                    const double mkp = PQP_UBF(10), vL = PQP_UBV, vU = PQP_UBF(4), vP = PQP_UBF(5);
                    const double gL = PQP_UBW * (2.0 * fmax(vL, -mkp) - vL);
                    const double gU = PQP_UBW * (2.0 * fmin(vU, mkp) - vU);
                    const double gP = PQP_UBF(6) * (2.0 * fmax(vP, 0.0) - vP);
                    double acc = PQP_UBSG * PQP_UBX + gL + gU;
                    for (int t = ub.t0; t <= ub.t1; ++t) acc += s.dsS()[t] * s.ex(2)[t + 1];
                    s.tr()[ub.pos] = acc;
                    tskp = (PQP_UBF(8) * PQP_UBF(7) + (gP + gL - gU)) * PQP_UBF(9);
                  }
                } else {
                if (st.live) {
                    zKB = clamp2(st.vKB, -pm.kmax, pm.kmax);
                    zSB = clamp2(st.vSB, 0.0, pm.margin);
                    zH1 = clamp2(st.vH1, st.lH1, st.uH1);
                    zH3 = clamp2(st.vH3, st.lH3, st.uH3);
                    z4m = fmin(st.vS4m, st.uS4m);
                    z4p = fmax(st.vS4p, st.lS4p);
                    z2m = fmin(st.vS2m, st.uS2m);
                    z2p = fmax(st.vS2p, st.lS2p);
                    const double gKB = st.WKB * (2.0 * zKB - st.vKB);
                    const double gSB = st.WSB * (2.0 * zSB - st.vSB);
                    const double gH1 = st.WH1 * (2.0 * zH1 - st.vH1);
                    const double gH3 = st.WH3 * (2.0 * zH3 - st.vH3);
                    const double g4m = st.WS4 * (2.0 * z4m - st.vS4m);
                    const double g4p = st.WS4 * (2.0 * z4p - st.vS4p);
                    const double g2m = st.WS2 * (2.0 * z2m - st.vS2m);
                    const double g2p = st.WS2 * (2.0 * z2p - st.vS2p);
                    const double s4 = g4m + g4p, s2 = g2m + g2p;
                    double ra = -gD0 + gH1 + gH3 + s4 + s2;
                    double rb = -gD1 + d1 * gH1 + d3 * gH3 + d4 * s4 + d2 * s2;
                    double rc = -gD2 + gKB;
                    const double rs = gSB - g4m + g4p - g2m + g2p;
                    if (!st.last) {
                        const double n0 = s.ex(0)[i + 1], n1 = s.ex(1)[i + 1], n2 = s.ex(2)[i + 1];
                        ra += n0 + st.q10 * n1;
                        rb += st.ds * n0 + n1;
                        rc += st.ds * n1 + n2;
                    } else {
                        ra += WEY * (2.0 * clamp2(vEY, -1.0, 1.0) - vEY);
                        rb += WEH * (2.0 * clamp2(vEH, lEH, uEH) - vEH);
                    }
                    s.tr()[st.pos] = st.sga * st.xa + ra;
                    s.tr()[st.pos + 1] = st.sgb * st.xb + rb;
                    s.tr()[st.pos + 2] = st.sgc * st.xc + rc;
                    tsl = (st.sgs * st.xs + rs) * st.ksinv;
                }
                if (ub.live) {
                    double acc = PQP_UBSG * PQP_UBX + PQP_UBW * (2.0 * clamp2(PQP_UBV, -kOsqpInfty, kOsqpInfty) - PQP_UBV);
                    if constexpr (kLean) {
#pragma unroll 1
                        for (int t = ub.t0; t <= ub.t1; ++t) acc += s.dsS()[t] * s.ex(2)[t + 1];
                    } else {
                        for (int t = ub.t0; t <= ub.t1; ++t) acc += s.dsS()[t] * s.ex(2)[t + 1];
                    }
                    s.tr()[ub.pos] = acc;
                }
                }
                PQP_BAR();
                PQP_PH(1)
                // ---- (b1) separator rhs g = r_S - T' r_I  (threads 0..3M-1; p fastest -> unit stride, conflict-free)
                if (tid < nS) {
                    const int r = kLean ? s.ixS()[kT + tid] : tid / M, p = tid - r * M;
                    const double *rI = s.tr() + p * d.CS + 3;
                    const double *Tl = s.T() + r * s.nv + p * d.CS + 3;
                    double a0 = rI[r - 3], a1 = 0.0, a2 = 0.0, a3 = 0.0;
#pragma unroll
                    for (int k = 0; k < IMAX; ++k) {
                        if (k & 1) a1 -= Tl[k] * rI[k];
                        else a0 -= Tl[k] * rI[k];
                    }
                    if (p > 0) {
                        const double *Tr = Tl + 3 * s.nv - d.CS;
                        const double *rJ = rI - d.CS;
#pragma unroll
                        for (int k = 0; k < IMAX; ++k) {
                            if (k & 1) a3 -= Tr[k] * rJ[k];
                            else a2 -= Tr[k] * rJ[k];
                        }
                    }
                    s.gS()[3 * p + r] = (a0 + a1) + (a2 + a3);
                }
                // 100-station class: only the separator product of (b2), on warps 0 and 1 (3M <= 51 threads), reads g_S,
                // so only those two warps wait for it (named barrier 1, 64 threads).  The row warps go straight on to
                // y = K_I^-1 r_I, which needs nothing but the rhs.  (The CPU emulator has no partial barrier: full one.)
#ifndef PQP_HOST_EMU
                if constexpr (kLean) {
                    static_assert(!kLean || 3 * MMAX <= 64, "the separator threads fit in warps 0 and 1");
                    if (wid < 2) asm volatile("bar.sync 1, 64;" ::: "memory");
                } else
#endif
                PQP_BAR();
                PQP_PH(2)
                if constexpr (kTwoLevel) {
                    // ---- (b1') reduced right-hand side of the even separators: g'_p = g_p - PL_p g_{p-1} - PR_p g_{p+1}
                    if (tid < nSr) {
                        const int pr = tid / 3, r = tid - 3 * pr, pe = 2 * pr;
                        const double *gS = s.gS();
                        const double *lvp = s.lv() + 36 * pe;
                        double a = gS[3 * pe + r];
                        if (pe > 0) a -= lvp[9 + 3 * r] * gS[3 * pe - 3] + lvp[10 + 3 * r] * gS[3 * pe - 2] + lvp[11 + 3 * r] * gS[3 * pe - 1];
                        if (pe + 1 < M) a -= lvp[18 + 3 * r] * gS[3 * pe + 3] + lvp[19 + 3 * r] * gS[3 * pe + 4] + lvp[20 + 3 * r] * gS[3 * pe + 5];
                        s.ex(4)[tid] = a;
                    }
                    PQP_BAR();
                }
                // ---- (b2) x_S = Sinv g on the first threads  ||  y = K_I^-1 r_I:
                //      dense interiors: row tasks (p, k) spread over all the OTHER threads of the CTA;
                //      otherwise M banded substitutions on the first M threads (and Sinv g on the warps after them).
                if constexpr (kDense) {
                    if (tid < nSr) {
                        const double *row = s.Sinv() + tid;
                        const double *gS = kTwoLevel ? s.ex(4) : s.gS();
                        double a0 = 0, a1 = 0, a2 = 0;
#pragma unroll 4
                        for (int k = 0; k < nSr; k += 3) {
                            a0 += row[k * nSr] * gS[k];
                            a1 += row[(k + 1) * nSr] * gS[k + 1];
                            a2 += row[(k + 2) * nSr] * gS[k + 2];
                        }
                        const int xo = kTwoLevel ? 6 * (tid / 3) + (tid % 3) : tid;   // even separator 2*(t/3) in full numbering
                        s.ex(3)[xo] = (a0 + a1) + a2;
                    }
                    if (tid >= yT0) dense_rows(tid - yT0, yQ, yNw);
                } else if (tid < kSolveT) {
                    if (solver) K2::local_solve2(s.tr() + lo, s.yv() + lo, s.fac() + sid, Mst);
                } else {
                    const int t = tid - kSolveT;
                    if (t < nSr) {
                        const double *row = s.Sinv() + t;
                        const double *gS = kTwoLevel ? s.ex(4) : s.gS();
                        double a0 = 0, a1 = 0, a2 = 0;
#pragma unroll 4
                        for (int k = 0; k < nSr; k += 3) {
                            a0 += row[k * nSr] * gS[k];
                            a1 += row[(k + 1) * nSr] * gS[k + 1];
                            a2 += row[(k + 2) * nSr] * gS[k + 2];
                        }
                        const int xo = kTwoLevel ? 6 * (t / 3) + (t % 3) : t;
                        s.ex(3)[xo] = (a0 + a1) + a2;
                    }
                }
                PQP_BAR();
                PQP_PH(3)
                if constexpr (kTwoLevel) {
                    // ---- (b2') odd separators: x_p = E_p (g_p - Off_{p-1}' x_{p-1} - Off_p x_{p+1})  (even entries are read,
                    //      odd ones written: no hazard inside the phase)
                    if (tid < 3 * (M / 2)) {
                        const int po = 2 * (tid / 3) + 1, r = tid % 3;
                        const double *gS = s.gS(), *xS = s.ex(3);
                        const double *Om = s.lv() + 36 * (po - 1) + 27, *E = s.lv() + 36 * po;
                        double t0 = gS[3 * po], t1 = gS[3 * po + 1], t2 = gS[3 * po + 2];
                        {
                            const double x0 = xS[3 * po - 3], x1 = xS[3 * po - 2], x2 = xS[3 * po - 1];
                            t0 -= Om[0] * x0 + Om[3] * x1 + Om[6] * x2;
                            t1 -= Om[1] * x0 + Om[4] * x1 + Om[7] * x2;
                            t2 -= Om[2] * x0 + Om[5] * x1 + Om[8] * x2;
                        }
                        if (po + 1 < M) {
                            const double *Op = s.lv() + 36 * po + 27;
                            const double x0 = xS[3 * po + 3], x1 = xS[3 * po + 4], x2 = xS[3 * po + 5];
                            t0 -= Op[0] * x0 + Op[1] * x1 + Op[2] * x2;
                            t1 -= Op[3] * x0 + Op[4] * x1 + Op[5] * x2;
                            t2 -= Op[6] * x0 + Op[7] * x1 + Op[8] * x2;
                        }
                        s.ex(3)[3 * po + r] = E[3 * r] * t0 + E[3 * r + 1] * t1 + E[3 * r + 2] * t2;
                    }
                    PQP_BAR();
                }
                // ---- (b3) x-tilde: separators take x_S, interiors y - T [x_Sp ; x_Sq]
                double ta = 0, tb = 0, tc = 0, tu = 0;
#define PQP_TX(q) ((s.yv()[q] - (Tq[q] * xl0 + Tq[nvs + (q)] * xl1 + Tq[2 * nvs + (q)] * xl2)) \
                   - (Tq[3 * nvs + (q)] * xr0 + Tq[4 * nvs + (q)] * xr1 + Tq[5 * nvs + (q)] * xr2))
                if (st.live) {
                    const int p = kLean ? s.ixS()[tid] : i / L;
                    if (st.sep) {
                        ta = s.ex(3)[3 * p]; tb = s.ex(3)[3 * p + 1]; tc = s.ex(3)[3 * p + 2];
                    } else {
                        const double *Tq = s.T();
                        const int nvs = s.nv;
                        const double xl0 = s.ex(3)[3 * p], xl1 = s.ex(3)[3 * p + 1], xl2 = s.ex(3)[3 * p + 2];
                        double xr0 = 0, xr1 = 0, xr2 = 0;
                        if (p + 1 < M) { xr0 = s.ex(3)[3 * p + 3]; xr1 = s.ex(3)[3 * p + 4]; xr2 = s.ex(3)[3 * p + 5]; }
                        ta = PQP_TX(st.pos); tb = PQP_TX(st.pos + 1); tc = PQP_TX(st.pos + 2);
                    }
                }
                if (ub.live) {
                    const int p = ub.pos / d.CS;
                    const double *Tq = s.T();
                    const int nvs = s.nv;
                    const double xl0 = s.ex(3)[3 * p], xl1 = s.ex(3)[3 * p + 1], xl2 = s.ex(3)[3 * p + 2];
                    double xr0 = 0, xr1 = 0, xr2 = 0;
                    if (p + 1 < M) { xr0 = s.ex(3)[3 * p + 3]; xr1 = s.ex(3)[3 * p + 4]; xr2 = s.ex(3)[3 * p + 5]; }
                    tu = PQP_TX(ub.pos);
                }
#undef PQP_TX
                // publish x-tilde in tr for the neighbours.  The rhs it overwrites is last read in (b2), before the barrier
                // that ends it, so the 100-station class publishes at once; the other classes keep their barrier here.
                if constexpr (!kLean) PQP_BAR();
                if (st.live) { s.tr()[st.pos] = ta; s.tr()[st.pos + 1] = tb; s.tr()[st.pos + 2] = tc; }
                if (ub.live) s.tr()[ub.pos] = tu;
                PQP_BAR();
                PQP_PH(4)
                // ---- (c) v += alpha (A xt - clamp(v)),  x = alpha xt + (1 - alpha) x
                if (st.live) {
                    double zD0 = -ta, zD1 = -tb, zD2 = -tc;
                    if (!st.first) {
                        const double at = s.tr()[st.posp], bt = s.tr()[st.posp + 1], ct = s.tr()[st.posp + 2];
                        const double ut = s.tr()[st.posup];
                        zD0 += at + st.dst * bt;
                        zD1 += st.qt * at + bt + st.dst * ct;
                        zD2 += ct + st.dst * ut;
                    }
                    st.vD0 += alpha * (zD0 - st.b0);
                    st.vD1 += alpha * (zD1 - st.b1);
                    st.vD2 += alpha * (zD2 - st.b2);
                    if constexpr (kKPC) {
                        const double e4 = ta + cS4 * tb;
                        st.vKL += alpha * ((tc + tsk) - zKB);
                        st.vKU += alpha * ((tc - tsk) - zKU);
                        st.vSB += alpha * (tsl - zSB);
                        st.vSK += alpha * (tsk - zSK);
                        st.vH1 += alpha * ((ta + cH1 * tb) - zH1);
                        st.vH3 += alpha * ((ta + cH3 * tb) - zH3);
                        st.vH4 += alpha * ((ta + cH4 * tb) - zH4);
                        st.vS4m += alpha * ((e4 - tsl) - z4m);
                        st.vS4p += alpha * ((e4 + tsl) - z4p);
                        if (st.last) {
                            vEY += alpha * (ta - clamp2(vEY, lEY, uEY));
                            vEH += alpha * (tb - clamp2(vEH, lEH, uEH));
                        }
                        st.xk = alpha * tsk + (1.0 - alpha) * st.xk;
                    } else {
                    const double e4 = ta + d4 * tb, e2 = ta + d2 * tb;
                    st.vKB += alpha * (tc - zKB);
                    st.vSB += alpha * (tsl - zSB);
                    st.vH1 += alpha * ((ta + d1 * tb) - zH1);
                    st.vH3 += alpha * ((ta + d3 * tb) - zH3);
                    st.vS4m += alpha * ((e4 - tsl) - z4m);
                    st.vS4p += alpha * ((e4 + tsl) - z4p);
                    st.vS2m += alpha * ((e2 - tsl) - z2m);
                    st.vS2p += alpha * ((e2 + tsl) - z2p);
                    if (st.last) {
                        vEY += alpha * (ta - clamp2(vEY, -1.0, 1.0));
                        vEH += alpha * (tb - clamp2(vEH, lEH, uEH));
                    }
                    }
                    st.xa = alpha * ta + (1.0 - alpha) * st.xa;
                    st.xb = alpha * tb + (1.0 - alpha) * st.xb;
                    st.xc = alpha * tc + (1.0 - alpha) * st.xc;
                    st.xs = alpha * tsl + (1.0 - alpha) * st.xs;
                }
                if (ub.live) {
                    if constexpr (kKPC) {
                        const double mkp = PQP_UBF(10), vL = PQP_UBV, vU = PQP_UBF(4), vP = PQP_UBF(5);
                        PQP_UBV = vL + alpha * ((tu + tskp) - fmax(vL, -mkp));
                        PQP_UBF(4) = vU + alpha * ((tu - tskp) - fmin(vU, mkp));
                        PQP_UBF(5) = vP + alpha * (tskp - fmax(vP, 0.0));
                        PQP_UBF(7) = alpha * tskp + (1.0 - alpha) * PQP_UBF(7);
                    } else {
                        PQP_UBV += alpha * (tu - clamp2(PQP_UBV, -kOsqpInfty, kOsqpInfty));
                    }
                    PQP_UBX = alpha * tu + (1.0 - alpha) * PQP_UBX;
                }
                PQP_PH(5)
                // ---- (d) residuals, termination, adaptive rho
                if constexpr (decltype(with_check)::value) {
#ifdef PQP_PHASE_TIMING
// lane 0 of every warp: 0 loads + x publish, 1 primal pass, 2 its barrier, 3 dual pass, 4 certificate, 5 reduction
#define PQP_CK(k) if (lane == 0) { const long long now_ = clock64(); ck_acc[k] += now_ - ck_t; ck_t = now_; }
                    if (lane == 0) ck_t = clock64();
#else
#define PQP_CK(k)
#endif
                    const bool can_check = pm.check_termination && (iter % pm.check_termination == 0);
                    const bool can_adapt = pm.adaptive_rho && pm.adaptive_rho_interval &&
                                           (iter % pm.adaptive_rho_interval == 0);
                    const bool chk = can_check || iter == pm.max_iter;
                    // the row / column scalings (and the parked dual direction) live in the global workspace: fetch them
                    // first, as independent loads, so that their L2 latency overlaps the barriers and the stencils below
                    const int iw = st.live ? i : 0;
                    double eW[kWE], dW[kWD], wo[kWR];
                    {
                        const double *w9g = ws + (size_t)kWE * iw;
                        const double *wDg = ws + oD + (size_t)kWD * iw;
#pragma unroll
                        for (int k = 0; k < kWE; ++k) eW[k] = w9g[k];
#pragma unroll
                        for (int k = 0; k < kWD; ++k) dW[k] = wDg[k];
#pragma unroll
                        for (int k = 0; k < kWR; ++k) wo[k] = chk ? wold[(size_t)k * N + iw] : 0.0;
                    }
                    // publish x (neighbours need station i-1 and the control) and read the scalings
                    c.sync();
                    if (st.live) { s.tr()[st.pos] = st.xa; s.tr()[st.pos + 1] = st.xb; s.tr()[st.pos + 2] = st.xc; }
                    if (ub.live) s.tr()[ub.pos] = PQP_UBX;
                    c.sync();
                    PQP_CK(0)
                    double pr = 0, nz = 0, nax = 0, prs = 0, nzs = 0, naxs = 0;
                    double dr = 0, npx = 0, naty = 0, drs = 0, npxs = 0, natys = 0;
                    const double cinv = 1.0 / cost_c;
#define PQP_ROW(AX, V, LO, HI, EE)                                                   \
    {                                                                                \
        const double ax_ = (AX), v_ = (V), z_ = clamp2(v_, (LO), (HI)), r_ = ax_ - z_; \
        const double e_ = (EE);                                                      \
        pr = fmax(pr, fabs(r_)); nz = fmax(nz, fabs(z_)); nax = fmax(nax, fabs(ax_)); \
        prs = fmax(prs, e_ * fabs(r_)); nzs = fmax(nzs, e_ * fabs(z_));              \
        naxs = fmax(naxs, e_ * fabs(ax_));                                           \
    }
#define PQP_DUAL(V, LO, HI, WW) ((WW) * ((V) - clamp2((V), (LO), (HI))) * cinv)
#define PQP_VAR(PX, ATY, DD)                                                          \
    {                                                                                 \
        const double px_ = (PX), aty_ = (ATY), r_ = px_ + aty_, cd_ = cost_c * (DD);  \
        dr = fmax(dr, fabs(r_)); npx = fmax(npx, fabs(px_)); naty = fmax(naty, fabs(aty_)); \
        drs = fmax(drs, cd_ * fabs(r_)); npxs = fmax(npxs, cd_ * fabs(px_));          \
        natys = fmax(natys, cd_ * fabs(aty_));                                        \
    }
                    double yD0 = 0, yD1 = 0, yD2 = 0;
                    if (st.live) {
                        double aD0 = -st.xa, aD1 = -st.xb, aD2 = -st.xc;
                        if (!st.first) {
                            const double at = s.tr()[st.posp], bt = s.tr()[st.posp + 1], ct = s.tr()[st.posp + 2];
                            const double ut = s.tr()[st.posup];
                            aD0 += at + st.dst * bt;
                            aD1 += st.qt * at + bt + st.dst * ct;
                            aD2 += ct + st.dst * ut;
                        }
                        PQP_ROW(aD0, st.vD0, st.b0, st.b0, eW[0])
                        PQP_ROW(aD1, st.vD1, st.b1, st.b1, eW[1])
                        PQP_ROW(aD2, st.vD2, st.b2, st.b2, eW[2])
                        if constexpr (kKPC) {
                            const double e4 = st.xa + cS4 * st.xb;
                            PQP_ROW(st.xc + st.xk, st.vKL, -st.mk, kOsqpInfty, eW[3])
                            PQP_ROW(st.xc - st.xk, st.vKU, -kOsqpInfty, st.mk, eW[3])
                            PQP_ROW(st.xs, st.vSB, 0.0, pm.margin, eW[4])
                            PQP_ROW(st.xk, st.vSK, 0.0, st.uSK, eW[9])
                            PQP_ROW(st.xa + cH1 * st.xb, st.vH1, st.lH1, st.uH1, eW[5])
                            PQP_ROW(st.xa + cH3 * st.xb, st.vH3, st.lH3, st.uH3, eW[6])
                            PQP_ROW(st.xa + cH4 * st.xb, st.vH4, st.lH4, st.uH4, eW[8])
                            PQP_ROW(e4 - st.xs, st.vS4m, -kOsqpInfty, st.uS4m, eW[7])
                            PQP_ROW(e4 + st.xs, st.vS4p, st.lS4p, kOsqpInfty, eW[7])
                        } else {
                        const double e4 = st.xa + d4 * st.xb, e2 = st.xa + d2 * st.xb;
                        PQP_ROW(st.xc, st.vKB, -pm.kmax, pm.kmax, eW[3])
                        PQP_ROW(st.xs, st.vSB, 0.0, pm.margin, eW[4])
                        PQP_ROW(st.xa + d1 * st.xb, st.vH1, st.lH1, st.uH1, eW[5])
                        PQP_ROW(st.xa + d3 * st.xb, st.vH3, st.lH3, st.uH3, eW[6])
                        PQP_ROW(e4 - st.xs, st.vS4m, -kOsqpInfty, st.uS4m, eW[7])
                        PQP_ROW(e4 + st.xs, st.vS4p, st.lS4p, kOsqpInfty, eW[7])
                        PQP_ROW(e2 - st.xs, st.vS2m, -kOsqpInfty, st.uS2m, eW[8])
                        PQP_ROW(e2 + st.xs, st.vS2p, st.lS2p, kOsqpInfty, eW[8])
                        }
                        if (st.last) {
                            PQP_ROW(st.xa, vEY, lEY, uEY, ws[oEnd])
                            PQP_ROW(st.xb, vEH, lEH, uEH, ws[oEnd + 1])
                        }
                        yD0 = PQP_DUAL(st.vD0, st.b0, st.b0, st.WD0);
                        yD1 = PQP_DUAL(st.vD1, st.b1, st.b1, st.WD1);
                        yD2 = PQP_DUAL(st.vD2, st.b2, st.b2, st.WD2);
                        s.ex(0)[i] = yD0; s.ex(1)[i] = yD1; s.ex(2)[i] = yD2;
                    }
                    if (ub.live) {
                        if constexpr (kKPC) {
                            const double mkp = PQP_UBF(10), xp = PQP_UBF(7);
                            PQP_ROW(PQP_UBX + xp, PQP_UBV, -mkp, kOsqpInfty, ws[oEU + tid])
                            PQP_ROW(PQP_UBX - xp, PQP_UBF(4), -kOsqpInfty, mkp, ws[oEU + tid])
                            PQP_ROW(xp, PQP_UBF(5), 0.0, kOsqpInfty, ws[oEU + ch + tid])
                        } else {
                            PQP_ROW(PQP_UBX, PQP_UBV, -kOsqpInfty, kOsqpInfty, ws[oEU + tid])
                        }
                    }
                    PQP_CK(1)
                    c.sync();
                    PQP_CK(2)
                    if constexpr (kKPC) {
                      if (st.live) {
                        const double yKL = PQP_DUAL(st.vKL, -st.mk, kOsqpInfty, st.WK);
                        const double yKU = PQP_DUAL(st.vKU, -kOsqpInfty, st.mk, st.WK);
                        const double ySB = PQP_DUAL(st.vSB, 0.0, pm.margin, st.WSB);
                        const double ySK = PQP_DUAL(st.vSK, 0.0, st.uSK, st.WSK);
                        const double yH1 = PQP_DUAL(st.vH1, st.lH1, st.uH1, st.WH1);
                        const double yH3 = PQP_DUAL(st.vH3, st.lH3, st.uH3, st.WH3);
                        const double yH4 = PQP_DUAL(st.vH4, st.lH4, st.uH4, st.WH4);
                        const double y4m = PQP_DUAL(st.vS4m, -kOsqpInfty, st.uS4m, st.WS4);
                        const double y4p = PQP_DUAL(st.vS4p, st.lS4p, kOsqpInfty, st.WS4);
                        const double s4 = y4m + y4p;
                        double ra = -yD0 + yH1 + yH3 + yH4 + s4;
                        double rb = -yD1 + cH1 * yH1 + cH3 * yH3 + cH4 * yH4 + cS4 * s4;
                        double rc = -yD2 + yKL + yKU;
                        const double rs = ySB - y4m + y4p;
                        const double rk = ySK + yKL - yKU;
                        if (!st.last) {
                            const double n0 = s.ex(0)[i + 1], n1 = s.ex(1)[i + 1], n2 = s.ex(2)[i + 1];
                            ra += n0 + st.q10 * n1;
                            rb += st.ds * n0 + n1;
                            rc += st.ds * n1 + n2;
                        } else {
                            ra += PQP_DUAL(vEY, lEY, uEY, WEY);
                            rb += PQP_DUAL(vEH, lEH, uEH, WEH);
                        }
                        PQP_VAR(pm.w_pq * st.xa, ra, dW[0])
                        PQP_VAR(0.0, rb, dW[1])
                        PQP_VAR(pm.w_c * st.xc, rc, dW[2])
                        PQP_VAR(pm.w_s * st.xs, rs, dW[3])
                        PQP_VAR(500.0 * st.xk, rk, dW[4])
                      }
                      if (ub.live) {
                        const double mkp = PQP_UBF(10);
                        const double yL = PQP_DUAL(PQP_UBV, -mkp, kOsqpInfty, PQP_UBW);
                        const double yU = PQP_DUAL(PQP_UBF(4), -kOsqpInfty, mkp, PQP_UBW);
                        const double yP = PQP_DUAL(PQP_UBF(5), 0.0, kOsqpInfty, PQP_UBF(6));
                        double aty = yL + yU;
                        for (int t = ub.t0; t <= ub.t1; ++t) aty += s.dsS()[t] * s.ex(2)[t + 1];
                        PQP_VAR((keep * pm.w_cr) * PQP_UBX, aty, ws[oDu + tid])
                        PQP_VAR((25000.0 * keep) * PQP_UBF(7), yP + yL - yU, ws[oDu + ch + tid])
                      }
                    } else {
                    if (st.live) {
                        const double yKB = PQP_DUAL(st.vKB, -pm.kmax, pm.kmax, st.WKB);
                        const double ySB = PQP_DUAL(st.vSB, 0.0, pm.margin, st.WSB);
                        const double yH1 = PQP_DUAL(st.vH1, st.lH1, st.uH1, st.WH1);
                        const double yH3 = PQP_DUAL(st.vH3, st.lH3, st.uH3, st.WH3);
                        const double y4m = PQP_DUAL(st.vS4m, -kOsqpInfty, st.uS4m, st.WS4);
                        const double y4p = PQP_DUAL(st.vS4p, st.lS4p, kOsqpInfty, st.WS4);
                        const double y2m = PQP_DUAL(st.vS2m, -kOsqpInfty, st.uS2m, st.WS2);
                        const double y2p = PQP_DUAL(st.vS2p, st.lS2p, kOsqpInfty, st.WS2);
                        const double s4 = y4m + y4p, s2 = y2m + y2p;
                        double ra = -yD0 + yH1 + yH3 + s4 + s2;
                        double rb = -yD1 + d1 * yH1 + d3 * yH3 + d4 * s4 + d2 * s2;
                        double rc = -yD2 + yKB;
                        const double rs = ySB - y4m + y4p - y2m + y2p;
                        if (!st.last) {
                            const double n0 = s.ex(0)[i + 1], n1 = s.ex(1)[i + 1], n2 = s.ex(2)[i + 1];
                            ra += n0 + st.q10 * n1;
                            rb += st.ds * n0 + n1;
                            rc += st.ds * n1 + n2;
                        } else {
                            ra += PQP_DUAL(vEY, -1.0, 1.0, WEY);
                            rb += PQP_DUAL(vEH, lEH, uEH, WEH);
                        }
                        PQP_VAR(pm.w_pq * st.xa, ra, dW[0])
                        PQP_VAR(0.0, rb, dW[1])
                        PQP_VAR(pm.w_c * st.xc, rc, dW[2])
                        PQP_VAR(pm.w_s * st.xs, rs, dW[3])
                    }
                    if (ub.live) {
                        double aty = PQP_DUAL(PQP_UBV, -kOsqpInfty, kOsqpInfty, PQP_UBW);
                        for (int t = ub.t0; t <= ub.t1; ++t) aty += s.dsS()[t] * s.ex(2)[t + 1];
                        PQP_VAR((keep * pm.w_cr) * PQP_UBX, aty, ws[oDu + tid])
                    }
                    }
#undef PQP_ROW
#undef PQP_DUAL
#undef PQP_VAR
                    // ---- primal-infeasibility certificate (OSQP is_primal_infeasible) in unscaled terms:
                    // g = W (w_new - w_old) = E delta_y, projected on the cone of the finite bounds;
                    // ||g||_inf, u'g+ + l'g-, ||A'g||_inf.  The control rows are free (g = 0).
                    PQP_CK(3)
                    double c_nrm = 0, c_lhs = 0, c_cert = 0;
                    if (chk) {
#define PQP_G(V, LO, HI, WW, WO) ((WW) * (((V) - clamp2((V), (LO), (HI))) - (WO)))
#define PQP_ACC(G, LO, HI) { const double g_ = (G); c_nrm = fmax(c_nrm, fabs(g_)); c_lhs += (HI) * fmax(g_, 0.0) + (LO) * fmin(g_, 0.0); }
                        double gD0 = 0, gD1 = 0, gD2 = 0;
                        if (st.live) {
                            gD0 = st.WD0 * ((st.vD0 - st.b0) - wo[0]);
                            gD1 = st.WD1 * ((st.vD1 - st.b1) - wo[1]);
                            gD2 = st.WD2 * ((st.vD2 - st.b2) - wo[2]);
                        }
                        c.sync();   // the dual-residual pass has consumed ex(0..2)
                        if (st.live) { s.ex(0)[i] = gD0; s.ex(1)[i] = gD1; s.ex(2)[i] = gD2; }
                        c.sync();
                        if constexpr (kKPC) {
                          // project a row's g on the cone of its finite bounds and accumulate ||g||, u'g+ + l'g-
                          auto cone = [&](double g, double l_, double u_) {
                              const bool ui = u_ >= kOsqpInfty, li = l_ <= -kOsqpInfty;
                              if (ui) g = li ? 0.0 : fmin(g, 0.0);
                              else if (li) g = fmax(g, 0.0);
                              c_nrm = fmax(c_nrm, fabs(g));
                              c_lhs += (ui ? 0.0 : u_) * fmax(g, 0.0) + (li ? 0.0 : l_) * fmin(g, 0.0);
                              return g;
                          };
                          if (st.live) {
                            const double gKL = cone(PQP_G(st.vKL, -st.mk, kOsqpInfty, st.WK, wo[3]), -st.mk, kOsqpInfty);
                            const double gKU = cone(PQP_G(st.vKU, -kOsqpInfty, st.mk, st.WK, wo[4]), -kOsqpInfty, st.mk);
                            const double gSB = cone(PQP_G(st.vSB, 0.0, pm.margin, st.WSB, wo[5]), 0.0, pm.margin);
                            const double gSK = cone(PQP_G(st.vSK, 0.0, st.uSK, st.WSK, wo[6]), 0.0, st.uSK);
                            const double gH1 = cone(PQP_G(st.vH1, st.lH1, st.uH1, st.WH1, wo[7]), st.lH1, st.uH1);
                            const double gH3 = cone(PQP_G(st.vH3, st.lH3, st.uH3, st.WH3, wo[8]), st.lH3, st.uH3);
                            const double gH4 = cone(PQP_G(st.vH4, st.lH4, st.uH4, st.WH4, wo[9]), st.lH4, st.uH4);
                            const double g4m = cone(PQP_G(st.vS4m, -kOsqpInfty, st.uS4m, st.WS4, wo[10]), -kOsqpInfty, st.uS4m);
                            const double g4p = cone(PQP_G(st.vS4p, st.lS4p, kOsqpInfty, st.WS4, wo[11]), st.lS4p, kOsqpInfty);
                            PQP_ACC(gD0, st.b0, st.b0) PQP_ACC(gD1, st.b1, st.b1) PQP_ACC(gD2, st.b2, st.b2)
                            const double s4 = g4m + g4p;
                            double ra = -gD0 + gH1 + gH3 + gH4 + s4;
                            double rb = -gD1 + cH1 * gH1 + cH3 * gH3 + cH4 * gH4 + cS4 * s4;
                            double rc = -gD2 + gKL + gKU;
                            const double rs = gSB - g4m + g4p;
                            const double rk = gSK + gKL - gKU;
                            if (!st.last) {
                                const double n0 = s.ex(0)[i + 1], n1 = s.ex(1)[i + 1], n2 = s.ex(2)[i + 1];
                                ra += n0 + st.q10 * n1;
                                rb += st.ds * n0 + n1;
                                rc += st.ds * n1 + n2;
                            } else {
                                ra += cone(PQP_G(vEY, lEY, uEY, WEY, wold[kWR * N]), lEY, uEY);
                                rb += cone(PQP_G(vEH, lEH, uEH, WEH, wold[kWR * N + 1]), lEH, uEH);
                            }
                            c_cert = fmax(fmax(fmax(fabs(ra), fabs(rb)), fmax(fabs(rc), fabs(rs))), fabs(rk));
                          }
                          if (ub.live) {
                            const double mkp = PQP_UBF(10);
                            const double *wc = wold + kWR * N + 2 + tid;
                            const double gL = cone(PQP_G(PQP_UBV, -mkp, kOsqpInfty, PQP_UBW, wc[0]), -mkp, kOsqpInfty);
                            const double gU = cone(PQP_G(PQP_UBF(4), -kOsqpInfty, mkp, PQP_UBW, wc[ch]), -kOsqpInfty, mkp);
                            const double gP = cone(PQP_G(PQP_UBF(5), 0.0, kOsqpInfty, PQP_UBF(6), wc[2 * ch]), 0.0, kOsqpInfty);
                            double aty = gL + gU;
                            for (int t = ub.t0; t <= ub.t1; ++t) aty += s.dsS()[t] * s.ex(2)[t + 1];
                            c_cert = fmax(c_cert, fmax(fabs(aty), fabs(gP + gL - gU)));
                          }
                        } else {
                        if (st.live) {
                            const double gKB = PQP_G(st.vKB, -pm.kmax, pm.kmax, st.WKB, wo[3]);
                            const double gSB = PQP_G(st.vSB, 0.0, pm.margin, st.WSB, wo[4]);
                            const double gH1 = PQP_G(st.vH1, st.lH1, st.uH1, st.WH1, wo[5]);
                            const double gH3 = PQP_G(st.vH3, st.lH3, st.uH3, st.WH3, wo[6]);
                            // one-sided rows: l = -inf keeps the positive part, u = +inf the negative part
                            const double g4m = fmax(PQP_G(st.vS4m, -kOsqpInfty, st.uS4m, st.WS4, wo[7]), 0.0);
                            const double g4p = fmin(PQP_G(st.vS4p, st.lS4p, kOsqpInfty, st.WS4, wo[8]), 0.0);
                            const double g2m = fmax(PQP_G(st.vS2m, -kOsqpInfty, st.uS2m, st.WS2, wo[9]), 0.0);
                            const double g2p = fmin(PQP_G(st.vS2p, st.lS2p, kOsqpInfty, st.WS2, wo[10]), 0.0);
                            PQP_ACC(gD0, st.b0, st.b0) PQP_ACC(gD1, st.b1, st.b1) PQP_ACC(gD2, st.b2, st.b2)
                            PQP_ACC(gKB, -pm.kmax, pm.kmax) PQP_ACC(gSB, 0.0, pm.margin)
                            PQP_ACC(gH1, st.lH1, st.uH1) PQP_ACC(gH3, st.lH3, st.uH3)
                            PQP_ACC(g4m, 0.0, st.uS4m) PQP_ACC(g4p, st.lS4p, 0.0)
                            PQP_ACC(g2m, 0.0, st.uS2m) PQP_ACC(g2p, st.lS2p, 0.0)
                            const double s4 = g4m + g4p, s2 = g2m + g2p;
                            double ra = -gD0 + gH1 + gH3 + s4 + s2;
                            double rb = -gD1 + d1 * gH1 + d3 * gH3 + d4 * s4 + d2 * s2;
                            double rc = -gD2 + gKB;
                            const double rs = gSB - g4m + g4p - g2m + g2p;
                            if (!st.last) {
                                const double n0 = s.ex(0)[i + 1], n1 = s.ex(1)[i + 1], n2 = s.ex(2)[i + 1];
                                ra += n0 + st.q10 * n1;
                                rb += st.ds * n0 + n1;
                                rc += st.ds * n1 + n2;
                            } else {
                                const double gEY = PQP_G(vEY, -1.0, 1.0, WEY, wold[kWR * N]);
                                double gEH = PQP_G(vEH, lEH, uEH, WEH, wold[kWR * N + 1]);
                                PQP_ACC(gEY, -1.0, 1.0)
                                if (uEH >= kOsqpInfty) gEH = (lEH <= -kOsqpInfty) ? 0.0 : fmin(gEH, 0.0);
                                else if (lEH <= -kOsqpInfty) gEH = fmax(gEH, 0.0);
                                PQP_ACC(gEH, (lEH <= -kOsqpInfty ? 0.0 : lEH), (uEH >= kOsqpInfty ? 0.0 : uEH))
                                ra += gEY;
                                rb += gEH;
                            }
                            c_cert = fmax(fmax(fabs(ra), fabs(rb)), fmax(fabs(rc), fabs(rs)));
                        }
                        if (ub.live) {
                            double aty = 0.0;
                            for (int t = ub.t0; t <= ub.t1; ++t) aty += s.dsS()[t] * s.ex(2)[t + 1];
                            c_cert = fmax(c_cert, fabs(aty));
                        }
                        }
#undef PQP_G
#undef PQP_ACC
                    }
                    PQP_CK(4)
                    {
                        // the 14 maxima and (checks only) the certificate's sum u'g+ + l'g- over the CTA in ONE shared
                        // exchange: warp butterflies, one slot row of 16 per warp, and the cross-warp combine unrolled
                        // over the compile-time warp count.  Same operations in the same order as Cta::max_n and
                        // Cta::sum (warp 0's partial first, then warps 1, 2, ...), so the same bits.
                        double red[14] = {pr, nz, nax, prs, nzs, naxs, dr, npx, naty, drs, npxs, natys, c_nrm, c_cert};
                        static_assert(NW > 1 && 16 * NW <= kCtaScratch, "one slot row of 16 per warp");
#pragma unroll
                        for (int k = 0; k < 14; ++k) red[k] = c.w.max(red[k]);
                        if (chk) c_lhs = c.w.sum(c_lhs);
                        double *const sc = c.scratch;
                        if (lane == 0) {
#pragma unroll
                            for (int k = 0; k < 14; ++k) sc[wid * 16 + k] = red[k];
                            sc[wid * 16 + 14] = c_lhs;
                        }
                        c.cs.sync();
#pragma unroll
                        for (int k = 0; k < 14; ++k) {
                            double r = sc[k];
#pragma unroll
                            for (int q = 1; q < NW; ++q) r = fmax(r, sc[q * 16 + k]);
                            red[k] = r;
                        }
                        if (chk) {
                            double r = sc[14];
#pragma unroll
                            for (int q = 1; q < NW; ++q) r += sc[q * 16 + 14];
                            c_lhs = r;
                        }
                        c.cs.sync();
                        pr = red[0]; nz = red[1]; nax = red[2]; prs = red[3]; nzs = red[4]; naxs = red[5];
                        dr = red[6]; npx = red[7]; naty = red[8]; drs = red[9]; npxs = red[10]; natys = red[11];
                        c_nrm = red[12]; c_cert = red[13];
                    }
                    PQP_CK(5)
#undef PQP_CK
                    // No residual or certificate is carried across iterations (registers): the 10x
                    // re-check OSQP does when max_iter is reached is decided right here.
                    const double pri_res = pr, dua_res = dr;
                    const double pri_nrm = fmax(nz, nax), dua_nrm = fmax(npx, naty);
                    if (chk) {
                        // OSQP check_termination; q = 0, so the dual-infeasibility test (q'dx < 0) never fires
                        const bool prim_ok = pri_res < pm.eps_abs + pm.eps_rel * pri_nrm;
                        if (pri_res > kOsqpInfty || dua_res > kOsqpInfty) status = PQP_NON_CVX;
                        else if (prim_ok && dua_res < pm.eps_abs + pm.eps_rel * dua_nrm) status = PQP_SOLVED;
                        else if (!prim_ok && primal_infeasible(c_nrm, c_lhs, c_cert, pm.eps_prim_inf))
                            status = PQP_PRIMAL_INFEASIBLE;
                        if (status == PQP_UNSOLVED && iter == pm.max_iter) {
                            const bool prim_ok10 = pri_res < 10 * pm.eps_abs + 10 * pm.eps_rel * pri_nrm;
                            if (prim_ok10 && dua_res < 10 * pm.eps_abs + 10 * pm.eps_rel * dua_nrm) status = PQP_SOLVED_INACCURATE;
                            else if (!prim_ok10 && primal_infeasible(c_nrm, c_lhs, c_cert, 10 * pm.eps_prim_inf))
                                status = PQP_PRIMAL_INFEASIBLE_INACCURATE;
                            else status = PQP_MAX_ITER_REACHED;
                        }
                    }
                    if (status == PQP_UNSOLVED && can_adapt) {
                        const double pn = prs / (fmax(nzs, naxs) + 1e-10);
                        const double dn = drs / (fmax(npxs, natys) + 1e-10);
                        double rho_new = rho * sqrt(pn / (dn + 1e-10));
                        rho_new = fmin(fmax(rho_new, kRhoMin), kRhoMax);
                        if (rho_new > rho * pm.adaptive_rho_tolerance || rho_new < rho / pm.adaptive_rho_tolerance) {
                            const double ratio = rho / rho_new;   // y is kept: w = E^-1 y / rho_row rescales
                            double v, z;
#define PQP_RESC(V, LO, HI) v = (V); z = clamp2(v, (LO), (HI)); (V) = z + (v - z) * ratio;
                            st.vD0 = st.b0 + (st.vD0 - st.b0) * ratio;
                            st.vD1 = st.b1 + (st.vD1 - st.b1) * ratio;
                            st.vD2 = st.b2 + (st.vD2 - st.b2) * ratio;
                            if constexpr (kKPC) {
                                PQP_RESC(st.vKL, -st.mk, kOsqpInfty)
                                PQP_RESC(st.vKU, -kOsqpInfty, st.mk)
                                PQP_RESC(st.vSK, 0.0, st.uSK)
                                PQP_RESC(st.vH4, st.lH4, st.uH4)
                                if (ub.live) {
                                    const double mkp = PQP_UBF(10);
                                    PQP_RESC(PQP_UBV, -mkp, kOsqpInfty)
                                    PQP_RESC(PQP_UBF(4), -kOsqpInfty, mkp)
                                    PQP_RESC(PQP_UBF(5), 0.0, kOsqpInfty)
                                }
                            } else {
                                PQP_RESC(st.vKB, -pm.kmax, pm.kmax)
                                PQP_RESC(st.vS2m, -kOsqpInfty, st.uS2m)
                                PQP_RESC(st.vS2p, st.lS2p, kOsqpInfty)
                            }
                            PQP_RESC(st.vSB, 0.0, pm.margin)
                            PQP_RESC(st.vH1, st.lH1, st.uH1)
                            PQP_RESC(st.vH3, st.lH3, st.uH3)
                            PQP_RESC(st.vS4m, -kOsqpInfty, st.uS4m)
                            PQP_RESC(st.vS4p, st.lS4p, kOsqpInfty)
                            if (st.last) {
                                PQP_RESC(vEY, lEY, uEY)
                                PQP_RESC(vEH, lEH, uEH)
                            }
#undef PQP_RESC
                            rho = rho_new;
                            c.sync();
#ifdef PQP_PHASE_TIMING
                            {   // (counted in ph_refactor, not in ph_check)
                                const long long t0_ = clock64();
                                if (!refactor()) status = PQP_NON_CVX;
                                const long long dt_ = clock64() - t0_;
                                ph_refactor += dt_; ph_check -= dt_; ++ph_nref;
                            }
#else
                            if (!refactor()) status = PQP_NON_CVX;
#endif
                        }
                    }
#ifdef PQP_PHASE_TIMING
                    ph_check += clock64() - ph_t;   // (a refactorisation it triggered is subtracted above)
#endif
                }
            };
#undef PQP_BAR
            // first iteration after `it` that needs the checked form
            auto next_event = [&](int it) {
                int k = pm.max_iter;
                if (pm.check_termination > 0) { const int q = (it / pm.check_termination + 1) * pm.check_termination; k = q < k ? q : k; }
                if (pm.adaptive_rho && pm.adaptive_rho_interval > 0) {
                    const int q = (it / pm.adaptive_rho_interval + 1) * pm.adaptive_rho_interval;
                    k = q < k ? q : k;
                }
                return k;
            };
            if constexpr (kLean) { s.ixS()[tid] = i / L; s.ixS()[kT + tid] = tid / M; }   // (each thread reads back its own)
            iter = first_event ? 0 : 1;
            if (first_event && is_check(1)) {
                for (int k = tid; k < kWR * N + 2 + (kKPC ? 3 * ch : 0); k += kT) wold[k] = 0.0;
                c.sync();
            }
            while (status == PQP_UNSOLVED && iter < pm.max_iter) {
                const int ev = next_event(iter);
                while (iter + 1 < ev) {
                    ++iter;
                    step(std::false_type{});
                }
                if (ev > 1 && is_check(ev)) park_w();
                ++iter;
                step(std::true_type{});
                alpha_ev = alpha_pm;
            }
            // (max_iter < 1, which OSQP's settings check refuses: no iteration ran)
            if (status == PQP_UNSOLVED) status = PQP_SOLVED_INACCURATE;
            if (status == PQP_INVALID_PROBLEM) iter = 0;
        }
#ifdef PQP_PHASE_TIMING
        if (kPhTime && bv.debug && (tid & 31) == 0 && wid < 2 && status != PQP_INVALID_PROBLEM) {
            const double *acc = s.ex(5) + 8 * (wid & 1);
            for (int k = 0; k < 7; ++k) bv.debug[(2 * (size_t)prob + wid) * 8 + k] = (long long)acc[k];
            bv.debug[(2 * (size_t)prob + wid) * 8 + 7] = clock64() - ph_kernel_t0;
            if (wid == 0) {
                long long *g = bv.debug + 16 * 65536 + 4 * (size_t)prob;
                g[0] = ph_scale; g[1] = ph_refactor; g[2] = ph_check; g[3] = ph_nref;
                long long *g2 = bv.debug + 20 * 65536 + 8 * (size_t)prob;
                for (int k = 0; k < 8; ++k) g2[k] = rt_acc[k];
            }
        }
#endif
#ifdef PQP_PHASE_TIMING
        if (kPhTime && bv.debug && lane == 0 && wid < 4 && status != PQP_INVALID_PROBLEM) {
            long long *g3 = bv.debug + 32 * 65536 + 32 * (size_t)prob + 8 * wid;
            for (int k = 0; k < 6; ++k) g3[k] = ck_acc[k];
        }
#endif
        // ---- epilogue: getOptimizedPath, solver_kp_as_input.cpp:26-43
        const bool has_sol = (status == PQP_SOLVED || status == PQP_SOLVED_INACCURATE || status == PQP_MAX_ITER_REACHED);
        c.sync();
        double *px = s.ex(0), *py = s.ex(1), *seg = s.ex(2);
        if (st.live) {
            double ey = qnan, ephi = qnan, kk = qnan;
            if (has_sol) { ey = st.xa; ephi = st.xb; kk = st.xc; }
            const double angle = ref[i].z;
            const double new_angle = constraint_angle(angle + 1.57079632679489661923);
            const double tx = ref[i].x + ey * cos(new_angle);
            const double ty = ref[i].y + ey * sin(new_angle);
            out[i].x = tx; out[i].y = ty; out[i].z = angle + ephi; out[i].k = kk;
            out[i].v = 0.0; out[i].a = 0.0;
            px[i] = tx;
            py[i] = ty;
            if (bv.out_frenet) {
                double *f = bv.out_frenet + 3 * (size_t)(off + i);
                f[0] = ey; f[1] = ephi; f[2] = kk;
            }
        }
        c.sync();
        if (st.live) {
            double sg = 0.0;
            if (i > 0) {
                const double dx = px[i] - px[i - 1], dy = py[i] - py[i - 1];
                sg = sqrt(dx * dx + dy * dy);
            }
            seg[i] = sg;
        }
        c.sync();
        if (tid == 0) {
            double acc = 0.0;  // sequential: same association order as the reference's running sum
            for (int k = 0; k < N; ++k) {
                acc += seg[k];
                out[k].s = acc;
            }
            bv.status[prob] = status;
            if (bv.iters) bv.iters[prob] = iter;
        }
        c.sync();
    }
#undef PQP_F
#undef vEY
#undef vEH
#undef WEY
#undef WEH
#undef lEH
#undef uEH
#undef PQP_UBV
#undef PQP_UBW
#undef PQP_UBX
#undef PQP_UBSG
#undef PQP_UBF
};

}  // namespace pqp
