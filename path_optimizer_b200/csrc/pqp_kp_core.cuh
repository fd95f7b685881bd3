// pqp_kp_core.cuh -- one warp solves one "KP" path QP entirely on chip.
//
// Replaces, for one path:  SolverKpAsInput::setHessianMatrix / setConstraintMatrix
// (reference src/solver/solver_kp_as_input.cpp:45-203), the OSQP setup + ADMM loop the
// reference runs through osqp-eigen (src/solver/solver.cpp:66-74) and
// SolverKpAsInput::getOptimizedPath (solver_kp_as_input.cpp:26-43).
//
// Nothing is materialised: P, A, l, u exist only as per-station coefficients.  The iteration is
// OSQP's, rewritten in unscaled variables with per-row weights W = rho_row*E^2 and per-variable
// sigma_v = sigma/D^2 (E, D, c = OSQP's Ruiz scalings), which is algebraically identical to
// OSQP's scaled iteration (see DESIGN.md "The recurrence"):
//     v_r   = z_r + w_r                  (one stored value per row; z = clamp(v), w = v - z,
//                                          OSQP's scaled dual is y_r = rho_r E_r w_r)
//     rhs   = sigma_v x + A' W (2 clamp(v) - v)
//     (cP + diag(sigma_v) + A' W A) xt = rhs          <- reduced KKT, banded, SPD
//     v    += alpha (A xt - clamp(v));   x = alpha xt + (1 - alpha) x
// Variables are ordered station by station (e_y, e_phi, kappa)_i with each held control u_j placed
// after station j*keep + keep/2, which makes the reduced KKT banded (half-bandwidth <= 7 for
// keep <= 4).  The slack s_i decouples exactly (its two soft rows carry equal weights) and the
// second N slack variables of the reference appear in no constraint and stay 0.
//
// Linear solves are partitioned across the lanes of the warp: stations 0, L, 2L, ... are
// separators (3 unknowns each), lane p owns the interior between separator p and p+1, factors /
// solves it privately (banded LDL'), and a block-tridiagonal Schur system over the separators ties
// the lanes together.
#pragma once
#include "pqp_device.cuh"

#if defined(__CUDACC__) && !defined(PQP_HOST_EMU)
#define PQP_HD __host__ __device__ __forceinline__
#else
#define PQP_HD inline
#endif

namespace pqp {

// Global-memory workspace of one path (BatchView::workspace): 16 doubles per station + kWsPerPath
// for the scaling vectors the v2/v3 kernels keep out of shared memory (E: 9N + ch + 2, D: nv, N),
// plus 16 doubles per station for w = v - clamp(v) of the previous iterate, parked only on
// iterations that end in a termination check (11N + 2 used): region = 32 N + kWsPerPath.
constexpr int kWsPerPath = 2048;
constexpr int kWsPerStation = 32;
PQP_HD size_t kp2_ws_doubles(size_t total_points, size_t batch) { return kWsPerStation * total_points + (size_t)kWsPerPath * batch; }
PQP_HD double *kp_ws_base(double *workspace, int off, int prob) {
    return workspace + (size_t)off * kWsPerStation + (size_t)prob * kWsPerPath;
}
PQP_HD double *kp_ws_wold(double *ws, int N) { return ws + 16 * (size_t)N + kWsPerPath; }

struct KpDims {
    int N, keep, ch, h, nred, bw, L, M;
};

// solver_kp_as_input.cpp:17-23 sizes + the layout constants of this implementation.
PQP_HD KpDims kp_dims(int N, int keep) {
    KpDims d;
    d.N = N;
    d.keep = keep;
    d.ch = (N + keep - 2) / keep;
    d.h = keep / 2;
    d.nred = 3 * N + d.ch;
    int bw = 5;
    if (3 * (keep - d.h) > bw) bw = 3 * (keep - d.h);
    if (3 * d.h + 1 > bw) bw = 3 * d.h + 1;
    d.bw = bw;
    int L = keep * ((N - 1 + 31 * keep - 1) / (31 * keep));
    if (L < 2) L = 2;
    d.L = L;
    d.M = (N - 1) / L + 1;
    return d;
}

// number of held controls whose home station is < i
PQP_HD int kp_cnt_before(const KpDims &d, int i) {
    int r = i - d.h;
    if (r <= 0) return 0;
    int c = (r - 1) / d.keep + 1;
    return c < d.ch ? c : d.ch;
}
PQP_HD int kp_gx(const KpDims &d, int i) { return 3 * i + kp_cnt_before(d, i); }
PQP_HD int kp_gu(const KpDims &d, int j) {
    int home = j * d.keep + d.h;
    if (home > d.N - 1) home = d.N - 1;
    return 3 * (home + 1) + j;
}

// Shared-memory layout (in doubles).  All arrays are [field][station]; addresses are computed
// arithmetically from the base so that the layout costs no registers.
//   5 arrays of nred : xr tr tmp Dr sgr
//   39 arrays of N   : see the indices below
//   2 arrays of ch   : vUB EUB ; 4 scalars: vEnd[2] EEnd[2]
//   band [(bw+1)*nred] ; red [kRedStride*32]
constexpr int kRedStride = 48;
// Shared-memory layout.  The Ruiz scalings (row factors E of the 9 per-station row kinds, column factors D) are read
// at scaling time, in the row weights and at residual checks; they normally sit in shared memory next to the rest, but
// for paths too long for that (N > ~340 stations) they move to the path's global workspace (`in_ws`), which takes the
// one-warp kernel to ~420 stations.
constexpr int kKpNrArrays = 4;    // xr, tr, tmp, sgr            [nred each]
constexpr int kKpNArrays = 29;    // per-station arrays kept in shared memory in both layouts
constexpr int kKpEArrays = 10;    // ED[3], EKB, ESB, EH1, EH3, ES4, ES2, Dsl   [N each]  (+ Dr [nred])
struct KpSmem {
    double *base;
    double *ebase;   // E arrays + Dsl: shared memory or workspace
    double *drbase;  // Dr
    int N, ch, nred, bwp1;
    bool in_ws;
#define PQP_F_NR(name, k) \
    PQP_DEV double *name() const { return base + (k) * nred; }
#define PQP_F_N(name, k) \
    PQP_DEV double *name() const { return base + kKpNrArrays * nred + (k) * N; }
#define PQP_F_E(name, k) \
    PQP_DEV double *name() const { return ebase + (k) * N; }
    PQP_F_NR(xr, 0)   // iterate, reduced unknowns in g-order
    PQP_F_NR(tr, 1)   // rhs / x-tilde
    PQP_F_NR(tmp, 2)  // second vector (interior correction solve, scratch)
    PQP_F_NR(sgr, 3)  // sigma / D^2
    PQP_DEV double *Dr() const { return drbase; }   // Ruiz D
    PQP_F_N(xs, 0) PQP_F_N(ts, 1)
    PQP_F_N(vD, 2)    // [3][N] v = z + w of the dynamics rows
    PQP_F_N(vKB, 5) PQP_F_N(vSB, 6) PQP_F_N(vH1, 7) PQP_F_N(vH3, 8)
    PQP_F_N(vS4m, 9) PQP_F_N(vS4p, 10) PQP_F_N(vS2m, 11) PQP_F_N(vS2p, 12)
    PQP_F_E(ED, 0)    // [3][N] Ruiz E of the dynamics rows
    PQP_F_E(EKB, 3) PQP_F_E(ESB, 4) PQP_F_E(EH1, 5) PQP_F_E(EH3, 6) PQP_F_E(ES4, 7) PQP_F_E(ES2, 8)
    PQP_F_E(Dsl, 9)
    PQP_F_N(sgs, 13)
    PQP_F_N(ds, 14) PQP_F_N(q10, 15) PQP_F_N(kds, 16)  // ds_i, -kappa_i^2 ds_i, ds_i kappa_i
    PQP_F_N(lH1, 17) PQP_F_N(uH1, 18) PQP_F_N(lH3, 19) PQP_F_N(uH3, 20)
    PQP_F_N(uS4m, 21) PQP_F_N(lS4p, 22) PQP_F_N(uS2m, 23) PQP_F_N(lS2p, 24)
    PQP_F_N(gD, 25)   // [3][N] weighted dynamics-row values for the A' gather
    PQP_F_N(ksinv, 28)
#undef PQP_F_NR
#undef PQP_F_N
#undef PQP_F_E
    PQP_DEV double *tail() const { return base + kKpNrArrays * nred + kKpNArrays * N; }
    PQP_DEV double *vUB() const { return tail(); }
    PQP_DEV double *EUB() const { return tail() + ch; }
    PQP_DEV double *vEnd() const { return tail() + 2 * ch; }
    PQP_DEV double *EEnd() const { return tail() + 2 * ch + 2; }
    PQP_DEV double *band() const { return tail() + 2 * ch + 4; }
    PQP_DEV double *red() const { return band() + bwp1 * nred; }
    PQP_DEV double *escr() const { return red() + kRedStride * 32; }   // E arrays + Dr when they stay in shared memory
};

PQP_HD size_t kp_smem_doubles(const KpDims &d, bool in_ws = false) {
    return (size_t)kKpNrArrays * d.nred + (size_t)kKpNArrays * d.N + 2 * (size_t)d.ch + 4 +
           (size_t)(d.bw + 1) * d.nred + (size_t)kRedStride * 32 +
           (in_ws ? 0 : (size_t)kKpEArrays * d.N + (size_t)d.nred);
}

// `ws` = the path's workspace region (kp_ws_base); used for the scalings when in_ws
PQP_DEV void kp_smem_carve(const KpDims &d, double *base, KpSmem &s, bool in_ws, double *ws) {
    s.base = base; s.N = d.N; s.ch = d.ch; s.nred = d.nred; s.bwp1 = d.bw + 1;
    s.in_ws = in_ws;
    s.ebase = in_ws ? ws : s.escr();
    s.drbase = s.ebase + (size_t)kKpEArrays * d.N;
}

// ---- per-problem context ------------------------------------------------------------------------
struct KpCtx {
    KpDims d;
    KpSmem s;
    const DevParams *pm;
    double x0[3];
    double lEH, uEH;   // end-heading window
    double c;          // OSQP cost scaling
    double Dt;         // scaling of the dead second-slack columns
    double rho;
    int lo, hi, gsep;  // this lane's interior g-range and separator start (lane < M)
};

#define PQP_B(g, dd) s.band()[(g) * (bw + 1) + (dd)]

// Thread-local banded LDL' of K[lo:hi, lo:hi] in place (rows >= hi are left untouched).
// Returns 0 on a non-positive pivot.
PQP_DEV int kp_local_factor(const KpCtx &cx, int lo, int hi) {
    const KpSmem &s = cx.s;
    const int bw = cx.d.bw;
    int ok = 1;
    for (int j = lo; j < hi; ++j) {
        const double dj = PQP_B(j, 0);
        if (!(dj > 0.0)) ok = 0;
        const double dinv = 1.0 / dj;
        int R = hi - 1 - j;
        if (R > bw) R = bw;
        for (int r = 1; r <= R; ++r) {
            const double kr = PQP_B(j + r, r);
            for (int cc = 1; cc <= r; ++cc) PQP_B(j + r, r - cc) -= kr * (PQP_B(j + cc, cc) * dinv);
        }
        for (int r = 1; r <= R; ++r) PQP_B(j + r, r) *= dinv;
        PQP_B(j, 0) = dinv;
    }
    return ok;
}

// Thread-local solve K[lo:hi,lo:hi] x = v (in place) with the factor above.
PQP_DEV void kp_local_solve(const KpCtx &cx, double *v, int lo, int hi) {
    const KpSmem &s = cx.s;
    const int bw = cx.d.bw;
    for (int g = lo; g < hi; ++g) {
        double acc = v[g];
        int dm = g - lo;
        if (dm > bw) dm = bw;
        for (int dd = 1; dd <= dm; ++dd) acc -= PQP_B(g, dd) * v[g - dd];
        v[g] = acc;
    }
    for (int g = hi - 1; g >= lo; --g) {
        double acc = v[g] * PQP_B(g, 0);
        int dm = hi - 1 - g;
        if (dm > bw) dm = bw;
        for (int dd = 1; dd <= dm; ++dd) acc -= PQP_B(g + dd, dd) * v[g + dd];
        v[g] = acc;
    }
}

// symmetric positive definite 3x3 inverse (row-major 9) via LDL'
PQP_DEV void inv3_spd(const double *a, double *o) {
    const double d0 = a[0];
    const double l10 = a[3] / d0, l20 = a[6] / d0;
    const double d1 = a[4] - l10 * a[3];
    const double l21 = (a[7] - l20 * a[3]) / d1;
    const double d2 = a[8] - l20 * a[6] - l21 * (a[7] - l20 * a[3]);
    // inverse of L (unit lower): m10 = -l10, m21 = -l21, m20 = l10*l21 - l20
    const double m10 = -l10, m21 = -l21, m20 = l10 * l21 - l20;
    const double i0 = 1.0 / d0, i1 = 1.0 / d1, i2 = 1.0 / d2;
    // inv = M' diag(i) M
    o[0] = i0 + m10 * m10 * i1 + m20 * m20 * i2;
    o[1] = o[3] = m10 * i1 + m20 * m21 * i2;
    o[2] = o[6] = m20 * i2;
    o[4] = i1 + m21 * m21 * i2;
    o[5] = o[7] = m21 * i2;
    o[8] = i2;
}

// W of the rows of station i for the current rho ------------------------------------------------
struct KpRowW {
    double D0, D1, D2, KB, SB, H1, H3, S4, S2;
};
PQP_DEV double kp_w_eq(double E, double rho) { return (kRhoEqOverIneq * rho) * E * E; }
PQP_DEV double kp_w_box(double E, double lo, double hi, double rho) {
    return rho_bar(E * lo, E * hi, rho) * E * E;
}
PQP_DEV KpRowW kp_row_weights(const KpCtx &cx, int i, double rho) {
    const KpSmem &s = cx.s;
    const int N = cx.d.N;
    KpRowW w;
    w.D0 = kp_w_eq(s.ED()[i], rho);
    w.D1 = kp_w_eq(s.ED()[N + i], rho);
    w.D2 = kp_w_eq(s.ED()[2 * N + i], rho);
    w.KB = kp_w_box(s.EKB()[i], -cx.pm->kmax, cx.pm->kmax, rho);
    w.SB = kp_w_box(s.ESB()[i], 0.0, cx.pm->margin, rho);
    w.H1 = kp_w_box(s.EH1()[i], s.lH1()[i], s.uH1()[i], rho);
    w.H3 = kp_w_box(s.EH3()[i], s.lH3()[i], s.uH3()[i], rho);
    w.S4 = kp_w_box(s.ES4()[i], -kOsqpInfty, s.uS4m()[i], rho);
    w.S2 = kp_w_box(s.ES2()[i], -kOsqpInfty, s.uS2m()[i], rho);
    return w;
}
PQP_DEV double kp_w_ub(const KpCtx &cx, int j, double rho) {
    return kp_w_box(cx.s.EUB()[j], -kOsqpInfty, kOsqpInfty, rho);
}
PQP_DEV double kp_w_ey(const KpCtx &cx, double rho) { return kp_w_box(cx.s.EEnd()[0], -1.0, 1.0, rho); }
PQP_DEV double kp_w_eh(const KpCtx &cx, double rho) { return kp_w_box(cx.s.EEnd()[1], cx.lEH, cx.uEH, rho); }

// bound of the dynamics (equality) rows of station i
PQP_DEV void kp_dyn_bounds(const KpCtx &cx, int i, double &b0, double &b1, double &b2) {
    if (i == 0) {
        b0 = -cx.x0[0]; b1 = -cx.x0[1]; b2 = -cx.x0[2];
    } else {
        b0 = 0.0; b1 = cx.s.kds()[i - 1]; b2 = 0.0;
    }
}

// ---- Ruiz equilibration + cost scaling (OSQP scale_data), matrix free ------------------------
PQP_DEV void kp_scale(Warp &w, KpCtx &cx) {
    KpSmem &s = cx.s;
    const KpDims &d = cx.d;
    const int N = d.N, ch = d.ch, keep = d.keep, lane = w.lane();
    const DevParams &pm = *cx.pm;
    // temporaries alias the (not yet used) band area
    double *fDr = s.band(), *fDs = fDr + d.nred, *fE = fDs + N;  // fE: 9N + ch + 2
    for (int g = lane; g < d.nred; g += 32) s.Dr()[g] = 1.0;
    for (int i = lane; i < N; i += 32) {
        s.Dsl()[i] = 1.0;
        s.ED()[i] = s.ED()[N + i] = s.ED()[2 * N + i] = 1.0;
        s.EKB()[i] = s.ESB()[i] = s.EH1()[i] = s.EH3()[i] = s.ES4()[i] = s.ES2()[i] = 1.0;
    }
    for (int j = lane; j < ch; j += 32) s.EUB()[j] = 1.0;
    if (lane == 0) s.EEnd()[0] = s.EEnd()[1] = 1.0;
    cx.c = 1.0;
    cx.Dt = 1.0;
    w.sync();
    const double ad1 = fabs(pm.d1), ad2 = fabs(pm.d2), ad3 = fabs(pm.d3), ad4 = fabs(pm.d4);
    for (int sweep = 0; sweep < pm.scaling; ++sweep) {
        const double c = cx.c;
        for (int i = lane; i < N; i += 32) {
            const int ga = kp_gx(d, i);
            const double Da = s.Dr()[ga], Db = s.Dr()[ga + 1], Dc = s.Dr()[ga + 2], Dsv = s.Dsl()[i];
            const double e0 = s.ED()[i], e1 = s.ED()[N + i], e2 = s.ED()[2 * N + i];
            const double eKB = s.EKB()[i], eSB = s.ESB()[i], eH1 = s.EH1()[i], eH3 = s.EH3()[i];
            const double eS4 = s.ES4()[i], eS2 = s.ES2()[i];
            const bool last = (i == N - 1);
            // column norms of [P; A]
            double Aa = fmax(fmax(e0, eH1), fmax(eH3, fmax(eS4, eS2)));
            double Ab = fmax(fmax(e1, eH1 * ad1), fmax(eH3 * ad3, fmax(eS4 * ad4, eS2 * ad2)));
            double Ac = fmax(e2, eKB);
            if (!last) {
                const double e0n = s.ED()[i + 1], e1n = s.ED()[N + i + 1], e2n = s.ED()[2 * N + i + 1];
                const double dsi = s.ds()[i], aq = fabs(s.q10()[i]);
                Aa = fmax(Aa, fmax(e0n, e1n * aq));
                Ab = fmax(Ab, fmax(e0n * dsi, e1n));
                Ac = fmax(Ac, fmax(e1n * dsi, e2n));
            } else {
                Aa = fmax(Aa, s.EEnd()[0]);
                Ab = fmax(Ab, s.EEnd()[1]);
            }
            const double As = fmax(eSB, fmax(eS4, eS2));
            const double na = fmax(c * pm.w_pq * Da * Da, Aa * Da);
            const double nb = Ab * Db;
            const double nc = fmax(c * pm.w_c * Dc * Dc, Ac * Dc);
            const double ns = fmax(c * pm.w_s * Dsv * Dsv, As * Dsv);
            fDr[ga] = 1.0 / sqrt(limit_scaling(na));
            fDr[ga + 1] = 1.0 / sqrt(limit_scaling(nb));
            fDr[ga + 2] = 1.0 / sqrt(limit_scaling(nc));
            fDs[i] = 1.0 / sqrt(limit_scaling(ns));
            // row norms of A
            double r0, r1, r2;
            if (i == 0) {
                r0 = e0 * Da; r1 = e1 * Db; r2 = e2 * Dc;
            } else {
                const int t = i - 1, gt = kp_gx(d, t);
                const double Dat = s.Dr()[gt], Dbt = s.Dr()[gt + 1], Dct = s.Dr()[gt + 2];
                const double Dut = s.Dr()[kp_gu(d, t / keep)];
                const double dst = s.ds()[t], aqt = fabs(s.q10()[t]);
                r0 = e0 * fmax(Da, fmax(Dat, dst * Dbt));
                r1 = e1 * fmax(fmax(Db, aqt * Dat), fmax(Dbt, dst * Dct));
                r2 = e2 * fmax(Dc, fmax(Dct, dst * Dut));
            }
            fE[i] = 1.0 / sqrt(limit_scaling(r0));
            fE[N + i] = 1.0 / sqrt(limit_scaling(r1));
            fE[2 * N + i] = 1.0 / sqrt(limit_scaling(r2));
            fE[3 * N + i] = 1.0 / sqrt(limit_scaling(eKB * Dc));
            fE[4 * N + i] = 1.0 / sqrt(limit_scaling(eSB * Dsv));
            fE[5 * N + i] = 1.0 / sqrt(limit_scaling(eH1 * fmax(Da, ad1 * Db)));
            fE[6 * N + i] = 1.0 / sqrt(limit_scaling(eH3 * fmax(Da, ad3 * Db)));
            fE[7 * N + i] = 1.0 / sqrt(limit_scaling(eS4 * fmax(Da, fmax(ad4 * Db, Dsv))));
            fE[8 * N + i] = 1.0 / sqrt(limit_scaling(eS2 * fmax(Da, fmax(ad2 * Db, Dsv))));
            if (last) {
                fE[9 * N + ch] = 1.0 / sqrt(limit_scaling(s.EEnd()[0] * Da));
                fE[9 * N + ch + 1] = 1.0 / sqrt(limit_scaling(s.EEnd()[1] * Db));
            }
        }
        for (int j = lane; j < ch; j += 32) {
            const int gu = kp_gu(d, j);
            const double Du = s.Dr()[gu];
            double Au = s.EUB()[j];
            int t1 = j * keep + keep - 1;
            if (t1 > N - 2) t1 = N - 2;
            for (int t = j * keep; t <= t1; ++t) Au = fmax(Au, s.ED()[2 * N + t + 1] * s.ds()[t]);
            const double nu = fmax(c * (keep * pm.w_cr) * Du * Du, Au * Du);
            fDr[gu] = 1.0 / sqrt(limit_scaling(nu));
            fE[9 * N + j] = 1.0 / sqrt(limit_scaling(s.EUB()[j] * Du));
        }
        const double fDt = 1.0 / sqrt(limit_scaling(c * pm.w_s * cx.Dt * cx.Dt));
        w.sync();
        for (int g = lane; g < d.nred; g += 32) s.Dr()[g] *= fDr[g];
        for (int i = lane; i < N; i += 32) {
            s.Dsl()[i] *= fDs[i];
            s.ED()[i] *= fE[i]; s.ED()[N + i] *= fE[N + i]; s.ED()[2 * N + i] *= fE[2 * N + i];
            s.EKB()[i] *= fE[3 * N + i]; s.ESB()[i] *= fE[4 * N + i];
            s.EH1()[i] *= fE[5 * N + i]; s.EH3()[i] *= fE[6 * N + i];
            s.ES4()[i] *= fE[7 * N + i]; s.ES2()[i] *= fE[8 * N + i];
        }
        for (int j = lane; j < ch; j += 32) s.EUB()[j] *= fE[9 * N + j];
        if (lane == 0) {
            s.EEnd()[0] *= fE[9 * N + ch];
            s.EEnd()[1] *= fE[9 * N + ch + 1];
        }
        cx.Dt *= fDt;
        w.sync();
        // cost scaling: c <- c / max(mean column norm of P, 1)   (||q|| = 0 is limited to 1)
        double part = 0.0;
        for (int i = lane; i < N; i += 32) {
            const int ga = kp_gx(d, i);
            const double Da = s.Dr()[ga], Dc = s.Dr()[ga + 2], Dsv = s.Dsl()[i];
            part += c * pm.w_pq * Da * Da + c * pm.w_c * Dc * Dc + c * pm.w_s * Dsv * Dsv +
                    c * pm.w_s * cx.Dt * cx.Dt;
        }
        for (int j = lane; j < ch; j += 32) {
            const double Du = s.Dr()[kp_gu(d, j)];
            part += c * (keep * pm.w_cr) * Du * Du;
        }
        const double mean = w.sum(part) / (double)(5 * N + ch);
        double ct = fmax(mean, 1.0);
        ct = limit_scaling(ct);
        cx.c = c * (1.0 / ct);
        w.sync();
    }
    // sigma_v = sigma / D_v^2
    for (int g = lane; g < d.nred; g += 32) s.sgr()[g] = pm.sigma / (s.Dr()[g] * s.Dr()[g]);
    for (int i = lane; i < N; i += 32) s.sgs()[i] = pm.sigma / (s.Dsl()[i] * s.Dsl()[i]);
    w.sync();
}

// ---- reduced KKT assembly + partitioned factorisation ----------------------------------------
// returns 0 if a pivot was not positive (status NON_CVX)
PQP_DEV int kp_factor(Warp &w, KpCtx &cx) {
    KpSmem &s = cx.s;
    const KpDims &d = cx.d;
    const int N = d.N, ch = d.ch, keep = d.keep, bw = d.bw, lane = w.lane();
    const DevParams &pm = *cx.pm;
    const double rho = cx.rho, c = cx.c;
    const size_t nb = (size_t)(bw + 1) * d.nred;
    for (size_t k = lane; k < nb; k += 32) s.band()[k] = 0.0;
    w.sync();
    for (int i = lane; i < N; i += 32) {
        const int ga = kp_gx(d, i);
        const KpRowW W = kp_row_weights(cx, i, rho);
        const bool last = (i == N - 1);
        double N0 = 0, N1 = 0, N2 = 0, dsi = 0, q = 0;
        if (!last) {
            N0 = kp_w_eq(s.ED()[i + 1], rho);
            N1 = kp_w_eq(s.ED()[N + i + 1], rho);
            N2 = kp_w_eq(s.ED()[2 * N + i + 1], rho);
            dsi = s.ds()[i];
            q = s.q10()[i];
        }
        const double d1 = pm.d1, d2 = pm.d2, d3 = pm.d3, d4 = pm.d4;
        double da = c * pm.w_pq + s.sgr()[ga] + W.D0 + N0 + N1 * q * q + W.H1 + W.H3 + 2.0 * W.S4 + 2.0 * W.S2;
        double db = s.sgr()[ga + 1] + W.D1 + N0 * dsi * dsi + N1 + W.H1 * d1 * d1 + W.H3 * d3 * d3 +
                    2.0 * W.S4 * d4 * d4 + 2.0 * W.S2 * d2 * d2;
        const double dc = c * pm.w_c + s.sgr()[ga + 2] + W.D2 + N1 * dsi * dsi + N2 + W.KB;
        if (last) {
            da += kp_w_ey(cx, rho);
            db += kp_w_eh(cx, rho);
        }
        PQP_B(ga, 0) = da;
        PQP_B(ga + 1, 0) = db;
        PQP_B(ga + 2, 0) = dc;
        PQP_B(ga + 1, 1) = N0 * dsi + N1 * q + W.H1 * d1 + W.H3 * d3 + 2.0 * W.S4 * d4 + 2.0 * W.S2 * d2;
        PQP_B(ga + 2, 2) = N1 * q * dsi;
        PQP_B(ga + 2, 1) = N1 * dsi;
        if (i >= 1) {
            const int t = i - 1;
            const int off = ga - kp_gx(d, t);  // 3 or 4
            const double dst = s.ds()[t], qt = s.q10()[t];
            PQP_B(ga, off) = -W.D0;
            PQP_B(ga, off - 1) = -W.D0 * dst;
            PQP_B(ga + 1, off + 1) = -W.D1 * qt;
            PQP_B(ga + 1, off) = -W.D1;
            PQP_B(ga + 1, off - 1) = -W.D1 * dst;
            PQP_B(ga + 2, off) = -W.D2;
        }
        s.ksinv()[i] = 1.0 / (c * pm.w_s + s.sgs()[i] + W.SB + 2.0 * W.S4 + 2.0 * W.S2);
    }
    for (int j = lane; j < ch; j += 32) {
        const int gu = kp_gu(d, j);
        double du = c * (keep * pm.w_cr) + s.sgr()[gu] + kp_w_ub(cx, j, rho);
        int i1 = j * keep + keep;
        if (i1 > N - 1) i1 = N - 1;
        for (int ii = j * keep; ii <= i1; ++ii) {
            double val = 0.0;
            if (ii >= 1 && (ii - 1) / keep == j) {
                const double wv = kp_w_eq(s.ED()[2 * N + ii], rho), dst = s.ds()[ii - 1];
                val -= wv * dst;
                du += wv * dst * dst;
            }
            if (ii <= N - 2 && ii / keep == j) val += kp_w_eq(s.ED()[2 * N + ii + 1], rho) * s.ds()[ii];
            const int gc = kp_gx(d, ii) + 2;
            if (gc < gu) PQP_B(gu, gu - gc) = val;
            else PQP_B(gc, gc - gu) = val;
        }
        PQP_B(gu, 0) = du;
    }
    w.sync();
    // --- F1: private LDL' of each interior
    int ok = 1;
    const bool act = lane < d.M;
    double *R = s.red() + (size_t)kRedStride * lane;  // [0:9) Dg/Sinv, [9:18) Off, [18:27) G, [27:36) A, [36:45) C, [45:48) g
    if (act) ok = kp_local_factor(cx, cx.lo, cx.hi);
    w.sync();
    // --- F2: Schur complement pieces.  A = K[S_p,I] K_I^-1 K[I,S_p], C = K[S_q,I] K_I^-1 K[I,S_q],
    //         Off = -K[S_p,I] K_I^-1 K[I,S_q]   (q = p+1)
    if (act) {
        const int lo = cx.lo, hi = cx.hi, gs = cx.gsep, gq = hi;  // right separator starts at hi
        const bool has_right = (lane + 1 < d.M);
        for (int k = 9; k < 18; ++k) R[k] = 0.0;   // Off := 0
        for (int k = 27; k < 45; ++k) R[k] = 0.0;  // A, C := 0
        for (int col = 0; col < 6; ++col) {
            const bool left = col < 3;
            if (!left && !has_right) break;
            const int sc = left ? gs + col : gq + (col - 3);
            for (int g = lo; g < hi; ++g) {
                double v = 0.0;
                if (left) { if (g - sc <= bw) v = PQP_B(g, g - sc); }
                else { if (sc - g <= bw) v = PQP_B(sc, sc - g); }
                s.tmp()[g] = v;
            }
            kp_local_solve(cx, s.tmp(), lo, hi);
            for (int r = 0; r < 3; ++r) {
                // row of K[S_p, I] . w
                double accL = 0.0, accR = 0.0;
                const int sl = gs + r, sr = gq + r;
                for (int g = lo; g < hi && g - sl <= bw; ++g) accL += PQP_B(g, g - sl) * s.tmp()[g];
                if (has_right) {
                    int g0 = sr - bw;
                    if (g0 < lo) g0 = lo;
                    for (int g = g0; g < hi; ++g) accR += PQP_B(sr, sr - g) * s.tmp()[g];
                }
                if (left) {
                    R[27 + r * 3 + col] = accL;          // A[r][col]
                    R[9 + col * 3 + r] = -accR;          // Off[col][r] = -(K[S_q,I] w_col)[r]
                } else {
                    R[36 + r * 3 + (col - 3)] = accR;    // C[r][col]
                }
            }
        }
    }
    w.sync();
    if (act) {
        const int gs = cx.gsep;
        const double *Cprev = s.red() + (size_t)kRedStride * (lane - 1) + 36;
        for (int r = 0; r < 3; ++r)
            for (int cc = 0; cc < 3; ++cc) {
                const int hi_ = r > cc ? r : cc, lo_ = r > cc ? cc : r;
                double v = PQP_B(gs + hi_, hi_ - lo_) - R[27 + r * 3 + cc];
                if (lane > 0) v -= Cprev[r * 3 + cc];
                R[r * 3 + cc] = v;
            }
    }
    w.sync();
    // --- F3: block LDL' of the separator system (sequential, lane 0)
    if (lane == 0) {
        double Sch[9], Sinv[9];
        for (int k = 0; k < 9; ++k) Sch[k] = s.red()[k];
        for (int p = 0; p < d.M; ++p) {
            double *Rp = s.red() + (size_t)kRedStride * p;
            if (!(Sch[0] > 0.0)) ok = 0;
            inv3_spd(Sch, Sinv);
            for (int k = 0; k < 9; ++k) Rp[k] = Sinv[k];
            if (p + 1 < d.M) {
                double *Rn = Rp + kRedStride;
                const double *Off = Rp + 9;
                // G_{p+1} = Off' Sinv ; Sch_{p+1} = Dg_{p+1} - G_{p+1} Off
                for (int r = 0; r < 3; ++r)
                    for (int cc = 0; cc < 3; ++cc) {
                        double a = 0.0;
                        for (int k = 0; k < 3; ++k) a += Off[k * 3 + r] * Sinv[k * 3 + cc];
                        Rn[18 + r * 3 + cc] = a;
                    }
                for (int r = 0; r < 3; ++r)
                    for (int cc = 0; cc < 3; ++cc) {
                        double a = Rn[r * 3 + cc];
                        for (int k = 0; k < 3; ++k) a -= Rn[18 + r * 3 + k] * Off[k * 3 + cc];
                        Sch[r * 3 + cc] = a;
                    }
            }
        }
    }
    ok = !w.any(!ok);
    w.sync();
    return ok;
}

// Solve K xt = rhs.  rhs / solution in s.tr() (reduced unknowns) and s.ts() (slack).
PQP_DEV void kp_solve(Warp &w, KpCtx &cx) {
    KpSmem &s = cx.s;
    const KpDims &d = cx.d;
    const int N = d.N, bw = d.bw, lane = w.lane();
    const bool act = lane < d.M;
    const int lo = cx.lo, hi = cx.hi, gs = cx.gsep;
    const bool has_right = (lane + 1 < d.M);
    double *R = s.red() + (size_t)kRedStride * lane;
    for (int i = lane; i < N; i += 32) s.ts()[i] *= s.ksinv()[i];
    if (act) kp_local_solve(cx, s.tr(), lo, hi);
    w.sync();
    if (act) {
        // g_p = r_S - K[S_p, I_{p-1}] y - K[S_p, I_p] y
        for (int r = 0; r < 3; ++r) {
            const int sg = gs + r;
            double acc = s.tr()[sg];
            if (lane > 0) {
                int g0 = sg - bw;
                for (int g = g0 < 0 ? 0 : g0; g < gs; ++g) acc -= PQP_B(sg, sg - g) * s.tr()[g];
            }
            for (int g = lo; g < hi && g - sg <= bw; ++g) acc -= PQP_B(g, g - sg) * s.tr()[g];
            R[45 + r] = acc;
        }
    }
    w.sync();
    if (lane == 0) {
        // block forward / backward substitution over the separators
        for (int p = 1; p < d.M; ++p) {
            double *Rp = s.red() + (size_t)kRedStride * p;
            const double *gp = Rp - kRedStride + 45;
            for (int r = 0; r < 3; ++r)
                Rp[45 + r] -= Rp[18 + r * 3] * gp[0] + Rp[18 + r * 3 + 1] * gp[1] + Rp[18 + r * 3 + 2] * gp[2];
        }
        double xn[3] = {0, 0, 0};
        for (int p = d.M - 1; p >= 0; --p) {
            double *Rp = s.red() + (size_t)kRedStride * p;
            double t[3];
            for (int r = 0; r < 3; ++r) {
                t[r] = Rp[45 + r];
                if (p + 1 < d.M)
                    t[r] -= Rp[9 + r * 3] * xn[0] + Rp[9 + r * 3 + 1] * xn[1] + Rp[9 + r * 3 + 2] * xn[2];
            }
            for (int r = 0; r < 3; ++r) xn[r] = Rp[r * 3] * t[0] + Rp[r * 3 + 1] * t[1] + Rp[r * 3 + 2] * t[2];
            const int sg = kp_gx(d, p * d.L);
            s.tr()[sg] = xn[0]; s.tr()[sg + 1] = xn[1]; s.tr()[sg + 2] = xn[2];
        }
    }
    w.sync();
    if (act) {
        // interior correction: K_I delta = -K[I,S_p] x_p - K[I,S_q] x_q
        const int gq = hi;
        for (int g = lo; g < hi; ++g) {
            double acc = 0.0;
            for (int r = 0; r < 3; ++r) {
                const int sg = gs + r;
                if (g - sg <= bw) acc -= PQP_B(g, g - sg) * s.tr()[sg];
            }
            if (has_right)
                for (int r = 0; r < 3; ++r) {
                    const int sg = gq + r;
                    if (sg - g <= bw) acc -= PQP_B(sg, sg - g) * s.tr()[sg];
                }
            s.tmp()[g] = acc;
        }
        kp_local_solve(cx, s.tmp(), lo, hi);
        for (int g = lo; g < hi; ++g) s.tr()[g] += s.tmp()[g];
    }
    w.sync();
}

// The 11 row values (A x)_r of station i for the vector (vr, vs).
struct KpRows {
    double D0, D1, D2, KB, SB, H1, H3, S4m, S4p, S2m, S2p;
};
PQP_DEV KpRows kp_apply_A(const KpCtx &cx, int i, const double *vr, const double *vs) {
    const KpSmem &s = cx.s;
    const KpDims &d = cx.d;
    const DevParams &pm = *cx.pm;
    const int ga = kp_gx(d, i);
    const double a = vr[ga], b = vr[ga + 1], cc = vr[ga + 2], sl = vs[i];
    KpRows r;
    r.D0 = -a; r.D1 = -b; r.D2 = -cc;
    if (i >= 1) {
        const int t = i - 1, gt = kp_gx(d, t);
        const double at = vr[gt], bt = vr[gt + 1], ct = vr[gt + 2], ut = vr[kp_gu(d, t / d.keep)];
        const double dst = s.ds()[t];
        r.D0 += at + dst * bt;
        r.D1 += s.q10()[t] * at + bt + dst * ct;
        r.D2 += ct + dst * ut;
    }
    r.KB = cc;
    r.SB = sl;
    r.H1 = a + pm.d1 * b;
    r.H3 = a + pm.d3 * b;
    const double e4 = a + pm.d4 * b, e2 = a + pm.d2 * b;
    r.S4m = e4 - sl; r.S4p = e4 + sl;
    r.S2m = e2 - sl; r.S2p = e2 + sl;
    return r;
}

// A' gather for station i: given the row values of station i (own rows, in `o`) and the dynamics
// row values of station i+1 (through s.gD()), produce the components for (a, b, c, s).
PQP_DEV void kp_apply_At(const KpCtx &cx, int i, const KpRows &o, double gEY, double gEH,
                         double &ra, double &rb, double &rc, double &rs) {
    const KpSmem &s = cx.s;
    const DevParams &pm = *cx.pm;
    const int N = cx.d.N;
    const double s4 = o.S4m + o.S4p, s2 = o.S2m + o.S2p;
    ra = -o.D0 + o.H1 + o.H3 + s4 + s2;
    rb = -o.D1 + pm.d1 * o.H1 + pm.d3 * o.H3 + pm.d4 * s4 + pm.d2 * s2;
    rc = -o.D2 + o.KB;
    rs = o.SB - o.S4m + o.S4p - o.S2m + o.S2p;
    if (i < N - 1) {
        const double n0 = s.gD()[i + 1], n1 = s.gD()[N + i + 1], n2 = s.gD()[2 * N + i + 1];
        const double dsi = s.ds()[i];
        ra += n0 + s.q10()[i] * n1;
        rb += dsi * n0 + n1;
        rc += dsi * n1 + n2;
    } else {
        ra += gEY;
        rb += gEH;
    }
}

// ---- the whole per-path solve --------------------------------------------------------------------
// `smem` must hold kp_smem_doubles(dims) doubles.  Returns through view.{status,iters,out_*}.
PQP_DEV void kp_solve_path(Warp &w, const DevParams &prm, const BatchView &bv, int prob, double *smem,
                           size_t smem_doubles) {
    const int lane = w.lane();
    const int N = bv.n_points[prob];
    const int off = bv.offsets[prob];
    const pqp_state *ref = bv.ref + off;
    const pqp_station_bounds *bnd = bv.bounds + off;
    pqp_state *out = bv.out_states + off;
    // keep_control_steps_: solver.cpp:21-27 + solver_kp_as_input.cpp:17 (in double, as the reference)
    int keep = 1;
    {
        double interval = 0.0;   // std::max: a NaN interval is skipped
        for (int i = 1; i < N && i < 10; ++i) {
            const double dd = ref[i].s - ref[i - 1].s;
            interval = interval < dd ? dd : interval;
        }
        const double q = 1.2 / interval;
        keep = (q < 2147483647.0) ? (int)q : 2147483647;
        if (!(q == q)) keep = 0;
        if (keep < 1) keep = 1;
    }
    int bad = (N < 2) || (keep > 10);
    KpCtx cx;
    cx.pm = &prm;
    cx.d = kp_dims(N < 2 ? 2 : N, keep > 10 ? 10 : keep);
    // long paths: the scalings go to the workspace (needs one: 10 N + nred <= 16 N + kWsPerPath doubles)
    const bool in_ws = !bad && kp_smem_doubles(cx.d) > smem_doubles && bv.workspace != nullptr;
    if (!bad && kp_smem_doubles(cx.d, in_ws) > smem_doubles) bad = 1;
    if (bad) {
        if (lane == 0) {
            bv.status[prob] = PQP_INVALID_PROBLEM;
            if (bv.iters) bv.iters[prob] = 0;
        }
        const double qnan = nan("");
        for (int i = lane; i < N; i += 32) {
            out[i].x = out[i].y = out[i].z = out[i].k = out[i].s = qnan;
            out[i].v = out[i].a = 0.0;
            if (bv.out_frenet) {
                double *f = bv.out_frenet + 3 * (size_t)(off + i);
                f[0] = f[1] = f[2] = qnan;
            }
        }
        return;
    }
    const KpDims &d = cx.d;
    kp_smem_carve(d, smem, cx.s, in_ws, bv.workspace ? kp_ws_base(bv.workspace, off, prob) : nullptr);
    KpSmem &s = cx.s;
    const int ch = d.ch;
    const DevParams &pm = *cx.pm;
    cx.x0[0] = bv.x0[3 * (size_t)prob];
    cx.x0[1] = bv.x0[3 * (size_t)prob + 1];
    cx.x0[2] = bv.x0[3 * (size_t)prob + 2];
    // end-heading window, solver_kp_as_input.cpp:193-201
    cx.lEH = -kOsqpInfty;
    cx.uEH = kOsqpInfty;
    if (pm.constraint_end_heading) {
        const double pi = 3.14159265358979323846;
        const double end_psi = constraint_angle(bv.end_heading[prob] - ref[N - 1].z);
        if (end_psi < 70 * pi / 180) {
            cx.lEH = end_psi - 5 * pi / 180;
            cx.uEH = end_psi + 5 * pi / 180;
        }
    }
    // partition
    cx.lo = cx.hi = cx.gsep = 0;
    if (lane < d.M) {
        cx.gsep = kp_gx(d, lane * d.L);
        cx.lo = cx.gsep + 3;
        cx.hi = (lane + 1 < d.M) ? kp_gx(d, (lane + 1) * d.L) : d.nred;
    }
    // ---- load the per-station coefficients (setConstraintMatrix :84-98, :166-187)
    int invalid = 0;
    for (int i = lane; i < N; i += 32) {
        const double kap = ref[i].k;
        if (i < N - 1) {
            const double dsv = ref[i + 1].s - ref[i].s;
            s.ds()[i] = dsv;
            s.q10()[i] = -(kap * kap) * dsv;
            s.kds()[i] = dsv * kap;
            // the dynamics rows' constant is NaN exactly when ds (ref_kp - ref_kp) is (see pqp_kp_core3.cuh)
            const double rkp = (ref[i + 1].k - kap) / dsv;
            if (!(dsv * (rkp - rkp) == 0.0)) invalid = 1;
        } else {
            s.ds()[i] = 0.0; s.q10()[i] = 0.0; s.kds()[i] = 0.0;
        }
        const pqp_station_bounds bb = bnd[i];
        s.lH1()[i] = bb.c0_lb; s.uH1()[i] = bb.c0_ub;
        s.lH3()[i] = bb.c2_lb; s.uH3()[i] = bb.c2_ub;
        s.uS4m()[i] = bb.c3_ub - pm.margin; s.lS4p()[i] = bb.c3_lb + pm.margin;
        s.uS2m()[i] = bb.c1_ub - pm.margin; s.lS2p()[i] = bb.c1_lb + pm.margin;
        if (!(bb.c0_lb <= bb.c0_ub) || !(bb.c2_lb <= bb.c2_ub)) invalid = 1;
        // one-sided rows: -1e30 <= u and l <= 1e30 must hold too (NaN guard)
        if (!(-kOsqpInfty <= s.uS4m()[i]) || !(s.lS4p()[i] <= kOsqpInfty) || !(-kOsqpInfty <= s.uS2m()[i]) ||
            !(s.lS2p()[i] <= kOsqpInfty))
            invalid = 1;
    }
    if (!(0.0 <= pm.margin) || !(-pm.kmax <= pm.kmax) || !(cx.lEH <= cx.uEH)) invalid = 1;
    invalid = w.any(invalid);
    w.sync();

    int status = PQP_UNSOLVED;
    int iter = 0;
    if (invalid) {
        status = PQP_INVALID_PROBLEM;
    } else {
        kp_scale(w, cx);
        // cold start (x = z = y = 0).  OSQP's first iteration from zero has rhs = 0, hence
        // xt = 0, x = 0, v = 0 (z = clamp(0), w = -clamp(0)): it is accounted for as iter = 1.
        for (int g = lane; g < d.nred; g += 32) s.xr()[g] = 0.0;
        for (int i = lane; i < N; i += 32) {
            s.xs()[i] = 0.0;
            s.vD()[i] = s.vD()[N + i] = s.vD()[2 * N + i] = 0.0;
            s.vKB()[i] = s.vSB()[i] = s.vH1()[i] = s.vH3()[i] = 0.0;
            s.vS4m()[i] = s.vS4p()[i] = s.vS2m()[i] = s.vS2p()[i] = 0.0;
        }
        for (int j = lane; j < ch; j += 32) s.vUB()[j] = 0.0;
        if (lane == 0) s.vEnd()[0] = s.vEnd()[1] = 0.0;
        cx.rho = fmin(fmax(pm.rho, kRhoMin), kRhoMax);
        w.sync();
        // a slack pair whose rows fall in different rho classes is refused (see pqp_kp_core3.cuh, pqp.h)
        int split = 0;
        for (int i = lane; i < N; i += 32)
            if (kp_w_box(s.ES4()[i], -kOsqpInfty, s.uS4m()[i], 1.0) != kp_w_box(s.ES4()[i], s.lS4p()[i], kOsqpInfty, 1.0) ||
                kp_w_box(s.ES2()[i], -kOsqpInfty, s.uS2m()[i], 1.0) != kp_w_box(s.ES2()[i], s.lS2p()[i], kOsqpInfty, 1.0))
                split = 1;
        if (w.any(split)) status = PQP_INVALID_PROBLEM;
        else if (!kp_factor(w, cx)) status = PQP_NON_CVX;
        const double alpha = pm.alpha;
        Residuals res{};   // of the last check
        // (without a workspace -- test harnesses of this core alone -- infeasibility is not detected)
        double *wold = bv.workspace ? kp_ws_wold(kp_ws_base(bv.workspace, off, prob), N) : nullptr;
        iter = 0;
        while (status == PQP_UNSOLVED && iter < pm.max_iter) {
            ++iter;
            const double rho = cx.rho;
            // iterations that end in a termination check first park w = v - clamp(v): the check needs
            // delta_y = W (w_new - w_old) (OSQP update_y / is_primal_infeasible)
            const bool chk = wold && ((pm.check_termination && (iter % pm.check_termination == 0)) || iter == pm.max_iter);
            if (iter == 1) {
                // OSQP's first iteration from x = z = y = 0 ends at the cold start (x = 0, v = 0: z = clamp(0),
                // y = -rho clamp(0)).  Its check and rho adaptation still run in (d), on w_old = y_0 / rho = 0.
                if (chk) for (int k = lane; k < 11 * N + 2; k += 32) wold[k] = 0.0;
                w.sync();
            } else {
                // ---- (a) rhs = sigma_v x + A' W (2 clamp(v) - v)
                for (int i = lane; i < N; i += 32) {
                    const KpRowW W = kp_row_weights(cx, i, rho);
                    double b0, b1, b2;
                    kp_dyn_bounds(cx, i, b0, b1, b2);
                    s.gD()[i] = W.D0 * (2.0 * b0 - s.vD()[i]);
                    s.gD()[N + i] = W.D1 * (2.0 * b1 - s.vD()[N + i]);
                    s.gD()[2 * N + i] = W.D2 * (2.0 * b2 - s.vD()[2 * N + i]);
                }
                w.sync();
                for (int i = lane; i < N; i += 32) {
                    const KpRowW W = kp_row_weights(cx, i, rho);
                    KpRows g;
                    g.D0 = s.gD()[i]; g.D1 = s.gD()[N + i]; g.D2 = s.gD()[2 * N + i];
                    double v;
                    v = s.vKB()[i]; g.KB = W.KB * (2.0 * clampd(v, -pm.kmax, pm.kmax) - v);
                    v = s.vSB()[i]; g.SB = W.SB * (2.0 * clampd(v, 0.0, pm.margin) - v);
                    v = s.vH1()[i]; g.H1 = W.H1 * (2.0 * clampd(v, s.lH1()[i], s.uH1()[i]) - v);
                    v = s.vH3()[i]; g.H3 = W.H3 * (2.0 * clampd(v, s.lH3()[i], s.uH3()[i]) - v);
                    v = s.vS4m()[i]; g.S4m = W.S4 * (2.0 * clampd(v, -kOsqpInfty, s.uS4m()[i]) - v);
                    v = s.vS4p()[i]; g.S4p = W.S4 * (2.0 * clampd(v, s.lS4p()[i], kOsqpInfty) - v);
                    v = s.vS2m()[i]; g.S2m = W.S2 * (2.0 * clampd(v, -kOsqpInfty, s.uS2m()[i]) - v);
                    v = s.vS2p()[i]; g.S2p = W.S2 * (2.0 * clampd(v, s.lS2p()[i], kOsqpInfty) - v);
                    double gEY = 0, gEH = 0;
                    if (i == N - 1) {
                        v = s.vEnd()[0]; gEY = kp_w_ey(cx, rho) * (2.0 * clampd(v, -1.0, 1.0) - v);
                        v = s.vEnd()[1]; gEH = kp_w_eh(cx, rho) * (2.0 * clampd(v, cx.lEH, cx.uEH) - v);
                    }
                    double ra, rb, rc, rs;
                    kp_apply_At(cx, i, g, gEY, gEH, ra, rb, rc, rs);
                    const int ga = kp_gx(d, i);
                    s.tr()[ga] = s.sgr()[ga] * s.xr()[ga] + ra;
                    s.tr()[ga + 1] = s.sgr()[ga + 1] * s.xr()[ga + 1] + rb;
                    s.tr()[ga + 2] = s.sgr()[ga + 2] * s.xr()[ga + 2] + rc;
                    s.ts()[i] = s.sgs()[i] * s.xs()[i] + rs;
                }
                for (int j = lane; j < ch; j += 32) {
                    const int gu = kp_gu(d, j);
                    const double v = s.vUB()[j];
                    double acc = s.sgr()[gu] * s.xr()[gu] +
                                 kp_w_ub(cx, j, rho) * (2.0 * clampd(v, -kOsqpInfty, kOsqpInfty) - v);
                    int t1 = j * d.keep + d.keep - 1;
                    if (t1 > N - 2) t1 = N - 2;
                    for (int t = j * d.keep; t <= t1; ++t) acc += s.ds()[t] * s.gD()[2 * N + t + 1];
                    s.tr()[gu] = acc;
                }
                w.sync();
                // ---- (b) reduced KKT solve
                kp_solve(w, cx);
                if (chk) {
                    for (int i = lane; i < N; i += 32) {
                        double b0, b1, b2, v;
                        kp_dyn_bounds(cx, i, b0, b1, b2);
                        double *wo = wold + i;
                        wo[0] = s.vD()[i] - b0; wo[N] = s.vD()[N + i] - b1; wo[2 * N] = s.vD()[2 * N + i] - b2;
                        v = s.vKB()[i]; wo[3 * N] = v - clampd(v, -pm.kmax, pm.kmax);
                        v = s.vSB()[i]; wo[4 * N] = v - clampd(v, 0.0, pm.margin);
                        v = s.vH1()[i]; wo[5 * N] = v - clampd(v, s.lH1()[i], s.uH1()[i]);
                        v = s.vH3()[i]; wo[6 * N] = v - clampd(v, s.lH3()[i], s.uH3()[i]);
                        v = s.vS4m()[i]; wo[7 * N] = v - clampd(v, -kOsqpInfty, s.uS4m()[i]);
                        v = s.vS4p()[i]; wo[8 * N] = v - clampd(v, s.lS4p()[i], kOsqpInfty);
                        v = s.vS2m()[i]; wo[9 * N] = v - clampd(v, -kOsqpInfty, s.uS2m()[i]);
                        v = s.vS2p()[i]; wo[10 * N] = v - clampd(v, s.lS2p()[i], kOsqpInfty);
                        if (i == N - 1) {
                            v = s.vEnd()[0]; wold[11 * N] = v - clampd(v, -1.0, 1.0);
                            v = s.vEnd()[1]; wold[11 * N + 1] = v - clampd(v, cx.lEH, cx.uEH);
                        }
                    }
                }
                // ---- (c) v += alpha (A xt - clamp(v)),  x = alpha xt + (1 - alpha) x
                for (int i = lane; i < N; i += 32) {
                    const KpRows zt = kp_apply_A(cx, i, s.tr(), s.ts());
                    double b0, b1, b2, v;
                    kp_dyn_bounds(cx, i, b0, b1, b2);
                    s.vD()[i] += alpha * (zt.D0 - b0);
                    s.vD()[N + i] += alpha * (zt.D1 - b1);
                    s.vD()[2 * N + i] += alpha * (zt.D2 - b2);
                    v = s.vKB()[i]; s.vKB()[i] = v + alpha * (zt.KB - clampd(v, -pm.kmax, pm.kmax));
                    v = s.vSB()[i]; s.vSB()[i] = v + alpha * (zt.SB - clampd(v, 0.0, pm.margin));
                    v = s.vH1()[i]; s.vH1()[i] = v + alpha * (zt.H1 - clampd(v, s.lH1()[i], s.uH1()[i]));
                    v = s.vH3()[i]; s.vH3()[i] = v + alpha * (zt.H3 - clampd(v, s.lH3()[i], s.uH3()[i]));
                    v = s.vS4m()[i]; s.vS4m()[i] = v + alpha * (zt.S4m - clampd(v, -kOsqpInfty, s.uS4m()[i]));
                    v = s.vS4p()[i]; s.vS4p()[i] = v + alpha * (zt.S4p - clampd(v, s.lS4p()[i], kOsqpInfty));
                    v = s.vS2m()[i]; s.vS2m()[i] = v + alpha * (zt.S2m - clampd(v, -kOsqpInfty, s.uS2m()[i]));
                    v = s.vS2p()[i]; s.vS2p()[i] = v + alpha * (zt.S2p - clampd(v, s.lS2p()[i], kOsqpInfty));
                    if (i == N - 1) {
                        const int ga = kp_gx(d, i);
                        v = s.vEnd()[0]; s.vEnd()[0] = v + alpha * (s.tr()[ga] - clampd(v, -1.0, 1.0));
                        v = s.vEnd()[1]; s.vEnd()[1] = v + alpha * (s.tr()[ga + 1] - clampd(v, cx.lEH, cx.uEH));
                    }
                }
                for (int j = lane; j < ch; j += 32) {
                    const double v = s.vUB()[j];
                    s.vUB()[j] = v + alpha * (s.tr()[kp_gu(d, j)] - clampd(v, -kOsqpInfty, kOsqpInfty));
                }
                w.sync();
                for (int g = lane; g < d.nred; g += 32) s.xr()[g] = alpha * s.tr()[g] + (1.0 - alpha) * s.xr()[g];
                for (int i = lane; i < N; i += 32) s.xs()[i] = alpha * s.ts()[i] + (1.0 - alpha) * s.xs()[i];
                w.sync();
            }
            // ---- (d) residuals, termination, adaptive rho
            const bool can_check = pm.check_termination && (iter % pm.check_termination == 0);
            const bool can_adapt = pm.adaptive_rho && pm.adaptive_rho_interval &&
                                   (iter % pm.adaptive_rho_interval == 0);
            if (can_check || can_adapt || iter == pm.max_iter) {
                // primal side: r = A x - z with z = clamp(v); unscaled dual y = W w / c, w = v - z.
                // Pass 1 accumulates the primal norms and publishes the dynamics-row duals (the only
                // duals a neighbouring station needs); pass 2 recomputes the station-local duals.
                double pr = 0, nz = 0, nax = 0, prs = 0, nzs = 0, naxs = 0;
                const double cinv = 1.0 / cx.c;
#define PQP_ROW(AX, V, LO, HI, EE)                                                   \
    {                                                                                \
        const double ax_ = (AX), v_ = (V), z_ = clampd(v_, (LO), (HI)), r_ = ax_ - z_; \
        const double e_ = (EE);                                                      \
        pr = fmax(pr, fabs(r_)); nz = fmax(nz, fabs(z_)); nax = fmax(nax, fabs(ax_)); \
        prs = fmax(prs, e_ * fabs(r_)); nzs = fmax(nzs, e_ * fabs(z_));              \
        naxs = fmax(naxs, e_ * fabs(ax_));                                           \
    }
#define PQP_DUAL(V, LO, HI, WW) ((WW) * ((V) - clampd((V), (LO), (HI))) * cinv)
                for (int i = lane; i < N; i += 32) {
                    const KpRowW W = kp_row_weights(cx, i, rho);
                    const KpRows ax = kp_apply_A(cx, i, s.xr(), s.xs());
                    double b0, b1, b2;
                    kp_dyn_bounds(cx, i, b0, b1, b2);
                    PQP_ROW(ax.D0, s.vD()[i], b0, b0, s.ED()[i])
                    PQP_ROW(ax.D1, s.vD()[N + i], b1, b1, s.ED()[N + i])
                    PQP_ROW(ax.D2, s.vD()[2 * N + i], b2, b2, s.ED()[2 * N + i])
                    PQP_ROW(ax.KB, s.vKB()[i], -pm.kmax, pm.kmax, s.EKB()[i])
                    PQP_ROW(ax.SB, s.vSB()[i], 0.0, pm.margin, s.ESB()[i])
                    PQP_ROW(ax.H1, s.vH1()[i], s.lH1()[i], s.uH1()[i], s.EH1()[i])
                    PQP_ROW(ax.H3, s.vH3()[i], s.lH3()[i], s.uH3()[i], s.EH3()[i])
                    PQP_ROW(ax.S4m, s.vS4m()[i], -kOsqpInfty, s.uS4m()[i], s.ES4()[i])
                    PQP_ROW(ax.S4p, s.vS4p()[i], s.lS4p()[i], kOsqpInfty, s.ES4()[i])
                    PQP_ROW(ax.S2m, s.vS2m()[i], -kOsqpInfty, s.uS2m()[i], s.ES2()[i])
                    PQP_ROW(ax.S2p, s.vS2p()[i], s.lS2p()[i], kOsqpInfty, s.ES2()[i])
                    s.gD()[i] = PQP_DUAL(s.vD()[i], b0, b0, W.D0);
                    s.gD()[N + i] = PQP_DUAL(s.vD()[N + i], b1, b1, W.D1);
                    s.gD()[2 * N + i] = PQP_DUAL(s.vD()[2 * N + i], b2, b2, W.D2);
                    if (i == N - 1) {
                        const int ga = kp_gx(d, i);
                        PQP_ROW(s.xr()[ga], s.vEnd()[0], -1.0, 1.0, s.EEnd()[0])
                        PQP_ROW(s.xr()[ga + 1], s.vEnd()[1], cx.lEH, cx.uEH, s.EEnd()[1])
                    }
                }
                for (int j = lane; j < ch; j += 32)
                    PQP_ROW(s.xr()[kp_gu(d, j)], s.vUB()[j], -kOsqpInfty, kOsqpInfty, s.EUB()[j])
                w.sync();
                // dual side: (P x + A' y)_v per variable; P is diagonal
                double dr = 0, npx = 0, naty = 0, drs = 0, npxs = 0, natys = 0;
                const double cc = cx.c;
#define PQP_VAR(PX, ATY, DD)                                                          \
    {                                                                                 \
        const double px_ = (PX), aty_ = (ATY), r_ = px_ + aty_, cd_ = cc * (DD);      \
        dr = fmax(dr, fabs(r_)); npx = fmax(npx, fabs(px_)); naty = fmax(naty, fabs(aty_)); \
        drs = fmax(drs, cd_ * fabs(r_)); npxs = fmax(npxs, cd_ * fabs(px_));          \
        natys = fmax(natys, cd_ * fabs(aty_));                                        \
    }
                for (int i = lane; i < N; i += 32) {
                    const int ga = kp_gx(d, i);
                    const KpRowW W = kp_row_weights(cx, i, rho);
                    KpRows y;
                    y.D0 = s.gD()[i]; y.D1 = s.gD()[N + i]; y.D2 = s.gD()[2 * N + i];
                    y.KB = PQP_DUAL(s.vKB()[i], -pm.kmax, pm.kmax, W.KB);
                    y.SB = PQP_DUAL(s.vSB()[i], 0.0, pm.margin, W.SB);
                    y.H1 = PQP_DUAL(s.vH1()[i], s.lH1()[i], s.uH1()[i], W.H1);
                    y.H3 = PQP_DUAL(s.vH3()[i], s.lH3()[i], s.uH3()[i], W.H3);
                    y.S4m = PQP_DUAL(s.vS4m()[i], -kOsqpInfty, s.uS4m()[i], W.S4);
                    y.S4p = PQP_DUAL(s.vS4p()[i], s.lS4p()[i], kOsqpInfty, W.S4);
                    y.S2m = PQP_DUAL(s.vS2m()[i], -kOsqpInfty, s.uS2m()[i], W.S2);
                    y.S2p = PQP_DUAL(s.vS2p()[i], s.lS2p()[i], kOsqpInfty, W.S2);
                    double yEY = 0, yEH = 0;
                    if (i == N - 1) {
                        yEY = PQP_DUAL(s.vEnd()[0], -1.0, 1.0, kp_w_ey(cx, rho));
                        yEH = PQP_DUAL(s.vEnd()[1], cx.lEH, cx.uEH, kp_w_eh(cx, rho));
                    }
                    double ra, rb, rc, rs;
                    kp_apply_At(cx, i, y, yEY, yEH, ra, rb, rc, rs);
                    PQP_VAR(pm.w_pq * s.xr()[ga], ra, s.Dr()[ga])
                    PQP_VAR(0.0, rb, s.Dr()[ga + 1])
                    PQP_VAR(pm.w_c * s.xr()[ga + 2], rc, s.Dr()[ga + 2])
                    PQP_VAR(pm.w_s * s.xs()[i], rs, s.Dsl()[i])
                }
                for (int j = lane; j < ch; j += 32) {
                    const int gu = kp_gu(d, j);
                    double aty = PQP_DUAL(s.vUB()[j], -kOsqpInfty, kOsqpInfty, kp_w_ub(cx, j, rho));
                    int t1 = j * d.keep + d.keep - 1;
                    if (t1 > N - 2) t1 = N - 2;
                    for (int t = j * d.keep; t <= t1; ++t) aty += s.ds()[t] * s.gD()[2 * N + t + 1];
                    PQP_VAR((d.keep * pm.w_cr) * s.xr()[gu], aty, s.Dr()[gu])
                }
#undef PQP_ROW
#undef PQP_DUAL
#undef PQP_VAR
                // ---- primal-infeasibility certificate (OSQP is_primal_infeasible) in unscaled terms:
                // g = W (w_new - w_old) = E delta_y projected on the cone of the finite bounds;
                // ||g||_inf, u'g+ + l'g-, ||A'g||_inf.  The control rows are free (g = 0).
                if (chk) {
                    double c_nrm = 0, c_lhs = 0, c_cert = 0;
#define PQP_G(V, LO, HI, WW, WO) ((WW) * (((V) - clampd((V), (LO), (HI))) - (WO)))
#define PQP_ACC(G, LO, HI) { const double g_ = (G); c_nrm = fmax(c_nrm, fabs(g_)); c_lhs += (HI) * fmax(g_, 0.0) + (LO) * fmin(g_, 0.0); }
                    w.sync();   // the dual-residual pass has consumed gD
                    for (int i = lane; i < N; i += 32) {
                        const KpRowW W = kp_row_weights(cx, i, rho);
                        double b0, b1, b2;
                        kp_dyn_bounds(cx, i, b0, b1, b2);
                        const double *wo = wold + i;
                        s.gD()[i] = W.D0 * ((s.vD()[i] - b0) - wo[0]);
                        s.gD()[N + i] = W.D1 * ((s.vD()[N + i] - b1) - wo[N]);
                        s.gD()[2 * N + i] = W.D2 * ((s.vD()[2 * N + i] - b2) - wo[2 * N]);
                    }
                    w.sync();
                    for (int i = lane; i < N; i += 32) {
                        const KpRowW W = kp_row_weights(cx, i, rho);
                        double b0, b1, b2;
                        kp_dyn_bounds(cx, i, b0, b1, b2);
                        const double *wo = wold + i;
                        KpRows g;
                        g.D0 = s.gD()[i]; g.D1 = s.gD()[N + i]; g.D2 = s.gD()[2 * N + i];
                        g.KB = PQP_G(s.vKB()[i], -pm.kmax, pm.kmax, W.KB, wo[3 * N]);
                        g.SB = PQP_G(s.vSB()[i], 0.0, pm.margin, W.SB, wo[4 * N]);
                        g.H1 = PQP_G(s.vH1()[i], s.lH1()[i], s.uH1()[i], W.H1, wo[5 * N]);
                        g.H3 = PQP_G(s.vH3()[i], s.lH3()[i], s.uH3()[i], W.H3, wo[6 * N]);
                        // one-sided rows: l = -inf keeps the positive part, u = +inf the negative part
                        g.S4m = fmax(PQP_G(s.vS4m()[i], -kOsqpInfty, s.uS4m()[i], W.S4, wo[7 * N]), 0.0);
                        g.S4p = fmin(PQP_G(s.vS4p()[i], s.lS4p()[i], kOsqpInfty, W.S4, wo[8 * N]), 0.0);
                        g.S2m = fmax(PQP_G(s.vS2m()[i], -kOsqpInfty, s.uS2m()[i], W.S2, wo[9 * N]), 0.0);
                        g.S2p = fmin(PQP_G(s.vS2p()[i], s.lS2p()[i], kOsqpInfty, W.S2, wo[10 * N]), 0.0);
                        PQP_ACC(g.D0, b0, b0) PQP_ACC(g.D1, b1, b1) PQP_ACC(g.D2, b2, b2)
                        PQP_ACC(g.KB, -pm.kmax, pm.kmax) PQP_ACC(g.SB, 0.0, pm.margin)
                        PQP_ACC(g.H1, s.lH1()[i], s.uH1()[i]) PQP_ACC(g.H3, s.lH3()[i], s.uH3()[i])
                        PQP_ACC(g.S4m, 0.0, s.uS4m()[i]) PQP_ACC(g.S4p, s.lS4p()[i], 0.0)
                        PQP_ACC(g.S2m, 0.0, s.uS2m()[i]) PQP_ACC(g.S2p, s.lS2p()[i], 0.0)
                        double gEY = 0, gEH = 0;
                        if (i == N - 1) {
                            gEY = PQP_G(s.vEnd()[0], -1.0, 1.0, kp_w_ey(cx, rho), wold[11 * N]);
                            gEH = PQP_G(s.vEnd()[1], cx.lEH, cx.uEH, kp_w_eh(cx, rho), wold[11 * N + 1]);
                            if (cx.uEH >= kOsqpInfty) gEH = (cx.lEH <= -kOsqpInfty) ? 0.0 : fmin(gEH, 0.0);
                            else if (cx.lEH <= -kOsqpInfty) gEH = fmax(gEH, 0.0);
                            PQP_ACC(gEY, -1.0, 1.0)
                            PQP_ACC(gEH, (cx.lEH <= -kOsqpInfty ? 0.0 : cx.lEH), (cx.uEH >= kOsqpInfty ? 0.0 : cx.uEH))
                        }
                        double ra, rb, rc, rs;
                        kp_apply_At(cx, i, g, gEY, gEH, ra, rb, rc, rs);
                        c_cert = fmax(c_cert, fmax(fmax(fabs(ra), fabs(rb)), fmax(fabs(rc), fabs(rs))));
                    }
                    for (int j = lane; j < ch; j += 32) {
                        double aty = 0.0;
                        int t1 = j * d.keep + d.keep - 1;
                        if (t1 > N - 2) t1 = N - 2;
                        for (int t = j * d.keep; t <= t1; ++t) aty += s.ds()[t] * s.gD()[2 * N + t + 1];
                        c_cert = fmax(c_cert, fabs(aty));
                    }
#undef PQP_G
#undef PQP_ACC
                    res.inf_nrm = w.max(c_nrm); res.inf_cert = w.max(c_cert); res.inf_lhs = w.sum(c_lhs);
                }
                pr = w.max(pr); nz = w.max(nz); nax = w.max(nax);
                prs = w.max(prs); nzs = w.max(nzs); naxs = w.max(naxs);
                dr = w.max(dr); npx = w.max(npx); naty = w.max(naty);
                drs = w.max(drs); npxs = w.max(npxs); natys = w.max(natys);
                w.sync();
                res.pri_res = pr; res.dua_res = dr;
                res.pri_nrm = fmax(nz, nax); res.dua_nrm = fmax(npx, naty);
                if (can_check || iter == pm.max_iter) status = termination_verdict(pm, res);
                if (status == PQP_UNSOLVED && can_adapt) {
                    const double rho_new = rho_estimate(rho, prs, drs, fmax(nzs, naxs), fmax(npxs, natys));
                    if (rho_changed(pm, rho_new, rho)) {
                        // y is kept, rho changes: w = E^-1 y / rho_row scales by rho/rho_new on every
                        // row whose rho follows the setting (free rows have w = 0).
                        const double ratio = rho / rho_new;
                        for (int i = lane; i < N; i += 32) {
                            double b0, b1, b2, v, z;
                            kp_dyn_bounds(cx, i, b0, b1, b2);
                            s.vD()[i] = b0 + (s.vD()[i] - b0) * ratio;
                            s.vD()[N + i] = b1 + (s.vD()[N + i] - b1) * ratio;
                            s.vD()[2 * N + i] = b2 + (s.vD()[2 * N + i] - b2) * ratio;
#define PQP_RESC(V, LO, HI) v = (V); z = clampd(v, (LO), (HI)); (V) = z + (v - z) * ratio;
                            PQP_RESC(s.vKB()[i], -pm.kmax, pm.kmax)
                            PQP_RESC(s.vSB()[i], 0.0, pm.margin)
                            PQP_RESC(s.vH1()[i], s.lH1()[i], s.uH1()[i])
                            PQP_RESC(s.vH3()[i], s.lH3()[i], s.uH3()[i])
                            PQP_RESC(s.vS4m()[i], -kOsqpInfty, s.uS4m()[i])
                            PQP_RESC(s.vS4p()[i], s.lS4p()[i], kOsqpInfty)
                            PQP_RESC(s.vS2m()[i], -kOsqpInfty, s.uS2m()[i])
                            PQP_RESC(s.vS2p()[i], s.lS2p()[i], kOsqpInfty)
                            if (i == N - 1) {
                                PQP_RESC(s.vEnd()[0], -1.0, 1.0)
                                PQP_RESC(s.vEnd()[1], cx.lEH, cx.uEH)
                            }
#undef PQP_RESC
                        }
                        cx.rho = rho_new;
                        w.sync();
                        if (!kp_factor(w, cx)) status = PQP_NON_CVX;
                    }
                }
            }
        }
        if (status == PQP_UNSOLVED) status = max_iter_verdict(pm, res);
    }
    // ---- epilogue: getOptimizedPath, solver_kp_as_input.cpp:26-43
    const bool has_sol = has_solution(status);
    const double nanv = nan("");
    for (int i = lane; i < N; i += 32) {
        double ey = nanv, ephi = nanv, kk = nanv, tx, ty;
        if (has_sol) {
            const int ga = kp_gx(d, i);
            ey = s.xr()[ga]; ephi = s.xr()[ga + 1]; kk = s.xr()[ga + 2];
        }
        optimized_station(ref[i], ey, ephi, kk, out[i], tx, ty);
        s.tr()[i] = tx;        // (tr/ts are free now)
        s.tmp()[i] = ty;
        store_frenet(bv.out_frenet, off + i, ey, ephi, kk);
    }
    w.sync();
    for (int i = lane; i < N; i += 32) {
        double seg = 0.0;
        if (i > 0) {
            const double dx = s.tr()[i] - s.tr()[i - 1], dy = s.tmp()[i] - s.tmp()[i - 1];
            seg = sqrt(dx * dx + dy * dy);
        }
        s.ts()[i] = seg;
    }
    w.sync();
    if (lane == 0) {
        double acc = 0.0;  // sequential, same association order as the reference's running sum
        for (int i = 0; i < N; ++i) {
            acc += s.ts()[i];
            out[i].s = acc;
        }
        bv.status[prob] = status;
        if (bv.iters) bv.iters[prob] = iter;
    }
    w.sync();
}

#undef PQP_B
}  // namespace pqp
