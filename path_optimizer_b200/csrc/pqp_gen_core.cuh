// pqp_gen_core.cuh -- generic banded path-QP kernel: one warp solves one QP given as sparse data in
// BAND ORDER.  It serves the formulations that have no hand-specialised kernel yet:
//   "K"   SolverKAsInput               reference src/solver/solver_k_as_input.cpp:14-207
//   "KPC" SolverKpAsInputConstrained   reference src/solver/solver_kp_as_input_constrained.cpp:13-221
// The host (pqp_forms.h) restates the reference's setHessianMatrix / setConstraintMatrix as sparse
// rows (<= 4 entries per row, as every row of these formulations has), orders the unknowns station
// by station so that the reduced KKT  cP + sigma D^-2 + A' W A  is banded, and marks S-unknown
// separators (one station's unknowns) every L stations: S = 3 for "K" and "KPC", S = 4 for the TENSION2
// smoothing QP of pqp_smooth_reference_device, whose four chains x, y, theta, k admit no 3-unknown separator, and
// S = 9 (three stations) for the TENSION smoothing QP of pqp_smooth_reference_tension_device, whose reduced KKT has
// half-bandwidth 9 in the band order (x_i, y_i, d_i) and whose P records six partners per unknown (NP = 6).
// The TENSION2 QP also has a linear cost term q (kLinear); the others have q = 0.  The device part is formulation-agnostic:
// OSQP's Ruiz scaling / rho classes / ADMM recurrence / termination / adaptive rho exactly as in
// pqp_kp_core.cuh (same unscaled-weighted form, same partitioned banded LDL'), with the stencils
// replaced by ELL row gathers and CSC column gathers.
#pragma once
#include "pqp_kp_core.cuh"

namespace pqp {

constexpr int kGenMeta = 16;
// meta[b]: 0 n (unknowns, band order)  1 m (rows)  2 n_den (n + dead variables: denominator of OSQP's
//          cost-scaling mean)  3 bw  4 M (separators)  5 N (stations)  6 station offset
//          7 offset into n-arrays  8 offset into m-arrays  9 offset into CSC entry arrays
//          10 offset into csc_ptr (= offn + b)
struct GenView {
    int batch;
    const int32_t *meta;
    const int32_t *A_col;    // [sum m][4], -1 = empty
    const double *A_val;     // [sum m][4]
    const double *l, *u;     // [sum m]
    const double *Pd;        // [sum n] diagonal of P
    const int32_t *Po_idx;   // [sum n][NP] band position of an off-diagonal partner, -1 = none (NP: gen_solve_qp)
    const double *Po_val;    // [sum n][NP]
    const int32_t *csc_ptr;  // [sum (n+1)]
    const int32_t *csc_row;  // [sum nnz]
    const double *csc_val;   // [sum nnz]
    const int32_t *sep;      // [B][32] band position of separator p
    const int32_t *out_idx;  // [sum N][3] band positions of (e_y, e_phi, k) of each station
    const pqp_state *ref;    // [sum N]
    pqp_state *out_states;   // [sum N]
    double *out_frenet;      // [sum N][3] or nullptr
    int32_t *status, *iters; // [B]
};

// Per-lane reduction record of an S-wide separator: [0, S^2) Dg / Sinv (S = 3) or its LDL' factors (S > 3), [S^2, 2S^2) Off, [2S^2, 3S^2) G,
// [3S^2, 4S^2) A, [4S^2, 5S^2) C, [5S^2, 5S^2 + S) g.  S = 3 gives kRedStride.
template <int S> constexpr int kGenRedStride = 5 * S * S + S;
static_assert(kGenRedStride<3> == kRedStride, "width-3 record");

template <int S = 3>
PQP_HD size_t gen_smem_doubles(int n, int m, int bw) {
    return 5 * (size_t)n + 4 * (size_t)m + (size_t)(bw + 1) * n + (size_t)kGenRedStride<S> * 32;
}

// LDL' of an SPD S x S block a (row-major) into f: the unit lower factor below the diagonal, 1 / d on it.  The width-4
// separator chain keeps these factors and solves with them: an explicit inverse of its Schur blocks, which are far worse
// conditioned than the QP's KKT system when the cost scaling c is small (UTM-sized coordinates, a large deviation
// weight), loses up to all digits of the x-step there (DESIGN.md §9).
template <int S> PQP_DEV void gen_ldl_spd(const double *a, double *f) {
    double d[S];
    for (int j = 0; j < S; ++j) {
        double dj = a[j * S + j];
        for (int k = 0; k < j; ++k) dj -= f[j * S + k] * f[j * S + k] * d[k];
        d[j] = dj;
        const double rj = 1.0 / dj;
        f[j * S + j] = rj;
        for (int i = j + 1; i < S; ++i) {
            double v = a[i * S + j];
            for (int k = 0; k < j; ++k) v -= f[i * S + k] * f[j * S + k] * d[k];
            f[i * S + j] = v * rj;
        }
    }
}
// x = (L D L')^-1 b for the factors of gen_ldl_spd (x may alias b).
template <int S> PQP_DEV void gen_ldl_solve(const double *f, const double *b, double *x) {
    double y[S];
    for (int i = 0; i < S; ++i) {
        double v = b[i];
        for (int k = 0; k < i; ++k) v -= f[i * S + k] * y[k];
        y[i] = v;
    }
    for (int i = 0; i < S; ++i) y[i] *= f[i * S + i];
    for (int i = S - 1; i >= 0; --i) {
        double v = y[i];
        for (int k = i + 1; k < S; ++k) v -= f[k * S + i] * x[k];
        x[i] = v;
    }
}

struct GenCtx {
    int n, m, bw, M;
    double *D, *xr, *tr, *tmp, *sg, *v, *E, *W, *wold, *band, *red;
    const int32_t *A_col, *csc_ptr, *csc_row, *sep, *Po_idx;
    const double *A_val, *l, *u, *Pd, *Po_val, *csc_val;
    int lo, hi, gsep;
};

#define PQP_GB(g, dd) cx.band[(size_t)(g) * (cx.bw + 1) + (dd)]

// a[0] b[0] + a[1] b[1] + ... in that order (S = 3: the expression the width-3 core always had)
template <int S> PQP_DEV double gen_dot(const double *a, const double *b) {
    if constexpr (S == 3) {
        return a[0] * b[0] + a[1] * b[1] + a[2] * b[2];
    } else {
        double acc = a[0] * b[0];
        for (int k = 1; k < S; ++k) acc += a[k] * b[k];
        return acc;
    }
}

PQP_DEV int gen_local_factor(const GenCtx &cx, int lo, int hi) {
    const int bw = cx.bw;
    int ok = 1;
    for (int j = lo; j < hi; ++j) {
        const double dj = PQP_GB(j, 0);
        if (!(dj > 0.0)) ok = 0;
        const double dinv = 1.0 / dj;
        int R = hi - 1 - j;
        if (R > bw) R = bw;
        for (int r = 1; r <= R; ++r) {
            const double kr = PQP_GB(j + r, r);
            for (int cc = 1; cc <= r; ++cc) PQP_GB(j + r, r - cc) -= kr * (PQP_GB(j + cc, cc) * dinv);
        }
        for (int r = 1; r <= R; ++r) PQP_GB(j + r, r) *= dinv;
        PQP_GB(j, 0) = dinv;
    }
    return ok;
}
PQP_DEV void gen_local_solve(const GenCtx &cx, double *v, int lo, int hi) {
    const int bw = cx.bw;
    for (int g = lo; g < hi; ++g) {
        double acc = v[g];
        int dm = g - lo;
        if (dm > bw) dm = bw;
        for (int dd = 1; dd <= dm; ++dd) acc -= PQP_GB(g, dd) * v[g - dd];
        v[g] = acc;
    }
    for (int g = hi - 1; g >= lo; --g) {
        double acc = v[g] * PQP_GB(g, 0);
        int dm = hi - 1 - g;
        if (dm > bw) dm = bw;
        for (int dd = 1; dd <= dm; ++dd) acc -= PQP_GB(g + dd, dd) * v[g + dd];
        v[g] = acc;
    }
}

// band assembly (one thread per band row, deterministic) + partitioned factorisation
template <int S, int NP>
PQP_DEV int gen_factor(Warp &w, GenCtx &cx, double cost_c) {
    constexpr int RS = kGenRedStride<S>, S2 = S * S;
    const int n = cx.n, bw = cx.bw, lane = w.lane();
    for (int j = lane; j < n; j += 32) {
        for (int dd = 0; dd <= bw; ++dd) PQP_GB(j, dd) = 0.0;
        double dg = cost_c * cx.Pd[j] + cx.sg[j];
        for (int q = 0; q < NP; ++q) {
            const int k = cx.Po_idx[NP * j + q];
            if (k >= 0 && k < j) PQP_GB(j, j - k) += cost_c * cx.Po_val[NP * j + q];
        }
        for (int e = cx.csc_ptr[j]; e < cx.csc_ptr[j + 1]; ++e) {
            const int r = cx.csc_row[e];
            const double wa = cx.W[r] * cx.csc_val[e];
            dg += wa * cx.csc_val[e];
            for (int t = 0; t < 4; ++t) {
                const int k = cx.A_col[4 * r + t];
                if (k >= 0 && k < j) PQP_GB(j, j - k) += wa * cx.A_val[4 * r + t];
            }
        }
        PQP_GB(j, 0) = dg;
    }
    w.sync();
    int ok = 1;
    const bool act = lane < cx.M;
    double *R = cx.red + (size_t)RS * lane;
    if (act) ok = gen_local_factor(cx, cx.lo, cx.hi);
    w.sync();
    if (act) {
        const int lo = cx.lo, hi = cx.hi, gs = cx.gsep, gq = hi;
        const bool has_right = (lane + 1 < cx.M);
        for (int k = S2; k < 2 * S2; ++k) R[k] = 0.0;
        for (int k = 3 * S2; k < 5 * S2; ++k) R[k] = 0.0;
        for (int col = 0; col < 2 * S; ++col) {
            const bool left = col < S;
            if (!left && !has_right) break;
            const int sc = left ? gs + col : gq + (col - S);
            for (int g = lo; g < hi; ++g) {
                double vv = 0.0;
                if (left) { if (g - sc <= bw) vv = PQP_GB(g, g - sc); }
                else { if (sc - g <= bw) vv = PQP_GB(sc, sc - g); }
                cx.tmp[g] = vv;
            }
            gen_local_solve(cx, cx.tmp, lo, hi);
            for (int r = 0; r < S; ++r) {
                double accL = 0.0, accR = 0.0;
                const int sl = gs + r, sr = gq + r;
                for (int g = lo; g < hi && g - sl <= bw; ++g) accL += PQP_GB(g, g - sl) * cx.tmp[g];
                if (has_right) {
                    int g0 = sr - bw;
                    if (g0 < lo) g0 = lo;
                    for (int g = g0; g < hi; ++g) accR += PQP_GB(sr, sr - g) * cx.tmp[g];
                }
                if (left) { R[3 * S2 + r * S + col] = accL; R[S2 + col * S + r] = -accR; }
                else R[4 * S2 + r * S + (col - S)] = accR;
            }
        }
    }
    w.sync();
    if (act) {
        const int gs = cx.gsep;
        const double *Cprev = cx.red + (size_t)RS * (lane - 1) + 4 * S2;
        for (int r = 0; r < S; ++r)
            for (int cc = 0; cc < S; ++cc) {
                const int hi_ = r > cc ? r : cc, lo_ = r > cc ? cc : r;
                double vv = PQP_GB(gs + hi_, hi_ - lo_) - R[3 * S2 + r * S + cc];
                if (lane > 0) vv -= Cprev[r * S + cc];
                R[r * S + cc] = vv;
            }
    }
    w.sync();
    if (lane == 0) {
        double Sch[S2], Sinv[S2];
        for (int k = 0; k < S2; ++k) Sch[k] = cx.red[k];
        for (int p = 0; p < cx.M; ++p) {
            double *Rp = cx.red + (size_t)RS * p;
            if (!(Sch[0] > 0.0)) ok = 0;
            if constexpr (S == 3) {
                inv3_spd(Sch, Sinv);
                for (int k = 0; k < S2; ++k) Rp[k] = Sinv[k];
            } else {
                gen_ldl_spd<S>(Sch, Rp);   // Dg holds the block's LDL' factors (gen_solve solves with them)
            }
            if (p + 1 < cx.M) {
                double *Rn = Rp + RS;
                const double *Off = Rp + S2;
                if constexpr (S == 3) {
                    for (int r = 0; r < S; ++r)
                        for (int cc = 0; cc < S; ++cc) {
                            double a = 0.0;
                            for (int k = 0; k < S; ++k) a += Off[k * S + r] * Sinv[k * S + cc];
                            Rn[2 * S2 + r * S + cc] = a;
                        }
                } else {
                    // row r of G = column r of Off solved against the block
                    for (int r = 0; r < S; ++r) {
                        double o[S];
                        for (int k = 0; k < S; ++k) o[k] = Off[k * S + r];
                        gen_ldl_solve<S>(Rp, o, Rn + 2 * S2 + r * S);
                    }
                }
                for (int r = 0; r < S; ++r)
                    for (int cc = 0; cc < S; ++cc) {
                        double a = Rn[r * S + cc];
                        for (int k = 0; k < S; ++k) a -= Rn[2 * S2 + r * S + k] * Off[k * S + cc];
                        Sch[r * S + cc] = a;
                    }
            }
        }
    }
    ok = !w.any(!ok);
    w.sync();
    return ok;
}

template <int S>
PQP_DEV void gen_solve(Warp &w, GenCtx &cx) {
    constexpr int RS = kGenRedStride<S>, S2 = S * S;
    const int bw = cx.bw, lane = w.lane();
    const bool act = lane < cx.M;
    const int lo = cx.lo, hi = cx.hi, gs = cx.gsep;
    const bool has_right = (lane + 1 < cx.M);
    double *R = cx.red + (size_t)RS * lane;
    if (act) gen_local_solve(cx, cx.tr, lo, hi);
    w.sync();
    if (act) {
        const int plo = lane > 0 ? cx.sep[lane - 1] + S : 0;
        for (int r = 0; r < S; ++r) {
            const int sg = gs + r;
            double acc = cx.tr[sg];
            if (lane > 0) {
                int g0 = sg - bw;
                if (g0 < plo) g0 = plo;
                for (int g = g0; g < gs; ++g) acc -= PQP_GB(sg, sg - g) * cx.tr[g];
            }
            for (int g = lo; g < hi && g - sg <= bw; ++g) acc -= PQP_GB(g, g - sg) * cx.tr[g];
            R[5 * S2 + r] = acc;
        }
    }
    w.sync();
    if (lane == 0) {
        for (int p = 1; p < cx.M; ++p) {
            double *Rp = cx.red + (size_t)RS * p;
            const double *gp = Rp - RS + 5 * S2;
            for (int r = 0; r < S; ++r) Rp[5 * S2 + r] -= gen_dot<S>(Rp + 2 * S2 + r * S, gp);
        }
        double xn[S] = {};
        for (int p = cx.M - 1; p >= 0; --p) {
            double *Rp = cx.red + (size_t)RS * p;
            double t[S];
            for (int r = 0; r < S; ++r) {
                t[r] = Rp[5 * S2 + r];
                if (p + 1 < cx.M) t[r] -= gen_dot<S>(Rp + S2 + r * S, xn);
            }
            if constexpr (S == 3) {
                for (int r = 0; r < S; ++r) xn[r] = gen_dot<S>(Rp + r * S, t);
            } else {
                gen_ldl_solve<S>(Rp, t, xn);
            }
            const int sg = cx.sep[p];
            for (int r = 0; r < S; ++r) cx.tr[sg + r] = xn[r];
        }
    }
    w.sync();
    if (act) {
        const int gq = hi;
        for (int g = lo; g < hi; ++g) {
            double acc = 0.0;
            for (int r = 0; r < S; ++r) {
                const int sg = gs + r;
                if (g - sg <= bw) acc -= PQP_GB(g, g - sg) * cx.tr[sg];
            }
            if (has_right)
                for (int r = 0; r < S; ++r) {
                    const int sg = gq + r;
                    if (sg - g <= bw) acc -= PQP_GB(sg, sg - g) * cx.tr[sg];
                }
            cx.tmp[g] = acc;
        }
        gen_local_solve(cx, cx.tmp, lo, hi);
        for (int g = lo; g < hi; ++g) cx.tr[g] += cx.tmp[g];
    }
    w.sync();
}
#undef PQP_GB

PQP_DEV double gen_row_dot(const GenCtx &cx, int r, const double *x) {
    double a = 0.0;
    for (int t = 0; t < 4; ++t) {
        const int k = cx.A_col[4 * r + t];
        if (k >= 0) a += cx.A_val[4 * r + t] * x[k];
    }
    return a;
}

// OSQP is_dual_infeasible on the certificate (||dx||, q'dx, ||P dx||, max A dx over rows with a finite upper bound,
// max -A dx over rows with a finite lower bound), in unscaled terms.
PQP_DEV bool dual_infeasible(double nrm, double qdx, double pdx, double adx_up, double adx_lo, double eps) {
    return nrm > eps && qdx < -eps * nrm && pdx < eps * nrm && adx_up <= eps * nrm && adx_lo <= eps * nrm;
}

// One QP of the batch.  S: separator width (gv.sep marks S-unknown blocks).  kLinear: the cost has a linear term, q
// [sum n] in band order at the path's n-offset, which enters OSQP's cost scaling (||c D q||), the x-step right-hand side
// (-c q), the dual residual and its norm, OSQP's first iteration (from x = z = y = 0 the x-step sees -c q alone and
// z_prev = 0), and OSQP's dual-infeasibility test (is_dual_infeasible: the step dx of a check iteration with
// q'dx < -eps ||dx||, ||P dx|| < eps ||dx|| and A dx within eps ||dx|| of the recession cone of the bounds, all in
// unscaled terms, eps = eps_dual_inf).  It runs after the SOLVED and primal-infeasibility tests, when the dual residual
// fails, in the exact check (PQP_DUAL_INFEASIBLE) and in the x10 re-check at max_iter (PQP_DUAL_INFEASIBLE_INACCURATE).
// dx is parked in tmp, which gen_solve leaves free until the next solve.  With q = 0, q'dx < 0 never holds.
// NP: the off-diagonal P partners recorded per unknown (Po_idx / Po_val rows): 2 for the formulations above, 6 for the
// TENSION smoothing QP, whose x and y chains couple every unknown to three neighbours on each side.
template <int S = 3, bool kLinear = false, int NP = 2>
PQP_DEV void gen_solve_qp(Warp &w, const DevParams &pm, const GenView &gv, int prob, double *smem, size_t smem_cap,
                          const double *q = nullptr) {
    const int lane = w.lane();
    const int32_t *meta = gv.meta + (size_t)kGenMeta * prob;
    const int n = meta[0], m = meta[1], n_den = meta[2], bw = meta[3], M = meta[4], N = meta[5];
    const int offN = meta[6], offn = meta[7], offm = meta[8], offz = meta[9], offp = meta[10];
    const pqp_state *ref = gv.ref + offN;
    pqp_state *out = gv.out_states + offN;
    const double qnan = nan("");
    GenCtx cx;
    cx.n = n; cx.m = m; cx.bw = bw; cx.M = M;
    cx.A_col = gv.A_col + 4 * (size_t)offm; cx.A_val = gv.A_val + 4 * (size_t)offm;
    cx.l = gv.l + offm; cx.u = gv.u + offm; cx.Pd = gv.Pd + offn;
    cx.Po_idx = gv.Po_idx + NP * (size_t)offn; cx.Po_val = gv.Po_val + NP * (size_t)offn;
    cx.csc_ptr = gv.csc_ptr + offp; cx.csc_row = gv.csc_row + offz; cx.csc_val = gv.csc_val + offz;
    cx.sep = gv.sep + 32 * (size_t)prob;
    const double *qv = kLinear ? q + offn : nullptr;
    int status = PQP_UNSOLVED, iter = 0;
    bool bad = (n < 1 || m < 1 || M < 1 || M > 32 || bw < 1 || bw > kMaxBand || gen_smem_doubles<S>(n, m, bw) > smem_cap);
    if (!bad) {
        double *p = smem;
        cx.D = p; p += n; cx.xr = p; p += n; cx.tr = p; p += n; cx.tmp = p; p += n; cx.sg = p; p += n;
        cx.v = p; p += m; cx.E = p; p += m; cx.W = p; p += m; cx.wold = p; p += m;
        cx.band = p; p += (size_t)(bw + 1) * n; cx.red = p;
        cx.lo = cx.hi = cx.gsep = 0;
        if (lane < M) {
            cx.gsep = cx.sep[lane];
            cx.lo = cx.gsep + S;
            cx.hi = (lane + 1 < M) ? cx.sep[lane + 1] : n;
        }
        // osqp_setup validate_data: l <= u
        int invalid = 0;
        for (int r = lane; r < m; r += 32) if (!(cx.l[r] <= cx.u[r])) invalid = 1;
        invalid = w.any(invalid);
        if (invalid) status = PQP_INVALID_PROBLEM;
    } else {
        status = PQP_INVALID_PROBLEM;
    }
    double cost_c = 1.0;
    if (status == PQP_UNSOLVED) {
        // ---- Ruiz equilibration + cost scaling (scratch: tmp = column factors, W = row factors)
        for (int j = lane; j < n; j += 32) cx.D[j] = 1.0;
        for (int r = lane; r < m; r += 32) cx.E[r] = 1.0;
        double Dt = 1.0;   // dead variables have P = 0 and no rows: their scaling stays 1
        (void)Dt;
        w.sync();
        for (int sweep = 0; sweep < pm.scaling; ++sweep) {
            for (int j = lane; j < n; j += 32) {
                const double Dj = cx.D[j];
                double nrm = cost_c * fabs(cx.Pd[j]) * Dj * Dj;
                for (int q = 0; q < NP; ++q) {
                    const int k = cx.Po_idx[NP * j + q];
                    if (k >= 0) nrm = fmax(nrm, cost_c * fabs(cx.Po_val[NP * j + q]) * Dj * cx.D[k]);
                }
                double an = 0.0;
                for (int e = cx.csc_ptr[j]; e < cx.csc_ptr[j + 1]; ++e)
                    an = fmax(an, fabs(cx.csc_val[e]) * cx.E[cx.csc_row[e]]);
                nrm = fmax(nrm, an * Dj);
                cx.tmp[j] = 1.0 / sqrt(limit_scaling(nrm));
            }
            for (int r = lane; r < m; r += 32) {
                double an = 0.0;
                for (int t = 0; t < 4; ++t) {
                    const int k = cx.A_col[4 * r + t];
                    if (k >= 0) an = fmax(an, fabs(cx.A_val[4 * r + t]) * cx.D[k]);
                }
                cx.W[r] = 1.0 / sqrt(limit_scaling(an * cx.E[r]));
            }
            w.sync();
            for (int j = lane; j < n; j += 32) cx.D[j] *= cx.tmp[j];
            for (int r = lane; r < m; r += 32) cx.E[r] *= cx.W[r];
            w.sync();
            double part = 0.0;
            for (int j = lane; j < n; j += 32) {
                const double Dj = cx.D[j];
                double nrm = cost_c * fabs(cx.Pd[j]) * Dj * Dj;
                for (int q = 0; q < NP; ++q) {
                    const int k = cx.Po_idx[NP * j + q];
                    if (k >= 0) nrm = fmax(nrm, cost_c * fabs(cx.Po_val[NP * j + q]) * Dj * cx.D[k]);
                }
                part += nrm;
            }
            const double mean = w.sum(part) / (double)n_den;
            double ct;
            if constexpr (kLinear) {
                double qn = 0.0;
                for (int j = lane; j < n; j += 32) qn = fmax(qn, fabs(cost_c * cx.D[j] * qv[j]));
                ct = fmax(mean, limit_scaling(w.max(qn)));
            } else {
                ct = fmax(mean, 1.0);
            }
            ct = limit_scaling(ct);
            cost_c = cost_c * (1.0 / ct);
            w.sync();
        }
        for (int j = lane; j < n; j += 32) { cx.sg[j] = pm.sigma / (cx.D[j] * cx.D[j]); cx.xr[j] = 0.0; }
        for (int r = lane; r < m; r += 32) cx.v[r] = 0.0;
        double rho = fmin(fmax(pm.rho, kRhoMin), kRhoMax);
        for (int r = lane; r < m; r += 32) cx.W[r] = rho_bar(cx.E[r] * cx.l[r], cx.E[r] * cx.u[r], rho) * cx.E[r] * cx.E[r];
        w.sync();
        if (!gen_factor<S, NP>(w, cx, cost_c)) status = PQP_NON_CVX;
        const double alpha = pm.alpha;
        Residuals res{};   // of the last check
        // dual-infeasibility certificate of the last check (kLinear), at eps_dual_inf and at 10 eps_dual_inf
        bool di_1 = false, di_10 = false;
        (void)di_1; (void)di_10;
        iter = 0;
        while (status == PQP_UNSOLVED && iter < pm.max_iter) {
            ++iter;
            // iterations that end in a termination check first park w = v - clamp(v): the check needs
            // delta_y = W (w_new - w_old) (OSQP update_y / is_primal_infeasible)
            const bool chk = (pm.check_termination && (iter % pm.check_termination == 0)) || iter == pm.max_iter;
            if (iter == 1 && !kLinear) {
                // OSQP's first iteration from x = z = y = 0 ends at the cold start (x = 0, v = 0: z = clamp(0),
                // y = -rho clamp(0)).  Its check and rho adaptation still run below, on w_old = y_0 / rho = 0.
                if (chk) for (int r = lane; r < m; r += 32) cx.wold[r] = 0.0;
            } else {
                // g_r = W (2 clamp(v) - v) parked in tmp-sized? no: m may exceed n -> reuse E? E is needed.
                // rhs_j = sigma_j x_j + sum_{r in col j} a_rj W_r (2 clamp(v_r) - v_r), gathered per column
                for (int j = lane; j < n; j += 32) {
                    double acc = cx.sg[j] * cx.xr[j];
                    if (!kLinear || iter > 1)
                        for (int e = cx.csc_ptr[j]; e < cx.csc_ptr[j + 1]; ++e) {
                            const int r = cx.csc_row[e];
                            const double vv = cx.v[r];
                            acc += cx.csc_val[e] * (cx.W[r] * (2.0 * clampd(vv, cx.l[r], cx.u[r]) - vv));
                        }
                    if constexpr (kLinear) acc -= cost_c * qv[j];
                    cx.tr[j] = acc;
                }
                w.sync();
                gen_solve<S>(w, cx);
                for (int r = lane; r < m; r += 32) {
                    const double vv = cx.v[r];
                    const double zz = (kLinear && iter == 1) ? 0.0 : clampd(vv, cx.l[r], cx.u[r]);
                    if (chk) cx.wold[r] = vv - zz;
                    cx.v[r] = vv + alpha * (gen_row_dot(cx, r, cx.tr) - zz);
                }
                if constexpr (kLinear) {
                    for (int j = lane; j < n; j += 32) {
                        const double xn = alpha * cx.tr[j] + (1.0 - alpha) * cx.xr[j];
                        if (chk) cx.tmp[j] = xn - cx.xr[j];
                        cx.xr[j] = xn;
                    }
                } else {
                    for (int j = lane; j < n; j += 32) cx.xr[j] = alpha * cx.tr[j] + (1.0 - alpha) * cx.xr[j];
                }
            }
            w.sync();
            const bool can_check = pm.check_termination && (iter % pm.check_termination == 0);
            const bool can_adapt = pm.adaptive_rho && pm.adaptive_rho_interval && (iter % pm.adaptive_rho_interval == 0);
            if (can_check || can_adapt || iter == pm.max_iter) {
                double pr = 0, nz = 0, nax = 0, prs = 0, nzs = 0, naxs = 0;
                const double cinv = 1.0 / cost_c;
                for (int r = lane; r < m; r += 32) {
                    const double ax = gen_row_dot(cx, r, cx.xr), vv = cx.v[r], z = clampd(vv, cx.l[r], cx.u[r]);
                    const double rr = ax - z, e = cx.E[r];
                    pr = fmax(pr, fabs(rr)); nz = fmax(nz, fabs(z)); nax = fmax(nax, fabs(ax));
                    prs = fmax(prs, e * fabs(rr)); nzs = fmax(nzs, e * fabs(z)); naxs = fmax(naxs, e * fabs(ax));
                }
                double dr = 0, npx = 0, naty = 0, drs = 0, npxs = 0, natys = 0, nq = 0, nqs = 0;
                for (int j = lane; j < n; j += 32) {
                    double px = cx.Pd[j] * cx.xr[j];
                    for (int q = 0; q < NP; ++q) {
                        const int k = cx.Po_idx[NP * j + q];
                        if (k >= 0) px += cx.Po_val[NP * j + q] * cx.xr[k];
                    }
                    double aty = 0.0;
                    for (int e = cx.csc_ptr[j]; e < cx.csc_ptr[j + 1]; ++e) {
                        const int r = cx.csc_row[e];
                        const double vv = cx.v[r];
                        aty += cx.csc_val[e] * (cx.W[r] * (vv - clampd(vv, cx.l[r], cx.u[r])) * cinv);
                    }
                    double rr = px + aty;
                    const double cd = cost_c * cx.D[j];
                    if constexpr (kLinear) {
                        rr = qv[j] + px + aty;
                        nq = fmax(nq, fabs(qv[j]));
                        nqs = fmax(nqs, cd * fabs(qv[j]));
                    }
                    dr = fmax(dr, fabs(rr)); npx = fmax(npx, fabs(px)); naty = fmax(naty, fabs(aty));
                    drs = fmax(drs, cd * fabs(rr)); npxs = fmax(npxs, cd * fabs(px)); natys = fmax(natys, cd * fabs(aty));
                }
                pr = w.max(pr); nz = w.max(nz); nax = w.max(nax); prs = w.max(prs); nzs = w.max(nzs); naxs = w.max(naxs);
                dr = w.max(dr); npx = w.max(npx); naty = w.max(naty); drs = w.max(drs); npxs = w.max(npxs); natys = w.max(natys);
                if constexpr (kLinear) {
                    nq = w.max(nq); nqs = w.max(nqs);
                    npx = fmax(npx, nq); npxs = fmax(npxs, nqs);   // OSQP's dual norm: max(||q||, ||Px||, ||A'y||)
                }
                w.sync();
                // ---- primal-infeasibility certificate (OSQP is_primal_infeasible) in unscaled terms:
                // g = W (w_new - w_old) = E delta_y projected on the cone of the finite (scaled) bounds;
                // ||g||_inf, u'g+ + l'g-, ||A'g||_inf.  g overwrites wold.
                if (chk) {
                    double c_nrm = 0, c_lhs = 0, c_cert = 0;
                    for (int r = lane; r < m; r += 32) {
                        const double vv = cx.v[r], lr = cx.l[r], ur = cx.u[r];
                        double g = cx.W[r] * ((vv - clampd(vv, lr, ur)) - cx.wold[r]);
                        const bool u_inf = cx.E[r] * ur > kOsqpInfty * kMinScaling;
                        const bool l_inf = cx.E[r] * lr < -kOsqpInfty * kMinScaling;
                        if (u_inf) g = l_inf ? 0.0 : fmin(g, 0.0);
                        else if (l_inf) g = fmax(g, 0.0);
                        cx.wold[r] = g;
                        c_nrm = fmax(c_nrm, fabs(g));
                        c_lhs += ur * fmax(g, 0.0) + lr * fmin(g, 0.0);
                    }
                    w.sync();
                    for (int j = lane; j < n; j += 32) {
                        double aty = 0.0;
                        for (int e = cx.csc_ptr[j]; e < cx.csc_ptr[j + 1]; ++e) aty += cx.csc_val[e] * cx.wold[cx.csc_row[e]];
                        c_cert = fmax(c_cert, fabs(aty));
                    }
                    res.inf_nrm = w.max(c_nrm); res.inf_cert = w.max(c_cert); res.inf_lhs = w.sum(c_lhs);
                    w.sync();
                }
                if constexpr (kLinear) {
                    if (chk) {
                        double dn = 0, qd = 0, pd = 0, au = -INFINITY, al = -INFINITY;
                        for (int j = lane; j < n; j += 32) {
                            const double dx = cx.tmp[j];
                            double p = cx.Pd[j] * dx;
                            for (int q = 0; q < NP; ++q) {
                                const int k = cx.Po_idx[NP * j + q];
                                if (k >= 0) p += cx.Po_val[NP * j + q] * cx.tmp[k];
                            }
                            dn = fmax(dn, fabs(dx)); qd += qv[j] * dx; pd = fmax(pd, fabs(p));
                        }
                        for (int r = lane; r < m; r += 32) {
                            const double ad = gen_row_dot(cx, r, cx.tmp);
                            if (cx.E[r] * cx.u[r] < kOsqpInfty * kMinScaling) au = fmax(au, ad);
                            if (cx.E[r] * cx.l[r] > -kOsqpInfty * kMinScaling) al = fmax(al, -ad);
                        }
                        dn = w.max(dn); qd = w.sum(qd); pd = w.max(pd); au = w.max(au); al = w.max(al);
                        di_1 = dual_infeasible(dn, qd, pd, au, al, pm.eps_dual_inf);
                        di_10 = dual_infeasible(dn, qd, pd, au, al, 10 * pm.eps_dual_inf);
                        w.sync();
                    }
                }
                res.pri_res = pr; res.dua_res = dr; res.pri_nrm = fmax(nz, nax); res.dua_nrm = fmax(npx, naty);
                if (can_check || iter == pm.max_iter) {
                    status = termination_verdict(pm, res);
                    if constexpr (kLinear)
                        if (status == PQP_UNSOLVED && !(res.dua_res < pm.eps_abs + pm.eps_rel * res.dua_nrm) &&
                            di_1)
                            status = PQP_DUAL_INFEASIBLE;
                }
                if (status == PQP_UNSOLVED && can_adapt) {
                    const double rho_new = rho_estimate(rho, prs, drs, fmax(nzs, naxs), fmax(npxs, natys));
                    if (rho_changed(pm, rho_new, rho)) {
                        for (int r = lane; r < m; r += 32) {
                            const double El = cx.E[r] * cx.l[r], Eu = cx.E[r] * cx.u[r];
                            const double ro = rho_bar(El, Eu, rho), rn = rho_bar(El, Eu, rho_new);
                            const double vv = cx.v[r], z = clampd(vv, cx.l[r], cx.u[r]);
                            cx.v[r] = z + (vv - z) * (ro / rn);   // y kept, w = E^-1 y / rho_row
                            cx.W[r] = rn * cx.E[r] * cx.E[r];
                        }
                        rho = rho_new;
                        w.sync();
                        if (!gen_factor<S, NP>(w, cx, cost_c)) status = PQP_NON_CVX;
                    }
                }
            }
        }
        if (status == PQP_UNSOLVED) {
            status = max_iter_verdict(pm, res);
            if constexpr (kLinear)
                if (status == PQP_MAX_ITER_REACHED && !(res.dua_res < 10 * pm.eps_abs + 10 * pm.eps_rel * res.dua_nrm) &&
                    di_10)
                    status = PQP_DUAL_INFEASIBLE_INACCURATE;
        }
    }
    // ---- epilogue: getOptimizedPath (solver_k_as_input.cpp:22-44, ..._constrained.cpp:26-43)
    const bool has_sol = has_solution(status);
    const int32_t *oi = gv.out_idx + 3 * (size_t)offN;
    w.sync();
    double *px = bad ? nullptr : cx.tr, *py = bad ? nullptr : cx.tmp;
    for (int i = lane; i < N; i += 32) {
        double ey = qnan, ephi = qnan, kk = qnan, tx, ty;
        if (has_sol) { ey = cx.xr[oi[3 * i]]; ephi = cx.xr[oi[3 * i + 1]]; kk = cx.xr[oi[3 * i + 2]]; }
        optimized_station(ref[i], ey, ephi, kk, out[i], tx, ty);
        out[i].s = qnan;
        if (px) { px[i] = tx; py[i] = ty; }
        store_frenet(gv.out_frenet, offN + i, ey, ephi, kk);
    }
    w.sync();
    if (lane == 0) {
        if (px) {
            double acc = 0.0;
            for (int i = 0; i < N; ++i) {
                if (i > 0) {
                    const double dx = px[i] - px[i - 1], dy = py[i] - py[i - 1];
                    acc += sqrt(dx * dx + dy * dy);
                }
                out[i].s = acc;
            }
        }
        gv.status[prob] = status;
        if (gv.iters) gv.iters[prob] = iter;
    }
    w.sync();
}

}  // namespace pqp
