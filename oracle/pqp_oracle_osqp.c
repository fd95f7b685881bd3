/*
 * pqp_oracle_osqp.c -- CPU ORACLE (test infrastructure, not product code; see pqp_oracle.h).
 *
 * Restatement of the OSQP algorithm that the reference calls through osqp-eigen at
 * src/solver/solver.cpp:66-74 (setHessianMatrix .. initSolver .. solve .. getSolution).
 * OSQP itself is a third-party dependency that is NOT under /root/reference (cloned un-pinned
 * by scripts/install_deps.sh:102; 0.6.x era) -- this file follows its published algorithm
 * [Stellato, Banjac, Goulart, Bemporad, Boyd: "OSQP: an operator splitting solver for quadratic
 * programs", Math. Prog. Comp. 12 (2020)] and documented 0.6.x behaviour:
 *   - modified Ruiz equilibration of the KKT matrix + cost scaling, `scaling` (=10) sweeps,
 *     scaling factors limited to [1e-4, 1e4];
 *   - rho vector: 1e3*rho on equality rows (u-l < 1e-4), 1e-6 on rows free on both sides
 *     (|bound| > 1e30*1e-4), rho elsewhere;
 *   - x~,nu from the quasi-definite KKT system [[P+sigma I, A'],[A, -diag(1/rho)]] solved by a
 *     sparse LDL' without pivoting (QDLDL in OSQP; here an up-looking LDL' after T. Davis,
 *     "Algorithm 849", with an exact minimum-degree ordering instead of AMD);
 *   - relaxation alpha, projection onto [l,u], dual update;
 *   - residual / tolerance formulas in UNSCALED form (scaled_termination = 0), checked every
 *     `check_termination` (=25) iterations, strict "<";
 *   - primal/dual infeasibility certificates on delta_y / delta_x;
 *   - adaptive rho: rho <- rho*sqrt(rp_norm/rd_norm) on scaled residuals, applied when it
 *     leaves [rho/5, 5 rho], KKT refactorised.  OSQP picks the adaptation interval from
 *     wall-clock timing; here it is the explicit pqp_params.adaptive_rho_interval.
 * PARITY UNPINNED: no real OSQP is available in this environment to pin these rules.
 */
#include "pqp_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>
#include "pqp_oracle_arena.h"   /* malloc / calloc / free of this file go through the per-thread arena when it is on */

#define OSQP_INFTY 1e30
#define RHO_MIN 1e-06
#define RHO_MAX 1e06
#define RHO_EQ_OVER_RHO_INEQ 1e03
#define RHO_TOL 1e-04
#define MIN_SCALING 1e-04
#define MAX_SCALING 1e+04

#define c_max(a, b) (((a) > (b)) ? (a) : (b))
#define c_min(a, b) (((a) < (b)) ? (a) : (b))
#define c_absval(x) (((x) < 0) ? -(x) : (x))

typedef struct {
    int nrow, ncol;
    int *p;   /* column pointers, ncol+1 */
    int *i;   /* row indices */
    double *x;
} csc;

static csc *csc_from_triplets(int nrow, int ncol, int nnz, const int *ti, const int *tj,
                              const double *tv) {
    csc *M = (csc *)calloc(1, sizeof(csc));
    M->nrow = nrow; M->ncol = ncol;
    M->p = (int *)calloc((size_t)ncol + 1, sizeof(int));
    M->i = (int *)malloc(sizeof(int) * (size_t)(nnz > 0 ? nnz : 1));
    M->x = (double *)malloc(sizeof(double) * (size_t)(nnz > 0 ? nnz : 1));
    for (int k = 0; k < nnz; ++k) M->p[tj[k] + 1]++;
    for (int j = 0; j < ncol; ++j) M->p[j + 1] += M->p[j];
    int *next = (int *)malloc(sizeof(int) * (size_t)(ncol + 1));
    memcpy(next, M->p, sizeof(int) * (size_t)(ncol + 1));
    for (int k = 0; k < nnz; ++k) {
        int d = next[tj[k]]++;
        M->i[d] = ti[k];
        M->x[d] = tv[k];
    }
    free(next);
    return M;
}
static void csc_free(csc *M) {
    if (!M) return;
    free(M->p); free(M->i); free(M->x); free(M);
}

/* y = A x ; y (+)= A' x ; inf norms ------------------------------------------------------------ */
static void mat_vec(const csc *A, const double *x, double *y) { /* y = A x */
    for (int i = 0; i < A->nrow; ++i) y[i] = 0;
    for (int j = 0; j < A->ncol; ++j)
        for (int k = A->p[j]; k < A->p[j + 1]; ++k) y[A->i[k]] += A->x[k] * x[j];
}
static void mat_tpose_vec(const csc *A, const double *x, double *y) { /* y = A' x */
    for (int j = 0; j < A->ncol; ++j) {
        double s = 0;
        for (int k = A->p[j]; k < A->p[j + 1]; ++k) s += A->x[k] * x[A->i[k]];
        y[j] = s;
    }
}
static void sym_triu_vec(const csc *P, const double *x, double *y) { /* y = P x, P upper stored */
    for (int i = 0; i < P->ncol; ++i) y[i] = 0;
    for (int j = 0; j < P->ncol; ++j)
        for (int k = P->p[j]; k < P->p[j + 1]; ++k) {
            int i = P->i[k];
            y[i] += P->x[k] * x[j];
            if (i != j) y[j] += P->x[k] * x[i];
        }
}
static double vec_norm_inf(const double *v, int n) {
    double m = 0;
    for (int i = 0; i < n; ++i) { double a = c_absval(v[i]); if (a > m) m = a; }
    return m;
}
static double vec_scaled_norm_inf(const double *S, const double *v, int n) {
    double m = 0;
    for (int i = 0; i < n; ++i) { double a = c_absval(S[i] * v[i]); if (a > m) m = a; }
    return m;
}
static void limit_scaling(double *D, int n) {
    for (int i = 0; i < n; ++i) {
        D[i] = D[i] < MIN_SCALING ? 1.0 : D[i];
        D[i] = D[i] > MAX_SCALING ? MAX_SCALING : D[i];
    }
}

/* ---- exact minimum-degree ordering of a symmetric pattern (stand-in for AMD) ---------------- */
typedef struct { int *v; int n, cap; } ivec;
static void iv_push(ivec *a, int x) {
    if (a->n == a->cap) { a->cap = a->cap ? 2 * a->cap : 8; a->v = (int *)realloc(a->v, sizeof(int) * (size_t)a->cap); }
    a->v[a->n++] = x;
}
static int iv_has(const ivec *a, int x) { for (int k = 0; k < a->n; ++k) if (a->v[k] == x) return 1; return 0; }
static void iv_remove(ivec *a, int x) {
    for (int k = 0; k < a->n; ++k) if (a->v[k] == x) { a->v[k] = a->v[--a->n]; return; }
}
static void min_degree_order(int nn, const int *Kp, const int *Ki, int *perm) {
    ivec *adj = (ivec *)calloc((size_t)nn, sizeof(ivec));
    for (int j = 0; j < nn; ++j)
        for (int k = Kp[j]; k < Kp[j + 1]; ++k) {
            int i = Ki[k];
            if (i != j && !iv_has(&adj[i], j)) { iv_push(&adj[i], j); iv_push(&adj[j], i); }
        }
    char *done = (char *)calloc((size_t)nn, 1);
    for (int step = 0; step < nn; ++step) {
        int best = -1, bestdeg = 1 << 30;
        for (int v = 0; v < nn; ++v)
            if (!done[v] && adj[v].n < bestdeg) { bestdeg = adj[v].n; best = v; }
        perm[step] = best;
        done[best] = 1;
        ivec *S = &adj[best];
        for (int a = 0; a < S->n; ++a) iv_remove(&adj[S->v[a]], best);
        for (int a = 0; a < S->n; ++a)
            for (int b = a + 1; b < S->n; ++b) {
                int u = S->v[a], w = S->v[b];
                if (!iv_has(&adj[u], w)) { iv_push(&adj[u], w); iv_push(&adj[w], u); }
            }
    }
    for (int v = 0; v < nn; ++v) free(adj[v].v);
    free(adj);
    free(done);
}

/* ---- symbolic structure of the permuted KKT, cached per sparsity pattern -------------------- */
typedef struct {
    int n, m, nn;          /* nn = n + m */
    int p_nnz, a_nnz;
    int *p_i, *p_j, *a_i, *a_j; /* pattern key */
    int *perm, *iperm;     /* perm[new] = old */
    int *Kp, *Ki;          /* permuted upper-triangular KKT pattern (CSC) */
    int knz;
    int *pos_P, *pos_A;    /* triplet k -> position in K values */
    int *pos_sigma;        /* i < n -> position of (i,i) */
    int *pos_rho;          /* j < m -> position of (n+j,n+j) */
    int *parent, *Lp;      /* etree and L column pointers */
    int lnz;
} symbolic;

static void symbolic_free(symbolic *S) {
    if (!S) return;
    free(S->p_i); free(S->p_j); free(S->a_i); free(S->a_j);
    free(S->perm); free(S->iperm); free(S->Kp); free(S->Ki);
    free(S->pos_P); free(S->pos_A); free(S->pos_sigma); free(S->pos_rho);
    free(S->parent); free(S->Lp);
    free(S);
}
static int symbolic_matches(const symbolic *S, const oqp_problem *qp) {
    if (!S) return 0;
    return S && S->n == qp->n && S->m == qp->m && S->p_nnz == qp->p_nnz && S->a_nnz == qp->a_nnz &&
           !memcmp(S->p_i, qp->p_i, sizeof(int) * (size_t)qp->p_nnz) &&
           !memcmp(S->p_j, qp->p_j, sizeof(int) * (size_t)qp->p_nnz) &&
           !memcmp(S->a_i, qp->a_i, sizeof(int) * (size_t)qp->a_nnz) &&
           !memcmp(S->a_j, qp->a_j, sizeof(int) * (size_t)qp->a_nnz);
}
static int *dup_int(const int *a, int n) {
    int *r = (int *)malloc(sizeof(int) * (size_t)(n > 0 ? n : 1));
    memcpy(r, a, sizeof(int) * (size_t)n);
    return r;
}

typedef struct { int r, c, src; } kent; /* src: >=0 P triplet, -1-k A triplet, sigma/rho encoded */
static int kent_cmp(const void *a, const void *b) {
    const kent *x = (const kent *)a, *y = (const kent *)b;
    if (x->c != y->c) return x->c - y->c;
    return x->r - y->r;
}

static symbolic *symbolic_build(const oqp_problem *qp) {
    const int n = qp->n, m = qp->m, nn = n + m;
    symbolic *S = (symbolic *)calloc(1, sizeof(symbolic));
    S->n = n; S->m = m; S->nn = nn; S->p_nnz = qp->p_nnz; S->a_nnz = qp->a_nnz;
    S->p_i = dup_int(qp->p_i, qp->p_nnz); S->p_j = dup_int(qp->p_j, qp->p_nnz);
    S->a_i = dup_int(qp->a_i, qp->a_nnz); S->a_j = dup_int(qp->a_j, qp->a_nnz);
    /* unpermuted upper-triangular KKT entries: P(i,j) i<=j ; A(r,c) -> (c, n+r) ; diagonals */
    const int tot = qp->p_nnz + qp->a_nnz + nn;
    kent *E = (kent *)malloc(sizeof(kent) * (size_t)tot);
    int e = 0;
    /* codes for src: [0,p_nnz) P ; [p_nnz, p_nnz+a_nnz) A ; then n sigma ; then m rho */
    for (int k = 0; k < qp->p_nnz; ++k) { E[e].r = qp->p_i[k]; E[e].c = qp->p_j[k]; E[e].src = k; e++; }
    for (int k = 0; k < qp->a_nnz; ++k) { E[e].r = qp->a_j[k]; E[e].c = n + qp->a_i[k]; E[e].src = qp->p_nnz + k; e++; }
    for (int i = 0; i < nn; ++i) { E[e].r = i; E[e].c = i; E[e].src = qp->p_nnz + qp->a_nnz + i; e++; }
    /* ordering on the unpermuted pattern */
    {
        int *cp = (int *)calloc((size_t)nn + 1, sizeof(int));
        int *ci = (int *)malloc(sizeof(int) * (size_t)tot);
        for (int k = 0; k < tot; ++k) cp[E[k].c + 1]++;
        for (int j = 0; j < nn; ++j) cp[j + 1] += cp[j];
        int *nx = dup_int(cp, nn + 1);
        for (int k = 0; k < tot; ++k) ci[nx[E[k].c]++] = E[k].r;
        S->perm = (int *)malloc(sizeof(int) * (size_t)nn);
        min_degree_order(nn, cp, ci, S->perm);
        free(cp); free(ci); free(nx);
    }
    S->iperm = (int *)malloc(sizeof(int) * (size_t)nn);
    for (int k = 0; k < nn; ++k) S->iperm[S->perm[k]] = k;
    /* permute, keep upper triangle, sort, merge duplicates */
    for (int k = 0; k < tot; ++k) {
        int r = S->iperm[E[k].r], c = S->iperm[E[k].c];
        if (r > c) { int t = r; r = c; c = t; }
        E[k].r = r; E[k].c = c;
    }
    qsort(E, (size_t)tot, sizeof(kent), kent_cmp);
    S->Kp = (int *)calloc((size_t)nn + 1, sizeof(int));
    S->Ki = (int *)malloc(sizeof(int) * (size_t)tot);
    S->pos_P = (int *)malloc(sizeof(int) * (size_t)(qp->p_nnz > 0 ? qp->p_nnz : 1));
    S->pos_A = (int *)malloc(sizeof(int) * (size_t)(qp->a_nnz > 0 ? qp->a_nnz : 1));
    S->pos_sigma = (int *)malloc(sizeof(int) * (size_t)n);
    S->pos_rho = (int *)malloc(sizeof(int) * (size_t)(m > 0 ? m : 1));
    int knz = 0;
    for (int k = 0; k < tot; ++k) {
        if (k == 0 || E[k].r != E[k - 1].r || E[k].c != E[k - 1].c) {
            S->Ki[knz] = E[k].r;
            S->Kp[E[k].c + 1]++;
            knz++;
        }
        int pos = knz - 1, s = E[k].src;
        if (s < qp->p_nnz) S->pos_P[s] = pos;
        else if (s < qp->p_nnz + qp->a_nnz) S->pos_A[s - qp->p_nnz] = pos;
        else if (s < qp->p_nnz + qp->a_nnz + n) S->pos_sigma[s - qp->p_nnz - qp->a_nnz] = pos;
        else S->pos_rho[s - qp->p_nnz - qp->a_nnz - n] = pos;
    }
    for (int j = 0; j < nn; ++j) S->Kp[j + 1] += S->Kp[j];
    S->knz = knz;
    free(E);
    /* elimination tree and column counts of L (up-looking LDL', Davis Alg. 849) */
    S->parent = (int *)malloc(sizeof(int) * (size_t)nn);
    S->Lp = (int *)calloc((size_t)nn + 1, sizeof(int));
    int *flag = (int *)malloc(sizeof(int) * (size_t)nn);
    int *lnzc = (int *)calloc((size_t)nn, sizeof(int));
    for (int k = 0; k < nn; ++k) {
        S->parent[k] = -1;
        flag[k] = k;
        for (int p = S->Kp[k]; p < S->Kp[k + 1]; ++p) {
            int i = S->Ki[p];
            if (i < k) {
                for (; flag[i] != k; i = S->parent[i]) {
                    if (S->parent[i] == -1) S->parent[i] = k;
                    lnzc[i]++;
                    flag[i] = k;
                }
            }
        }
    }
    for (int k = 0; k < nn; ++k) S->Lp[k + 1] = S->Lp[k] + lnzc[k];
    S->lnz = S->Lp[nn];
    free(flag); free(lnzc);
    return S;
}

/* ---- numeric LDL' --------------------------------------------------------------------------- */
typedef struct {
    const symbolic *S;
    double *Kx;            /* values of permuted KKT */
    int *Li; double *Lx;   /* L (unit lower, strict part) */
    double *D, *Dinv;
    int *Lnz, *pattern, *flag;
    double *Y, *w;
} ldl;

static ldl *ldl_alloc(const symbolic *S) {
    ldl *F = (ldl *)calloc(1, sizeof(ldl));
    F->S = S;
    F->Kx = (double *)calloc((size_t)S->knz, sizeof(double));
    F->Li = (int *)malloc(sizeof(int) * (size_t)(S->lnz > 0 ? S->lnz : 1));
    F->Lx = (double *)malloc(sizeof(double) * (size_t)(S->lnz > 0 ? S->lnz : 1));
    F->D = (double *)malloc(sizeof(double) * (size_t)S->nn);
    F->Dinv = (double *)malloc(sizeof(double) * (size_t)S->nn);
    F->Lnz = (int *)malloc(sizeof(int) * (size_t)S->nn);
    F->pattern = (int *)malloc(sizeof(int) * (size_t)S->nn);
    F->flag = (int *)malloc(sizeof(int) * (size_t)S->nn);
    F->Y = (double *)calloc((size_t)S->nn, sizeof(double));
    F->w = (double *)malloc(sizeof(double) * (size_t)S->nn);
    return F;
}
static void ldl_free(ldl *F) {
    if (!F) return;
    free(F->Kx); free(F->Li); free(F->Lx); free(F->D); free(F->Dinv);
    free(F->Lnz); free(F->pattern); free(F->flag); free(F->Y); free(F->w);
    free(F);
}
static int ldl_factor(ldl *F) {
    const symbolic *S = F->S;
    const int nn = S->nn;
    const int *Kp = S->Kp, *Ki = S->Ki, *Lp = S->Lp, *parent = S->parent;
    for (int k = 0; k < nn; ++k) {
        int top = nn;
        F->Y[k] = 0;
        F->flag[k] = k;
        F->Lnz[k] = 0;
        for (int p = Kp[k]; p < Kp[k + 1]; ++p) {
            int i = Ki[p];
            F->Y[i] += F->Kx[p];
            int len = 0;
            for (; F->flag[i] != k; i = parent[i]) {
                F->pattern[len++] = i;
                F->flag[i] = k;
            }
            while (len > 0) F->pattern[--top] = F->pattern[--len];
        }
        F->D[k] = F->Y[k];
        F->Y[k] = 0;
        for (; top < nn; ++top) {
            int i = F->pattern[top];
            double yi = F->Y[i];
            F->Y[i] = 0;
            int p2 = Lp[i] + F->Lnz[i];
            for (int p = Lp[i]; p < p2; ++p) F->Y[F->Li[p]] -= F->Lx[p] * yi;
            double lki = yi * F->Dinv[i];
            F->D[k] -= lki * yi;
            F->Li[p2] = k;
            F->Lx[p2] = lki;
            F->Lnz[i]++;
        }
        if (F->D[k] == 0.0) return -1;
        F->Dinv[k] = 1.0 / F->D[k];
    }
    return 0;
}
/* solve K sol = b (both in ORIGINAL ordering) */
static void ldl_solve(ldl *F, const double *b, double *sol) {
    const symbolic *S = F->S;
    const int nn = S->nn;
    double *w = F->w;
    for (int k = 0; k < nn; ++k) w[k] = b[S->perm[k]];
    for (int j = 0; j < nn; ++j) {
        double wj = w[j];
        for (int p = S->Lp[j]; p < S->Lp[j + 1]; ++p) w[F->Li[p]] -= F->Lx[p] * wj;
    }
    for (int j = 0; j < nn; ++j) w[j] *= F->Dinv[j];
    for (int j = nn - 1; j >= 0; --j) {
        double wj = w[j];
        for (int p = S->Lp[j]; p < S->Lp[j + 1]; ++p) wj -= F->Lx[p] * w[F->Li[p]];
        w[j] = wj;
    }
    for (int k = 0; k < nn; ++k) sol[S->perm[k]] = w[k];
}

/* Symbolic cache.  Paths of one batch that share (formulation, N, keep, zero pattern) share the sparsity
 * pattern; the analysis (ordering + elimination tree) is immutable once built, so one copy is shared by all
 * threads.  (OSQP redoes AMD + symbolic factorisation in every osqp_setup; sharing it only makes the CPU
 * baseline faster, i.e. errs on the generous side.)  A mixed-length batch (BASELINE config 5: 351 different
 * lengths) has one pattern per length: the cache holds 1024 of them, and an analysis is BUILT OUTSIDE the
 * lock so that threads working on different lengths do not wait for each other.  Entries are never freed. */
#include <pthread.h>
#define SYM_CACHE 1024
static symbolic *g_sym[SYM_CACHE];
static int g_sym_n = 0, g_sym_next = 0;
static pthread_mutex_t g_sym_mu = PTHREAD_MUTEX_INITIALIZER;
static __thread const symbolic *tls_sym = NULL;

static const symbolic *symbolic_lookup_locked(const oqp_problem *qp) {
    for (int k = 0; k < g_sym_n; ++k)
        if (symbolic_matches(g_sym[k], qp)) return g_sym[k];
    return NULL;
}

static const symbolic *symbolic_get(const oqp_problem *qp) {
    if (symbolic_matches(tls_sym, qp)) return tls_sym;
    pthread_mutex_lock(&g_sym_mu);
    const symbolic *found = symbolic_lookup_locked(qp);
    pthread_mutex_unlock(&g_sym_mu);
    if (!found) {
        const int arena_state = oa_suspend();   /* the analysis outlives this solve and is shared by all threads */
        symbolic *S = symbolic_build(qp);
        oa_resume(arena_state);
        pthread_mutex_lock(&g_sym_mu);
        found = symbolic_lookup_locked(qp);     /* another thread may have built the same pattern meanwhile */
        if (!found) {
            if (g_sym_n < SYM_CACHE) g_sym[g_sym_n++] = S;
            else { g_sym[g_sym_next] = S; g_sym_next = (g_sym_next + 1) % SYM_CACHE; } /* full: overwrite round robin (the old entry leaks; bounded use) */
            found = S;
            S = NULL;
        }
        pthread_mutex_unlock(&g_sym_mu);
        if (S) {
            const int st = oa_suspend();
            symbolic_free(S);
            oa_resume(st);
        }
    }
    tls_sym = found;
    return found;
}

/* ---- the solver ----------------------------------------------------------------------------- */
typedef struct {
    int n, m;
    csc *P, *A;            /* scaled in place */
    double *q, *l, *u;     /* scaled */
    double *D, *E, *Dinv, *Einv;
    double c, cinv;
    double *rho_vec, *rho_inv_vec;
    int *constr_type;
    double rho;
    double *x, *z, *y, *x_prev, *z_prev, *xz_tilde, *rhs;
    double *Ax, *Px, *Aty, *delta_x, *delta_y, *Adelta_x, *Atdelta_y, *Pdelta_x;
    int has_q;   /* q != 0: only then can the dual-infeasibility test fire, and only then are its margins noted */
    double *D_temp, *D_temp_A, *E_temp;
    double margin;         /* smallest relative gap of a value from its threshold in the checks since the last reset */
} work;

/* relative distance of a compared value from its threshold: a verdict closer than rounding is a coin flip */
static void note_gap(work *w, double a, double b) {
    const double d = c_max(c_absval(a), c_absval(b));
    w->margin = c_min(w->margin, d > 0 ? c_absval(a - b) / d : 0.0);
}

static void scale_data(work *w, int sweeps) {
    const int n = w->n, m = w->m;
    for (int i = 0; i < n; ++i) { w->D[i] = 1; w->Dinv[i] = 1; }
    for (int i = 0; i < m; ++i) { w->E[i] = 1; w->Einv[i] = 1; }
    w->c = 1.0;
    for (int it = 0; it < sweeps; ++it) {
        /* inf-norms of the columns of [[P, A'],[A, 0]] */
        for (int j = 0; j < n; ++j) { w->D_temp[j] = 0; w->D_temp_A[j] = 0; }
        for (int j = 0; j < n; ++j)
            for (int k = w->P->p[j]; k < w->P->p[j + 1]; ++k) {
                int i = w->P->i[k];
                double a = c_absval(w->P->x[k]);
                w->D_temp[j] = c_max(w->D_temp[j], a);
                if (i != j) w->D_temp[i] = c_max(w->D_temp[i], a);
            }
        for (int i = 0; i < m; ++i) w->E_temp[i] = 0;
        for (int j = 0; j < n; ++j)
            for (int k = w->A->p[j]; k < w->A->p[j + 1]; ++k) {
                double a = c_absval(w->A->x[k]);
                w->D_temp_A[j] = c_max(w->D_temp_A[j], a);
                w->E_temp[w->A->i[k]] = c_max(w->E_temp[w->A->i[k]], a);
            }
        for (int j = 0; j < n; ++j) w->D_temp[j] = c_max(w->D_temp[j], w->D_temp_A[j]);
        limit_scaling(w->D_temp, n);
        limit_scaling(w->E_temp, m);
        for (int j = 0; j < n; ++j) w->D_temp[j] = 1.0 / sqrt(w->D_temp[j]);
        for (int i = 0; i < m; ++i) w->E_temp[i] = 1.0 / sqrt(w->E_temp[i]);
        /* P <- D P D, A <- E A D, q <- D q */
        for (int j = 0; j < n; ++j)
            for (int k = w->P->p[j]; k < w->P->p[j + 1]; ++k)
                w->P->x[k] *= w->D_temp[w->P->i[k]] * w->D_temp[j];
        for (int j = 0; j < n; ++j)
            for (int k = w->A->p[j]; k < w->A->p[j + 1]; ++k)
                w->A->x[k] *= w->E_temp[w->A->i[k]] * w->D_temp[j];
        for (int j = 0; j < n; ++j) w->q[j] *= w->D_temp[j];
        for (int j = 0; j < n; ++j) w->D[j] *= w->D_temp[j];
        for (int i = 0; i < m; ++i) w->E[i] *= w->E_temp[i];
        /* cost scaling: c_temp = 1 / max(mean col-norm of P, ||q||_inf) */
        for (int j = 0; j < n; ++j) w->D_temp[j] = 0;
        for (int j = 0; j < n; ++j)
            for (int k = w->P->p[j]; k < w->P->p[j + 1]; ++k) {
                int i = w->P->i[k];
                double a = c_absval(w->P->x[k]);
                w->D_temp[j] = c_max(w->D_temp[j], a);
                if (i != j) w->D_temp[i] = c_max(w->D_temp[i], a);
            }
        double c_temp = 0;
        for (int j = 0; j < n; ++j) c_temp += w->D_temp[j];
        c_temp /= n;
        double inf_norm_q = vec_norm_inf(w->q, n);
        limit_scaling(&inf_norm_q, 1);
        c_temp = c_max(c_temp, inf_norm_q);
        limit_scaling(&c_temp, 1);
        c_temp = 1.0 / c_temp;
        for (int k = 0; k < w->P->p[n]; ++k) w->P->x[k] *= c_temp;
        for (int j = 0; j < n; ++j) w->q[j] *= c_temp;
        w->c *= c_temp;
    }
    w->cinv = 1.0 / w->c;
    for (int j = 0; j < n; ++j) w->Dinv[j] = 1.0 / w->D[j];
    for (int i = 0; i < m; ++i) w->Einv[i] = 1.0 / w->E[i];
    for (int i = 0; i < m; ++i) { w->l[i] *= w->E[i]; w->u[i] *= w->E[i]; }
}

static void set_rho_vec(work *w) {
    w->rho = c_min(c_max(w->rho, RHO_MIN), RHO_MAX);
    for (int i = 0; i < w->m; ++i) {
        if ((w->l[i] < -OSQP_INFTY * MIN_SCALING) && (w->u[i] > OSQP_INFTY * MIN_SCALING)) {
            w->constr_type[i] = -1;
            w->rho_vec[i] = RHO_MIN;
        } else if (w->u[i] - w->l[i] < RHO_TOL) {
            w->constr_type[i] = 1;
            w->rho_vec[i] = RHO_EQ_OVER_RHO_INEQ * w->rho;
        } else {
            w->constr_type[i] = 0;
            w->rho_vec[i] = w->rho;
        }
        w->rho_inv_vec[i] = 1.0 / w->rho_vec[i];
    }
}

static void kkt_fill(const work *w, const oqp_problem *qp, ldl *F, double sigma,
                     const int *p_map, const int *a_map) {
    const symbolic *S = F->S;
    memset(F->Kx, 0, sizeof(double) * (size_t)S->knz);
    for (int k = 0; k < qp->p_nnz; ++k) F->Kx[S->pos_P[k]] += w->P->x[p_map[k]];
    for (int k = 0; k < qp->a_nnz; ++k) F->Kx[S->pos_A[k]] += w->A->x[a_map[k]];
    for (int i = 0; i < w->n; ++i) F->Kx[S->pos_sigma[i]] += sigma;
    for (int j = 0; j < w->m; ++j) F->Kx[S->pos_rho[j]] += -w->rho_inv_vec[j];
}

/* triplet k -> index into the CSC value array built by csc_from_triplets (same stable order) */
static int *triplet_to_csc_map(int ncol, int nnz, const int *tj) {
    int *cnt = (int *)calloc((size_t)ncol + 1, sizeof(int));
    int *map = (int *)malloc(sizeof(int) * (size_t)(nnz > 0 ? nnz : 1));
    for (int k = 0; k < nnz; ++k) cnt[tj[k] + 1]++;
    for (int j = 0; j < ncol; ++j) cnt[j + 1] += cnt[j];
    for (int k = 0; k < nnz; ++k) map[k] = cnt[tj[k]]++;
    free(cnt);
    return map;
}

static double *dalloc(int n) { return (double *)calloc((size_t)(n > 0 ? n : 1), sizeof(double)); }

static double compute_pri_res(work *w, const double *x, const double *z) {
    mat_vec(w->A, x, w->Ax);
    for (int i = 0; i < w->m; ++i) w->z_prev[i] = w->Ax[i] - z[i];
    return vec_scaled_norm_inf(w->Einv, w->z_prev, w->m);
}
static double compute_dua_res(work *w, const double *x, const double *y) {
    sym_triu_vec(w->P, x, w->Px);
    mat_tpose_vec(w->A, y, w->Aty);
    for (int i = 0; i < w->n; ++i) w->x_prev[i] = w->q[i] + w->Px[i] + w->Aty[i];
    return w->cinv * vec_scaled_norm_inf(w->Dinv, w->x_prev, w->n);
}
static double compute_pri_tol(const work *w, double eps_abs, double eps_rel) {
    double a = vec_scaled_norm_inf(w->Einv, w->z, w->m);
    double b = vec_scaled_norm_inf(w->Einv, w->Ax, w->m);
    return eps_abs + eps_rel * c_max(a, b);
}
static double compute_dua_tol(const work *w, double eps_abs, double eps_rel) {
    double a = vec_scaled_norm_inf(w->Dinv, w->q, w->n);
    double b = vec_scaled_norm_inf(w->Dinv, w->Aty, w->n);
    double c = vec_scaled_norm_inf(w->Dinv, w->Px, w->n);
    double mx = c_max(c_max(a, b), c);
    return eps_abs + eps_rel * (w->cinv * mx);
}
static int is_primal_infeasible(work *w, double eps_prim_inf) {
    const int m = w->m, n = w->n;
    for (int i = 0; i < m; ++i) {
        if (w->u[i] > OSQP_INFTY * MIN_SCALING) {
            if (w->l[i] < -OSQP_INFTY * MIN_SCALING) w->delta_y[i] = 0.0;
            else w->delta_y[i] = c_min(w->delta_y[i], 0.0);
        } else if (w->l[i] < -OSQP_INFTY * MIN_SCALING) {
            w->delta_y[i] = c_max(w->delta_y[i], 0.0);
        }
    }
    double norm_delta_y = vec_scaled_norm_inf(w->E, w->delta_y, m);
    note_gap(w, norm_delta_y, eps_prim_inf);
    if (norm_delta_y > eps_prim_inf) {
        double ineq_lhs = 0;
        for (int i = 0; i < m; ++i)
            ineq_lhs += w->u[i] * c_max(w->delta_y[i], 0) + w->l[i] * c_min(w->delta_y[i], 0);
        note_gap(w, ineq_lhs, -eps_prim_inf * norm_delta_y);
        if (ineq_lhs < -eps_prim_inf * norm_delta_y) {
            mat_tpose_vec(w->A, w->delta_y, w->Atdelta_y);
            const double cert = vec_scaled_norm_inf(w->Dinv, w->Atdelta_y, n);
            note_gap(w, cert, eps_prim_inf * norm_delta_y);
            return cert < eps_prim_inf * norm_delta_y;
        }
    }
    return 0;
}
static int is_dual_infeasible(work *w, double eps_dual_inf) {
    const int m = w->m, n = w->n;
    double norm_delta_x = vec_scaled_norm_inf(w->D, w->delta_x, n);
    double cost_scaling = w->c;
    if (!w->has_q) return 0;   /* q'dx = 0 is never below -eps ||dx|| c */
    note_gap(w, norm_delta_x, eps_dual_inf);
    if (norm_delta_x > eps_dual_inf) {
        double qdx = 0;
        for (int i = 0; i < n; ++i) qdx += w->q[i] * w->delta_x[i];
        note_gap(w, qdx, -cost_scaling * eps_dual_inf * norm_delta_x);
        if (qdx < -cost_scaling * eps_dual_inf * norm_delta_x) {
            sym_triu_vec(w->P, w->delta_x, w->Pdelta_x);
            const double pdx = vec_scaled_norm_inf(w->Dinv, w->Pdelta_x, n);
            note_gap(w, pdx, cost_scaling * eps_dual_inf * norm_delta_x);
            if (pdx < cost_scaling * eps_dual_inf * norm_delta_x) {
                mat_vec(w->A, w->delta_x, w->Adelta_x);
                for (int i = 0; i < m; ++i) w->Adelta_x[i] *= w->Einv[i];
                double up = -INFINITY, lo = -INFINITY;   /* the rows closest to breaking the certificate */
                for (int i = 0; i < m; ++i) {
                    if (w->u[i] < OSQP_INFTY * MIN_SCALING) up = c_max(up, w->Adelta_x[i]);
                    if (w->l[i] > -OSQP_INFTY * MIN_SCALING) lo = c_max(lo, -w->Adelta_x[i]);
                }
                if (up > -INFINITY) note_gap(w, up, eps_dual_inf * norm_delta_x);
                if (lo > -INFINITY) note_gap(w, lo, eps_dual_inf * norm_delta_x);
                for (int i = 0; i < m; ++i) {
                    if (((w->u[i] < OSQP_INFTY * MIN_SCALING) && (w->Adelta_x[i] > eps_dual_inf * norm_delta_x)) ||
                        ((w->l[i] > -OSQP_INFTY * MIN_SCALING) && (w->Adelta_x[i] < -eps_dual_inf * norm_delta_x)))
                        return 0;
                }
                return 1;
            }
        }
    }
    return 0;
}

/* returns 1 when the algorithm should stop; sets *status */
static int check_termination(work *w, const pqp_params *prm, double pri_res, double dua_res,
                             int approximate, int *status) {
    double eps_abs = prm->eps_abs, eps_rel = prm->eps_rel;
    double eps_prim_inf = prm->eps_prim_inf, eps_dual_inf = prm->eps_dual_inf;
    int prim_res_check = 0, dual_res_check = 0, prim_inf_check = 0, dual_inf_check = 0;
    if (approximate) { eps_abs *= 10; eps_rel *= 10; eps_prim_inf *= 10; eps_dual_inf *= 10; }
    if (pri_res > OSQP_INFTY || dua_res > OSQP_INFTY) { *status = PQP_NON_CVX; return 1; }
    if (w->m == 0) prim_res_check = 1;
    else {
        double eps_prim = compute_pri_tol(w, eps_abs, eps_rel);
        note_gap(w, pri_res, eps_prim);
        if (pri_res < eps_prim) prim_res_check = 1;
        else prim_inf_check = is_primal_infeasible(w, eps_prim_inf);
    }
    double eps_dual = compute_dua_tol(w, eps_abs, eps_rel);
    note_gap(w, dua_res, eps_dual);
    if (dua_res < eps_dual) dual_res_check = 1;
    else dual_inf_check = is_dual_infeasible(w, eps_dual_inf);
    if (prim_res_check && dual_res_check) { *status = approximate ? PQP_SOLVED_INACCURATE : PQP_SOLVED; return 1; }
    if (prim_inf_check) { *status = approximate ? PQP_PRIMAL_INFEASIBLE_INACCURATE : PQP_PRIMAL_INFEASIBLE; return 1; }
    if (dual_inf_check) { *status = approximate ? PQP_DUAL_INFEASIBLE_INACCURATE : PQP_DUAL_INFEASIBLE; return 1; }
    return 0;
}

/* OSQP 0.6 validate_settings (auxil.c), on the settings pqp_params carries; written so that a NaN fails */
static int settings_valid(const pqp_params *p) {
    if (!(p->rho > 0) || !(p->sigma > 0) || !(p->alpha > 0) || !(p->alpha < 2)) return 0;
    if (!(p->max_iter > 0)) return 0;
    if (!(p->eps_abs >= 0) || !(p->eps_rel >= 0) || (p->eps_abs == 0 && p->eps_rel == 0)) return 0;
    if (!(p->eps_prim_inf > 0) || !(p->eps_dual_inf > 0)) return 0;
    if (p->scaling < 0 || p->check_termination < 0) return 0;
    if (p->adaptive_rho != 0 && p->adaptive_rho != 1) return 0;
    if (p->adaptive_rho_interval < 0 || !(p->adaptive_rho_tolerance >= 1)) return 0;
    return 1;
}

static double compute_rho_estimate(const work *w) {
    double pri_res = vec_norm_inf(w->z_prev, w->m);   /* scaled residuals left there by compute_*_res */
    double dua_res = vec_norm_inf(w->x_prev, w->n);
    double pri_norm = c_max(vec_norm_inf(w->z, w->m), vec_norm_inf(w->Ax, w->m));
    pri_res /= (pri_norm + 1e-10);
    double dua_norm = c_max(c_max(vec_norm_inf(w->q, w->n), vec_norm_inf(w->Aty, w->n)),
                            vec_norm_inf(w->Px, w->n));
    dua_res /= (dua_norm + 1e-10);
    double rho_estimate = w->rho * sqrt(pri_res / (dua_res + 1e-10));
    return c_min(c_max(rho_estimate, RHO_MIN), RHO_MAX);
}

int oracle_osqp_solve(const pqp_params *prm, const oqp_problem *qp, double *x_out, double *y_out,
                      oqp_info *info, double *trace, int trace_cap) {
    const int n = qp->n, m = qp->m;
    oqp_info local;
    if (!info) info = &local;
    memset(info, 0, sizeof(*info));
    info->status = PQP_UNSOLVED;
    /* osqp_setup refuses settings that fail validate_settings and bounds with l > u (validate_data) */
    int refused = !settings_valid(prm);
    for (int i = 0; i < m && !refused; ++i) refused = !(qp->l[i] <= qp->u[i]);
    if (refused) {
        info->status = PQP_INVALID_PROBLEM;
        for (int k = 0; k < n; ++k) x_out[k] = NAN;
        if (y_out) for (int k = 0; k < m; ++k) y_out[k] = NAN;
        return info->status;
    }
    work W;
    work *w = &W;
    memset(w, 0, sizeof(W));
    w->n = n; w->m = m;
    w->P = csc_from_triplets(n, n, qp->p_nnz, qp->p_i, qp->p_j, qp->p_v);
    w->A = csc_from_triplets(m, n, qp->a_nnz, qp->a_i, qp->a_j, qp->a_v);
    int *p_map = triplet_to_csc_map(n, qp->p_nnz, qp->p_j);
    int *a_map = triplet_to_csc_map(n, qp->a_nnz, qp->a_j);
    w->q = dalloc(n); w->l = dalloc(m); w->u = dalloc(m);
    memcpy(w->q, qp->q, sizeof(double) * (size_t)n);
    for (int i = 0; i < n; ++i) w->has_q |= qp->q[i] != 0.0;
    memcpy(w->l, qp->l, sizeof(double) * (size_t)m);
    memcpy(w->u, qp->u, sizeof(double) * (size_t)m);
    w->D = dalloc(n); w->Dinv = dalloc(n); w->E = dalloc(m); w->Einv = dalloc(m);
    w->rho_vec = dalloc(m); w->rho_inv_vec = dalloc(m);
    w->constr_type = (int *)calloc((size_t)(m > 0 ? m : 1), sizeof(int));
    w->x = dalloc(n); w->z = dalloc(m); w->y = dalloc(m);
    w->x_prev = dalloc(n); w->z_prev = dalloc(m);
    w->xz_tilde = dalloc(n + m); w->rhs = dalloc(n + m);
    w->Ax = dalloc(m); w->Px = dalloc(n); w->Aty = dalloc(n);
    w->delta_x = dalloc(n); w->delta_y = dalloc(m);
    w->Adelta_x = dalloc(m); w->Atdelta_y = dalloc(n); w->Pdelta_x = dalloc(n);
    w->D_temp = dalloc(n); w->D_temp_A = dalloc(n); w->E_temp = dalloc(m);

    if (prm->scaling > 0) scale_data(w, prm->scaling);
    else {
        for (int i = 0; i < n; ++i) { w->D[i] = w->Dinv[i] = 1; }
        for (int i = 0; i < m; ++i) { w->E[i] = w->Einv[i] = 1; }
        w->c = w->cinv = 1;
    }
    w->rho = prm->rho;
    set_rho_vec(w);

    const symbolic *sym = symbolic_get(qp);
    ldl *F = ldl_alloc(sym);
    info->kkt_n = sym->nn;
    info->kkt_lnz = sym->lnz;
    kkt_fill(w, qp, F, prm->sigma, p_map, a_map);
    int status = PQP_UNSOLVED;
    int iter = 0;
    double pri_res = 0, dua_res = 0;
    if (ldl_factor(F) != 0) {
        status = PQP_NON_CVX;
    } else {
        const double alpha = prm->alpha, sigma = prm->sigma;
        int can_check = 0;
        for (iter = 1; iter <= prm->max_iter; ++iter) {
            /* swap: x_prev <- x, z_prev <- z */
            double *t;
            t = w->x; w->x = w->x_prev; w->x_prev = t;
            t = w->z; w->z = w->z_prev; w->z_prev = t;
            /* update_xz_tilde */
            for (int i = 0; i < n; ++i) w->rhs[i] = sigma * w->x_prev[i] - w->q[i];
            for (int i = 0; i < m; ++i) w->rhs[n + i] = w->z_prev[i] - w->rho_inv_vec[i] * w->y[i];
            ldl_solve(F, w->rhs, w->xz_tilde);
            /* z_tilde = rhs_z + rho_inv * nu  (QDLDL solve_linsys: b[n+j] += rho_inv*sol[n+j]) */
            for (int i = 0; i < m; ++i) w->xz_tilde[n + i] = w->rhs[n + i] + w->rho_inv_vec[i] * w->xz_tilde[n + i];
            /* update_x */
            for (int i = 0; i < n; ++i) {
                w->x[i] = alpha * w->xz_tilde[i] + (1.0 - alpha) * w->x_prev[i];
                w->delta_x[i] = w->x[i] - w->x_prev[i];
            }
            /* update_z */
            for (int i = 0; i < m; ++i) {
                double v = alpha * w->xz_tilde[n + i] + (1.0 - alpha) * w->z_prev[i] + w->rho_inv_vec[i] * w->y[i];
                w->z[i] = c_min(c_max(v, w->l[i]), w->u[i]);
            }
            /* update_y */
            for (int i = 0; i < m; ++i) {
                w->delta_y[i] = w->rho_vec[i] * (alpha * w->xz_tilde[n + i] + (1.0 - alpha) * w->z_prev[i] - w->z[i]);
                w->y[i] += w->delta_y[i];
            }
            can_check = prm->check_termination && (iter % prm->check_termination == 0);
            if (can_check) {
                pri_res = compute_pri_res(w, w->x, w->z);
                dua_res = compute_dua_res(w, w->x, w->y);
                if (trace) {
                    int row = iter / prm->check_termination - 1;
                    if (row < trace_cap)
                        for (int i = 0; i < n; ++i) trace[(size_t)row * n + i] = w->D[i] * w->x[i];
                }
                w->margin = INFINITY;
                if (check_termination(w, prm, pri_res, dua_res, 0, &status)) break;
            }
            if (prm->adaptive_rho && prm->adaptive_rho_interval &&
                (iter % prm->adaptive_rho_interval == 0)) {
                if (!can_check) {
                    pri_res = compute_pri_res(w, w->x, w->z);
                    dua_res = compute_dua_res(w, w->x, w->y);
                }
                double rho_new = compute_rho_estimate(w);
                if (rho_new > w->rho * prm->adaptive_rho_tolerance ||
                    rho_new < w->rho / prm->adaptive_rho_tolerance) {
                    w->rho = c_min(c_max(rho_new, RHO_MIN), RHO_MAX);
                    for (int i = 0; i < m; ++i) {
                        if (w->constr_type[i] == 0) {
                            w->rho_vec[i] = w->rho;
                            w->rho_inv_vec[i] = 1.0 / w->rho;
                        } else if (w->constr_type[i] == 1) {
                            w->rho_vec[i] = RHO_EQ_OVER_RHO_INEQ * w->rho;
                            w->rho_inv_vec[i] = 1.0 / w->rho_vec[i];
                        }
                    }
                    kkt_fill(w, qp, F, sigma, p_map, a_map);
                    if (ldl_factor(F) != 0) { status = PQP_NON_CVX; break; }
                    info->rho_updates++;
                }
            }
        }
        if (iter > prm->max_iter) iter = prm->max_iter;
        if (status == PQP_UNSOLVED) {
            if (!can_check) {
                pri_res = compute_pri_res(w, w->x, w->z);
                dua_res = compute_dua_res(w, w->x, w->y);
                w->margin = INFINITY;
                check_termination(w, prm, pri_res, dua_res, 0, &status);
            }
            if (status == PQP_UNSOLVED) {
                if (!check_termination(w, prm, pri_res, dua_res, 1, &status)) status = PQP_MAX_ITER_REACHED;
            }
        }
    }
    info->status = status;
    info->iters = iter;
    info->rho_final = w->rho;
    info->pri_res = pri_res;
    info->dua_res = dua_res;
    info->margin = w->margin;
    /* store_solution: unscale; NaN when the status carries no solution */
    if (status == PQP_SOLVED || status == PQP_SOLVED_INACCURATE || status == PQP_MAX_ITER_REACHED) {
        for (int i = 0; i < n; ++i) x_out[i] = w->D[i] * w->x[i];
        if (y_out) for (int i = 0; i < m; ++i) y_out[i] = w->cinv * w->E[i] * w->y[i];
        /* objective 1/2 x'Px + q'x, unscaled */
        sym_triu_vec(w->P, w->x, w->Px);
        double obj = 0;
        for (int i = 0; i < n; ++i) obj += 0.5 * w->x[i] * w->Px[i] + w->q[i] * w->x[i];
        info->obj_val = obj * w->cinv;
    } else {
        for (int i = 0; i < n; ++i) x_out[i] = NAN;
        if (y_out) for (int i = 0; i < m; ++i) y_out[i] = NAN;
        info->obj_val = NAN;
    }
    ldl_free(F);
    free(p_map); free(a_map);
    csc_free(w->P); csc_free(w->A);
    free(w->q); free(w->l); free(w->u); free(w->D); free(w->Dinv); free(w->E); free(w->Einv);
    free(w->rho_vec); free(w->rho_inv_vec); free(w->constr_type);
    free(w->x); free(w->z); free(w->y); free(w->x_prev); free(w->z_prev); free(w->xz_tilde); free(w->rhs);
    free(w->Ax); free(w->Px); free(w->Aty); free(w->delta_x); free(w->delta_y);
    free(w->Adelta_x); free(w->Atdelta_y); free(w->Pdelta_x);
    free(w->D_temp); free(w->D_temp_A); free(w->E_temp);
    return status;
}
