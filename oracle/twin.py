"""Independent numpy/scipy twin of the CPU oracle (TEST INFRASTRUCTURE, not product code).

Purpose: the C oracle (pqp_oracle_*.c) is what the CUDA path is judged against, and no real OSQP
exists in this environment to pin it (PARITY UNPINNED, see pqp_oracle.h).  This twin re-derives
the same two things by a different route so that an implementation slip in the C code shows up:

  * assembly: written in the reference's own dense-block style (numpy dense matrices filled
    block by block like the Eigen code in src/solver/solver_*.cpp), then compared entry by entry
    with the C oracle's triplets;
  * OSQP recurrence: scipy.sparse + SuperLU (partial pivoting) on the KKT matrix instead of the
    C oracle's pivot-free LDL', vectorised numpy for everything else.

It also offers a KKT-certificate checker and a tight-tolerance "optimum" solve.
"""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

INFTY = 1e30
RHO_MIN, RHO_MAX, RHO_EQ_OVER_RHO_INEQ, RHO_TOL = 1e-6, 1e6, 1e3, 1e-4
MIN_SCALING, MAX_SCALING = 1e-4, 1e4


def constraint_angle(a):
    """tools.hpp:24-35"""
    while a > np.pi:
        a -= 2 * np.pi
    while a < -np.pi:
        a += 2 * np.pi
    return a


def keep_control_steps(ref):
    """solver.cpp:21-27 + solver_kp_as_input.cpp:17.  std::max skips a NaN interval; int(1.2 / interval) saturates at
    INT_MAX (a zero interval) as pqp_keep_control_steps does."""
    if len(ref) < 2:
        return 1
    interval = 0.0
    for i in range(1, min(len(ref), 10)):
        d = float(ref["s"][i]) - float(ref["s"][i - 1])
        interval = d if interval < d else interval
    with np.errstate(divide="ignore"):
        q = float(np.float64(1.2) / np.float64(interval))
    keep = 0 if q != q else (int(q) if q < 2147483647.0 else 2147483647)
    return max(keep, 1)


def _end_window(prm, end_heading, ref):
    lo, hi = -INFTY, INFTY
    if prm.constraint_end_heading:
        end_psi = constraint_angle(end_heading - float(ref["z"][-1]))
        if end_psi < 70 * np.pi / 180:
            lo, hi = end_psi - 5 * np.pi / 180, end_psi + 5 * np.pi / 180
    return lo, hi


def assemble_kp(prm, ref, bounds, x0, end_heading):
    """solver_kp_as_input.cpp:13-203 in dense-block style.  Returns (P, q, A, l, u) dense."""
    N = len(ref)
    keep = keep_control_steps(ref)
    ch = (N + keep - 2) // keep
    ns, nc, nsl = 3 * N, ch, 2 * N
    n, m = ns + nc + nsl, 11 * N + ch + 2
    H = np.zeros((n, n))
    for i in range(N):
        H[3 * i, 3 * i] += prm.KP_deviation_weight
        H[3 * i + 2, 3 * i + 2] += prm.KP_curvature_weight
        H[ns + nc + i, ns + nc + i] += prm.KP_slack_weight
        H[ns + nc + N + i, ns + nc + N + i] += prm.KP_slack_weight
    for j in range(ch):
        H[ns + j, ns + j] += keep * prm.KP_curvature_rate_weight
    vars_b = 3 * N
    coll_b = vars_b + 2 * N + ch
    end_b = coll_b + 6 * N
    cons = np.zeros((m, n))
    cons[np.arange(ns), np.arange(ns)] = -1
    a = np.zeros((3, 3)); a[0, 1] = 1; a[1, 2] = 1
    bvec = np.array([0.0, 0.0, 1.0])
    lo = np.zeros(m); up = np.zeros(m)
    for i in range(N - 1):
        ref_k = float(ref["k"][i])
        ds = float(ref["s"][i + 1]) - float(ref["s"][i])
        ref_kp = (float(ref["k"][i + 1]) - ref_k) / ds
        a[1, 0] = -ref_k ** 2
        cons[3 * (i + 1):3 * (i + 1) + 3, 3 * i:3 * i + 3] = a * ds + np.eye(3)
        cons[3 * (i + 1):3 * (i + 1) + 3, ns + i // keep] = bvec * ds
        c = np.array([0.0, 0.0, ref_kp]); ref_state = np.array([0.0, 0.0, ref_k])
        c_i = ds * (c - a @ ref_state - bvec * ref_kp)
        lo[3 * (i + 1):3 * (i + 1) + 3] = -c_i
        up[3 * (i + 1):3 * (i + 1) + 3] = -c_i
    for i in range(N):
        cons[vars_b + i, 3 * i + 2] = 1
        cons[vars_b + N + ch + i, ns + nc + i] = 1
    for j in range(ch):
        cons[vars_b + N + j, ns + j] = 1
    for i in range(N):
        cons[coll_b + 2 * i:coll_b + 2 * i + 2, 3 * i:3 * i + 2] = [[1, prm.d1], [1, prm.d3]]
        for blk, d, sgn in ((2, prm.d4, -1), (3, prm.d4, 1), (4, prm.d2, -1), (5, prm.d2, 1)):
            r = coll_b + blk * N + i
            cons[r, 3 * i:3 * i + 2] = [1, d]
            cons[r, ns + nc + i] = sgn
    cons[end_b, ns - 3] = 1
    cons[end_b + 1, ns - 2] = 1
    lo[0:3] = -np.asarray(x0); up[0:3] = -np.asarray(x0)
    kmax = np.tan(prm.max_steering_angle) / prm.wheel_base
    mg = prm.expected_safety_margin
    for i in range(N):
        lo[vars_b + i], up[vars_b + i] = -kmax, kmax
        lo[vars_b + N + ch + i], up[vars_b + N + ch + i] = 0, mg
    lo[vars_b + N:vars_b + N + ch] = -INFTY
    up[vars_b + N:vars_b + N + ch] = INFTY
    for i in range(N):
        b = bounds[i]
        lo[coll_b + 2 * i], up[coll_b + 2 * i] = b["c0_lb"], b["c0_ub"]
        lo[coll_b + 2 * i + 1], up[coll_b + 2 * i + 1] = b["c2_lb"], b["c2_ub"]
        up[coll_b + 2 * N + i] = b["c3_ub"] - mg; lo[coll_b + 2 * N + i] = -INFTY
        lo[coll_b + 3 * N + i] = b["c3_lb"] + mg; up[coll_b + 3 * N + i] = INFTY
        up[coll_b + 4 * N + i] = b["c1_ub"] - mg; lo[coll_b + 4 * N + i] = -INFTY
        lo[coll_b + 5 * N + i] = b["c1_lb"] + mg; up[coll_b + 5 * N + i] = INFTY
    lo[end_b], up[end_b] = -1, 1
    lo[end_b + 1], up[end_b + 1] = _end_window(prm, end_heading, ref)
    return H, np.zeros(n), cons, lo, up


def assemble_k(prm, ref, bounds, x0, end_heading):
    """solver_k_as_input.cpp:14-207 in dense-block style (its own Eigen block fills, one numpy statement each).
    Variables [(e_phi, e_y)_i ; delta_i ; slack_i]; returns (P, q, A, l, u) dense."""
    N = len(ref)
    state, control, slack = 2 * N, N - 1, N
    n, m = 4 * N - 1, 11 * N - 1
    w_c, w_cr, w_pq, w_e = prm.K_curvature_weight, prm.K_curvature_rate_weight, prm.K_deviation_weight, prm.KP_slack_weight
    H = np.zeros((n, n))
    Q = np.array([[0.0, 0.0], [0.0, w_pq]])
    R = np.zeros((control, control))
    for i in range(control):            # :60-72
        for j in range(control):
            if i == j:
                R[i, j] = (w_c + w_cr) if (i == 0 or i == control - 1) else (w_cr * 2 + w_c)
            elif i == j - 1 or i == j + 1:
                R[i, j] = -w_cr
    for i in range(N):
        H[2 * i:2 * i + 2, 2 * i:2 * i + 2] = Q
    H[2 * N:2 * N + control, 2 * N:2 * N + control] = R
    H[3 * N - 1:3 * N - 1 + slack, 3 * N - 1:3 * N - 1 + slack] = np.eye(slack) * w_e
    cons = np.zeros((m, n))
    cons[np.arange(2 * N), np.arange(2 * N)] = -1                      # :112-114
    lo = np.zeros(m); up = np.zeros(m)
    for i in range(N - 1):                                              # setDynamicMatrix :89-103
        ref_k = float(ref["k"][i])
        ref_s = float(ref["s"][i + 1]) - float(ref["s"][i])
        ref_delta = np.arctan(ref_k * prm.wheel_base)
        a = np.array([[1.0, -ref_s * ref_k ** 2], [ref_s, 1.0]])
        b = np.array([ref_s / prm.wheel_base / np.cos(ref_delta) ** 2, 0.0])
        cons[2 * (i + 1):2 * (i + 1) + 2, 2 * i:2 * i + 2] = a
        cons[2 * (i + 1):2 * (i + 1) + 2, 2 * N + i] = b
    cons[2 * N + np.arange(n), np.arange(n)] = 1                         # :124-126
    coll = np.array([[prm.d1, 1.0], [prm.d3, 1.0], [prm.d4, 1.0]])       # :129-136
    for i in range(N):
        cons[6 * N - 1 + 3 * i:6 * N - 1 + 3 * i + 3, 2 * i:2 * i + 2] = coll
        cons[9 * N - 1 + i, 2 * i:2 * i + 2] = [prm.d2, 1.0]
        cons[10 * N - 1 + i, 2 * i:2 * i + 2] = [prm.d2, 1.0]
    cons[9 * N - 1:10 * N - 1, 3 * N - 1:4 * N - 1] = -np.eye(N)
    cons[10 * N - 1:11 * N - 1, 3 * N - 1:4 * N - 1] = np.eye(N)
    # bounds :151-206
    lo[0:2] = [-x0[1], -x0[0]]; up[0:2] = lo[0:2]
    for i in range(N - 1):
        ds = float(ref["s"][i + 1]) - float(ref["s"][i])
        steer = np.arctan(float(ref["k"][i]) * prm.wheel_base)
        c = ds * steer / prm.wheel_base / np.cos(steer) ** 2
        lo[2 + 2 * i], up[2 + 2 * i] = c, c
    lo[2 * N:4 * N] = -INFTY; up[2 * N:4 * N] = INFTY
    if prm.constraint_end_heading:
        end_psi = constraint_angle(end_heading - float(ref["z"][-1]))
        if end_psi < 70 * np.pi / 180:
            lo[2 * N + 2 * N - 2] = end_psi - 5 * np.pi / 180
            up[2 * N + 2 * N - 2] = end_psi + 5 * np.pi / 180
    lo[4 * N:5 * N - 1] = -prm.max_steering_angle; up[4 * N:5 * N - 1] = prm.max_steering_angle
    lo[5 * N - 1:6 * N - 1] = 0; up[5 * N - 1:6 * N - 1] = prm.expected_safety_margin
    for i in range(N):
        bd = bounds[i]
        up[6 * N - 1 + 3 * i:6 * N - 1 + 3 * i + 3] = [bd["c0_ub"], bd["c2_ub"], bd["c3_ub"]]
        lo[6 * N - 1 + 3 * i:6 * N - 1 + 3 * i + 3] = [bd["c0_lb"], bd["c2_lb"], bd["c3_lb"]]
        up[9 * N - 1 + i] = bd["c1_ub"] - prm.expected_safety_margin
        lo[10 * N - 1 + i] = bd["c1_lb"] + prm.expected_safety_margin
    up[10 * N - 1:11 * N - 1] = INFTY
    lo[9 * N - 1:10 * N - 1] = -INFTY
    return H, np.zeros(n), cons, lo, up


def assemble_kpc(prm, ref, bounds, x0, end_heading, max_k, max_kp):
    """solver_kp_as_input_constrained.cpp:13-221 in dense-block style.  keep_control_steps_ = 4 (:17).
    Returns (P, q, A, l, u) dense."""
    N = len(ref)
    keep = 4
    ch = (N + keep - 2) // keep
    ns, nc, nsl = 3 * N, ch, 3 * N
    n, m = ns + nc + nsl, 12 * N + 3 * ch + 2
    H = np.zeros((n, n))
    w_k_slack, w_kp_slack = 500.0, 25000.0
    for i in range(N):                                                   # :54-59
        H[3 * i, 3 * i] += prm.KP_deviation_weight
        H[3 * i + 2, 3 * i + 2] += prm.KP_curvature_weight
        H[ns + nc + i, ns + nc + i] += prm.KP_slack_weight
        H[ns + nc + N + i, ns + nc + N + i] += w_k_slack
    for j in range(ch):                                                  # :60-64
        H[ns + j, ns + j] += keep * prm.KP_curvature_rate_weight
        H[ns + nc + 2 * N + j, ns + nc + 2 * N + j] += w_kp_slack * keep
    kl_b = 3 * N; ku_b = kl_b + N; kpl_b = ku_b + N; kpu_b = kpl_b + ch
    slack_b = kpu_b + ch; coll_b = slack_b + 2 * N + ch; end_b = coll_b + 5 * N
    cons = np.zeros((m, n))
    cons[np.arange(ns), np.arange(ns)] = -1
    a = np.zeros((3, 3)); a[0, 1] = 1; a[1, 2] = 1
    bvec = np.array([0.0, 0.0, 1.0])
    lo = np.zeros(m); up = np.zeros(m)
    for i in range(N - 1):                                               # :86-102
        ref_k = float(ref["k"][i])
        ds = float(ref["s"][i + 1]) - float(ref["s"][i])
        ref_kp = (float(ref["k"][i + 1]) - ref_k) / ds
        a[1, 0] = -ref_k ** 2
        cons[3 * (i + 1):3 * (i + 1) + 3, 3 * i:3 * i + 3] = a * ds + np.eye(3)
        cons[3 * (i + 1):3 * (i + 1) + 3, ns + i // keep] = bvec * ds
        c = np.array([0.0, 0.0, ref_kp]); ref_state = np.array([0.0, 0.0, ref_k])
        c_i = ds * (c - a @ ref_state - bvec * ref_kp)
        lo[3 * (i + 1):3 * (i + 1) + 3] = -c_i
        up[3 * (i + 1):3 * (i + 1) + 3] = -c_i
    for i in range(N):                                                   # :106-113
        cons[kl_b + i, 3 * i + 2] = 1
        cons[kl_b + i, ns + nc + N + i] = 1
        cons[ku_b + i, 3 * i + 2] = 1
        cons[ku_b + i, ns + nc + N + i] = -1
        cons[slack_b + i, ns + nc + i] = 1
        cons[slack_b + N + i, ns + nc + N + i] = 1
    for j in range(ch):                                                  # :115-121
        cons[kpl_b + j, ns + j] = 1
        cons[kpl_b + j, ns + nc + 2 * N + j] = 1
        cons[kpu_b + j, ns + j] = 1
        cons[kpu_b + j, ns + nc + 2 * N + j] = -1
        cons[slack_b + 2 * N + j, ns + nc + 2 * N + j] = 1
    coll = np.array([[1.0, prm.d1], [1.0, prm.d2], [1.0, prm.d4]])       # :124-131
    for i in range(N):
        cons[coll_b + 3 * i:coll_b + 3 * i + 3, 3 * i:3 * i + 2] = coll
        cons[coll_b + 3 * N + i, 3 * i:3 * i + 2] = [1.0, prm.d3]
        cons[coll_b + 3 * N + i, ns + nc + i] = -1
        cons[coll_b + 4 * N + i, 3 * i:3 * i + 2] = [1.0, prm.d3]
        cons[coll_b + 4 * N + i, ns + nc + i] = 1
    cons[end_b, ns - 3] = 1
    cons[end_b + 1, ns - 2] = 1
    lo[0:3] = -np.asarray(x0); up[0:3] = -np.asarray(x0)
    kmax = np.tan(prm.max_steering_angle) / prm.wheel_base
    mg = prm.expected_safety_margin
    for i in range(N):                                                   # :160-172
        lo[kl_b + i], up[kl_b + i] = -max_k[i], INFTY
        lo[ku_b + i], up[ku_b + i] = -INFTY, max_k[i]
        lo[slack_b + i], up[slack_b + i] = 0, mg
        lo[slack_b + N + i], up[slack_b + N + i] = 0, max(kmax - max_k[i], 0.0)
    for j in range(ch):                                                  # :173-182
        lo[kpl_b + j], up[kpl_b + j] = -max_kp[j], INFTY
        lo[kpu_b + j], up[kpu_b + j] = -INFTY, max_kp[j]
        lo[slack_b + 2 * N + j], up[slack_b + 2 * N + j] = 0, INFTY
    for i in range(N):                                                   # :185-200
        bd = bounds[i]
        up[coll_b + 3 * i:coll_b + 3 * i + 3] = [bd["c0_ub"], bd["c1_ub"], bd["c3_ub"]]
        lo[coll_b + 3 * i:coll_b + 3 * i + 3] = [bd["c0_lb"], bd["c1_lb"], bd["c3_lb"]]
        up[coll_b + 3 * N + i] = bd["c2_ub"] - mg; lo[coll_b + 3 * N + i] = -INFTY
        lo[coll_b + 4 * N + i] = bd["c2_lb"] + mg; up[coll_b + 4 * N + i] = INFTY
    lo[end_b], up[end_b] = -INFTY, INFTY                                 # :204-205: end e_y is not constrained
    lo[end_b + 1], up[end_b + 1] = _end_window(prm, end_heading, ref)
    return H, np.zeros(n), cons, lo, up


def _limit(v):
    v = np.where(v < MIN_SCALING, 1.0, v)
    return np.where(v > MAX_SCALING, MAX_SCALING, v)


def _rel_gap(a, b):
    """Relative distance of a compared value from its threshold (0 when the comparison is a coin flip)."""
    d = max(abs(a), abs(b))
    return abs(a - b) / d if d > 0 else 0.0


def osqp_twin(prm, P, q, A, l, u, eps=None, max_iter=None, trace_every=0):
    """OSQP 0.6.x recurrence on dense/sparse (P full symmetric, A), through the end of osqp_solve: the checks inside
    the loop, the exact check after it when the last iteration was not a check iteration, and the re-check with
    eps_abs, eps_rel and eps_prim_inf x 10 when nothing has stopped the run.  Returns dict(x, y, iters, status,
    rho_updates, rho, trace, decision): x and y are NaN when the status carries no solution (store_solution), and
    `decision` holds the residuals and tolerances of the deciding check(s) with `margin`, the smallest relative gap
    between a compared value and its threshold there."""
    P = sp.csc_matrix(P); A = sp.csc_matrix(A)
    n, m = P.shape[0], A.shape[0]
    q = np.array(q, dtype=float); l = np.array(l, dtype=float); u = np.array(u, dtype=float)
    eps_abs = prm.eps_abs if eps is None else eps
    eps_rel = prm.eps_rel if eps is None else eps
    max_iter = prm.max_iter if max_iter is None else max_iter
    if np.any(l > u) or max_iter < 1:
        return dict(x=np.full(n, np.nan), y=np.full(m, np.nan), iters=0, status=-100, rho_updates=0)
    D = np.ones(n); E = np.ones(m); c = 1.0
    for _ in range(prm.scaling):
        absP, absA = abs(P), abs(A)
        colP = np.asarray(absP.max(axis=0).todense()).ravel()
        colA = np.asarray(absA.max(axis=0).todense()).ravel() if m else np.zeros(n)
        rowA = np.asarray(absA.max(axis=1).todense()).ravel() if m else np.zeros(0)
        Dt = 1.0 / np.sqrt(_limit(np.maximum(colP, colA)))
        Et = 1.0 / np.sqrt(_limit(rowA))
        P = sp.diags(Dt) @ P @ sp.diags(Dt)
        A = sp.diags(Et) @ A @ sp.diags(Dt)
        q = Dt * q
        D *= Dt; E *= Et
        colP = np.asarray(abs(P).max(axis=0).todense()).ravel()
        ct = max(colP.mean(), float(_limit(np.array([np.abs(q).max()]))[0]))
        ct = 1.0 / float(_limit(np.array([ct]))[0])
        P = P * ct; q = q * ct; c *= ct
    P = sp.csc_matrix(P); A = sp.csc_matrix(A)
    l = E * l; u = E * u
    rho = min(max(prm.rho, RHO_MIN), RHO_MAX)
    ctype = np.zeros(m, dtype=int)
    free = (l < -INFTY * MIN_SCALING) & (u > INFTY * MIN_SCALING)
    eq = ~free & (u - l < RHO_TOL)
    ctype[free] = -1; ctype[eq] = 1

    def rho_vector(r):
        v = np.full(m, r)
        v[ctype == 1] = RHO_EQ_OVER_RHO_INEQ * r
        v[ctype == -1] = RHO_MIN
        return v

    def factor(rv):
        K = sp.bmat([[P + prm.sigma * sp.identity(n), A.T], [A, -sp.diags(1.0 / rv)]], format="csc")
        return spla.splu(K)

    rho_vec = rho_vector(rho)
    lu = factor(rho_vec)
    x = np.zeros(n); z = np.zeros(m); y = np.zeros(m); dy = np.zeros(m)
    Dinv, Einv, cinv = 1.0 / D, 1.0 / E, 1.0 / c
    ninf = lambda v: np.abs(v).max() if len(v) else 0.0  # noqa: E731
    uinf, linf = u > INFTY * MIN_SCALING, l < -INFTY * MIN_SCALING

    def residuals():
        Ax = A @ x; Px = P @ x; Aty = A.T @ y
        return dict(Ax=Ax, Px=Px, Aty=Aty, rp=Ax - z, rd=q + Px + Aty,
                    pri_res=ninf(Einv * (Ax - z)), dua_res=cinv * ninf(Dinv * (q + Px + Aty)))

    def check(r, approximate, gaps):
        """check_termination(work, approximate): a status, or None to go on.  q = 0 for this path, so the dual
        infeasibility certificate is dead.  Appends the relative gap of every comparison it makes to `gaps`."""
        k = 10.0 if approximate else 1.0
        ea, er, ep = k * eps_abs, k * eps_rel, k * prm.eps_prim_inf
        if r["pri_res"] > INFTY or r["dua_res"] > INFTY:
            return -7
        eps_p = ea + er * max(ninf(Einv * z), ninf(Einv * r["Ax"]))
        eps_d = ea + er * cinv * max(ninf(Dinv * q), ninf(Dinv * r["Aty"]), ninf(Dinv * r["Px"]))
        r.update(eps_pri=eps_p, eps_dua=eps_d)
        prim_ok = r["pri_res"] < eps_p
        dua_ok = r["dua_res"] < eps_d
        gaps += [_rel_gap(r["pri_res"], eps_p), _rel_gap(r["dua_res"], eps_d)]
        if prim_ok and dua_ok:
            return 2 if approximate else 1
        if not prim_ok:
            # primal infeasibility certificate on delta y, projected onto the polar of the bounds' recession cone
            d = dy.copy()
            d[uinf & linf] = 0
            d[uinf & ~linf] = np.minimum(d[uinf & ~linf], 0)
            d[~uinf & linf] = np.maximum(d[~uinf & linf], 0)
            nd = ninf(E * d)
            gaps.append(_rel_gap(nd, ep))
            if nd > ep:
                lhs = np.sum(u * np.maximum(d, 0) + l * np.minimum(d, 0))
                gaps.append(_rel_gap(lhs, -ep * nd))
                if lhs < -ep * nd:
                    cert = ninf(Dinv * (A.T @ d))
                    gaps.append(_rel_gap(cert, ep * nd))
                    if cert < ep * nd:
                        return 3 if approximate else -3
        return None

    status, rho_updates, it = None, 0, 0
    trace = []
    r, gaps = None, []
    can_check = False
    for it in range(1, max_iter + 1):
        xp, zp = x, z
        rhs = np.concatenate([prm.sigma * xp - q, zp - y / rho_vec])
        sol = lu.solve(rhs)
        xt = sol[:n]
        zt = rhs[n:] + sol[n:] / rho_vec
        x = prm.alpha * xt + (1 - prm.alpha) * xp
        zr = prm.alpha * zt + (1 - prm.alpha) * zp
        z = np.minimum(np.maximum(zr + y / rho_vec, l), u)
        dy = rho_vec * (zr - z)
        y = y + dy
        can_check = bool(prm.check_termination) and it % prm.check_termination == 0
        can_adapt = prm.adaptive_rho and prm.adaptive_rho_interval and it % prm.adaptive_rho_interval == 0
        if can_check or can_adapt:
            r = residuals()
        if can_check:
            if trace_every and (it // prm.check_termination) % trace_every == 0:
                trace.append(D * x)
            gaps = []
            status = check(r, False, gaps)
            if status is not None:
                break
        if can_adapt:
            pn = ninf(r["rp"]) / (max(ninf(z), ninf(r["Ax"])) + 1e-10)
            dn = ninf(r["rd"]) / (max(ninf(q), ninf(r["Aty"]), ninf(r["Px"])) + 1e-10)
            rho_new = min(max(rho * np.sqrt(pn / (dn + 1e-10)), RHO_MIN), RHO_MAX)
            if rho_new > rho * prm.adaptive_rho_tolerance or rho_new < rho / prm.adaptive_rho_tolerance:
                rho = rho_new
                rho_vec = rho_vector(rho)
                lu = factor(rho_vec)
                rho_updates += 1
    exact = None
    if status is None:
        if not can_check:                   # the last iteration was not a check iteration: check it exactly now
            r, gaps = residuals(), []
            status = check(r, False, gaps)
        if status is None:                  # max_iter reached: the 10x re-check
            exact = dict(pri_res=r["pri_res"], dua_res=r["dua_res"], eps_pri=r["eps_pri"], eps_dua=r["eps_dua"])
            status = check(r, True, gaps)
            if status is None:
                status = -2
    decision = dict(pri_res=r["pri_res"], dua_res=r["dua_res"], eps_pri=r.get("eps_pri"), eps_dua=r.get("eps_dua"),
                    exact=exact, margin=min(gaps) if gaps else np.inf)
    has_sol = status in (1, 2, -2)
    return dict(x=D * x if has_sol else np.full(n, np.nan), y=cinv * E * y if has_sol else np.full(m, np.nan),
                iters=it, status=status, rho_updates=rho_updates, rho=rho, trace=np.array(trace), decision=decision)


def kkt_certificate(P, q, A, l, u, x, y):
    """Optimality residuals of (x, y) for min 1/2x'Px+q'x, l<=Ax<=u (unscaled):
    returns dict(primal, dual, comp): max bound violation, ||Px+q+A'y||_inf and the worst
    complementarity slack |min(y+,u-Ax)|, |min(y-,Ax-l)|."""
    Ax = A @ x
    primal = max(np.max(np.maximum(Ax - u, 0)), np.max(np.maximum(l - Ax, 0)))
    dual = np.max(np.abs(P @ x + q + A.T @ y))
    yp, ym = np.maximum(y, 0), np.maximum(-y, 0)
    fin_u, fin_l = u < 1e29, l > -1e29
    comp_u = np.max(np.minimum(yp[fin_u], np.abs(u[fin_u] - Ax[fin_u]))) if fin_u.any() else 0.0
    comp_l = np.max(np.minimum(ym[fin_l], np.abs(Ax[fin_l] - l[fin_l]))) if fin_l.any() else 0.0
    bad_inf = max(np.max(yp[~fin_u]) if (~fin_u).any() else 0.0, np.max(ym[~fin_l]) if (~fin_l).any() else 0.0)
    return dict(primal=float(primal), dual=float(dual), comp=float(max(comp_u, comp_l, bad_inf)))
