"""Named verdict cases: every way OSQP 0.6 ends a run, picked from the oracle (TEST DATA).

OSQP decides a run's status at three places: at a check iteration (every check_termination-th), at max_iter with an
exact check when the last iteration was not a check iteration, and then, when neither has stopped the run, with
eps_abs, eps_rel and eps_prim_inf x 10.  The verdicts are discrete: a kernel that takes the wrong branch is wrong by a
whole status while its iterates still match.  These cases put each path into one named branch:

    solved_check / solved_final                            PQP_SOLVED at a check iteration / at an off-grid max_iter
    solved_inaccurate_check / solved_inaccurate_final      PQP_SOLVED_INACCURATE at max_iter on / off the check grid
    infeasible_check / infeasible_final                    PQP_PRIMAL_INFEASIBLE (exact certificate)
    infeasible_inaccurate_check / ..._final                PQP_PRIMAL_INFEASIBLE_INACCURATE (the 10x certificate)
    max_iter_check / max_iter_final                        PQP_MAX_ITER_REACHED

under every schedule of SCHEDULES.  Nothing is tuned by hand: a run's trajectory does not depend on check_termination,
so the oracle first runs the path with a check at every iteration, which gives the first iteration k1 where an exact
verdict holds; max_iter values below k1 then end in the 10x re-check (or MAX_ITER_REACHED), k1 itself off the check
grid ends in the final exact check, and a long run ends at a check iteration.  Each candidate is confirmed by running the
oracle on it.  A case whose deciding comparison lies closer than MIN_MARGIN (relative) to its threshold is dropped and
counted: its verdict would be a rounding coin flip, not a property of the kernel."""
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from oracle import oracle

MAX_ITER = 4000
MIN_MARGIN = 1e-9
RHO_MIN, RHO_MAX = 1e-6, 1e6

# name: (check_termination, adaptive_rho_interval, adaptive_rho).  "c25_a7": the adaptive interval does not divide the
# check interval, so max_iter can be an adaptation iteration that is not a check iteration.
SCHEDULES = {
    "c25_a25": (25, 25, 1), "c25_a7": (25, 7, 1), "c10_a25": (10, 25, 1), "c1_a1": (1, 1, 1), "c25_fixed": (25, 25, 0),
    "c0_a25": (0, 25, 1), "c0_a7": (0, 7, 1), "c0_a1": (0, 1, 1), "c0_fixed": (0, 25, 0),
}
FAMILY = {1: "solved", 2: "solved_inaccurate", -3: "infeasible", 3: "infeasible_inaccurate", -2: "max_iter"}
BRANCHES = sorted(f"{f}_{g}" for f in FAMILY.values() for g in ("check", "final"))

# Settings cases, each run through every branch under the "c25_a25" schedule: the near-1 tolerance regime (eps_abs =
# eps_rel = 0.5 and 1 are 5 and 10 after the x10) and large certificate tolerances.
SETTINGS = {
    "eps_0.5": dict(eps_abs=0.5, eps_rel=0.5),
    "eps_1": dict(eps_abs=1.0, eps_rel=1.0),
    "eps_prim_inf_0.1": dict(eps_prim_inf=0.1),
    "eps_prim_inf_1": dict(eps_prim_inf=1.0),
}


def infeasible(batch):
    """A copy of `batch` no path of which can be satisfied, in every formulation: the vehicle starts on the reference
    line (the x0 rows fix e_y = 0) while the hard rows of circles 0 and 2 demand an offset of 0.6..1.5 m everywhere."""
    b = dict(batch, bounds=batch["bounds"].copy(), x0=batch["x0"].copy())
    for f in ("c0", "c2"):
        b["bounds"][f + "_lb"] = 0.6
        b["bounds"][f + "_ub"] = 1.5
    b["x0"][:, 0] = 0.0
    return b


def kpc_limits(p, batch):
    """KPC limits (updateLimits through the oracle) from a speed profile without standstill, so that every limit is
    finite: a DBL_MAX bound scaled by E > 1 makes the oracle's certificate NaN (tests/test_gpu_envelope.py)."""
    ref = batch["ref"].copy()
    idx = np.arange(len(ref))
    ref["v"] = 4.0 + 3.0 * np.sin(idx * 0.05)
    ref["a"] = 0.5 * np.cos(idx * 0.05)
    return oracle.update_limits(p, ref)


def base_params(form, kind):
    """The settings a path kind ("feasible" / "infeasible") starts from.  The oracle certifies this infeasible
    corridor late in "K" (about 1900 iterations at eps_prim_inf 1e-4) and not within 4000 in "KPC"; eps_prim_inf 1e-2
    and 0.1 bring their certificates to a few hundred and about a thousand iterations."""
    p = oracle.default_params()
    if kind == "infeasible" and form != 0:
        p.eps_prim_inf = 1e-2 if form == 1 else 0.1
    return p


def params(base, schedule, max_iter, **over):
    check, interval, adaptive = SCHEDULES[schedule]
    p = base.copy()
    p.check_termination, p.adaptive_rho_interval, p.adaptive_rho, p.max_iter = check, interval, adaptive, max_iter
    for k, v in over.items():
        setattr(p, k, v)
    return p


def _solve(p, form, path, mk, mkp):
    r = oracle.solve_qp(p, form, path["ref"], path["bounds"], path["x0"], path["end_heading"], mk, mkp)
    return r["info"]


def _candidates(check, interval, adaptive, k1):
    """max_iter values to try, in order: a long run when there are checks (an exact verdict at a check iteration), k1
    (the final exact check when k1 is off the grid), the grid points and the off-grid points just below k1 (the 10x
    re-check), and small grid and off-grid values from 3 on (MAX_ITER_REACHED; 1 and 2 are covered by
    tests/envelope.py).  Off-grid values that are adaptation iterations come first."""
    on = (lambda t: check > 0 and t % check == 0)
    adapt = (lambda t: adaptive and interval > 0 and t % interval == 0)
    below = [t for t in range(k1 - 1, max(k1 - 60, 2), -1)]
    small = list(range(3, min(k1, 80)))
    out = ([MAX_ITER] if check > 0 else []) + [k1]
    out += [t for t in below if on(t)][:3]
    out += sorted([t for t in below if not on(t)], key=lambda t: not adapt(t))[:3]
    out += [t for t in small if on(t)][:3]
    out += sorted([t for t in small if not on(t)], key=lambda t: not adapt(t))[:3]
    return list(dict.fromkeys(out))


def pick(base, form, path, mk=None, mkp=None, schedules=SCHEDULES, over=None, label=""):
    """The cases of one path (a dict of one path's ref, bounds, x0, end_heading; mk, mkp its KPC limits): one per
    (schedule, branch) the path reaches.  Returns (cases, dropped): each case a dict(schedule, branch, params, status,
    iters, margin, rho_final, rho_updates, adapt_not_check)."""
    over = over or {}
    cases, dropped = [], 0
    for s in schedules:
        check, interval, adaptive = SCHEDULES[s]
        first = _solve(params(base, s, MAX_ITER, **dict(over, check_termination=1)), form, path, mk, mkp)
        if first.status not in (1, -3):
            continue
        seen = set()
        for t in _candidates(check, interval, adaptive, first.iters):
            p = params(base, s, t, **over)
            info = _solve(p, form, path, mk, mkp)
            if info.status not in FAMILY:
                continue
            grid = check > 0 and info.iters % check == 0
            if not grid and info.iters != t:
                continue
            branch = f"{FAMILY[info.status]}_{'check' if grid else 'final'}"
            if branch in seen:
                continue
            seen.add(branch)
            if not info.margin >= MIN_MARGIN:
                dropped += 1
                continue
            cases.append(dict(label=label, schedule=s, branch=branch, params=p, status=int(info.status),
                              iters=int(info.iters), margin=float(info.margin), rho_final=float(info.rho_final),
                              rho_updates=int(info.rho_updates),
                              adapt_not_check=bool(adaptive and interval and info.iters % interval == 0 and not grid)))
    return cases, dropped


def rho_clamp_path(batch):
    """A copy of `batch` whose QP x = 0 solves exactly: straight reference (kappa = 0), zero initial error, the goal
    heading along the reference, and corridors around the centre line.  Its first iteration leaves no primal residual,
    so OSQP's rho estimate is 0 and an adaptation there lands exactly on RHO_MIN."""
    b = dict(batch, ref=batch["ref"].copy(), bounds=batch["bounds"].copy(), x0=np.zeros_like(batch["x0"]))
    b["ref"]["k"] = 0.0
    b["ref"]["z"] = 0.0
    b["end_heading"] = np.zeros_like(batch["end_heading"])
    for f in ("c0", "c1", "c2", "c3"):
        b["bounds"][f + "_lb"] = -2.0
        b["bounds"][f + "_ub"] = 2.0
    return b


def batch_cases(form, batch, kinds=("feasible", "infeasible"), schedules=SCHEDULES, settings=SETTINGS, threads=1):
    """Every case of every path of `batch` in formulation `form`, both path kinds, every schedule, and the settings
    cases under "c25_a25".  Returns (cases, dropped, batches): each case carries `kind` and `path` (its index in
    batches[kind])."""
    jobs, batches = [], {}
    for kind in kinds:
        b = batch if kind == "feasible" else infeasible(batch)
        base = base_params(form, kind)
        mk, mkp = kpc_limits(base, b) if form == 2 else (None, None)
        batches[kind] = (b, mk, mkp)
        o = b["offsets"]
        for i in range(len(b["n_points"])):
            path = dict(ref=np.ascontiguousarray(b["ref"][o[i]:o[i + 1]]),
                        bounds=np.ascontiguousarray(b["bounds"][o[i]:o[i + 1]]), x0=b["x0"][i],
                        end_heading=float(b["end_heading"][i]))
            lim = (None, None) if mk is None else (np.ascontiguousarray(mk[o[i]:o[i + 1]]),
                                                   np.ascontiguousarray(mkp[o[i]:o[i + 1]]))
            jobs.append((kind, i, base, path, lim, schedules, None, ""))
            for name, over in settings.items():
                jobs.append((kind, i, base, path, lim, ("c25_a25",), over, name))

    def run(j):
        kind, i, base, path, lim, sch, over, label = j
        cs, dr = pick(base, form, path, *lim, schedules=sch, over=over, label=label)
        for c in cs:
            c.update(kind=kind, path=i)
        return cs, dr
    with ThreadPoolExecutor(max_workers=max(1, threads)) as ex:     # (ctypes releases the GIL in the oracle)
        results = list(ex.map(run, jobs))
    cases = [c for cs, _ in results for c in cs]
    return cases, sum(d for _, d in results), batches


# Settings OSQP 0.6's validate_settings refuses (osqp_setup fails, the reference's solve() returns false): one entry
# per rule, each a dict of pqp_params overrides on the defaults.
NAN = float("nan")
ILLEGAL = {
    "rho_0": dict(rho=0.0), "rho_neg": dict(rho=-0.1), "rho_nan": dict(rho=NAN),
    "sigma_0": dict(sigma=0.0), "sigma_nan": dict(sigma=NAN),
    "alpha_0": dict(alpha=0.0), "alpha_2": dict(alpha=2.0), "alpha_nan": dict(alpha=NAN),
    "max_iter_0": dict(max_iter=0), "max_iter_neg": dict(max_iter=-1),
    "eps_abs_neg": dict(eps_abs=-1e-3), "eps_abs_nan": dict(eps_abs=NAN),
    "eps_rel_neg": dict(eps_rel=-1e-3), "eps_rel_nan": dict(eps_rel=NAN),
    "eps_both_0": dict(eps_abs=0.0, eps_rel=0.0),
    "eps_prim_inf_0": dict(eps_prim_inf=0.0), "eps_prim_inf_nan": dict(eps_prim_inf=NAN),
    "eps_dual_inf_0": dict(eps_dual_inf=0.0), "eps_dual_inf_nan": dict(eps_dual_inf=NAN),
    "scaling_neg": dict(scaling=-1), "check_termination_neg": dict(check_termination=-1),
    "adaptive_rho_2": dict(adaptive_rho=2), "adaptive_rho_neg": dict(adaptive_rho=-1),
    "adaptive_rho_interval_neg": dict(adaptive_rho_interval=-1),
    "adaptive_rho_tolerance_0.5": dict(adaptive_rho_tolerance=0.5), "adaptive_rho_tolerance_nan": dict(adaptive_rho_tolerance=NAN),
}


def legal(p):
    """validate_settings restated on the fields of pqp_params (comparisons written so that a NaN fails)."""
    return bool(p.rho > 0 and p.sigma > 0 and 0 < p.alpha < 2 and p.max_iter > 0 and p.eps_abs >= 0 and p.eps_rel >= 0
                and not (p.eps_abs == 0 and p.eps_rel == 0) and p.eps_prim_inf > 0 and p.eps_dual_inf > 0
                and p.scaling >= 0 and p.check_termination >= 0 and p.adaptive_rho in (0, 1)
                and p.adaptive_rho_interval >= 0 and p.adaptive_rho_tolerance >= 1)


def one_per_branch(cases):
    """The cases a slow runner (the CPU emulator) takes: for every (kind, branch), the shortest case overall, the
    shortest without termination checks (check_termination 0), the shortest with fixed rho, and the shortest whose
    max_iter is an adaptation iteration but not a check iteration."""
    picks = {}
    tags = {"any": lambda c: True, "check0": lambda c: c["params"].check_termination == 0,
            "fixed_rho": lambda c: c["params"].adaptive_rho == 0, "adapt_not_check": lambda c: c["adapt_not_check"]}
    for c in sorted(cases, key=lambda c: c["iters"]):
        for tag, f in tags.items():
            if f(c):
                picks.setdefault((c["kind"], c["branch"], tag), c)
    return list({id(c): c for c in picks.values()}.values())
