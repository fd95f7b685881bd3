"""ctypes loader for the CPU oracle (``oracle/_build/libpqp_oracle.so``).

TEST INFRASTRUCTURE, not product code: only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / ``--impl reference`` leg may import this.  PARITY UNPINNED (see pqp_oracle.h).
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(_HERE))
from path_optimizer_b200.abi import BOUNDS_DTYPE, STATE_DTYPE, DistanceMap, Params, ptr  # noqa: E402

_LIB_PATH = os.path.join(_HERE, "_build", "libpqp_oracle.so")


class OqpInfo(C.Structure):
    _fields_ = [("status", C.c_int), ("iters", C.c_int), ("rho_updates", C.c_int),
                ("rho_final", C.c_double), ("pri_res", C.c_double), ("dua_res", C.c_double),
                ("obj_val", C.c_double), ("kkt_n", C.c_int), ("kkt_lnz", C.c_int), ("margin", C.c_double)]


class OqpProblem(C.Structure):
    _fields_ = [("n", C.c_int), ("m", C.c_int), ("p_nnz", C.c_int), ("a_nnz", C.c_int),
                ("p_i", C.POINTER(C.c_int)), ("p_j", C.POINTER(C.c_int)), ("p_v", C.POINTER(C.c_double)),
                ("a_i", C.POINTER(C.c_int)), ("a_j", C.POINTER(C.c_int)), ("a_v", C.POINTER(C.c_double)),
                ("q", C.POINTER(C.c_double)), ("l", C.POINTER(C.c_double)), ("u", C.POINTER(C.c_double))]


def build(force=False):
    """(Re)build the oracle library with the committed Makefile when missing or stale."""
    srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith((".c", ".h"))]
    srcs.append(os.path.join(os.path.dirname(_HERE), "include", "pqp.h"))
    srcs.append(os.path.join(os.path.dirname(_HERE), "include", "pqp_env.h"))
    stale = (not os.path.exists(_LIB_PATH)
             or any(os.path.getmtime(s) > os.path.getmtime(_LIB_PATH) for s in srcs))
    if force or stale:
        subprocess.run(["make", "-C", _HERE] + (["-B"] if force else []), check=True,
                       stdout=subprocess.DEVNULL)
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        L.oracle_params_default.argtypes = [C.POINTER(Params)]
        L.oracle_params_default.restype = None
        L.oracle_keep_control_steps.argtypes = [C.c_int, C.c_void_p, C.c_int]
        L.oracle_keep_control_steps.restype = C.c_int
        L.oracle_assemble.restype = C.POINTER(OqpProblem)
        L.oracle_assemble.argtypes = [C.POINTER(Params), C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_double, C.c_void_p, C.c_void_p]
        L.oracle_problem_free.argtypes = [C.POINTER(OqpProblem)]
        L.oracle_problem_free.restype = None
        L.oracle_osqp_solve.argtypes = [C.POINTER(Params), C.POINTER(OqpProblem), C.c_void_p,
                                        C.c_void_p, C.POINTER(OqpInfo), C.c_void_p, C.c_int]
        L.oracle_osqp_solve.restype = C.c_int
        L.oracle_extract.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.oracle_extract.restype = None
        L.oracle_solve_path.argtypes = [C.POINTER(Params), C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.POINTER(OqpInfo)]
        L.oracle_solve_path.restype = C.c_int
        L.oracle_solve_batch.argtypes = [C.POINTER(Params), C.c_int, C.c_int] + [C.c_void_p] * 11 + [C.c_int]
        L.oracle_solve_batch.restype = C.c_double
        # stages either side of the QP (pqp_oracle_env.c)
        vp, dm, pp = C.c_void_p, C.POINTER(DistanceMap), C.POINTER(Params)
        L.oracle_map_inside.argtypes = [dm, C.c_double, C.c_double]
        L.oracle_map_distance.argtypes = [dm, C.c_double, C.c_double]
        L.oracle_map_distance.restype = C.c_double
        L.oracle_spline_fit.argtypes = [C.c_int, vp, vp, vp]
        L.oracle_spline_eval.argtypes = [C.c_int, vp, vp, C.c_int, C.c_double]
        L.oracle_spline_eval.restype = C.c_double
        L.oracle_clearance_strict.argtypes = [pp, dm, C.c_double, C.c_double, C.c_double, vp]
        L.oracle_clearance_strict.restype = None
        L.oracle_update_bounds.argtypes = [pp, dm, C.c_int, C.c_int, vp, C.c_int, vp, vp, vp, vp]
        L.oracle_car_circles.argtypes = [pp, vp]
        L.oracle_update_limits.argtypes = [pp, C.c_int, C.c_int, vp, vp, vp]
        L.oracle_update_limits.restype = None
        L.oracle_car_circles.restype = None
        L.oracle_state_collision_free.argtypes = [pp, dm, vp]
        L.oracle_finish_raw.argtypes = [pp, dm, C.c_int, vp, C.c_int, C.POINTER(C.c_int)]
        L.oracle_densify.argtypes = [pp, dm, C.c_int, vp, C.c_double, C.c_int, C.c_int, vp, C.POINTER(C.c_int)]
        L.oracle_plan_path.argtypes = ([pp, dm] + [C.c_int] * 4 + [vp, C.c_int, vp, vp, vp, vp, C.c_double,
                                       C.c_double, C.c_int, C.c_int, vp, C.POINTER(C.c_int), C.POINTER(C.c_int),
                                       C.POINTER(C.c_int), vp])
        _lib = L
    return _lib


def default_params():
    p = Params()
    lib().oracle_params_default(C.byref(p))
    return p


def keep_control_steps(formulation, ref):
    ref = np.ascontiguousarray(ref, dtype=STATE_DTYPE)
    return lib().oracle_keep_control_steps(formulation, ptr(ref), len(ref))


def assemble(params, formulation, ref, bounds, x0, end_heading, max_k=None, max_kp=None):
    """Assembled QP of one path as numpy arrays (copies): dict(n, m, P=(i,j,v) upper, A=(i,j,v), q, l, u)."""
    ref = np.ascontiguousarray(ref, dtype=STATE_DTYPE)
    bounds = np.ascontiguousarray(bounds, dtype=BOUNDS_DTYPE)
    x0 = np.ascontiguousarray(x0, dtype=np.float64)
    qp = lib().oracle_assemble(C.byref(params), formulation, len(ref), ptr(ref), ptr(bounds), ptr(x0),
                               float(end_heading), ptr(max_k), ptr(max_kp))
    if not qp:
        raise ValueError("oracle_assemble refused the problem")
    q = qp.contents
    arr = lambda p, n, t: np.ctypeslib.as_array(p, shape=(n,)).astype(t).copy()  # noqa: E731
    out = dict(n=q.n, m=q.m,
               P=(arr(q.p_i, q.p_nnz, np.int64), arr(q.p_j, q.p_nnz, np.int64), arr(q.p_v, q.p_nnz, np.float64)),
               A=(arr(q.a_i, q.a_nnz, np.int64), arr(q.a_j, q.a_nnz, np.int64), arr(q.a_v, q.a_nnz, np.float64)),
               q=arr(q.q, q.n, np.float64), l=arr(q.l, q.m, np.float64), u=arr(q.u, q.m, np.float64))
    lib().oracle_problem_free(qp)
    return out


def solve_qp(params, formulation, ref, bounds, x0, end_heading, max_k=None, max_kp=None, trace_rows=0):
    """Assemble + OSQP-restatement solve of one path; returns dict(x, y, info, trace)."""
    ref = np.ascontiguousarray(ref, dtype=STATE_DTYPE)
    bounds = np.ascontiguousarray(bounds, dtype=BOUNDS_DTYPE)
    x0 = np.ascontiguousarray(x0, dtype=np.float64)
    qp = lib().oracle_assemble(C.byref(params), formulation, len(ref), ptr(ref), ptr(bounds), ptr(x0),
                               float(end_heading), ptr(max_k), ptr(max_kp))
    if not qp:
        raise ValueError("oracle_assemble refused the problem")
    n, m = qp.contents.n, qp.contents.m
    x = np.zeros(n)
    y = np.zeros(m)
    info = OqpInfo()
    trace = np.zeros((trace_rows, n)) if trace_rows else None
    lib().oracle_osqp_solve(C.byref(params), qp, ptr(x), ptr(y), C.byref(info), ptr(trace), trace_rows)
    lib().oracle_problem_free(qp)
    return dict(x=x, y=y, info=info, trace=trace, n=n, m=m)


def solve_batch(params, formulation, batch, threads=1, max_k=None, max_kp=None):
    """Batch driver (same layout as pqp_solve_batch).  Returns dict(states, frenet, status, iters, seconds)."""
    B = len(batch["n_points"])
    total = int(batch["offsets"][-1])
    ref = np.ascontiguousarray(batch["ref"], dtype=STATE_DTYPE)
    bounds = np.ascontiguousarray(batch["bounds"], dtype=BOUNDS_DTYPE)
    out = np.zeros(total, dtype=STATE_DTYPE)
    frenet = np.zeros((total, 3))
    status = np.zeros(B, dtype=np.int32)
    iters = np.zeros(B, dtype=np.int32)
    secs = lib().oracle_solve_batch(C.byref(params), formulation, B, ptr(batch["n_points"]), ptr(ref),
                                    ptr(bounds), ptr(batch["x0"]), ptr(batch["end_heading"]),
                                    ptr(max_k), ptr(max_kp), ptr(out), ptr(frenet), ptr(status),
                                    ptr(iters), int(threads))
    return dict(states=out, frenet=frenet, status=status, iters=iters, seconds=secs)


# ---------------------------------------------------------------------------------------------
# stages either side of the QP (pqp_oracle_env.c)
# ---------------------------------------------------------------------------------------------

def _dm(m):
    dist = np.ascontiguousarray(m["distance"], dtype=np.float32)
    return DistanceMap(ptr(dist), dist.shape[0], dist.shape[1], float(m["resolution"]), float(m["center_x"]),
                       float(m["center_y"])), dist   # keep `dist` alive with the struct


def map_distance(m, xy):
    dm, _keep = _dm(m)
    xy = np.asarray(xy, dtype=np.float64).reshape(-1, 2)
    L = lib()
    return np.array([L.oracle_map_distance(C.byref(dm), float(x), float(y)) for x, y in xy])


def spline_fit(t, y):
    t = np.ascontiguousarray(t, dtype=np.float64)
    y = np.ascontiguousarray(y, dtype=np.float64)
    coef = np.zeros((len(t), 4))
    if lib().oracle_spline_fit(len(t), ptr(t), ptr(y), ptr(coef)) != 0:
        raise ValueError("oracle_spline_fit refused the knots")
    return coef


def spline_eval(t, coef, at, order=0):
    t = np.ascontiguousarray(t, dtype=np.float64)
    coef = np.ascontiguousarray(coef, dtype=np.float64)
    L = lib()
    return np.array([L.oracle_spline_eval(len(t), ptr(t), ptr(coef), int(order), float(a)) for a in np.atleast_1d(at)])


def clearance_strict(params, m, x, y, z):
    dm, _keep = _dm(m)
    out = np.zeros(2)
    lib().oracle_clearance_strict(C.byref(params), C.byref(dm), float(x), float(y), float(z), ptr(out))
    return out


def _spl(splines, b):
    if splines is None:
        return 0, None, None, None
    ko = np.concatenate([[0], np.cumsum(splines["n_knots"])])
    lo, hi = int(ko[b]), int(ko[b + 1])
    return (hi - lo, np.ascontiguousarray(splines["knots"][lo:hi]), np.ascontiguousarray(splines["x_coef"][lo:hi]),
            np.ascontiguousarray(splines["y_coef"][lo:hi]))


def update_bounds(params, m, batch, mode=1, splines=None):
    """updateBounds[Improved] per path.  Returns dict(bounds, n_valid)."""
    dm, _keep = _dm(m)
    off = batch["offsets"]
    ref = np.ascontiguousarray(batch["ref"], dtype=STATE_DTYPE)
    bounds = np.zeros(len(ref), dtype=BOUNDS_DTYPE)
    n_valid = np.zeros(len(batch["n_points"]), dtype=np.int32)
    for b in range(len(n_valid)):
        nk, kn, xc, yc = _spl(splines, b)
        r = np.ascontiguousarray(ref[off[b]:off[b + 1]])
        o = np.zeros(len(r), dtype=BOUNDS_DTYPE)
        n_valid[b] = lib().oracle_update_bounds(C.byref(params), C.byref(dm), int(mode), len(r), ptr(r), nk, ptr(kn),
                                                ptr(xc), ptr(yc), ptr(o))
        bounds[off[b]:off[b + 1]] = o
    return dict(bounds=bounds, n_valid=n_valid)


def update_limits(params, ref, from_spline=False):
    """ReferencePathImpl::updateLimits -> (max_k, max_kp)."""
    ref = np.ascontiguousarray(ref, dtype=STATE_DTYPE)
    mk, mkp = np.zeros(len(ref)), np.zeros(len(ref))
    lib().oracle_update_limits(C.byref(params), int(bool(from_spline)), len(ref), ptr(ref), ptr(mk), ptr(mkp))
    return mk, mkp


def car_circles(params):
    c = np.zeros((7, 3))
    lib().oracle_car_circles(C.byref(params), ptr(c))
    return c


def check_states(params, m, states):
    dm, _keep = _dm(m)
    states = np.ascontiguousarray(states, dtype=STATE_DTYPE)
    L = lib()
    return np.array([L.oracle_state_collision_free(C.byref(params), C.byref(dm), ptr(states[i:i + 1]))
                     for i in range(len(states))], dtype=np.int32)


def finish_raw(params, m, n_points, paths, collision_check=True):
    dm, _keep = _dm(m)
    paths = np.array(paths, dtype=STATE_DTYPE)
    off = np.concatenate([[0], np.cumsum(n_points)])
    n_kept = np.zeros(len(n_points), dtype=np.int32)
    ok = np.zeros(len(n_points), dtype=np.int32)
    for b in range(len(n_points)):
        p = np.ascontiguousarray(paths[off[b]:off[b + 1]])
        nk = C.c_int(0)
        ok[b] = lib().oracle_finish_raw(C.byref(params), C.byref(dm), len(p), ptr(p), int(collision_check), C.byref(nk))
        n_kept[b] = nk.value
        paths[off[b]:off[b + 1]] = p
    return dict(states=paths, n_kept=n_kept, ok=ok)


def densify(params, m, n_points, paths, output_spacing=0.3, collision_check=True, max_out=512):
    dm, _keep = _dm(m)
    paths = np.ascontiguousarray(paths, dtype=STATE_DTYPE)
    off = np.concatenate([[0], np.cumsum(n_points)])
    B = len(n_points)
    out = np.zeros((B, max_out), dtype=STATE_DTYPE)
    n_out = np.zeros(B, dtype=np.int32)
    ok = np.zeros(B, dtype=np.int32)
    for b in range(B):
        p = np.ascontiguousarray(paths[off[b]:off[b + 1]])
        no = C.c_int(0)
        ok[b] = lib().oracle_densify(C.byref(params), C.byref(dm), len(p), ptr(p), float(output_spacing),
                                     int(collision_check), int(max_out), ptr(out[b]), C.byref(no))
        n_out[b] = no.value
    return dict(states=out, n_out=n_out, ok=ok)


def plan(params, m, batch, formulation=0, bounds_mode=1, splines=None, output_mode=0, output_spacing=0.3,
         collision_check=True, max_out=512):
    """solveWithoutSmoothing per path.  Same result layout as PathPlanner.plan."""
    dm, _keep = _dm(m)
    off = batch["offsets"]
    B = len(batch["n_points"])
    ref = np.ascontiguousarray(batch["ref"], dtype=STATE_DTYPE)
    total = len(ref)
    states = np.zeros(total, dtype=STATE_DTYPE) if output_mode == 0 else np.zeros((B, max_out), dtype=STATE_DTYPE)
    bounds = np.zeros(total, dtype=BOUNDS_DTYPE)
    n_out = np.zeros(B, dtype=np.int32)
    ok = np.zeros(B, dtype=np.int32)
    status = np.zeros(B, dtype=np.int32)
    iters = np.zeros(B, dtype=np.int32)
    for b in range(B):
        nk, kn, xc, yc = _spl(splines, b)
        r = np.ascontiguousarray(ref[off[b]:off[b + 1]])
        cap = max(len(r), max_out if output_mode == 1 else 0)
        o = np.zeros(cap, dtype=STATE_DTYPE)
        bo = np.zeros(len(r), dtype=BOUNDS_DTYPE)
        no, st, it = C.c_int(0), C.c_int(0), C.c_int(0)
        x0 = np.ascontiguousarray(batch["x0"][b], dtype=np.float64)
        ok[b] = lib().oracle_plan_path(C.byref(params), C.byref(dm), int(formulation), int(bounds_mode), int(output_mode),
                                       len(r), ptr(r), nk, ptr(kn), ptr(xc), ptr(yc), ptr(x0),
                                       float(batch["end_heading"][b]), float(output_spacing), int(collision_check),
                                       int(max_out), ptr(o), C.byref(no), C.byref(st), C.byref(it), ptr(bo))
        n_out[b], status[b], iters[b] = no.value, st.value, it.value
        if output_mode == 0:
            states[off[b]:off[b] + no.value] = o[:no.value]
        else:
            states[b, :no.value] = o[:no.value]
        bounds[off[b]:off[b + 1]] = bo
    return dict(states=states, n_out=n_out, ok=ok, status=status, iters=iters, bounds=bounds)
