"""Kernel shape classes as the library selects them (pqp_class_info_form, host logic: no device needed), the station
spacings that reach every KP class, and the partition-edge path lengths of a class.  Shared by the CPU class and
emulator tests and the GPU shape sweep, so that all of them follow the library's own class table."""
import ctypes as C

import numpy as np

from path_optimizer_b200 import _lib, synth
from path_optimizer_b200.abi import STATE_DTYPE

KP, K, KPC = 0, 1, 2
GENERIC = "pqp_kp_solve_kernel"

# Every class each formulation selects (pick_variant / class_for in pqp_capi.cu).  A class that drops out of the
# selection, or a new one, fails the coverage checks by name.  The compiled "KPC" class pqp_kp3_solve_kernel<23,7,4,17,KPC>
# is not selected at any length: <13,7,8,34,KPC> comes first in the table and takes every length it could (2..128).
CLASSES = {
    KP: ["pqp_kp3_solve_kernel<17,6,4,17>", "pqp_kp3_solve_kernel<23,7,4,17>", "pqp_kp3_solve_kernel<17,6,8,34>",
         "pqp_kp3_solve_kernel<23,7,8,34>", "pqp_kp3_solve_kernel<27,7,8,34>", "pqp_kp3_solve_kernel<27,7,10,34>",
         "pqp_kp3_solve_kernel<37,7,12,34>", "pqp_kp3_solve_kernel<37,7,13,34>", GENERIC],
    KPC: ["pqp_kp3_solve_kernel<13,7,8,34,KPC>", "pqp_kp3_solve_kernel<23,7,8,34,KPC>"],
    K: ["pqp_kk_solve_kernel<4>", "pqp_kk_solve_kernel<8>", "pqp_kk_solve_kernel<13>"],
}
UNSELECTED = ["pqp_kp3_solve_kernel<23,7,4,17,KPC>"]

# KP station spacings of the shape sweep, accumulated in double as a resampler makes them.  keep_control_steps is
# int(1.2 / interval) of the first ten intervals: 0.3 m gives 3 (4 for paths of 2..4 stations, whose intervals have not
# accumulated the rounding yet), 0.15 m gives 7 (8 for 2..4 stations); keep 5..10 run on the one-warp kernel.
SPACINGS = (0.3, 0.25, 0.5, 1.0, 0.2, 0.15, 0.11)


# The parity bar of the GPU tests: identical status and iteration count, 1e-8 on the Frenet and Cartesian states.  Past
# 1000 ADMM iterations the rounding differences between kernel and oracle (FMA contraction, summation order) grow with
# the iteration count while the discrete decisions stay the same: on an H100, a 162-station path at keep 10 agrees to
# 3e-13 after 400 iterations, 9e-11 after 800, 6e-8 after 1600 and 1.9e-7 at its 1775th, where both sides stop.
# Such long runs are held to 1e-6.
TOL, LONG_RUN_ITERS, LONG_RUN_TOL = 1e-8, 1000, 1e-6


def assert_matches(res, ref, idx, rows, n_points, what):
    """res: a whole-batch result; ref: the oracle's result for the paths idx of that batch, of n_points stations each
    (rows: their stations in the batch)."""
    idx, n_points = np.asarray(idx), np.asarray(n_points)
    bad = (res["status"][idx] != ref["status"]) | (res["iters"][idx] != ref["iters"])
    assert not bad.any(), (what, [(int(i), int(res["status"][i]), int(res["iters"][i])) for i in idx[bad]],
                           ref["status"][bad].tolist(), ref["iters"][bad].tolist())
    tol = np.repeat(np.where(ref["iters"] > LONG_RUN_ITERS, LONG_RUN_TOL, TOL), n_points)
    pairs = [("frenet", res["frenet"][rows], ref["frenet"], tol[:, None])]
    pairs += [(f, res["states"][f][rows], ref["states"][f], tol) for f in "xyzks"]
    ends = np.cumsum(n_points)
    for f, a, d, t in pairs:
        over = ~((np.abs(a - d) <= t) | (np.isnan(a) & np.isnan(d)))
        if over.ndim == 2:
            over = over.any(axis=1)
        paths = sorted({int(idx[j]) for j in np.searchsorted(ends, np.nonzero(over)[0], side="right")})
        assert not paths, (what, f, "paths", paths, float(np.nanmax(np.abs(a - d))))


def keep_of(form, ref):
    ref = np.ascontiguousarray(ref, dtype=STATE_DTYPE)
    return _lib.load().pqp_keep_control_steps(form, ref.ctypes.data_as(C.c_void_p), len(ref))


def class_of(form, n, keep):
    """(class name, ok): the class pqp_solve_batch launches a path of n stations on; ok False = PQP_INVALID_PROBLEM."""
    L = _lib.load()
    v, t, s = C.c_int(), C.c_int(), C.c_int64()
    rc = L.pqp_class_info_form(form, int(n), int(keep), 0, C.byref(v), C.byref(t), C.byref(s))
    return L.pqp_class_name(v.value).decode(), rc == 0


def device_class_of(nmax, keep_lo, keep_hi):
    """The one KP class pqp_solve_batch_device launches for every path of 2..nmax stations at keep_lo..keep_hi."""
    L = _lib.load()
    v, t, s = C.c_int(), C.c_int(), C.c_int64()
    rc = L.pqp_device_class_info(int(nmax), int(keep_lo), int(keep_hi), 0, C.byref(v), C.byref(t), C.byref(s))
    assert rc == 0, (nmax, keep_lo, keep_hi)
    return L.pqp_class_name(v.value).decode()


def compiled_classes():
    """Names of every kernel class in the library's table, in table order."""
    L = _lib.load()
    names = []
    while L.pqp_class_name(len(names)):
        names.append(L.pqp_class_name(len(names)).decode())
    return names


def max_points(form, keep):
    """Longest path the host-buffer entry solves at this keep (pqp_max_points_keep without a handle: the default
    227 KB shared-memory opt-in of an H100)."""
    n = 2
    while class_of(form, n + 1, keep)[1]:
        n += 1
    return n


def class_ranges(form, keep):
    """{class name: (first N, last N)} of every class the selection uses at this keep."""
    out = {}
    for n in range(2, max_points(form, keep) + 1):
        name, _ = class_of(form, n, keep)
        lo, hi = out.get(name, (n, n))
        out[name] = (min(lo, n), max(hi, n))
    return out


def kp_keeps():
    """The keep values the KP sweep spacings produce, path lengths 2..408."""
    ks = set()
    for ds in SPACINGS:
        for n in (2, 3, 4, 5, 408):
            ref = np.zeros(n, dtype=STATE_DTYPE)
            ref["s"] = synth._accumulate_s(n, ds)
            ks.add(keep_of(KP, ref))
    return sorted(ks)


def kp3_partition(n, keep, mmax):
    """(L, M, stations after the last separator) of a thread-per-station KP / KPC class: kp3_dims_raw in
    pqp_kp_core3.cuh -- separators every L stations (a multiple of keep), at most mmax of them."""
    L = max(keep * ((n - 1) // (mmax * keep) + 1), 2)
    M = (n - 1) // L + 1
    return L, M, (n - 1) - (M - 1) * L


def kk_partition(n, ms):
    """(L, M, stations after the last separator) of the SPIKE form of the K classes (Kk::sp_dims, pqp_kk_core.cuh)."""
    L = max((n + ms - 1) // ms, 2)
    M = (n - 1) // L + 1
    return L, M, (n - 1) - (M - 1) * L


def partition_edges(lo, hi, part):
    """Lengths in [lo, hi] where a partition goes wrong first.  `part(n)` -> (L, M, stations after the last separator).
    A change of M puts a new separator on the last station (a last interior of 0 stations); one station further the last
    interior has 1 station, one station before it is full.  Taken: both ends of the range; both sides of every change
    of L; both sides of the first and the last change of M at each L; the first change of M to an odd and to an even
    count."""
    changes = [n for n in range(lo + 1, hi + 1) if part(n)[:2] != part(n - 1)[:2]]
    picked = set()
    for L in sorted({part(n)[0] for n in range(lo, hi + 1)}):
        at_L = [n for n in changes if part(n)[0] == L and part(n - 1)[0] == L]
        picked.update(at_L[:1] + at_L[-1:])
    picked.update(n for n in changes if part(n)[0] != part(n - 1)[0])
    for parity in (0, 1):
        picked.update([n for n in changes if part(n)[1] % 2 == parity][:1])
    edges = {lo, hi}
    for n in picked:
        edges.update((n - 1, n, min(n + 1, hi)))
    return sorted(edges)
