"""Host-side mirror of the reference's solver interface on top of the C ABI (include/pqp.h).

Reference interface being mirrored (names, argument meaning, error behaviour):
  OsqpSolver::create(type, reference_path, vehicle_state, horizon)   src/solver/solver.cpp:30-44
  OsqpSolver::solve(std::vector<State>* optimized_path) -> bool      src/solver/solver.cpp:46-77
`create` returns None (and logs) for an unknown type string exactly like the reference returns
nullptr; `solve` returns False whenever OSQP's status would not be SOLVED (osqp-eigen semantics).

All numerics run in libpqp.so's sm_90a kernels; this module only marshals buffers.
"""
import ctypes as C
import logging

import numpy as np

from . import _lib
from .abi import (BOUNDS_DTYPE, FORMULATIONS, OK, SOLVED, STATE_DTYPE, Params, Stats, ptr)

log = logging.getLogger("path_optimizer_b200")


class PqpError(RuntimeError):
    pass


def default_params():
    """FLAGS_* defaults (planning_flags.cpp) + updateConfig() + OSQP defaults."""
    p = Params()
    _lib.load().pqp_params_default(C.byref(p))
    return p


def keep_control_steps(formulation, ref):
    ref = np.ascontiguousarray(ref, dtype=STATE_DTYPE)
    return _lib.load().pqp_keep_control_steps(int(formulation), ptr(ref), len(ref))


class BatchPathSolver:
    """A batch of independent path QPs per call: the batched form of OsqpSolver::solve."""

    def __init__(self, params=None, device=0, max_batch=1024, max_total_points=1024 * 128):
        self._L = _lib.load()
        self.params = params if params is not None else default_params()
        self._h = C.c_void_p()
        rc = self._L.pqp_create(C.byref(self._h), C.byref(self.params), int(device), int(max_batch),
                                int(max_total_points))
        if rc != OK:
            raise PqpError(f"pqp_create failed (rc={rc}): {_lib.last_error()}")
        self.device = device
        self.max_batch = max_batch
        self.max_total_points = max_total_points

    def close(self):
        if self._h:
            self._L.pqp_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_params(self, params):
        """Replace the parameter snapshot (pqp_set_params); settings OSQP refuses raise and leave the previous one."""
        rc = self._L.pqp_set_params(self._h, C.byref(params))
        if rc != OK:
            raise PqpError(f"pqp_set_params failed (rc={rc}): {_lib.last_error()}")
        self.params = params

    def set_param_sets(self, sets):
        """Replace the parameter sets (pqp_set_param_sets): a sequence of 1..64 Params, each already run through
        pqp_params_update_config.  solve(), solve_device() and the planner's plan calls pick a path's set with
        `param_index`; set 0 is what the calls without an index use.  A bad argument leaves the previous sets in place."""
        sets = list(sets)
        arr = (Params * max(len(sets), 1))(*sets)
        rc = self._L.pqp_set_param_sets(self._h, len(sets), arr)
        if rc != OK:
            raise PqpError(f"pqp_set_param_sets failed (rc={rc}): {_lib.last_error()}")
        self.params = sets[0]
        self.param_sets = sets

    @staticmethod
    def _param_index(param_index, B):
        pi = np.asarray(param_index)
        if pi.shape != (B,) or pi.dtype.kind not in "iu":
            raise ValueError(f"param_index: expected an integer array of shape ({B},), got {pi.dtype} {pi.shape}")
        return np.ascontiguousarray(pi, dtype=np.int32)

    @staticmethod
    def _forms(formulation, B):
        """None for one formulation for the whole batch (a name or an int: today's entries), else the per-path
        formulations as an int32 numpy array [B] (PQP_FORM_* values; a list of names maps an unknown name to -1, which
        fails its path).  A torch tensor is returned as it is, for the device entries to check."""
        if isinstance(formulation, (str, int, np.integer)):
            return None
        if type(formulation).__module__.startswith("torch"):
            return formulation
        f = list(formulation) if not isinstance(formulation, np.ndarray) else formulation
        if len(f) and isinstance(f[0], str):
            f = [FORMULATIONS.get(name, -1) for name in f]
        f = np.asarray(f)
        if f.shape != (B,) or f.dtype.kind not in "iu":
            raise ValueError(f"formulation: expected a name or an integer array / list of names of shape ({B},), "
                             f"got {f.dtype} {f.shape}")
        return np.ascontiguousarray(f, dtype=np.int32)

    def _forms_device(self, formulation, B, dev):
        """The per-path formulations as an int32 CUDA tensor [B] on `dev` (a tensor passes through unchanged, so that a
        graph replay reads the captured one); None for one formulation for the whole batch."""
        import torch
        f = self._forms(formulation, B)
        if f is None or isinstance(f, torch.Tensor):
            return f
        return torch.from_numpy(f).to(dev)

    @staticmethod
    def _form_mask(form_mask):
        """An int bitmask (1 << PQP_FORM_*; 0 = all three) or a collection of names / PQP_FORM_* values."""
        if isinstance(form_mask, (int, np.integer)):
            return int(form_mask)
        m = 0
        for f in form_mask:
            m |= 1 << (FORMULATIONS[f] if isinstance(f, str) else int(f))
        return m

    def max_points(self, formulation="KP"):
        return self._L.pqp_max_points(self._h, FORMULATIONS[formulation])

    def solve(self, batch, formulation="KP", want_frenet=True, out=None, max_k=None, max_kp=None, param_index=None):
        """batch: dict as produced by synth.* (host numpy arrays).  Returns dict(states, frenet,
        status, iters, ok, stats).  `out` may carry preallocated (e.g. pinned) output arrays.
        max_k / max_kp ([sum N] each) are the KPC limits (ReferencePath::getMaxKList / getMaxKpList).
        `param_index`: int32 [B], the parameter set (set_param_sets) every path is solved with (pqp_solve_batch_sets);
        None: set 0.  A path whose index is outside the sets reports status -100 with 0 iterations and NaN states.
        `formulation`: a name ("KP", "K", "KPC") for the whole batch, or one per path (pqp_solve_batch_forms): an int32
        array [B] of PQP_FORM_* values or a list of names.  Path b then gets what a call with its own formulation gives
        it; a value that is not a formulation fails its path as an out-of-range set index does."""
        n_points = np.ascontiguousarray(batch["n_points"], dtype=np.int32)
        B = len(n_points)
        forms = self._forms(formulation, B)
        form = 0 if forms is not None else FORMULATIONS[formulation] if isinstance(formulation, str) else int(formulation)
        total = int(n_points.sum())
        ref = np.ascontiguousarray(batch["ref"], dtype=STATE_DTYPE)
        bounds = np.ascontiguousarray(batch["bounds"], dtype=BOUNDS_DTYPE)
        x0 = np.ascontiguousarray(batch["x0"], dtype=np.float64)
        end_heading = np.ascontiguousarray(batch["end_heading"], dtype=np.float64)
        assert len(ref) == total and len(bounds) == total and x0.shape == (B, 3) and len(end_heading) == B
        out = out or {}
        states = out.get("states") if out.get("states") is not None else np.zeros(total, dtype=STATE_DTYPE)
        frenet = (out.get("frenet") if out.get("frenet") is not None else np.zeros((total, 3))) if want_frenet else None
        status = out.get("status") if out.get("status") is not None else np.zeros(B, dtype=np.int32)
        iters = out.get("iters") if out.get("iters") is not None else np.zeros(B, dtype=np.int32)
        stats = Stats()
        if max_k is not None:
            max_k = np.ascontiguousarray(max_k, dtype=np.float64)
            max_kp = np.ascontiguousarray(max_kp, dtype=np.float64)
            assert len(max_k) == total and len(max_kp) == total
        head = (self._h, form, B, ptr(n_points), ptr(ref), ptr(bounds), ptr(x0), ptr(end_heading), ptr(max_k), ptr(max_kp))
        tail = (ptr(states), ptr(frenet), ptr(status), ptr(iters), C.byref(stats))
        if forms is not None:
            pi = None if param_index is None else self._param_index(param_index, B)
            name = "pqp_solve_batch_forms"
            rc = self._L.pqp_solve_batch_forms(self._h, *head[2:], ptr(pi), ptr(forms), *tail)
        elif param_index is None:
            name, rc = "pqp_solve_batch", self._L.pqp_solve_batch(*head, *tail)
        else:
            pi = self._param_index(param_index, B)
            name, rc = "pqp_solve_batch_sets", self._L.pqp_solve_batch_sets(*head, ptr(pi), *tail)
        if rc != OK:
            raise PqpError(f"{name} failed (rc={rc}): {_lib.last_error()}")
        return dict(states=states, frenet=frenet, status=status, iters=iters, ok=(status == SOLVED), stats=stats)

    def _cuda_device(self):
        import torch
        return torch.device("cuda", int(self.device))

    def solve_device(self, n_points, offsets, ref, bounds, x0, end_heading, formulation="KP", max_n_points=0,
                     min_keep=0, max_keep=0, max_k=None, max_kp=None, want_frenet=True, out=None, stats=False,
                     param_index=None, n_param_sets=0, form_mask=0):
        """The batch as torch CUDA tensors on the solver's device (path_optimizer_b200.device): n_points int32 [B],
        offsets int32 [B + 1], ref float64 [T, 7], bounds float64 [T, 8], x0 float64 [B, 3], end_heading float64 [B],
        KPC limits float64 [T].  Every path runs on the kernel class solve() would choose for it, picked on the device
        (pqp_solve_batch_device_dispatch), with solve()'s results bit for bit.  Runs on torch.cuda.current_stream()
        without synchronising it (unless `stats`), so that after one warm-up call it can be captured in a CUDA graph.
        max_n_points / min_keep / max_keep (0 = unknown) only narrow the classes launched; a path outside them reports
        INVALID_PROBLEM.  `out` may carry the output tensors (states, frenet, status, iters).  Returns them as a dict.
        `param_index`: int32 [B] on the device, the parameter set of every path (pqp_solve_batch_device_dispatch_sets);
        None: set 0.  n_param_sets > 0 bounds the sets launched (an index at or past it reports INVALID_PROBLEM).
        `formulation` one per path (pqp_solve_batch_device_dispatch_forms): an int32 CUDA tensor [B] of PQP_FORM_*
        values (a graph replay reads the captured tensor), or an array / list of names, uploaded per call.
        `form_mask` (1 << PQP_FORM_* or a list of names; 0: all three) bounds the formulations launched; a path outside
        it reports INVALID_PROBLEM."""
        import torch
        from . import device as D
        dev = self._cuda_device()
        B, T = int(n_points.shape[0]), int(ref.shape[0])
        forms = self._forms_device(formulation, B, dev)
        form = 0 if forms is not None else FORMULATIONS[formulation] if isinstance(formulation, str) else int(formulation)
        out = dict(out or {})
        f64, i32 = torch.float64, torch.int32
        states = out.get("states")
        states = states if states is not None else torch.empty((T, D.STATE_COLS), dtype=f64, device=dev)
        frenet = out.get("frenet") if want_frenet else None
        if want_frenet and frenet is None:
            frenet = torch.empty((T, 3), dtype=f64, device=dev)
        status = out.get("status") if out.get("status") is not None else torch.empty(B, dtype=i32, device=dev)
        iters = out.get("iters") if out.get("iters") is not None else torch.empty(B, dtype=i32, device=dev)
        args = [D.check(n_points, "n_points", i32, (B,), dev), D.check(offsets, "offsets", i32, (B + 1,), dev),
                D.check(ref, "ref", f64, (T, D.STATE_COLS), dev), D.check(bounds, "bounds", f64, (T, D.BOUNDS_COLS), dev),
                D.check(x0, "x0", f64, (B, 3), dev), D.check(end_heading, "end_heading", f64, (B,), dev),
                D.check(max_k, "max_k", f64, (T,), dev), D.check(max_kp, "max_kp", f64, (T,), dev),
                D.check(states, "states", f64, (T, D.STATE_COLS), dev), D.check(frenet, "frenet", f64, (T, 3), dev),
                D.check(status, "status", i32, (B,), dev), D.check(iters, "iters", i32, (B,), dev)]
        st = Stats()
        tail = (torch.cuda.current_stream(dev).cuda_stream, C.byref(st) if stats else None)
        bounds_ = (self._h, form, B, T, int(max_n_points), int(min_keep), int(max_keep))
        if forms is not None:
            pi = D.check(param_index, "param_index", i32, (B,), dev)
            fm = D.check(forms, "formulation", i32, (B,), dev)
            name = "pqp_solve_batch_device_dispatch_forms"
            rc = self._L.pqp_solve_batch_device_dispatch_forms(self._h, *bounds_[2:], int(n_param_sets),
                                                               self._form_mask(form_mask), *args[:8], pi, fm, *args[8:],
                                                               *tail)
        elif param_index is None:
            name = "pqp_solve_batch_device_dispatch"
            rc = self._L.pqp_solve_batch_device_dispatch(*bounds_, *args, *tail)
        else:
            pi = D.check(param_index, "param_index", i32, (B,), dev)
            name = "pqp_solve_batch_device_dispatch_sets"
            rc = self._L.pqp_solve_batch_device_dispatch_sets(*bounds_, int(n_param_sets), *args[:8], pi, *args[8:], *tail)
        if rc != OK:
            raise PqpError(f"{name} failed (rc={rc}): {_lib.last_error()}")
        return dict(states=states, frenet=frenet, status=status, iters=iters, stats=st if stats else None)


class OsqpSolver:
    """Single-path adaptor with the reference's call shape (solver.hpp:31-36)."""

    _shared = {}

    def __init__(self, formulation, ref_states, bounds, init_error, start_k, end_heading, horizon,
                 params=None, device=0):
        self.formulation = formulation
        self.horizon = int(horizon)
        self._batch = dict(n_points=np.array([self.horizon], dtype=np.int32),
                           ref=np.ascontiguousarray(ref_states, dtype=STATE_DTYPE)[:self.horizon],
                           bounds=np.ascontiguousarray(bounds, dtype=BOUNDS_DTYPE)[:self.horizon],
                           x0=np.array([[init_error[0], init_error[1], start_k]], dtype=np.float64),
                           end_heading=np.array([end_heading], dtype=np.float64))
        # One shared handle per device, sized for the longest path the kernels take; the parameter snapshot is
        # (re)applied before every solve (the reference re-reads FLAGS_* on every solve), so an instance never
        # inherits another instance's parameters.
        self.params = params if params is not None else default_params()
        key = device
        if key not in OsqpSolver._shared:
            OsqpSolver._shared[key] = BatchPathSolver(self.params, device=device, max_batch=1, max_total_points=8192)
        self._solver = OsqpSolver._shared[key]

    @staticmethod
    def create(type_, ref_states, bounds, init_error, start_k, end_heading, horizon, params=None, device=0):
        """OsqpSolver::create: unknown type -> error log + None (solver.cpp:41-43)."""
        if type_ not in FORMULATIONS:
            log.error("No such solver!")
            return None
        return OsqpSolver(type_, ref_states, bounds, init_error, start_k, end_heading, horizon, params, device)

    def solve(self, optimized_path):
        """Fills `optimized_path` (a list) with horizon State records; returns the reference's bool."""
        try:
            self._solver.set_params(self.params)   # (settings osqp_setup refuses fail here)
            res = self._solver.solve(self._batch, self.formulation)
        except PqpError as e:   # the reference's solve() reports every failure through its bool
            log.error("QP failed: %s", e)
            return False
        if not bool(res["ok"][0]):
            return False
        optimized_path.clear()
        optimized_path.extend(res["states"])
        return True
