"""torch CUDA tensors in and out of the device-resident entry points (BatchPathSolver.solve_device,
PathPlanner.plan_device).  Records travel as float64 tensors: a state (x, y, z, k, s, v, a) is one row of 7, the
clearance bounds of a station (c0_ub, c0_lb, .., c3_lb) one row of 8; station counts, offsets, status and iteration
counts are int32.  torch is imported when a function here is first called."""
import numpy as np

from .abi import BOUNDS_DTYPE, STATE_DTYPE

STATE_COLS, BOUNDS_COLS = 7, 8


def _torch():
    import torch
    return torch


def records_to_tensor(a, cols, device):
    """A structured record array (STATE_DTYPE / BOUNDS_DTYPE) as a [len, cols] float64 tensor on `device`."""
    torch = _torch()
    flat = np.ascontiguousarray(a).view(np.float64).reshape(-1, cols)
    return torch.from_numpy(flat.copy()).to(device)


def tensor_to_records(t, dtype=STATE_DTYPE):
    """A [len, 7] (or [len, 8]) float64 tensor back to a structured numpy record array."""
    return np.ascontiguousarray(t.detach().cpu().numpy()).view(dtype).reshape(-1)


def batch_to_device(batch, device="cuda"):
    """A synth-style batch (n_points, ref, x0, end_heading, optional bounds / offsets) as device tensors."""
    torch = _torch()
    n = np.ascontiguousarray(batch["n_points"], dtype=np.int32)
    off = np.zeros(len(n) + 1, dtype=np.int32)
    np.cumsum(n, out=off[1:])
    out = dict(n_points=torch.from_numpy(n.copy()).to(device), offsets=torch.from_numpy(off).to(device),
               ref=records_to_tensor(np.asarray(batch["ref"], dtype=STATE_DTYPE), STATE_COLS, device),
               x0=torch.from_numpy(np.ascontiguousarray(batch["x0"], dtype=np.float64).reshape(-1, 3).copy()).to(device),
               end_heading=torch.from_numpy(np.ascontiguousarray(batch["end_heading"], dtype=np.float64).copy()).to(device))
    if batch.get("bounds") is not None:
        out["bounds"] = records_to_tensor(np.asarray(batch["bounds"], dtype=BOUNDS_DTYPE), BOUNDS_COLS, device)
    return out


def splines_to_device(splines, device="cuda"):
    """reference_splines() output as device tensors, with the knot counts turned into an exclusive prefix
    (knot_offsets [batch + 1])."""
    torch = _torch()
    nk = np.ascontiguousarray(splines["n_knots"], dtype=np.int32)
    koff = np.zeros(len(nk) + 1, dtype=np.int32)
    np.cumsum(nk, out=koff[1:])
    f64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64).copy()).to(device)  # noqa: E731
    return dict(knot_offsets=torch.from_numpy(koff).to(device), knots=f64(splines["knots"]),
                x_coef=f64(splines["x_coef"]).reshape(-1, 4), y_coef=f64(splines["y_coef"]).reshape(-1, 4))


def check(t, name, dtype, shape, device):
    """Raw pointer of a contiguous tensor of `dtype` and `shape` (-1: any) on `device`; None passes through."""
    torch = _torch()
    if t is None:
        return None
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.device != device:
        raise ValueError(f"{name}: expected a CUDA tensor on {device}")
    if t.dtype != dtype or not t.is_contiguous():
        raise ValueError(f"{name}: expected a contiguous {dtype} tensor, got {t.dtype}")
    if len(t.shape) != len(shape) or any(s != -1 and s != d for s, d in zip(shape, t.shape)):
        raise ValueError(f"{name}: expected shape {tuple(shape)}, got {tuple(t.shape)}")
    return t.data_ptr()
