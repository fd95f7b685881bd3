"""Named cases across the parameter envelope of pqp_params (TEST DATA).

Every discrete decision the kernels share with OSQP depends on parameter magnitudes: which stencil term wins the
matrix-free Ruiz norms, whether limit_scaling maps a norm to 1 or caps it, the cost scaling c, the rho class of a row
from its scaled bounds, the rho clamp at [1e-6, 1e6], the adaptive-rho rescale and the verdict at max_iter.  The rest of
the suite runs near the defaults (a 4.5-5.2 m car, weights within a decade of the flags, max_iter >= 25); these cases
move one group at a time to the ends of what a user of the reference can set, all inside OSQP's legal settings.

A case is a dict of pqp_params overrides (`params`, run through pqp_params_update_config as the reference's
updateConfig does) and, where the case is about the inputs, an `inputs` function that edits a batch in place.
`params(name)` and `apply(name, batch)` build them."""
import ctypes as C

import numpy as np

from oracle import oracle


def _curvature_near_kmax(b):
    """Reference curvature up to 0.95 of the robot's steering limit (tan(0.7) / 0.5 = 1.69 / m): kappa^2 ds is the
    largest term of the dynamics rows' norm."""
    o = b["offsets"]
    for i in range(len(b["n_points"])):
        n = o[i + 1] - o[i]
        b["ref"]["k"][o[i]:o[i + 1]] = 1.6 * np.sin(np.linspace(0.0, 3.0, n))


def _open_bounds(b):
    """Caller bounds of +-1e30 (OSQP's infinity): every third station has its rear circle row open above, every fifth
    open below, every seventh all four circle rows open on both sides (free rows: OSQP's RHO_MIN class).  (One row of a
    slack pair opened on its own is refused by the kernels: test_envelope.py::test_emu_one_open_side_of_a_slack_pair.)"""
    bb = b["bounds"]
    n = len(bb)
    idx = np.arange(n)
    bb["c0_ub"][idx % 3 == 1] = 1e30
    bb["c0_lb"][idx % 5 == 2] = -1e30
    both = idx % 7 == 3
    for f in ("c0", "c1", "c2", "c3"):
        bb[f + "_lb"][both] = -1e30
        bb[f + "_ub"][both] = 1e30


def _narrow_corridors(b):
    """Corridor rows 2e-4 and 2e-3 m wide by turns around the centre line (the x0 row starts inside): the scaled width
    of a circle row falls on both sides of RHO_TOL (1e-4), so the same row kind is an inequality at some stations and
    is treated as an equality (rho x 1e3) at others."""
    bb = b["bounds"]
    idx = np.arange(len(bb))
    half = np.where(idx % 2 == 0, 1e-4, 1e-3)
    for f in ("c0", "c2"):
        mid = 0.5 * (bb[f + "_lb"] + bb[f + "_ub"])
        bb[f + "_lb"] = mid - half
        bb[f + "_ub"] = mid + half
    b["x0"][:, 0] = 0.5 * (bb["c0_lb"][b["offsets"][:-1]] + bb["c0_ub"][b["offsets"][:-1]])


CASES = {
    # vehicles (pqp_params_update_config recomputes circle_radius and d1..d4)
    "robot": dict(params=dict(car_length=0.8, car_width=0.5, wheel_base=0.5, rear_axle_to_center=0.2,
                              max_steering_angle=0.7)),
    "truck": dict(params=dict(car_length=12.0, car_width=2.5, wheel_base=6.5, rear_axle_to_center=3.0)),
    "d2_zero": dict(params=dict(rear_axle_to_center=4.9 / 8)),           # d2 = -L/8 + r = 0 exactly
    "no_steering": dict(params=dict(max_steering_angle=0.0)),             # kappa box in the equality class
    "robot_kmax": dict(params=dict(car_length=0.8, car_width=0.5, wheel_base=0.5, rear_axle_to_center=0.2,
                                   max_steering_angle=0.7), inputs=_curvature_near_kmax),
    # margins
    "margin0": dict(params=dict(expected_safety_margin=0.0)),             # the SB row in the equality class
    "margin3": dict(params=dict(expected_safety_margin=3.0)),             # wider than half of some corridors
    # weights
    "weights_1e-3": dict(params=dict(KP_curvature_weight=1e-3, KP_curvature_rate_weight=1e-3, KP_deviation_weight=1e-3,
                                     KP_slack_weight=1e-3, K_curvature_weight=1e-3, K_curvature_rate_weight=1e-3,
                                     K_deviation_weight=1e-3)),           # c stays 1
    "weights_1e6": dict(params=dict(KP_curvature_weight=1e5, KP_curvature_rate_weight=1e6, KP_slack_weight=1e5,
                                    K_curvature_weight=1e5, K_curvature_rate_weight=1e6)),  # limit_scaling's cap
    "deviation_1e3": dict(params=dict(KP_deviation_weight=1e3, K_deviation_weight=1e3)),
    "slack_1e-5": dict(params=dict(KP_slack_weight=1e-5)),                # an unused slack's column norm -> 1
    # OSQP settings, inside OSQP's legal ranges
    "rho_1e-9": dict(params=dict(rho=1e-9)),                              # clamped to 1e-6 at setup
    "rho_1e7": dict(params=dict(rho=1e7)),                                # clamped to 1e6 at setup
    "alpha_0.05": dict(params=dict(alpha=0.05, max_iter=300)),
    "alpha_1.95": dict(params=dict(alpha=1.95)),
    "sigma_1e-9": dict(params=dict(sigma=1e-9)),
    "sigma_1e-1": dict(params=dict(sigma=1e-1)),
    "eps_abs_0": dict(params=dict(eps_abs=0.0, max_iter=300)),
    "eps_rel_0": dict(params=dict(eps_rel=0.0)),
    "scaling1": dict(params=dict(scaling=1)),
    "scaling40": dict(params=dict(scaling=40)),
    "every_iteration": dict(params=dict(check_termination=1, adaptive_rho_interval=1, adaptive_rho_tolerance=5.0)),
    "max_iter1": dict(params=dict(max_iter=1)),
    "max_iter2": dict(params=dict(max_iter=2)),
    # row classes
    "open_bounds": dict(params=dict(), inputs=_open_bounds),
    "narrow_rows": dict(params=dict(max_iter=400), inputs=_narrow_corridors),
}


def kpc_limits(b, p):
    """KPC limits (ReferencePathImpl::updateLimits through the oracle) from a speed profile with standstill stations
    every 11th (DBL_MAX limits: the curvature rows are free on that side); sets the batch's v and a."""
    total = int(b["offsets"][-1])
    b["ref"]["v"] = 4.0 + 3.0 * np.sin(np.arange(total) * 0.05)
    b["ref"]["a"] = 0.5 * np.cos(np.arange(total) * 0.05)
    b["ref"]["v"][::11] = 0.0
    return oracle.update_limits(p, b["ref"])


def params(name, base=None):
    """The case's pqp_params: the reference's defaults (or `base`) with the overrides, through pqp_params_update_config."""
    from path_optimizer_b200 import _lib
    p = oracle.default_params() if base is None else base.copy()
    for k, v in CASES[name]["params"].items():
        setattr(p, k, v)
    _lib.load().pqp_params_update_config(C.byref(p))
    return p


def apply(name, batch):
    """Edit `batch` in place with the case's inputs (no-op for a parameter-only case); returns it."""
    f = CASES[name].get("inputs")
    if f is not None:
        f(batch)
    return batch
