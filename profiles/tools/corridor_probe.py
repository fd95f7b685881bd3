"""Corridor search and post-smoothing on the device (pqp_post_smooth_device) against the host loop it replaces (one GPU
command; prints the card and its power limit first).

  python profiles/tools/corridor_probe.py [--reps 7] [--out FILE]

1. Stage time at 64, 1024 and 8192 config-3 lines (synth.map_reference_paths fitted on the device, on
   synth.disc_field_map, start at each line's first station) with the reference's default search flags: CUDA events
   around LAUNCHES back-to-back calls queued behind a device-side sleep, per call, median, min and max over --reps
   rounds after a warm-up call; torch.profiler's device time of each of the stage's kernels beside it.
2. The CPU restatement (oracle/corridor.py, one Python loop per path) on the same lines at 64 and 1024 paths.
3. Wall time of one graph-replayed cycle post-smooth + segment + fit + plan_device (KP, IMPROVED on the fitted
   splines, raw output) next to the segment + plan cycle of DESIGN.md §9 on the same lines, the two graphs replayed in
   alternating rounds after a warm-up: the config-1 map at 16 and 64 candidates (the benchmark polyline fitted with
   pqp_spline_fit and shifted sideways) and config-3 size (8192 lines); medians, min and max."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "profiles", "tools"))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from device_chain_probe import card, wall  # noqa: E402
from oracle import corridor as oc  # noqa: E402
from oracle import oracle as O  # noqa: E402
from path_optimizer_b200 import device, planner, synth  # noqa: E402
from segment_probe import config1_lines, lines  # noqa: E402

LAUNCHES = 10
MAX_LAYERS = 160
KERNELS = ("pqp_corridor_search_kernel", "pqp_gen_solve_kernel", "pqp_corridor_keep_kernel", "pqp_segment_scan_kernel",
           "pqp_corridor_copy_kernel", "pqp_fit_splines_kernel")


def spread(v):
    return dict(median_ms=statistics.median(v), min_ms=min(v), max_ms=max(v))


def time_stage(pl, spl, max_s, start, reps):
    ps = pl.post_smooth_device(spl, max_s, start, MAX_LAYERS)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    per = []
    for _ in range(reps):
        torch.cuda._sleep(2_000_000)
        e0.record()
        for _ in range(LAUNCHES):
            pl.post_smooth_device(spl, max_s, start, MAX_LAYERS, out=ps)
        e1.record()
        e1.synchronize()
        per.append(e0.elapsed_time(e1) / LAUNCHES)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            pl.post_smooth_device(spl, max_s, start, MAX_LAYERS, out=ps)
        torch.cuda.synchronize()
    prof_ms = {}
    for k in KERNELS:
        v = [e.device_time for e in prof.events() if k in e.name]
        prof_ms[k] = statistics.median(v) / 1e3 if v else None
    return ps, dict(events=spread(per), profiler_median_ms=prof_ms)


def host_loop(m, spl, max_s, start, reps):
    h = {k: v.cpu().numpy() for k, v in spl.items() if k != "ok"}
    st = device.tensor_to_records(start)
    ms = max_s.cpu().numpy()
    loop = []
    for _ in range(reps):
        t0 = time.perf_counter()
        oc.post_smooth_batch(h, ms, st, [m], O.default_params(), 1 << 30, max_layers=MAX_LAYERS)
        loop.append((time.perf_counter() - t0) * 1e3)
    return dict(oracle_loop_median_ms=statistics.median(loop), oracle_loop_min_ms=min(loop))


def stage_times(reps):
    out = {}
    m = synth.disc_field_map()
    pl = planner.PathPlanner(max_batch=8192, max_total_points=8192 * 256)
    pl.set_map(m)
    for B in (64, 1024, 8192):
        _, spl, max_s, start, _ = lines(pl, B)
        ps, t = time_stage(pl, spl, max_s, start, reps)
        out[f"{B}_paths"] = dict(kept=int(ps["ok"].sum()), knots=int(ps["knot_offsets"][-1]), **t)
        print(f"post-smooth stage, {B} lines: {json.dumps(out[f'{B}_paths'])}", flush=True)
        if B <= 1024:
            out[f"{B}_paths"]["host"] = host_loop(m, spl, max_s, start, reps=1 if B > 64 else 3)
            print(f"  host: {json.dumps(out[f'{B}_paths']['host'])}", flush=True)
    pl.close()
    return out


def cycle_pair(pl, spl, max_s, start, goal, max_n, reps):
    """Graphs of post-smooth + segment + fit + plan and of segment + plan on the same lines, replayed alternately."""
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
    rec = lambda a: t(np.ascontiguousarray(a).view(np.float64).reshape(len(a), -1))   # noqa: E731
    d = {k: t(v) for k, v in spl.items()} if isinstance(spl["knots"], np.ndarray) else spl
    ms = t(max_s) if isinstance(max_s, np.ndarray) else max_s
    st = rec(start) if isinstance(start, np.ndarray) else start
    gl = rec(goal) if isinstance(goal, np.ndarray) else goal

    def full(o=None):
        o = o or [None] * 4
        ps = pl.post_smooth_device(d, ms, st, MAX_LAYERS, out=o[0])
        sg = pl.segment_device(ps, ps["max_s"], st, gl, max_n, out=o[1])
        ft = pl.fit_splines_device(sg["offsets"], sg["ref"], out=o[2])
        mi = torch.where((ps["ok"] != 0) & (sg["ok"] != 0) & (ft["ok"] != 0), 0, -1).to(torch.int32)
        res = pl.plan_device(sg["n_points"], sg["offsets"], sg["ref"], sg["x0"], sg["end_heading"], max_n_points=max_n,
                             bounds_mode=planner.BOUNDS_IMPROVED, splines=ft, map_index=mi, out=o[3])
        return [ps, sg, ft, res]

    def short(o=None):
        o = o or [None] * 2
        sg = pl.segment_device(d, ms, st, gl, max_n, out=o[0])
        mi = torch.where(sg["ok"] != 0, 0, -1).to(torch.int32)
        res = pl.plan_device(sg["n_points"], sg["offsets"], sg["ref"], sg["x0"], sg["end_heading"], max_n_points=max_n,
                             bounds_mode=planner.BOUNDS_IMPROVED, splines=d, map_index=mi, out=o[1])
        return [sg, res]
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        of = full()
        of = full(of)
        os_ = short()
        os_ = short(os_)
    torch.cuda.synchronize()
    gf, gs = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    with torch.cuda.graph(gf):
        full(of)
    with torch.cuda.graph(gs):
        short(os_)
    gf.replay(); gs.replay()
    tf, ts = [], []
    for _ in range(reps):
        tf.append(wall(gf.replay))
        ts.append(wall(gs.replay))
    out = dict(paths=int(ms.shape[0]), post_smoothed=int(of[0]["ok"].sum()), stations=int(of[1]["offsets"][-1]),
               solved=int((of[3]["status"] == 1).sum()), post_smooth_segment_fit_plan=spread(tf),
               segment_plan=spread(ts))
    del gf, gs
    return out


def cycles(reps):
    out = {}
    for B in (16, 64):
        field, spl, ms, st, gl = config1_lines(B)
        pl = planner.PathPlanner(max_batch=B, max_total_points=B * 400)
        pl.set_map(field)
        out[f"config1_{B}_candidates"] = cycle_pair(pl, spl, ms, st, gl, 400, reps)
        print(f"config 1, {B} candidates:", json.dumps(out[f"config1_{B}_candidates"]), flush=True)
        pl.close()
    pl = planner.PathPlanner(max_batch=8192, max_total_points=8192 * 256)
    pl.set_map(synth.disc_field_map())
    _, spl, ms, st, gl = lines(pl, 8192)
    out["config3_8192"] = cycle_pair(pl, spl, ms, st, gl, 256, reps)
    print("config 3, 8192 lines:", json.dumps(out["config3_8192"]), flush=True)
    pl.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card())
    print("card, power limit:", res["card"], flush=True)
    side = torch.cuda.Stream()    # torch's default stream is the NULL stream, which the library takes for its own
    with torch.cuda.stream(side):
        res["post_smooth_stage"] = stage_times(a.reps)
    res["graph_cycle_wall_ms"] = cycles(a.reps)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
