"""Segmentation of smoothed reference lines on the device (pqp_segment_reference_device) against the host loop it
replaces (one GPU command; prints the card and its power limit first).

  python profiles/tools/segment_probe.py [--reps 7] [--out FILE]

1. Segment entry time alone (its three launches) at 64, 1024 and 8192 config-3 lines of 200 stations, segmented with
   the reference's default flags (spacings 0.15 / 0.3, dynamic): CUDA events around 20 back-to-back calls queued
   behind a device-side sleep, per call, median over --reps rounds; torch.profiler's device time of each kernel beside
   it.  Twice per size: with the goal at each line's last station (end distance 0, so the goal search does not run)
   and at 60 % of the line (the search walks back from the end to 8 m past the goal).  Then the longest goal search
   one path can run (a NaN goal, which never meets the break rule), timed on 2^16 lattice samples and scaled to the
   2^22 the length guard admits.
2. The CPU restatement (oracle/segment.py, one Python loop per path) on the same lines at 64 and 1024 paths, and the
   copies a host segmentation adds: the splines down, the segmented states up (torch copies, pinned host buffers).
3. Wall time of one graph-replayed cycle, segment + plan_device (KP, IMPROVED on the smoothed splines, raw output), on
   the config-1 map at 16 and 64 candidates (the benchmark polyline fitted with pqp_spline_fit and shifted sideways)
   and at config-3 size (8192 lines on synth.disc_field_map); median of --reps replays after a warm-up."""
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
from oracle import segment as oseg  # noqa: E402
from path_optimizer_b200 import device, planner, synth  # noqa: E402

N_ST = 200
LAUNCHES = 20
KERNELS = ("pqp_segment_count_kernel", "pqp_segment_scan_kernel", "pqp_segment_write_kernel")


def lines(pl, B, goal_at=1.0):
    """config-3 reference lines fitted on the device: splines, max_s, start (first station) and goal (the station at
    fraction goal_at of the line: 1.0 is the last station, where the goal search does not run; 0.6 lies inside the
    line, and the search walks back from the end until it is 8 m past the goal)."""
    dev = torch.device("cuda", 0)
    b = synth.map_reference_paths(B, N_ST)
    d = device.batch_to_device(b, dev)
    spl = pl.fit_splines_device(d["offsets"], d["ref"])
    first = d["offsets"][:-1].long()
    last = d["offsets"][1:].long() - 1
    goal = first + ((last - first).double() * goal_at).round().long()
    return b, spl, d["ref"][last, 4].contiguous(), d["ref"][first].contiguous(), d["ref"][goal].contiguous()


def time_entry(pl, spl, max_s, start, goal, max_n, reps):
    """Segment entry per call (CUDA events, LAUNCHES calls behind a device-side sleep) and torch.profiler's device time
    of each kernel; medians over reps."""
    from torch.profiler import ProfilerActivity, profile
    seg = pl.segment_device(spl, max_s, start, goal, max_n)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    per = []
    for _ in range(reps):
        torch.cuda._sleep(2_000_000)
        e0.record()
        for _ in range(LAUNCHES):
            pl.segment_device(spl, max_s, start, goal, max_n, out=seg)
        e1.record()
        e1.synchronize()
        per.append(e0.elapsed_time(e1) / LAUNCHES)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            pl.segment_device(spl, max_s, start, goal, max_n, out=seg)
        torch.cuda.synchronize()
    prof_ms = {k: statistics.median([e.device_time for e in prof.events() if k in e.name]) / 1e3 for k in KERNELS}
    return seg, dict(events_median_ms=statistics.median(per), events_min_ms=min(per), profiler_median_ms=prof_ms)


def kernel_times(reps):
    out = {}
    pl = planner.PathPlanner(max_batch=8192, max_total_points=8192 * 256)
    for B in (64, 1024, 8192):
        for name, goal_at in (("goal_at_end", 1.0), ("goal_inside", 0.6)):
            _, spl, max_s, start, goal = lines(pl, B, goal_at)
            seg, t = time_entry(pl, spl, max_s, start, goal, 256, reps)
            n = seg["n_points"].cpu().numpy()
            assert (seg["ok"] == 1).all(), int((seg["ok"] == 0).sum())
            key = f"{B}_paths_{name}"
            out[key] = dict(stations_mean=float(n.mean()), **t)
            print(f"segment entry, {B} lines, {name}: {json.dumps(out[key])}", flush=True)
            if B <= 1024 and goal_at == 1.0:
                out[key]["host"] = host_loop(spl, max_s, start, goal, seg, reps=3)
                print(f"  host: {json.dumps(out[key]['host'])}", flush=True)
    pl.close()
    return out


def longest_search(reps):
    """The longest goal search one path can run: a NaN goal never satisfies the break rule, so the search visits every
    lattice sample of max_s.  Timed at max_s = search_ds * 2^16 on one path (the walk behind it stops at the station
    cap), and scaled by 64 to the 2^22 samples the length guard still admits."""
    pl = planner.PathPlanner(max_batch=1, max_total_points=256)
    _, spl, _, start, goal = lines(pl, 1)
    goal = goal.clone()
    goal[:, :2] = float("nan")
    samples = 1 << 16
    max_s = torch.full((1,), 0.5 * samples, dtype=torch.float64, device=start.device)
    seg, t = time_entry(pl, spl, max_s, start, goal, 256, reps)
    assert int(seg["ok"][0]) == 0       # the walk of a 32 km line passes the station cap
    ms = t["profiler_median_ms"]["pqp_segment_count_kernel"]
    pl.close()
    return dict(samples=samples, count_kernel_ms=ms, us_per_sample=1e3 * ms / samples,
                extrapolated_2_22_samples_s=ms * 64 / 1e3)


def host_loop(spl, max_s, start, goal, seg, reps):
    """The oracle's Python loop on the same lines, and the copies a host segmentation adds."""
    h = {k: v.cpu().numpy() for k, v in spl.items() if k != "ok"}
    h["knot_offsets"] = spl["knot_offsets"].cpu().numpy()
    st, gl = (device.tensor_to_records(t) for t in (start, goal))
    ms = max_s.cpu().numpy()
    loop = []
    for _ in range(reps):
        t0 = time.perf_counter()
        o = oseg.segment_batch(h, ms, st, gl, 1 << 30)
        loop.append((time.perf_counter() - t0) * 1e3)
    T = int(o["offsets"][-1])
    down = [spl[k] for k in ("knot_offsets", "knots", "x_coef", "y_coef")]
    hbuf = [torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for t in down]
    up_h = torch.from_numpy(o["ref"]).pin_memory()
    up_d = torch.empty_like(up_h, device="cuda")

    def copies():
        for a, b in zip(hbuf, down):
            a.copy_(b, non_blocking=True)
        up_d.copy_(up_h, non_blocking=True)
    copy = [wall(copies) for _ in range(reps + 1)][1:]
    return dict(oracle_loop_median_ms=statistics.median(loop), copies_median_ms=statistics.median(copy), stations=T)


def config1_lines(B):
    from tests import segment_cases as sc
    c = sc.config1()
    t, xc, yc = c["spl"]
    ko = (np.arange(B + 1) * len(t)).astype(np.int32)
    ycs = np.concatenate([np.concatenate([yc[:, :3], yc[:, 3:] + dy], axis=1) for dy in np.linspace(-0.6, 0.6, B)])
    spl = dict(knot_offsets=ko, knots=np.tile(t, B), x_coef=np.tile(xc, (B, 1)), y_coef=ycs)
    st, gl = np.array([c["start"]] * B), np.array([c["goal"]] * B)
    return c["field"], spl, np.full(B, t[-1]), st, gl


def graph_cycle(pl, spl, max_s, start, goal, max_n, reps):
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
    rec = lambda a: t(np.ascontiguousarray(a).view(np.float64).reshape(len(a), -1))   # noqa: E731
    d = {k: t(v) for k, v in spl.items()} if isinstance(spl["knots"], np.ndarray) else spl
    ms = t(max_s) if isinstance(max_s, np.ndarray) else max_s
    st = rec(start) if isinstance(start, np.ndarray) else start
    gl = rec(goal) if isinstance(goal, np.ndarray) else goal
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        seg = pl.segment_device(d, ms, st, gl, max_n)
        zero = torch.zeros_like(seg["ok"])

        def cycle(seg_out=None, plan_out=None):
            s = pl.segment_device(d, ms, st, gl, max_n, out=seg_out)
            mi = torch.where(s["ok"] != 0, zero, -1)
            return s, pl.plan_device(s["n_points"], s["offsets"], s["ref"], s["x0"], s["end_heading"], max_n_points=max_n,
                                     bounds_mode=planner.BOUNDS_IMPROVED, splines=d, map_index=mi, out=plan_out)
        seg, res = cycle(seg)
    torch.cuda.synchronize()
    kept = int(seg["ok"].sum())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cycle(seg, res)
    g.replay()
    times = [wall(g.replay) for _ in range(reps)]
    solved = int((res["status"] == 1).sum())
    del g
    return dict(paths=int(ms.shape[0]), kept=kept, solved=solved, stations=int(seg["offsets"][-1]),
                median_ms=statistics.median(times), min_ms=min(times))


def cycles(reps):
    out = {}
    for B in (16, 64):
        field, spl, ms, st, gl = config1_lines(B)
        pl = planner.PathPlanner(max_batch=B, max_total_points=B * 400)
        pl.set_map(field)
        out[f"config1_{B}_candidates"] = graph_cycle(pl, spl, ms, st, gl, 400, reps)
        print(f"config 1, {B} candidates:", json.dumps(out[f"config1_{B}_candidates"]), flush=True)
        pl.close()
    pl = planner.PathPlanner(max_batch=8192, max_total_points=8192 * 256)
    pl.set_map(synth.disc_field_map())
    _, spl, ms, st, gl = lines(pl, 8192)
    out["config3_8192"] = graph_cycle(pl, spl, ms, st, gl, 256, reps)
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
        res["segment_entry_ms"] = kernel_times(a.reps)
        res["longest_goal_search"] = longest_search(3)
        print("longest goal search:", json.dumps(res["longest_goal_search"]), flush=True)
    res["graph_cycle_wall_ms"] = cycles(a.reps)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
