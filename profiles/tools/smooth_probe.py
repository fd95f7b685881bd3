"""Smoothing of raw reference polylines on the device (pqp_smooth_reference_device) against the host loop it replaces
(one GPU command; prints the card and its power limit first).

  python profiles/tools/smooth_probe.py [--reps 7] [--out FILE]

1. Stage time at 64, 1024 and 8192 config-1-like polylines (the benchmark's 100-point polyline, each copy shifted
   sideways by up to 0.5 m and its points jittered by up to 5 cm, seeded): CUDA events around 20 back-to-back calls
   queued behind a device-side sleep, per call, median over --reps rounds; torch.profiler's device time per call of
   each kernel beside it (pqp_fit_splines_kernel runs twice per call: the raw fit and the output fit), and the QP's
   iteration counts.
2. The CPU restatement (oracle/smooth.py, one Python loop per path) on the same polylines at 64 and 1024 paths.
3. Wall time of one graph-replayed cycle of the whole of PathOptimizer::solve from raw polylines -- smooth ->
   post-smooth -> segment -> fit -> plan_device (KP, IMPROVED bounds on the fitted splines) -- on the config-1 map at
   16 and 64 candidates; median of --reps replays after a warm-up."""
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
from oracle import oracle as O  # noqa: E402
from oracle import smooth as osm  # noqa: E402
from path_optimizer_b200 import planner  # noqa: E402
from tests import segment_cases, smooth_cases  # noqa: E402

LAUNCHES = 20
MAX_RAW, MAX_PTS, MAX_LAYERS = 64, 64, 64
KERNELS = ("pqp_smooth_sample_kernel", "pqp_fit_splines_kernel", "pqp_smooth_assemble_kernel", "pqp_gen4_solve_kernel",
           "pqp_smooth_keep_kernel", "pqp_segment_scan_kernel", "pqp_smooth_copy_kernel")


def polylines(B, seed=3):
    """B config-1-like polylines: points [B * 100, 7], offsets [B + 1]."""
    x, y = smooth_cases.config1()
    rng = np.random.default_rng(seed)
    n = len(x)
    pts = np.zeros((B * n, 7))
    for b in range(B):
        shift = rng.uniform(-0.5, 0.5)
        pts[b * n:(b + 1) * n, 0] = x + rng.uniform(-0.05, 0.05, n)
        pts[b * n:(b + 1) * n, 1] = y + shift + rng.uniform(-0.05, 0.05, n)
    return pts, np.arange(0, B * n + 1, n, dtype=np.int32)


def spread(v):
    return dict(median_ms=statistics.median(v), min_ms=min(v), max_ms=max(v))


def time_stage(pl, P, Of, reps):
    sm = pl.smooth_device(P, Of, MAX_RAW, MAX_PTS)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    per = []
    for _ in range(reps):
        torch.cuda._sleep(2_000_000)
        e0.record()
        for _ in range(LAUNCHES):
            pl.smooth_device(P, Of, MAX_RAW, MAX_PTS, out=sm)
        e1.record()
        e1.synchronize()
        per.append(e0.elapsed_time(e1) / LAUNCHES)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            pl.smooth_device(P, Of, MAX_RAW, MAX_PTS, out=sm)
        torch.cuda.synchronize()
    prof_ms = {}
    for k in KERNELS:
        v = [e.device_time for e in prof.events() if k in e.name]
        prof_ms[k] = sum(v) / reps / 1e3 if v else None
    it = sm["iters"].cpu().numpy()
    return sm, dict(events=spread(per), profiler_ms_per_call=prof_ms, iters_mean=float(it.mean()),
                    iters_max=int(it.max()), kept=int(sm["ok"].sum()))


def host_loop(pts, off, reps):
    loop = []
    for _ in range(reps):
        t0 = time.perf_counter()
        osm.smooth_batch(pts, off, O.default_params(), 1 << 30, MAX_RAW, MAX_PTS)
        loop.append((time.perf_counter() - t0) * 1e3)
    return dict(oracle_loop_median_ms=statistics.median(loop), oracle_loop_min_ms=min(loop))


def stage_times(reps):
    out = {}
    pl = planner.PathPlanner(max_batch=8192, max_total_points=8192 * 48)
    for B in (64, 1024, 8192):
        pts, off = polylines(B)
        P, Of = torch.from_numpy(pts).cuda(), torch.from_numpy(off).cuda()
        _, t = time_stage(pl, P, Of, reps)
        out[f"{B}_paths"] = t
        print(f"smooth stage, {B} polylines: {json.dumps(t)}", flush=True)
        if B <= 1024:
            t["host"] = host_loop(pts, off, reps=1 if B > 64 else 3)
            print(f"  host: {json.dumps(t['host'])}", flush=True)
    pl.close()
    return out


def cycle(B, reps):
    c = segment_cases.config1()
    pl = planner.PathPlanner(max_batch=B, max_total_points=B * 400)
    pl.set_maps([c["field"]])
    pts, off = polylines(B)
    P, Of = torch.from_numpy(pts).cuda(), torch.from_numpy(off).cuda()
    dev = torch.device("cuda", 0)
    st = torch.tensor(np.array([c["start"]] * B).view(np.float64).reshape(B, -1), device=dev)
    gl = torch.tensor(np.array([c["goal"]] * B).view(np.float64).reshape(B, -1), device=dev)

    def run(o_sm=None, o_ps=None, o_sg=None, o_ft=None, o_pr=None):
        sm = pl.smooth_device(P, Of, MAX_RAW, MAX_PTS, out=o_sm)
        ps = pl.post_smooth_device(sm, sm["max_s"], st, MAX_LAYERS, out=o_ps)
        sg = pl.segment_device(ps, ps["max_s"], st, gl, 400, out=o_sg)
        ft = pl.fit_splines_device(sg["offsets"], sg["ref"], out=o_ft)
        ok = (sm["ok"] != 0) & (ps["ok"] != 0) & (sg["ok"] != 0) & (ft["ok"] != 0)
        pr = pl.plan_device(sg["n_points"], sg["offsets"], sg["ref"], sg["x0"], sg["end_heading"], max_n_points=400,
                            bounds_mode=planner.BOUNDS_IMPROVED, splines=ft,
                            map_index=torch.where(ok, torch.zeros_like(sm["ok"]), torch.full_like(sm["ok"], -1)),
                            out=o_pr)
        return sm, ps, sg, ft, pr
    outs = run()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run(*outs)
    g.replay()
    times = [wall(g.replay) for _ in range(reps)]
    res = dict(wall_ms=spread(times), smoothed=int(outs[0]["ok"].sum()), planned=int((outs[4]["status"] == 1).sum()))
    del g
    pl.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card())
    print("card, power limit:", res["card"], flush=True)
    side = torch.cuda.Stream()    # torch's default stream is the NULL stream, which the library takes for its own
    with torch.cuda.stream(side):
        res["smooth_stage"] = stage_times(a.reps)
        res["graph_cycle"] = {}
        for B in (16, 64):
            res["graph_cycle"][f"config1_{B}_candidates"] = cycle(B, a.reps)
            print(f"full chain graph, config 1, {B} candidates:", json.dumps(res["graph_cycle"][f"config1_{B}_candidates"]),
                  flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
