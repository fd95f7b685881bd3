"""TENSION smoothing of raw reference polylines on the device (pqp_smooth_reference_tension_device), beside the
default TENSION2 stage on the same polylines (one GPU command; prints the card and its power limit first).

  python profiles/tools/tension_smooth_probe.py [--reps 7] [--out FILE]

1. Stage time at 64, 1024 and 8192 config-1-like polylines (smooth_probe.polylines) on the config-1 map: CUDA events
   around 20 back-to-back calls queued behind a device-side sleep, per call, median over --reps rounds; torch.profiler's
   device time per call of each kernel beside it, and the QP's iteration counts.  The TENSION2 stage is timed the same
   way for comparison.
2. Wall time of one graph-replayed cycle smooth(TENSION) -> post-smooth -> segment -> fit -> plan_device (KP, IMPROVED
   bounds on the fitted splines) on the config-1 map at 16 and 64 candidates; median of --reps replays after a
   warm-up."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "profiles", "tools"))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from device_chain_probe import card, wall  # noqa: E402
from path_optimizer_b200 import planner  # noqa: E402
from smooth_probe import LAUNCHES, MAX_LAYERS, MAX_PTS, MAX_RAW, polylines, spread  # noqa: E402
from tests import segment_cases  # noqa: E402

KERNELS = {"TENSION": ("pqp_smooth_sample_kernel", "pqp_fit_splines_kernel", "pqp_smooth_tension_assemble_kernel",
                       "pqp_gen9_solve_kernel", "pqp_smooth_keep_kernel", "pqp_segment_scan_kernel",
                       "pqp_smooth_copy_kernel"),
           "TENSION2": ("pqp_smooth_assemble_kernel", "pqp_gen4_solve_kernel")}


def time_stage(pl, P, Of, method, reps):
    def call(out=None):
        return pl.smooth_device(P, Of, MAX_RAW, MAX_PTS, method=method, out=out)
    sm = call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    per = []
    for _ in range(reps):
        torch.cuda._sleep(2_000_000)
        e0.record()
        for _ in range(LAUNCHES):
            call(sm)
        e1.record()
        e1.synchronize()
        per.append(e0.elapsed_time(e1) / LAUNCHES)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            call(sm)
        torch.cuda.synchronize()
    prof_ms = {}
    for k in KERNELS[method]:
        v = [e.device_time for e in prof.events() if k in e.name and (k != "pqp_smooth_assemble_kernel" or
                                                                      "tension" not in e.name)]
        prof_ms[k] = sum(v) / reps / 1e3 if v else None
    it = sm["iters"].cpu().numpy()
    return dict(events=spread(per), profiler_ms_per_call=prof_ms, iters_mean=float(it.mean()), iters_max=int(it.max()),
                kept=int(sm["ok"].sum()))


def stage_times(reps):
    out = {}
    pl = planner.PathPlanner(max_batch=8192, max_total_points=8192 * 48)
    pl.set_maps([segment_cases.config1()["field"]])
    for B in (64, 1024, 8192):
        pts, off = polylines(B)
        P, Of = torch.from_numpy(pts).cuda(), torch.from_numpy(off).cuda()
        for method in ("TENSION", "TENSION2"):
            t = time_stage(pl, P, Of, method, reps)
            out[f"{method}_{B}_paths"] = t
            print(f"{method} stage, {B} polylines: {json.dumps(t)}", flush=True)
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
        sm = pl.smooth_device(P, Of, MAX_RAW, MAX_PTS, method="TENSION", out=o_sm)
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
            print(f"TENSION chain graph, config 1, {B} candidates:",
                  json.dumps(res["graph_cycle"][f"config1_{B}_candidates"]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
