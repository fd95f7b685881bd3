"""The reference splines of IMPROVED bounds fitted on the device (pqp_fit_splines_device) against the host fit (one GPU
command; prints the card and its power limit first).

  python profiles/tools/spline_fit_probe.py [--reps 7] [--baseline-root DIR] [--out FILE]

1. Fit kernel time alone at 64, 1024 and 8192 paths x 200 stations (config-3 reference lines): CUDA events around 20
   back-to-back launches queued behind a device-side sleep (so no host gap is timed), per launch, median over --reps
   rounds; torch.profiler's device time of pqp_fit_splines_kernel beside it (a run of its own).
2. Wall time of one IMPROVED planning cycle (KP, raw output) on resident inputs, three ways:
     (a) host_fit      planner.reference_splines + device.splines_to_device + plan_device
                       (the copy of the reference lines to the host is not counted)
     (b) device_fit    fit_splines_device + plan_device
     (c) graph_replay  a CUDA graph replay of (b)
   for config 3 (8192 x 200 on synth.disc_field_map) and 16- and 64-candidate cycles on the config-1 map (the benchmark
   path shifted sideways, as profiles/tools/device_chain_probe.py builds them).  Every variant is warmed up, then the
   variants alternate for --reps rounds; medians are reported.
3. With --baseline-root: multi_map_probe.py's comparison of the existing entries of another checkout with its library
   built (e.g. the parent commit's) against this one: result digests and timings, each build in fresh processes,
   alternating."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "profiles", "tools"))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from device_chain_probe import alternate, card, wall  # noqa: E402
from path_optimizer_b200 import device, planner, synth  # noqa: E402

N_ST = 200
LAUNCHES = 20


def fit_kernel(reps):
    """On a side stream: torch's default stream is the NULL stream, which the library takes for the handle's own."""
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        return _fit_kernel(reps)


def _fit_kernel(reps):
    from torch.profiler import ProfilerActivity, profile
    dev = torch.device("cuda", 0)
    out = {}
    pl = planner.PathPlanner(max_batch=8192, max_total_points=8192 * N_ST)
    for B in (64, 1024, 8192):
        b = synth.map_reference_paths(B, N_ST)
        d = device.batch_to_device(b, dev)
        spl = pl.fit_splines_device(d["offsets"], d["ref"])
        torch.cuda.synchronize()
        assert (spl["ok"] == 1).all()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        per = []
        for _ in range(reps):
            torch.cuda._sleep(2_000_000)
            e0.record()
            for _ in range(LAUNCHES):
                pl.fit_splines_device(d["offsets"], d["ref"], out=spl)
            e1.record()
            e1.synchronize()
            per.append(e0.elapsed_time(e1) / LAUNCHES)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                pl.fit_splines_device(d["offsets"], d["ref"], out=spl)
            torch.cuda.synchronize()
        t = [e.device_time for e in prof.events() if "pqp_fit_splines_kernel" in e.name]
        assert len(t) == reps, len(t)
        out[f"{B}_paths"] = dict(events_median_ms=statistics.median(per), events_min_ms=min(per),
                                 profiler_median_ms=statistics.median(t) / 1e3)
        print(f"fit kernel, {B} x {N_ST}: {json.dumps(out[f'{B}_paths'])}", flush=True)
    pl.close()
    return out


def cycle_variants(pl, b, max_n, reps):
    dev = torch.device("cuda", 0)
    d = device.batch_to_device(b, dev)

    def plan(spl):
        return pl.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], max_n_points=max_n,
                              bounds_mode=planner.BOUNDS_IMPROVED, splines=spl)

    def host_fit():
        return plan(device.splines_to_device(planner.reference_splines(b), dev))
    spl = pl.fit_splines_device(d["offsets"], d["ref"])

    def device_fit():
        return plan(pl.fit_splines_device(d["offsets"], d["ref"], out=spl))
    # the two fits give the same paths, bit for bit (unsolved paths carry NaN states)
    a, c = host_fit(), device_fit()
    torch.cuda.synchronize()
    assert torch.equal(a["states"].view(torch.int64), c["states"].view(torch.int64))
    for k in ("status", "iters", "n_out", "ok"):
        assert torch.equal(a[k], c[k]), k
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        device_fit()
    res = alternate(dict(host_fit=lambda: wall(host_fit), device_fit=lambda: wall(device_fit),
                         graph_replay=lambda: wall(g.replay)), reps)
    del g
    return res


def config1_batch(B):
    g = np.load(os.path.join(ROOT, "tests", "golden", "config1_benchmark_map.npz"))
    field = dict(distance=g["map_distance"], rows=int(g["image_shape"][0]), cols=int(g["image_shape"][1]),
                 resolution=float(g["map_geo"][0]), center_x=float(g["map_geo"][1]), center_y=float(g["map_geo"][2]))
    n = int(g["n_points"][0])
    ref = np.concatenate([g["ref"]] * B)
    for i, dy in enumerate(np.linspace(-0.6, 0.6, B)):   # candidates: the benchmark path shifted sideways
        ref["y"][i * n:(i + 1) * n] += dy
    b = dict(n_points=np.full(B, n, dtype=np.int32), ref=ref, x0=np.repeat(g["x0"].reshape(1, 3), B, 0),
             end_heading=np.repeat(g["end_heading"], B))
    b["offsets"] = np.r_[0, np.cumsum(b["n_points"])].astype(np.int32)
    return field, b, n


def cycles(reps):
    out = {}
    pl = planner.PathPlanner(max_batch=8192, max_total_points=8192 * N_ST)
    pl.set_map(synth.disc_field_map())
    out["config3_8192x200"] = cycle_variants(pl, synth.map_reference_paths(8192, N_ST), N_ST, reps)
    print("config 3:", json.dumps(out["config3_8192x200"]), flush=True)
    pl.close()
    for B in (16, 64):
        field, b, n = config1_batch(B)
        pl = planner.PathPlanner(max_batch=B, max_total_points=B * n)
        pl.set_map(field)
        out[f"config1_{B}_candidates"] = cycle_variants(pl, b, n, reps)
        print(f"config 1, {B} candidates:", json.dumps(out[f"config1_{B}_candidates"]), flush=True)
        pl.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--baseline-root", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card())
    print("card, power limit:", res["card"], flush=True)
    res["fit_kernel_ms"] = fit_kernel(a.reps)
    res["improved_cycle_wall_ms"] = cycles(a.reps)
    if a.baseline_root:
        from multi_map_probe import regression
        res["existing_entries"] = regression(a.baseline_root, a.reps)
        print("existing entries:", json.dumps(res["existing_entries"]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
