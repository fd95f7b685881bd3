"""Many scenes in one plan call: pqp_set_maps + a map index per path against one scene at a time (one GPU command;
prints the card and its power limit first).

  python profiles/tools/multi_map_probe.py [--reps 7] [--sizes 16,64,256] [--baseline-root DIR] [--out FILE]

1. S scenes x 16 candidates x 200 stations (KP, simple bounds, raw output; scenes from synth.scene_map, 1100 x 250
   cells each), wall time per planning cycle of all S x 16 paths:
     (a) loop      pqp_set_map + pqp_plan_batch for each scene (what a caller does without map sets)
     (b) maps      pqp_set_maps once, then one pqp_plan_batch_maps per cycle
     (c) device    plan_device with a map index on resident inputs (pqp_plan_batch_device_maps)
     (d) graph     a CUDA graph replay of (c)
   Every variant is warmed up, then the variants alternate for --reps rounds; medians are reported.
2. The bounds stage of config 3's 8192 x 200 paths spread over 1, 8, 64 and 256 maps of 1.1 MB each (the H100's L2
   holds 50 MB), with the paths grouped by map and interleaved: the pqp_bounds_kernel time from torch.profiler's CUDA
   activity records (the chain has no separate timer for that stage), median over --reps calls of plan_device.
3. With --baseline-root: the existing entries of another checkout with its library built (e.g. the parent commit's;
   its path_optimizer_b200 package, libpqp.so, profiles/tools/device_chain_probe.py and tests/golden are used) against
   this one, each measured in a fresh process, the two alternating for --reps rounds: config 3 (8192 x 200) through
   pqp_plan_batch, plan_device and a graph replay, and 16- and 64-candidate cycles on the config-1 map
   (profiles/tools/device_chain_probe.py's workloads).  Each process also hashes the results of pqp_plan_batch on
   config 3 and of an improved-bounds, densified batch, so the two builds can be checked for identical outputs."""
import argparse
import hashlib
import json
import multiprocessing
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if "--worker-root" in sys.argv:   # the checkout a regression worker measures (its package and its probe helpers)
    ROOT = os.path.abspath(sys.argv[sys.argv.index("--worker-root") + 1])
sys.path.insert(0, os.path.join(ROOT, "profiles", "tools"))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from device_chain_probe import alternate, card, plan_three, small_cycles, wall  # noqa: E402
from path_optimizer_b200 import device, planner, synth  # noqa: E402

C_CAND, N_ST = 16, 200


def cycles(maps, S, reps):
    sub_maps, b, mi = synth.multi_map_batch(S, C_CAND, n=N_ST, first_maps=maps[:S])
    B, T = len(mi), int(b["offsets"][-1])
    scenes = [synth.slice_batch(b, m * C_CAND, (m + 1) * C_CAND) for m in range(S)]
    loop = planner.PathPlanner(max_batch=C_CAND, max_total_points=C_CAND * N_ST)
    pl = planner.PathPlanner(max_batch=B, max_total_points=T)
    pl.set_maps(sub_maps)
    dev = torch.device("cuda", 0)
    d = device.batch_to_device(b, dev)
    mi_t = torch.from_numpy(mi).to(dev)

    def run_loop():
        for m in range(S):
            loop.set_map(sub_maps[m])
            loop.plan(scenes[m])

    def run_dev():
        return pl.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], max_n_points=N_ST,
                              map_index=mi_t)
    run_dev()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run_dev()
    res = alternate(dict(loop_set_map_plan_batch=lambda: wall(run_loop),
                         set_maps_plan_batch_maps=lambda: wall(lambda: pl.plan(b, map_index=mi)),
                         plan_device_maps=lambda: wall(run_dev),
                         graph_replay=lambda: wall(g.replay)), reps)
    del g
    loop.close()
    pl.close()
    return res


def bounds_l2(maps, reps):
    from torch.profiler import ProfilerActivity, profile
    out = {}
    dev = torch.device("cuda", 0)
    pl = planner.PathPlanner(max_batch=8192, max_total_points=8192 * N_ST)
    for M in (1, 8, 64, 256):
        for order in ("grouped", "interleaved"):
            sub_maps, b, mi = synth.multi_map_batch(M, 8192 // M, n=N_ST, first_maps=maps[:M], order=order)
            pl.set_maps(sub_maps)
            d = device.batch_to_device(b, dev)
            mi_t = torch.from_numpy(mi).to(dev)

            def run():
                pl.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], max_n_points=N_ST,
                               map_index=mi_t)
            run()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(reps):
                    run()
                torch.cuda.synchronize()
            t = [e.device_time for e in prof.events() if "pqp_bounds_kernel" in e.name]
            assert len(t) == reps, len(t)
            out[f"{M}_maps_{order}"] = dict(median_ms=statistics.median(t) / 1e3, min_ms=min(t) / 1e3,
                                            map_mb=round(sum(m["distance"].nbytes for m in sub_maps) / 1e6, 1))
            print(f"bounds kernel, {M} maps, {order}: {json.dumps(out[f'{M}_maps_{order}'])}", flush=True)
    pl.close()
    return out


def _digest(r, keys=("states", "n_out", "ok", "status", "iters", "bounds")):
    h = hashlib.sha256()
    for k in keys:
        h.update(np.ascontiguousarray(r[k]).tobytes())
    return h.hexdigest()[:16]


def worker(reps):
    """One build's existing entries (the library PQP_LIB names): timings and result digests."""
    field = synth.disc_field_map()
    b = synth.map_reference_paths(8192, N_ST)
    pl = planner.PathPlanner(max_batch=8192, max_total_points=8192 * N_ST)
    pl.set_map(field)
    res = dict(config3_plan_wall_ms=plan_three(pl, b, reps=reps))
    res["digest_config3_simple_raw"] = _digest(pl.plan(b, want_bounds=True))
    w = synth.map_reference_paths(512, N_ST, first_path=9000, y_range=(-1.5, 1.5), heading_range=0.03,
                                  curvature_amp=0.01)
    r = pl.plan(w, bounds_mode=planner.BOUNDS_IMPROVED, splines=planner.reference_splines(w),
                output_mode=planner.OUTPUT_DENSIFY, max_out=256, want_bounds=True)
    r["states"] = np.concatenate([r["states"][i, :r["n_out"][i]] for i in range(512)])   # the reported samples
    res["digest_512_improved_densify"] = _digest(r)
    pl.close()
    res["config1_small_cycle_wall_ms"] = small_cycles(reps)
    print(json.dumps(res), flush=True)


def regression(baseline_root, reps):
    roots = dict(baseline=os.path.abspath(baseline_root), this=ROOT)
    runs = {k: [] for k in roots}
    env = {k: v for k, v in os.environ.items() if k != "PQP_LIB"}
    for _ in range(reps):
        for k, root in roots.items():
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "--worker-root", root,
                                "--reps", "3"], env=env, capture_output=True, text=True, check=True)
            runs[k].append(json.loads(p.stdout.strip().splitlines()[-1]))
    out = {}
    for k, rs in runs.items():
        med = lambda f: statistics.median(f(r) for r in rs)  # noqa: E731
        out[k] = dict(
            config3_plan_batch_ms=med(lambda r: r["config3_plan_wall_ms"]["plan_batch_host"]["median_ms"]),
            config3_plan_device_ms=med(lambda r: r["config3_plan_wall_ms"]["plan_device"]["median_ms"]),
            config3_graph_replay_ms=med(lambda r: r["config3_plan_wall_ms"]["graph_replay"]["median_ms"]),
            **{f"config1_{c}_{v}_ms": med(lambda r: r["config1_small_cycle_wall_ms"][f"{c}_candidates"][v]["median_ms"])
               for c in (16, 64) for v in ("plan_batch_host", "plan_device", "graph_replay")},
            digests=sorted({(r["digest_config3_simple_raw"], r["digest_512_improved_densify"]) for r in rs}))
    out["same_results"] = out["baseline"]["digests"] == out["this"]["digests"] and len(out["this"]["digests"]) == 1
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--sizes", default="16,64,256")
    ap.add_argument("--baseline-root", default=None)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--worker-root", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a.reps)
    res = dict(card=card())
    print("card, power limit:", res["card"], flush=True)
    sizes = [int(s) for s in a.sizes.split(",")]
    n_maps = max(sizes + [256])
    with multiprocessing.Pool(min(16, os.cpu_count() or 1)) as pool:
        maps = list(pool.starmap(synth.scene_map, [(k, synth.BASE_SEED) for k in range(n_maps)]))
    res["cycles_wall_ms"] = {}
    for S in sizes:
        res["cycles_wall_ms"][f"{S}_scenes"] = cycles(maps, S, a.reps)
        print(f"{S} scenes x {C_CAND} candidates:", json.dumps(res["cycles_wall_ms"][f"{S}_scenes"]), flush=True)
    res["bounds_kernel_config3"] = bounds_l2(maps, a.reps)
    if a.baseline_root:
        res["existing_entries"] = regression(a.baseline_root, a.reps)
        print("existing entries:", json.dumps(res["existing_entries"]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
