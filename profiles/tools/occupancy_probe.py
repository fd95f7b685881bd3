"""Distance maps built on the device from occupancy grids (pqp_set_maps_occupancy, pqp_set_maps_occupancy_device): one
GPU command; prints the card and its power limit first.

  python profiles/tools/occupancy_probe.py [--reps 7] [--sizes 16,64,256] [--baseline-root DIR] [--out FILE]

1. Transform kernel time per call (CUDA events around a same-layout pqp_set_maps_occupancy_device, which only launches
   the two transform kernels per 256 maps): 1, 16, 64 and 256 maps of 1100 x 250 cells, one 495 x 497 map (config 1),
   one 4096 x 4096 map.  Medians over --reps calls after a warm-up.
2. Wall time per planning cycle of S scenes x 16 candidates x 200 stations (KP, simple bounds, raw output) when every
   cycle starts from occupancy grids:
     (a) host_transform  cv2.distanceTransform(L2, MASK_PRECISE) * resolution per map on the host (the reference's
                         recipe; scipy's distance_transform_edt when cv2 is missing, reported as such) + pqp_set_maps +
                         plan_device
     (b) occupancy_host    pqp_set_maps_occupancy (host grids) + plan_device
     (c) occupancy_device  pqp_set_maps_occupancy_device (grids already on the device) + plan_device
     (d) graph             a CUDA graph replay of (c)
   Every variant is warmed up, then the variants alternate for --reps rounds; medians are reported.
3. With --baseline-root: multi_map_probe.py's regression of the existing entries (another checkout with its library
   built, e.g. the parent commit's, against this one; result digests and config 3 / config 1 timings, alternating, in
   fresh processes)."""
import argparse
import json
import multiprocessing
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

C_CAND, N_ST = 16, 200


def scene_occupancy(k, seed=synth.BASE_SEED):
    """The occupancy grid of synth.scene_map(k)."""
    if k % 4 == 1:
        return synth.disc_field_occupancy(resolution=0.25, seed=seed + k, center=(35.0 + 10.0 * (k % 7), -20.0 + 3.0 * (k % 5)))
    return synth.disc_field_occupancy(seed=seed + k)


def host_transform():
    try:
        import cv2

        def layer(occ, res):
            return cv2.distanceTransform(occ, cv2.DIST_L2, cv2.DIST_MASK_PRECISE) * np.float32(res)
        return "cv2", layer
    except ImportError:
        return "scipy", synth.distance_layer


def _dev_maps(occ):
    dev = torch.device("cuda", 0)
    return [dict(m, occupancy=torch.from_numpy(m["occupancy"]).to(dev)) for m in occ]


def kernel_times(occ_1100, reps):
    g = np.load(os.path.join(ROOT, "tests", "golden", "config1_benchmark_map.npz"))
    c1 = dict(occupancy=(g["map_distance"] != 0).astype(np.uint8), resolution=float(g["map_geo"][0]),
              center_x=float(g["map_geo"][1]), center_y=float(g["map_geo"][2]))
    big = dict(occupancy=(np.random.default_rng(3).random((4096, 4096)) >= 0.001).astype(np.uint8), resolution=0.1,
               center_x=0.0, center_y=0.0)
    cases = {f"{M}_maps_1100x250": occ_1100[:M] for M in (1, 16, 64, 256)}
    cases["1_map_495x497"] = [c1]
    cases["1_map_4096x4096"] = [big]
    pl = planner.PathPlanner(max_batch=1, max_total_points=N_ST)
    out = {}
    # a stream of its own: torch's default stream is the NULL stream, which the library reads as its handle's stream,
    # so events on it would not bracket the launches
    stream = torch.cuda.Stream()
    for name, maps in cases.items():
        dm = _dev_maps(maps)
        torch.cuda.synchronize()
        t = []
        with torch.cuda.stream(stream):
            pl.set_maps_occupancy_device(dm)   # lays the set out
            pl.set_maps_occupancy_device(dm)
            for _ in range(reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                pl.set_maps_occupancy_device(dm)
                e1.record()
                e1.synchronize()
                t.append(e0.elapsed_time(e1))
        out[name] = dict(median_ms=statistics.median(t), min_ms=min(t),
                         cells_per_us=round(sum(m["occupancy"].size for m in maps) / (statistics.median(t) * 1e3), 1))
        print(f"transform {name}: {json.dumps(out[name])}", flush=True)
        del dm
    pl.close()
    return out


def _graph(fn):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def cycles(occ, S, reps):
    occ = occ[:S]
    _, b, mi = synth.multi_map_batch(S, C_CAND, n=N_ST, first_maps=occ)
    B, T = len(mi), int(b["offsets"][-1])
    dev = torch.device("cuda", 0)
    d = device.batch_to_device(b, dev)
    mi_t = torch.from_numpy(mi).to(dev)
    dm = _dev_maps(occ)
    kind, layer = host_transform()
    pl = planner.PathPlanner(max_batch=B, max_total_points=T)

    def plan():
        return pl.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], max_n_points=N_ST,
                              map_index=mi_t)

    def host():
        pl.set_maps([dict(m, distance=layer(m["occupancy"], m["resolution"])) for m in occ])
        plan()

    def occ_host():
        pl.set_maps_occupancy(occ)
        plan()

    def occ_device():
        pl.set_maps_occupancy_device(dm)
        plan()
    occ_device()
    g = _graph(occ_device)
    # every variant leaves the same layout, so (c) and (d) stay on the launch-only path after (a) and (b)
    res = alternate({f"host_{kind}": lambda: wall(host), "occupancy_host": lambda: wall(occ_host),
                     "occupancy_device": lambda: wall(occ_device), "graph": lambda: wall(g.replay)}, reps)
    del g
    pl.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--sizes", default="16,64,256")
    ap.add_argument("--baseline-root", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card())
    print("card, power limit:", res["card"], flush=True)
    sizes = [int(s) for s in a.sizes.split(",") if s]   # --sizes "": transform times only
    with multiprocessing.Pool(min(16, os.cpu_count() or 1)) as pool:
        occ = pool.map(scene_occupancy, range(max(sizes + [256])))
    res["transform_kernel_ms"] = kernel_times(occ, a.reps)
    res["cycles_wall_ms"] = {}
    for S in sizes if a.sizes else []:
        res["cycles_wall_ms"][f"{S}_scenes"] = cycles(occ, S, a.reps)
        print(f"{S} scenes x {C_CAND} candidates:", json.dumps(res["cycles_wall_ms"][f"{S}_scenes"]), flush=True)
    if a.baseline_root:
        import multi_map_probe
        res["existing_entries"] = multi_map_probe.regression(a.baseline_root, a.reps)
        print("existing entries:", json.dumps(res["existing_entries"]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
