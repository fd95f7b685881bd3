"""Cost of the device-side class dispatch and of the device-resident plan chain (one GPU command; prints the card and
its power limit first).

  python profiles/tools/device_chain_probe.py [--reps 7] [--out FILE]

1. BASELINE config 5 shape (4096 paths x U{50..400} stations, KP): kernel time (CUDA events, pqp_stats.kernel_ms) of
   pqp_solve_batch_device_classes (classes from host copies of the lengths) against pqp_solve_batch_device_dispatch
   (classes picked on the device).  The difference is the dispatch kernel, the order fill and the CTAs past each
   class's last path.
2. Config 3 shape through the plan chain (8192 x 200 stations on the 1100 x 250 disc map): pqp_plan_batch (host
   buffers, host wall clock) against plan_device on resident inputs against a CUDA graph replay of plan_device.
3. A small planning cycle, 16 and 64 candidates on the config-1 map (the reference's benchmark path, shifted sideways):
   wall time per cycle for the same three.
Every variant is warmed up, then the variants alternate for --reps rounds; medians are reported."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import ctypes as C  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

from path_optimizer_b200 import device, planner, synth  # noqa: E402
from path_optimizer_b200.abi import Stats  # noqa: E402
from path_optimizer_b200.solver import BatchPathSolver  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def alternate(variants, reps):
    for fn in variants.values():   # warm-up
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in variants}
    for _ in range(reps):
        for k, fn in variants.items():
            times[k].append(fn())
    return {k: dict(median_ms=statistics.median(v), min_ms=min(v), max_ms=max(v)) for k, v in times.items()}


def config5(reps):
    B = 4096
    b = synth.curvy_corridors(B, n_points=synth.mixed_lengths(B, 50, 400), config=5)
    s = BatchPathSolver(max_batch=B, max_total_points=int(b["offsets"][-1]))
    dev = torch.device("cuda", 0)
    d = device.batch_to_device(b, dev)
    T = int(b["offsets"][-1])
    out = torch.empty((T, 7), dtype=torch.float64, device=dev)
    fr = torch.empty((T, 3), dtype=torch.float64, device=dev)
    st = torch.empty(B, dtype=torch.int32, device=dev)
    it = torch.empty(B, dtype=torch.int32, device=dev)
    hn = np.ascontiguousarray(b["n_points"], dtype=np.int32)
    hk = np.array([s._L.pqp_keep_control_steps(0, b["ref"][b["offsets"][i]:].ctypes.data_as(C.c_void_p), int(hn[i]))
                   for i in range(B)], dtype=np.int32)
    ptrs = [d[k].data_ptr() for k in ("n_points", "offsets", "ref", "bounds", "x0", "end_heading")] + [None, None] + \
           [out.data_ptr(), fr.data_ptr(), st.data_ptr(), it.data_ptr(), torch.cuda.current_stream().cuda_stream]

    def classes():
        stats = Stats()
        assert s._L.pqp_solve_batch_device_classes(s._h, 0, B, T, hn.ctypes.data_as(C.c_void_p),
                                                   hk.ctypes.data_as(C.c_void_p), *ptrs, C.byref(stats)) == 0
        return stats.kernel_ms

    def dispatch():
        stats = Stats()
        assert s._L.pqp_solve_batch_device_dispatch(s._h, 0, B, T, 400, 0, 0, *ptrs, C.byref(stats)) == 0
        return stats.kernel_ms
    res = alternate(dict(device_classes=classes, device_dispatch=dispatch), reps)
    a, b_ = res["device_classes"]["median_ms"], res["device_dispatch"]["median_ms"]
    res["dispatch_minus_classes_ms"] = b_ - a
    res["dispatch_minus_classes_pct"] = 100.0 * (b_ - a) / a
    s.close()
    return res


def plan_three(pl, b, splines=None, mode=planner.BOUNDS_SIMPLE, reps=7):
    dev = torch.device("cuda", 0)
    d = device.batch_to_device(b, dev)
    spl = device.splines_to_device(splines, dev) if splines is not None else None
    max_n = int(b["n_points"].max())

    def run_dev():
        return pl.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], max_n_points=max_n,
                              bounds_mode=mode, splines=spl)
    run_dev()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run_dev()
    res = alternate(dict(plan_batch_host=lambda: wall(lambda: pl.plan(b, bounds_mode=mode, splines=splines)),
                         plan_device=lambda: wall(run_dev),
                         graph_replay=lambda: wall(g.replay)), reps)
    del g
    return res


def config3(reps):
    field = synth.disc_field_map()
    b = synth.map_reference_paths(8192, 200)
    pl = planner.PathPlanner(max_batch=8192, max_total_points=8192 * 200)
    pl.set_map(field)
    res = plan_three(pl, b, reps=reps)
    pl.close()
    return res


def small_cycles(reps):
    g = np.load(os.path.join(ROOT, "tests", "golden", "config1_benchmark_map.npz"))
    field = dict(distance=g["map_distance"], rows=int(g["image_shape"][0]), cols=int(g["image_shape"][1]),
                 resolution=float(g["map_geo"][0]), center_x=float(g["map_geo"][1]), center_y=float(g["map_geo"][2]))
    n = int(g["n_points"][0])
    out = {}
    for B in (16, 64):
        ref = np.concatenate([g["ref"]] * B)
        for i, dy in enumerate(np.linspace(-0.6, 0.6, B)):   # candidates: the benchmark path shifted sideways
            ref["y"][i * n:(i + 1) * n] += dy
        b = dict(n_points=np.full(B, n, dtype=np.int32), ref=ref, x0=np.repeat(g["x0"].reshape(1, 3), B, 0),
                 end_heading=np.repeat(g["end_heading"], B))
        b["offsets"] = np.r_[0, np.cumsum(b["n_points"])].astype(np.int32)
        pl = planner.PathPlanner(max_batch=B, max_total_points=B * n)
        pl.set_map(field)
        out[f"{B}_candidates"] = plan_three(pl, b, reps=reps)
        pl.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card())
    print("card, power limit:", res["card"], flush=True)
    res["config5_4096_mixed_kernel_ms"] = config5(a.reps)
    print(json.dumps(res["config5_4096_mixed_kernel_ms"]), flush=True)
    res["config3_plan_wall_ms"] = config3(a.reps)
    print(json.dumps(res["config3_plan_wall_ms"]), flush=True)
    res["config1_small_cycle_wall_ms"] = small_cycles(a.reps)
    print(json.dumps(res["config1_small_cycle_wall_ms"]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
