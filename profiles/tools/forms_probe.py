"""Several formulations in one plan call: one formulation per path ("KP", "K", "KPC") against one call per formulation
(one GPU command; prints the card and its power limit first).

  python profiles/tools/forms_probe.py [--reps 7] [--sizes 16,64,256] [--baseline-root DIR] [--out FILE]

1. S scenes x 16 candidates x 200 stations (simple bounds, raw output; scenes from synth.scene_map, 1100 x 250 cells
   each, a map index per path), formulations assigned round robin over the paths, wall time per planning cycle:
     (a) split     three plan_device calls, one per formulation, each over its own resident paths
     (b) host      one pqp_plan_batch_forms
     (c) device    one plan_device(formulation=) on resident inputs (pqp_plan_batch_device_forms)
     (d) graph     a CUDA graph replay of (c)
   Every variant is warmed up, then the variants alternate for --reps rounds; medians are reported.
2. The cost of the mask: config 3 (8192 x 200 on the disc map), every path "KP": plain plan_device against
   plan_device(formulation=) with form_mask = "KP" only and with all three formulations.
3. With --baseline-root: multi_map_probe.py's regression of the existing entries, this checkout against another with
   its library built (e.g. the parent commit's)."""
import argparse
import json
import multiprocessing
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "profiles", "tools"))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from device_chain_probe import alternate, card, wall  # noqa: E402
from path_optimizer_b200 import device, planner, synth  # noqa: E402

C_CAND, N_ST = 16, 200
NAMES = ("KP", "K", "KPC")


def _speed_profile(b):
    """v, a fields that give the "KPC" limits something to bound."""
    t = np.arange(int(b["offsets"][-1]))
    b["ref"]["v"] = 4.0 + 3.0 * np.sin(t * 0.05)
    b["ref"]["a"] = 0.5 * np.cos(t * 0.05)
    return b


def cycles(maps, S, reps):
    sub_maps, b, mi = synth.multi_map_batch(S, C_CAND, n=N_ST, first_maps=maps[:S])
    b = _speed_profile(b)
    B, T = len(mi), int(b["offsets"][-1])
    forms = (np.arange(B) % 3).astype(np.int32)
    pl = planner.PathPlanner(max_batch=B, max_total_points=T)
    pl.set_maps(sub_maps)
    dev = torch.device("cuda", 0)
    d = device.batch_to_device(b, dev)
    mi_t, f_t = torch.from_numpy(mi).to(dev), torch.from_numpy(forms).to(dev)
    parts = []
    for f in range(3):
        idx = np.flatnonzero(forms == f)
        parts.append((NAMES[f], device.batch_to_device(synth.take_paths(b, idx), dev), torch.from_numpy(mi[idx]).to(dev)))

    def run_split():
        for name, dp, mp in parts:
            pl.plan_device(dp["n_points"], dp["offsets"], dp["ref"], dp["x0"], dp["end_heading"], max_n_points=N_ST,
                           formulation=name, map_index=mp)

    def run_dev():
        return pl.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"], max_n_points=N_ST,
                              formulation=f_t, map_index=mi_t)
    run_dev()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run_dev()
    res = alternate(dict(three_plan_device_calls=lambda: wall(run_split),
                         plan_batch_forms=lambda: wall(lambda: pl.plan(b, formulation=forms, map_index=mi)),
                         plan_device_forms=lambda: wall(run_dev),
                         graph_replay=lambda: wall(g.replay)), reps)
    del g
    pl.close()
    return res


def mask_cost(reps):
    b = synth.map_reference_paths(8192, N_ST)
    pl = planner.PathPlanner(max_batch=8192, max_total_points=8192 * N_ST)
    pl.set_map(synth.disc_field_map())
    dev = torch.device("cuda", 0)
    d = device.batch_to_device(b, dev)
    kp = torch.zeros(8192, dtype=torch.int32, device=dev)

    def run(**kw):
        return lambda: wall(lambda: pl.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"],
                                                   max_n_points=N_ST, **kw))
    res = alternate(dict(plan_device=run(), forms_mask_kp=run(formulation=kp, form_mask=1),
                         forms_mask_all=run(formulation=kp, form_mask=0)), reps)
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
    sizes = [int(s) for s in a.sizes.split(",")]
    with multiprocessing.Pool(min(16, os.cpu_count() or 1)) as pool:
        maps = list(pool.starmap(synth.scene_map, [(k, synth.BASE_SEED) for k in range(max(sizes))]))
    res["cycles_wall_ms"] = {}
    for S in sizes:
        res["cycles_wall_ms"][f"{S}_scenes"] = cycles(maps, S, a.reps)
        print(f"{S} scenes x {C_CAND} candidates:", json.dumps(res["cycles_wall_ms"][f"{S}_scenes"]), flush=True)
    res["mask_cost_config3"] = mask_cost(a.reps)
    print("config 3, every path KP:", json.dumps(res["mask_cost_config3"]), flush=True)
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
