"""Many parameter sets in one plan call: pqp_set_param_sets + a set index per path against one set at a time (one GPU
command; prints the card and its power limit first).

  python profiles/tools/param_sets_probe.py [--reps 7] [--sizes 4,16,64] [--baseline-root DIR] [--out FILE]

1. S sets (synth.param_sets) x 16 candidates x 200 stations on one map (KP, simple bounds, raw output), wall time per
   planning cycle of all S x 16 paths:
     (a) loop_host    pqp_set_params + pqp_plan_batch for each set (what a caller does without parameter sets)
     (b) loop_device  pqp_set_params + plan_device on the set's slice of resident inputs, for each set
     (c) loop_graph   one captured graph per set (captured after its pqp_set_params), replayed one after the other
     (d) sets_host    one pqp_plan_batch_sets call
     (e) sets_device  plan_device with a set index (pqp_plan_batch_device_sets)
     (f) sets_graph   a CUDA graph replay of (e)
   Every variant is warmed up, then the variants alternate for --reps rounds; medians are reported.
2. What the extra per-(set, class) grids cost when one set is used: plan_device with an all-zero index and
   n_param_sets = 1, 4, 16, 64 against the plain entry, on config 3 (8192 x 200) and on a 64-candidate cycle on the
   config-1 map, device and graph replay.
3. With --baseline-root: multi_map_probe.py's regression of the existing entries (another checkout with its library
   built, e.g. the parent commit's, against this one; result digests and config 3 / config 1 timings, alternating)."""
import argparse
import json
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


def _graph(fn):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def cycles(field, sets, S, reps):
    b = synth.map_reference_paths(S * C_CAND, N_ST)
    B, T = S * C_CAND, int(b["offsets"][-1])
    pi = np.repeat(np.arange(S, dtype=np.int32), C_CAND)
    parts = [synth.slice_batch(b, k * C_CAND, (k + 1) * C_CAND) for k in range(S)]
    dev = torch.device("cuda", 0)
    loop = planner.PathPlanner(max_batch=C_CAND, max_total_points=C_CAND * N_ST)
    pl = planner.PathPlanner(max_batch=B, max_total_points=T)
    for p in (loop, pl):
        p.set_map(field)
    pl.set_param_sets(sets[:S])
    dparts = [device.batch_to_device(x, dev) for x in parts]
    d = device.batch_to_device(b, dev)
    pi_t = torch.from_numpy(pi).to(dev)

    def dev_one(p, x, **kw):
        return p.plan_device(x["n_points"], x["offsets"], x["ref"], x["x0"], x["end_heading"], max_n_points=N_ST, **kw)

    def loop_host():
        for k in range(S):
            loop.set_params(sets[k])
            loop.plan(parts[k])

    def loop_device():
        for k in range(S):
            loop.set_params(sets[k])
            dev_one(loop, dparts[k])

    # one graph per set: each captures its set's parameters; they share the loop planner's scratch, so they run in turn
    graphs = []
    for k in range(S):
        loop.set_params(sets[k])
        graphs.append(_graph(lambda: dev_one(loop, dparts[k])))

    def loop_graph():
        for g in graphs:
            g.replay()

    run_sets = lambda: dev_one(pl, d, param_index=pi_t)   # noqa: E731
    gs = _graph(run_sets)
    res = alternate(dict(loop_host=lambda: wall(loop_host), loop_device=lambda: wall(loop_device),
                         loop_graph=lambda: wall(loop_graph), sets_host=lambda: wall(lambda: pl.plan(b, param_index=pi)),
                         sets_device=lambda: wall(run_sets), sets_graph=lambda: wall(gs.replay)), reps)
    del graphs, gs
    loop.close()
    pl.close()
    return res


def extra_grids(field, sets, b, reps):
    B = len(b["n_points"])
    dev = torch.device("cuda", 0)
    pl = planner.PathPlanner(max_batch=B, max_total_points=int(b["offsets"][-1]))
    pl.set_map(field)
    pl.set_param_sets(sets)
    d = device.batch_to_device(b, dev)
    zero = torch.zeros(B, dtype=torch.int32, device=dev)
    max_n = int(b["n_points"].max())

    def run(**kw):
        return lambda: pl.plan_device(d["n_points"], d["offsets"], d["ref"], d["x0"], d["end_heading"],
                                      max_n_points=max_n, **kw)
    fns = dict(plain=run())
    for ns in (1, 4, 16, 64):
        fns[f"sets_{ns}"] = run(param_index=zero, n_param_sets=ns)
    graphs = {k: _graph(f) for k, f in fns.items()}
    variants = {f"{k}_device": (lambda f=f: wall(f)) for k, f in fns.items()}
    variants.update({f"{k}_graph": (lambda g=g: wall(g.replay)) for k, g in graphs.items()})
    res = alternate(variants, reps)
    del graphs
    pl.close()
    return res


def config1_cycle(B):
    g = np.load(os.path.join(ROOT, "tests", "golden", "config1_benchmark_map.npz"))
    field = dict(distance=g["map_distance"], rows=int(g["image_shape"][0]), cols=int(g["image_shape"][1]),
                 resolution=float(g["map_geo"][0]), center_x=float(g["map_geo"][1]), center_y=float(g["map_geo"][2]))
    n = int(g["n_points"][0])
    ref = np.concatenate([g["ref"]] * B)
    for i, dy in enumerate(np.linspace(-0.6, 0.6, B)):
        ref["y"][i * n:(i + 1) * n] += dy
    b = dict(n_points=np.full(B, n, dtype=np.int32), ref=ref, x0=np.repeat(g["x0"].reshape(1, 3), B, 0),
             end_heading=np.repeat(g["end_heading"], B))
    b["offsets"] = np.r_[0, np.cumsum(b["n_points"])].astype(np.int32)
    return field, b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--sizes", default="4,16,64")
    ap.add_argument("--baseline-root", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card())
    print("card, power limit:", res["card"], flush=True)
    sizes = [int(s) for s in a.sizes.split(",")]
    sets = synth.param_sets(max(sizes + [64]))
    field = synth.disc_field_map()
    res["cycles_wall_ms"] = {}
    for S in sizes:
        res["cycles_wall_ms"][f"{S}_sets"] = cycles(field, sets, S, a.reps)
        print(f"{S} sets x {C_CAND} candidates:", json.dumps(res["cycles_wall_ms"][f"{S}_sets"]), flush=True)
    f1, b1 = config1_cycle(64)
    res["extra_grids_wall_ms"] = dict(
        config3_8192x200=extra_grids(field, sets, synth.map_reference_paths(8192, N_ST), a.reps),
        config1_64_candidates=extra_grids(f1, sets, b1, a.reps))
    print("extra grids:", json.dumps(res["extra_grids_wall_ms"]), flush=True)
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
