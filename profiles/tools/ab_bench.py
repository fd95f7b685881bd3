"""Diagnostic: A/B comparison of two (or more) builds of libpqp.so on the same GPU, through bench.py.

  python profiles/tools/ab_bench.py --lib parent=path/to/libpqp_parent.so --lib new=path_optimizer_b200/libpqp.so \
      --out DIR [--rounds 5] [--configs 2,4,5] [--dumps 2,3,4,5,2:KPC,2:K]

Each build is loaded by its own bench.py process (PQP_LIB selects the library; build an A/B library with
PQP_OBJ_SUFFIX / PQP_LIB_OUT, see path_optimizer_b200/build.py).  The timed runs ALTERNATE the builds round by round
(`--rounds` rounds of `bench.py --config C --no-extras` per config), so that drift of the shared card falls on both
alike; the first round of each config also dumps its outputs.  `--dumps` lists further config[:formulation] runs that
only dump.  Every dump of a build is compared byte for byte with the same dump of the first build.

Writes DIR/ab.json: the card (name, power limit), every bench line's value / ms_per_step / clocks, per build and config
the min / median / max, and the dump comparison; prints a short summary.  Exit code 1 when any dump differs."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip() if r.returncode == 0 else "unknown (nvidia-smi failed)"


def bench(lib, config, formulation, dump_dir, no_extras=True):
    env = dict(os.environ, PQP_LIB=os.path.abspath(lib))
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--config", str(config), "--formulation", formulation]
    if no_extras:
        cmd.append("--no-extras")
    if dump_dir:
        cmd += ["--dump-outputs", dump_dir]
    p = subprocess.run(cmd, env=env, capture_output=True, text=True)
    if p.returncode != 0:
        raise RuntimeError(f"bench.py failed with {lib}:\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
    line = json.loads([ln for ln in p.stdout.splitlines() if ln.startswith("{")][-1])
    return {"value": line["value"], "ms_per_step": line["ms_per_step"], "clocks": line.get("clocks"),
            "iters_per_solve_mean": line.get("iters_per_solve_mean")}


def same_files(a, b):
    names = sorted(set(os.listdir(a)) | set(os.listdir(b)))
    diff = []
    for n in names:
        pa, pb = os.path.join(a, n), os.path.join(b, n)
        if not (os.path.exists(pa) and os.path.exists(pb)):
            diff.append(n + " (missing)")
            continue
        with open(pa, "rb") as fa, open(pb, "rb") as fb:
            if fa.read() != fb.read():
                diff.append(n)
    return names, diff


def spread(xs):
    return {"min": min(xs), "median": statistics.median(xs), "max": max(xs), "n": len(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", required=True, help="NAME=path of a libpqp.so build (first = reference)")
    ap.add_argument("--out", required=True)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--configs", default="2")
    ap.add_argument("--dumps", default="", help="further config[:formulation] runs that only dump outputs")
    a = ap.parse_args()
    libs = [tuple(s.split("=", 1)) for s in a.lib]
    os.makedirs(a.out, exist_ok=True)
    res = {"card": card(), "libs": dict(libs), "runs": {}, "spread": {}, "dumps": {}}
    print("card, power limit, max SM clock:", res["card"], flush=True)
    dump_keys = []
    for cfg in [int(c) for c in a.configs.split(",") if c]:
        key = f"{cfg}:KP"
        dump_keys.append(key)
        for rnd in range(a.rounds):
            for name, lib in (libs if rnd % 2 == 0 else libs[::-1]):
                d = os.path.join(a.out, "dump", name, key.replace(":", "_")) if rnd == 0 else None
                r = bench(lib, cfg, "KP", d)
                res["runs"].setdefault(key, {}).setdefault(name, []).append(r)
                print(f"config {key} round {rnd} {name}: {r['ms_per_step']:.4f} ms/step  {r['value']:.0f} solves/s  "
                      f"clocks {json.dumps(r['clocks'])}", flush=True)
        res["spread"][key] = {name: {"ms_per_step": spread([r["ms_per_step"] for r in rs]),
                                     "value": spread([r["value"] for r in rs])}
                              for name, rs in res["runs"][key].items()}
    for spec in [s for s in a.dumps.split(",") if s]:
        cfg, _, form = spec.partition(":")
        key = f"{cfg}:{form or 'KP'}"
        if key in dump_keys:
            continue
        dump_keys.append(key)
        for name, lib in libs:
            bench(lib, int(cfg), form or "KP", os.path.join(a.out, "dump", name, key.replace(":", "_")))
    ok = True
    for key in dump_keys:
        ref_dir = os.path.join(a.out, "dump", libs[0][0], key.replace(":", "_"))
        for name, _ in libs[1:]:
            names, diff = same_files(ref_dir, os.path.join(a.out, "dump", name, key.replace(":", "_")))
            res["dumps"].setdefault(key, {})[name] = {"files": names, "differ": diff}
            ok = ok and not diff and bool(names)
            print(f"dump {key} {name} vs {libs[0][0]}: {len(names)} files, "
                  f"{'byte-identical' if not diff else 'DIFFER: ' + ', '.join(diff)}", flush=True)
    for key, per in res["spread"].items():
        for name, s in per.items():
            m = s["ms_per_step"]
            print(f"config {key} {name}: ms/step min {m['min']:.4f} median {m['median']:.4f} max {m['max']:.4f} (n={m['n']})")
    res["all_dumps_identical"] = ok
    with open(os.path.join(a.out, "ab.json"), "w") as f:
        json.dump(res, f, indent=1)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
