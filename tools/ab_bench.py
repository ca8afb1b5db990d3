#!/usr/bin/env python
"""A/B of two built trees with bench.py (development aid): runs `bench.py --gpus 1` from tree A, then from tree B, for
each configuration, `--pairs` times, alternating, and prints images/s and the per-kernel event times of every run, the
B/A ratio of every pair and the card's name and power limit.  The `--dump-outputs` arrays of the first pair of every
configuration are compared byte for byte.  Both trees must be built already (bench.py compiles nothing that is fresh).

usage: python tools/ab_bench.py TREE_A TREE_B [--configs p30,p10] [--pairs 3] [--steps 20] [--warmup 5]
                                [--env NAME=VALUE ...] [--env-b NAME=VALUE ...] [--out DIR]

TREE_A and TREE_B may be the same tree, to compare environment switches (--env-b applies to B's runs only)."""
import argparse, json, os, subprocess, sys, tempfile

ap = argparse.ArgumentParser()
ap.add_argument("a")
ap.add_argument("b")
ap.add_argument("--configs", default="p30")
ap.add_argument("--pairs", type=int, default=3)
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--warmup", type=int, default=5)
ap.add_argument("--env", action="append", default=[], help="NAME=VALUE for both trees' runs")
ap.add_argument("--env-b", action="append", default=[], help="NAME=VALUE for tree B's runs only")
ap.add_argument("--out", default=None, help="directory for the dumps and the JSON lines (default: a temporary one)")
args = ap.parse_args()
out = args.out or tempfile.mkdtemp(prefix="ab_bench_")
env = dict(os.environ, **dict(e.split("=", 1) for e in args.env))
env_b = dict(env, **dict(e.split("=", 1) for e in args.env_b))


def run(tree, cfg, tag, env):
    dump = os.path.join(out, tag)
    cmd = [sys.executable, "bench.py", "--gpus", "1", "--steps", str(args.steps), "--warmup", str(args.warmup),
           "--config", cfg, "--no-cpu-baseline", "--dump-outputs", dump]
    p = subprocess.run(cmd, cwd=tree, env=env, capture_output=True, text=True)
    line = [l for l in p.stdout.splitlines() if l.startswith("{")]
    if p.returncode or not line:
        sys.exit(f"{tag}: bench.py failed ({p.returncode})\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
    r = json.loads(line[-1])
    with open(os.path.join(out, "runs.jsonl"), "a") as f:
        f.write(json.dumps(dict(r, tag=tag)) + "\n")
    return r, dump


def same_dumps(da, db):
    names = sorted(os.listdir(da))
    if names != sorted(os.listdir(db)):
        return False
    return all(open(os.path.join(da, n), "rb").read() == open(os.path.join(db, n), "rb").read() for n in names)


print(f"A = {args.a}\nB = {args.b} {' '.join(args.env_b)}\nenv {args.env or '-'}; bench.py --steps {args.steps} --warmup {args.warmup}")
for cfg in args.configs.split(","):
    for i in range(args.pairs):
        ra, da = run(args.a, cfg, f"{cfg}_a{i}", env)
        rb, db = run(args.b, cfg, f"{cfg}_b{i}", env_b)
        if i == 0:
            d = ra["device"]
            print(f"[{cfg}] device {d['name']}, power limit {d['power_limit_w']} W; outputs A == B: {same_dumps(da, db)}")
        for t, r in (("A", ra), ("B", rb)):
            ks = ", ".join(f"{k} {v['ms']:.4f}" for k, v in r["kernels"].items())
            print(f"  {cfg} pair {i} {t}: {r['value']:.0f} images/s, {r['ms_per_pass']:.4f} ms/pass | {ks}")
        print(f"  {cfg} pair {i} B/A images/s: {rb['value'] / ra['value']:.4f}")
        sys.stdout.flush()
