#!/usr/bin/env python
"""Grouping a COCO-shaped batch: one call per image (what evaluate.py does through dropin) against one ragged call per
batch (spg_group_ragged).

Workload: --images synthetic images (seeded) at image resolution, shapes drawn from a fixed table of COCO val2017 sizes
with a long side of 640, 1-15 persons each; heat float32, paf float32 grouped as SPG_F32_AS_F64 (what a single-scale
predict() produces).  Maps are resident on the device before timing.

Modes, alternated round by round in one process:
  * loop:   per image group_device + fetch(1) (a host synchronisation per image);
  * ragged: per batch of B images group_ragged + fetch(B), B in --batches.
Reports images/s per mode (host clock around work that ends in a synchronise), then, in a separate pass under
torch.profiler, the kernel time of each mode and K1's algorithmic bytes (sum of 18*H*W*4 over the images) over K1's
kernel time as a share of 3.35 TB/s (H100 SXM HBM3 data sheet, 700 W), and the card's name and power limit.  Asserts
that both modes produce identical person arrays.

usage: python tools/bench_ragged.py [--images 64] [--rounds 5] [--batches 8,16,32,64] [--out profiles/ragged.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BPS = 3.35e12
SHAPES = [(480, 640), (640, 480), (427, 640), (640, 427), (426, 640), (612, 612), (375, 500), (500, 375), (360, 640),
          (640, 512)]


def card():
    import torch
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True).stdout.strip()
    except OSError:
        pl = "unknown"
    return torch.cuda.get_device_name(0), pl


def workload(n, seed=2027):
    from improved_body_parts_b200 import synth
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        H, W = SHAPES[int(rng.integers(len(SHAPES)))]
        heat, paf = synth.make_image(seed + i, H, W, int(rng.integers(1, 16)))
        out.append((heat, paf))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batches", default="8,16,32,64")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "ragged.json"))
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    from improved_body_parts_b200 import skeleton
    from improved_body_parts_b200.grouping import Grouper
    if not torch.cuda.is_available():
        raise SystemExit("bench_ragged needs a CUDA device")
    dev = torch.device("cuda:0")
    batches = [int(b) for b in a.batches.split(",") if int(b) <= a.images]
    t0 = time.time()
    host = workload(a.images)
    print(f"workload: {a.images} images, {time.time() - t0:.1f} s to synthesise", flush=True)
    maps = [(torch.from_numpy(h).to(dev)[None], torch.from_numpy(p).to(dev)[None]) for h, p in host]
    ext = [float(h.shape[1]) for h, _ in host]
    params = skeleton.default_params()
    caps = dict(max_h=640, max_w=640, max_peaks_per_part=128, max_cands_per_limb=4096, max_person_rows=128)
    g1 = Grouper(max_batch=1, **caps)  # dropin's handle
    gb = Grouper(max_batch=max(batches), **caps)

    def loop():
        res = []
        for (h, p), e in zip(maps, ext):
            g1.group_device(h, p, e, params, paf_as_f64=True)
            res.append(g1.fetch(1))
        return res

    def ragged(b):
        res = []
        for i0 in range(0, len(maps), b):
            gb.group_ragged(maps[i0:i0 + b], ext[i0:i0 + b], params, paf_as_f64=True)
            res.append(gb.fetch(len(maps[i0:i0 + b])))
        return res

    # identical person arrays
    ref = loop()
    for b in batches:
        got = ragged(b)
        for i in range(len(maps)):
            r, j = got[i // b], i % b
            P = int(ref[i].n_persons[0])
            assert int(r.status[j]) == int(ref[i].status[0]) == 0, (b, i)
            assert int(r.n_persons[j]) == P and np.array_equal(r.subset[j, :P], ref[i].subset[0, :P]) and \
                np.array_equal(r.people_xy[j, :P], ref[i].people_xy[0, :P]) and \
                np.array_equal(r.people_score[j, :P], ref[i].people_score[0, :P]), f"batch {b}: image {i} differs"
    print("outputs: ragged == loop for every batch size", flush=True)

    modes = [("loop", loop)] + [(f"ragged_b{b}", (lambda b=b: ragged(b))) for b in batches]
    for _, f in modes:  # warm-up
        f()
    times = {m: [] for m, _ in modes}
    for _ in range(a.rounds):
        for m, f in modes:
            torch.cuda.synchronize()
            t = time.perf_counter()
            f()
            torch.cuda.synchronize()
            times[m].append(time.perf_counter() - t)
    # kernel times in a separate pass
    kern = {}
    for m, f in modes:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            f()
            torch.cuda.synchronize()
        per = {}
        for ev in prof.key_averages():
            if ev.device_type is not None and "CUDA" in str(ev.device_type) and "kernel" in ev.key.lower():
                per[ev.key.split("(")[0].split("<")[0]] = per.get(ev.key.split("(")[0].split("<")[0], 0.0) + \
                    ev.device_time_total / 1e3
        kern[m] = per
    k1_bytes = sum(18 * h.shape[1] * h.shape[2] * 4 for h, _ in host)
    name, pl = card()
    res = {"card": name, "power_limit": pl, "images": a.images, "rounds": a.rounds, "k1_bytes": k1_bytes, "modes": {}}
    print(f"{name}, power limit {pl}; {a.images} images, K1 algorithmic bytes {k1_bytes / 1e6:.1f} MB")
    for m, _ in modes:
        ts = sorted(times[m])
        med = ts[len(ts) // 2]
        k = kern[m]
        k1 = sum(v for key, v in k.items() if "nms_peaks" in key)
        k2 = sum(v for key, v in k.items() if "limb_score" in key)
        ma = sum(v for key, v in k.items() if "match" in key or "assemble" in key)
        frac = k1_bytes / (k1 * 1e-3) / HBM_BPS if k1 > 0 else float("nan")
        res["modes"][m] = dict(images_per_s=a.images / med, spread=[a.images / ts[-1], a.images / ts[0]], wall_ms=med * 1e3,
                               k1_ms=k1, k2a_ms=k2, match_assemble_ms=ma, kernels_ms=k, k1_hbm_fraction=frac)
        print(f"  {m:>12}: {a.images / med:8.1f} images/s (min {a.images / ts[-1]:.1f}, max {a.images / ts[0]:.1f}); "
              f"kernels K1 {k1:.3f} ms, K2a {k2:.3f} ms, match_assemble {ma:.3f} ms; K1 {frac:.3f} of 3.35 TB/s")
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    g1.close()
    gb.close()


if __name__ == "__main__":
    main()
