#!/usr/bin/env python
"""predict() + grouping of a COCO-shaped image stream: per image (``dropin.predict``: a forward pass of the image and its
mirror and a post-network launch per image) against ``dropin.predict_batch`` (one forward pass per input size and chunk
of forward_batch images, one ragged post-network call per group).

Workload: --images seeded random uint8 images, shapes drawn from a fixed table of COCO val2017 sizes, at the reference's
settings (utils/config: boxsize 640, max_downsample 64, scale_search [1], rotation_search [0], stride 4), so every image
is resized to 640 rows and the images fall into a few network input sizes.  --scale-search and --rotation-search (comma
lists) select the reference's accuracy mode instead, e.g. 0.5,1,1.5,2 or 0,30,-30: every image then has one item per
(scale, angle), and the batched mode groups the items by input size (``dropin.plan_items``).  The network is imhn.IMHN with the
reference's random initialisation, bf16 autocast, channels-last, no CUDA graph.  The input stage is --input-stage
(default device: spg_prenet per image).  Every group of --group images is grouped with one ragged call
(``predict_many``'s batching).

Modes, alternated round by round after every mode has run once on every image (every shape warmed up):
  * per_image: predict per image;
  * fb{k}:     predict_batch with forward_batch k, k in --forward-batches.
Reports images/s per mode (host clock around work that ends in a device synchronise: the grouping's download), then, in
a separate pass under torch.profiler, the kernel time per mode split into network, pre-network, post-network and
grouping kernels, and the post-network kernels by name (the per-image launches against the ragged ones for the same
images).  Also the largest absolute difference between the per-image and the batched maps (and raw network outputs of
one input size): the network's numerics across batch sizes.  The card's name and power limit are read in the same run.

usage: python tools/bench_predict_batch.py [--images 48] [--group 16] [--rounds 3] [--forward-batches 2,4,8,16]
                                           [--scale-search 1] [--rotation-search 0]
                                           [--out profiles/predict_batch.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [(480, 640), (640, 480), (427, 640), (640, 427), (612, 612), (375, 500), (640, 640), (500, 375), (360, 640),
          (426, 640)]
MODEL_PARAMS_REF = dict(boxsize=640, stride=4, max_downsample=64, padValue=128)


def card():
    import torch
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True).stdout.strip()
    except OSError:
        pl = "unknown"
    return torch.cuda.get_device_name(0), pl


def kernel_class(name):
    if "postnet" in name:
        return "postnet"
    if "prenet" in name:
        return "prenet"
    if any(k in name for k in ("nms_peaks", "limb_score", "limb_match", "assemble")):
        return "grouping"
    return "network"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=48)
    ap.add_argument("--group", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--forward-batches", default="2,4,8,16")
    ap.add_argument("--input-stage", default="device", choices=("host", "device"))
    ap.add_argument("--scale-search", default="1", help="comma list (utils/config scale_search)")
    ap.add_argument("--rotation-search", default="0", help="comma list of angles (utils/config rotation_search)")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "predict_batch.json"))
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    from improved_body_parts_b200 import dropin, imhn, skeleton
    if not torch.cuda.is_available():
        raise SystemExit("bench_predict_batch needs a CUDA device")
    dropin.configure(device=0, limbs=dropin.LIMBS, input_stage=a.input_stage)
    rng = np.random.default_rng(2029)
    images = [rng.integers(0, 256, size=SHAPES[int(rng.integers(len(SHAPES)))] + (3,), dtype=np.uint8)
              for _ in range(a.images)]
    params = dict(skeleton.default_params(), scale_search=[float(v) for v in a.scale_search.split(",")],
                  rotation_search=[float(v) for v in a.rotation_search.split(",")])
    runner = imhn.Runner(imhn.IMHN().init_like_reference_(0), device="cuda:0", use_graph=False)

    def model(x):
        return [[runner(x)]]

    _, buckets = dropin.plan_items([im.shape[:2] for im in images], params, MODEL_PARAMS_REF)
    print(f"workload: {a.images} images, scale_search {params['scale_search']}, rotation_search "
          f"{params['rotation_search']}, input sizes {{(Hp, Wp): items}} = "
          f"{ {k: len(v) for k, v in buckets.items()} }", flush=True)
    groups = [list(range(i, min(i + a.group, a.images))) for i in range(0, a.images, a.group)]
    fbs = [int(k) for k in a.forward_batches.split(",")]

    def run(fb):
        out = []
        for idx in groups:
            if fb == 0:
                maps = [dropin.predict(images[i], params, model, MODEL_PARAMS_REF) for i in idx]
            else:
                maps = dropin.predict_batch([images[i] for i in idx], params, model, MODEL_PARAMS_REF, forward_batch=fb)
            out.append(dropin._people_of_batch(maps, [images[i].shape[0] for i in idx], params))
        return out

    modes = [("per_image", 0)] + [(f"fb{k}", k) for k in fbs]
    people = {m: run(fb) for m, fb in modes}  # warm-up: every shape and batch size once
    same_people = {m: people[m] == people["per_image"] for m, _ in modes}
    times = {m: [] for m, _ in modes}
    for _ in range(a.rounds):
        for m, fb in modes:
            torch.cuda.synchronize()
            t = time.perf_counter()
            run(fb)
            torch.cuda.synchronize()
            times[m].append(time.perf_counter() - t)
    # kernel times in a separate pass
    kern = {}
    for m, fb in modes:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run(fb)
            torch.cuda.synchronize()
        per = {}
        for ev in prof.key_averages():
            if ev.device_type is not None and "CUDA" in str(ev.device_type) and ev.device_time_total > 0 and \
                    not ev.key.startswith(("Memcpy", "Memset")):
                per[ev.key] = per.get(ev.key, 0.0) + ev.device_time_total / 1e3
        kern[m] = per
    # numerics: per-image against batched maps, and the raw network output of one input size
    with torch.no_grad():
        one = [dropin.predict(im, params, model, MODEL_PARAMS_REF) for im in images[:a.group]]
        bat = dropin.predict_batch(images[:a.group], params, model, MODEL_PARAMS_REF, forward_batch=max(fbs))
        map_diff = max(float((x.tensor - y.tensor).abs().max()) for p, q in zip(one, bat) for x, y in zip(p, q))
        (Hp, Wp), idx = max(buckets.items(), key=lambda kv: len(kv[1]))
        x = torch.rand((2 * min(len(idx), max(fbs)), Hp, Wp, 3), device="cuda:0", generator=torch.Generator("cuda:0").manual_seed(5))
        whole = runner(x).clone()
        pairs = torch.cat([runner(x[2 * j:2 * j + 2]).clone() for j in range(x.shape[0] // 2)])
        net_diff = float((whole - pairs).abs().max())
    name, pl = card()
    res = {"card": name, "power_limit": pl, "images": a.images, "group": a.group, "rounds": a.rounds,
           "input_stage": a.input_stage, "scale_search": params["scale_search"],
           "rotation_search": params["rotation_search"], "input_sizes": {f"{k[0]}x{k[1]}": len(v) for k, v in buckets.items()},
           "max_abs_diff_maps": map_diff, "max_abs_diff_network": net_diff, "network_diff_batch": list(x.shape),
           "modes": {}}
    print(f"{name}, power limit {pl}; {a.images} images in groups of {a.group}, input stage {a.input_stage}")
    print(f"max |per-image - batched|: maps {map_diff:.3g}, raw network output ({x.shape[0]} x {Hp}x{Wp}) {net_diff:.3g}")
    for m, _ in modes:
        ts = sorted(times[m])
        med = ts[len(ts) // 2]
        split = {}
        for key, v in kern[m].items():
            split[kernel_class(key)] = split.get(kernel_class(key), 0.0) + v
        post = {key.split("(")[0]: round(v, 4) for key, v in kern[m].items() if "postnet" in key}
        res["modes"][m] = dict(images_per_s=a.images / med, spread=[a.images / ts[-1], a.images / ts[0]], wall_ms=med * 1e3,
                               kernel_ms=split, postnet_kernels_ms=post, people_equal_per_image=same_people[m])
        print(f"  {m:>9}: {a.images / med:7.1f} images/s (min {a.images / ts[-1]:.1f}, max {a.images / ts[0]:.1f}); kernels "
              + ", ".join(f"{k} {v:.2f} ms" for k, v in sorted(split.items())) + f"; people == per_image: {same_people[m]}")
        print(f"             post-network kernels: {post}")
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
