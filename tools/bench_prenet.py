#!/usr/bin/env python
"""Cost of the pre-network stage (spg_prenet) against the host input path of predict(), on the reference's default
geometry: a 480x640 uint8 image at boxsize 640 (max_downsample 64, padValue 128), for four search settings.

Per setting it prints
  * the time of one spg_prenet call over all items: CUDA events around --iters calls after a warm-up (this includes
    the host's enqueue, which can bound it), and the kernels' own time from torch.profiler in a separate pass; the bytes
    the call must move (the pairs written, the source read, and for rotated items the scratch grid written and read) and
    that floor at 3.35 TB/s (H100 SXM HBM3 data sheet) as a share of the kernels' time;
  * the host path's time on the CPU of the host running the benchmark: dropin.predict's cv2 preparation of every item, and with the upload of
    each pair from pageable memory;
  * end-to-end dropin.predict with a stand-in model (a 4x4 average pool, expanded to 50 channels) for
    input_stage="host" against "device".
and the card's name and power limit.

The ragged setting (--only ragged, or all) builds the inputs of a batch as dropin.predict_batch does: the 16 COCO-shaped
images of tools/bench_predict_batch.py at boxsize 640, grouped by network input size (dropin.plan_items), each member
written into its slot of its size's batch tensor, under [1] x [0] and [0.5, 1, 1.5, 2] x [0, 30, -30].  It compares one
spg_prenet call per member against one spg_prenet_ragged call per input size: call time from CUDA events, kernel time
from torch.profiler in a separate pass, launches per batch, and the bytes-over-3.35 TB/s floor as a share of the kernels.

usage: python tools/bench_prenet.py [--iters 50] [--only all|single|ragged] [--out profiles/prenet/bench_prenet.json]"""
import argparse
import itertools
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

HBM_BPS = 3.35e12
RAGGED_SETTINGS = [([1.0], [0.0]), ([0.5, 1.0, 1.5, 2.0], [0.0, 30.0, -30.0])]
SETTINGS = [([1.0], [0.0]), ([1.0], [0.0, 30.0, -30.0]), ([0.5, 1.0, 1.5, 2.0], [0.0]), ([0.5, 1.0, 1.5, 2.0], [0.0, 30.0, -30.0])]
MODEL_PARAMS = dict(boxsize=640, stride=4, max_downsample=64, padValue=128)


def card():
    import torch
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True).stdout.strip()
    except OSError:
        pl = "unknown"
    return torch.cuda.get_device_name(0), pl


def host_items(image, multiplier, angles):
    """dropin.predict's host preparation (cv2) of every item; returns the pairs."""
    import cv2

    from improved_body_parts_b200 import dropin
    pairs = []
    for scale, angle in itertools.product(multiplier, angles):
        if scale * image.shape[0] > 2600 or scale * image.shape[1] > 3800:
            scale = min(2600 / image.shape[0], 3800 / image.shape[1])
        image_to_test = cv2.resize(image, (0, 0), fx=scale, fy=scale, interpolation=cv2.INTER_CUBIC)
        padded, _ = dropin.pad_right_down_corner(image_to_test, 64, 128)
        input_img = np.float32(padded / 255)
        if angle != 0:
            centre = (input_img.shape[0] / 2, input_img.shape[1] / 2)
            input_img = cv2.warpAffine(input_img, cv2.getRotationMatrix2D(centre, angle, 1), (0, 0))
        pairs.append(np.concatenate((input_img[None, ...], input_img[:, ::-1, :].copy()[None, ...]), axis=0))
    return pairs


def stand_in_model(x):
    import torch
    y = torch.nn.functional.avg_pool2d(x.permute(0, 3, 1, 2)[:, :1], 4)
    return [[y.expand(2, 50, y.shape[2], y.shape[3]).contiguous()]]


def timed(fn, iters, g):
    """(ms per call from CUDA events, {kernel: ms per call} from torch.profiler, launches per call) of fn()."""
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    call_ms = start.elapsed_time(end) / iters
    launches = g._lib.spg_launch_count(g._h)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    launches = (g._lib.spg_launch_count(g._h) - launches) / iters
    kernels = {}
    for ev in prof.key_averages():
        if "prenet" in ev.key:
            us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            kernels[ev.key.split("(")[0]] = us / 1e3 / iters
    return call_ms, kernels, launches


def ragged(iters, name, power):
    """The ragged setting: per-member spg_prenet calls against one spg_prenet_ragged call per network input size."""
    import torch

    from bench_predict_batch import SHAPES
    from improved_body_parts_b200 import dropin, skeleton
    from improved_body_parts_b200.grouping import Grouper
    rng = np.random.default_rng(2029)  # the first 16 images of tools/bench_predict_batch.py
    images = [rng.integers(0, 256, size=SHAPES[int(rng.integers(len(SHAPES)))] + (3,), dtype=np.uint8) for _ in range(16)]
    dev_imgs = [torch.from_numpy(im).cuda() for im in images]
    g = Grouper(max_batch=16, device=0)
    results = []
    for scale_search, angles in RAGGED_SETTINGS:
        params = dict(skeleton.default_params(), scale_search=scale_search, rotation_search=angles)
        plan, buckets = dropin.plan_items([im.shape[:2] for im in images], params, MODEL_PARAMS)
        xs = {key: torch.empty((2 * len(m), key[0], key[1], 3), dtype=torch.float32, device="cuda") for key, m in buckets.items()}
        nbytes = 0
        for (Hp, Wp), members in buckets.items():
            for i, t in members:
                # the pair written, the source read once; a rotated member's uint8 grid written and read
                nbytes += 2 * Hp * Wp * 3 * 4 + images[i].size + (2 * Hp * Wp * 3 if plan[i][t][2] != 0 else 0)

        def per_member():
            for key, members in buckets.items():
                for j, (i, t) in enumerate(members):
                    g.prenet(dev_imgs[i], [plan[i][t][0]], [plan[i][t][2]], max_downsample=64, pad_value=128,
                             out=[xs[key][2 * j:2 * j + 2]])

        def one_per_size():
            for key, members in buckets.items():
                g.prenet_ragged([(dev_imgs[i], plan[i][t][0], plan[i][t][2]) for i, t in members], max_downsample=64,
                                pad_value=128, out=[xs[key][2 * j:2 * j + 2] for j in range(len(members))])

        r = dict(setting="ragged", scale_search=scale_search, rotation_search=angles, images=16,
                 members=sum(len(m) for m in buckets.values()), input_sizes=len(buckets), bytes=nbytes,
                 hbm_floor_ms=nbytes / HBM_BPS * 1e3, device=name, power_limit=power)
        for label, fn in (("per_member", per_member), ("ragged", one_per_size)):
            call_ms, kernels, launches = timed(fn, iters, g)
            kern_ms = sum(kernels.values())
            r[label] = dict(call_ms=call_ms, kernel_ms=kern_ms, kernels=kernels, launches=launches,
                            share_of_hbm=r["hbm_floor_ms"] / kern_ms)
            print(f"ragged {scale_search} x {angles}: {r['members']} members in {len(buckets)} input sizes, {label}: "
                  f"call {call_ms:.3f} ms, kernels {kern_ms:.4f} ms ({launches:g} launches; "
                  + ", ".join(f"{k} {v:.4f}" for k, v in kernels.items())
                  + f"), floor {r['hbm_floor_ms']:.4f} ms = {r['hbm_floor_ms'] / kern_ms:.2f} of HBM")
        sys.stdout.flush()
        results.append(r)
        del xs
    g.close()
    return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--only", default="all", choices=("all", "single", "ragged"))
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "prenet", "bench_prenet.json"),
                    help="JSON results (default under profiles/, which git ignores)")
    args = ap.parse_args()
    import torch

    from improved_body_parts_b200 import dropin, skeleton
    from improved_body_parts_b200.grouping import Grouper
    if not torch.cuda.is_available():
        raise SystemExit("bench_prenet needs a CUDA device")
    name, power = card()
    print(f"device {name}, power limit {power}")
    rng = np.random.default_rng(0)
    image = rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)
    dev_img = torch.from_numpy(image).cuda()
    params = dict(skeleton.default_params())
    results = ragged(args.iters, name, power) if args.only in ("all", "ragged") else []
    g = Grouper(max_batch=1, device=0)
    for scale_search, angles in SETTINGS if args.only in ("all", "single") else []:
        multiplier = [x * 640 / 480 for x in scale_search]
        items = g.prenet(dev_img, multiplier, angles, max_downsample=64, pad_value=128)
        outs = [p for p, _, _ in items]
        nbytes = 0
        for (p, _, _), (_, angle) in zip(items, itertools.product(multiplier, angles)):
            # the pair written, the source read once; a rotated item's uint8 grid (Hp * Wp * 3 B) written and read
            nbytes += p.numel() * 4 + image.size + (p.numel() if angle != 0 else 0)
        for _ in range(5):
            g.prenet(dev_img, multiplier, angles, max_downsample=64, pad_value=128, out=outs)
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        for _ in range(args.iters):
            g.prenet(dev_img, multiplier, angles, max_downsample=64, pad_value=128, out=outs)
        end.record()
        end.synchronize()
        dev_ms = start.elapsed_time(end) / args.iters
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                g.prenet(dev_img, multiplier, angles, max_downsample=64, pad_value=128, out=outs)
            torch.cuda.synchronize()
        kernels = {}
        for ev in prof.key_averages():
            if "prenet" in ev.key:
                us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                kernels[ev.key] = dict(ms_per_launch=us / 1e3 / ev.count, launches_per_call=ev.count / args.iters)
        kern_ms = sum(k["ms_per_launch"] * k["launches_per_call"] for k in kernels.values())
        floor_ms = nbytes / HBM_BPS * 1e3
        # host path: preparation, and preparation + pageable upload
        host_items(image, multiplier, angles)
        reps = 5
        t0 = time.perf_counter()
        for _ in range(reps):
            host_items(image, multiplier, angles)
        host_ms = (time.perf_counter() - t0) / reps * 1e3
        t0 = time.perf_counter()
        for _ in range(reps):
            for p in host_items(image, multiplier, angles):
                torch.from_numpy(p).cuda()
            torch.cuda.synchronize()
        host_up_ms = (time.perf_counter() - t0) / reps * 1e3
        # end to end
        p = dict(params, scale_search=scale_search, rotation_search=angles)
        e2e = {}
        for stage in ("host", "device"):
            dropin.predict(image, p, stand_in_model, MODEL_PARAMS, 19, 30, None, input_stage=stage)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(reps):
                dropin.predict(image, p, stand_in_model, MODEL_PARAMS, 19, 30, None, input_stage=stage)
            torch.cuda.synchronize()
            e2e[stage] = (time.perf_counter() - t0) / reps * 1e3
        r = dict(scale_search=scale_search, rotation_search=angles, items=len(items), call_ms=dev_ms, kernel_ms=kern_ms,
                 kernels=kernels, bytes=nbytes, hbm_floor_ms=floor_ms, share_of_hbm=floor_ms / kern_ms,
                 host_prep_ms=host_ms, host_prep_upload_ms=host_up_ms, predict_host_ms=e2e["host"],
                 predict_device_ms=e2e["device"], device=name, power_limit=power)
        results.append(r)
        ks = ", ".join(f"{k} {v['ms_per_launch']:.4f} ms x {v['launches_per_call']:g}" for k, v in kernels.items())
        print(f"{scale_search} x {angles}: {len(items)} items | call {dev_ms:.3f} ms, kernels {kern_ms:.4f} ms ({ks}), "
              f"{nbytes / 1e6:.1f} MB, floor {floor_ms:.4f} ms = {floor_ms / kern_ms:.2f} of HBM | host prep {host_ms:.1f} ms, "
              f"+ upload {host_up_ms:.1f} ms | predict host {e2e['host']:.1f} ms, device {e2e['device']:.1f} ms")
        sys.stdout.flush()
    g.close()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
