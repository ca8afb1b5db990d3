#!/usr/bin/env python
"""A single stream of frames through ``dropin.FrameStream`` (one CUDA graph per slot and frame shape) against
``dropin.predict`` + ``dropin.group`` per frame, alternated round by round in the same run.

Workload: --frames seeded random uint8 frames, shapes drawn from a fixed table of COCO val2017 sizes, at the reference's
settings (boxsize 640, max_downsample 64, stride 4; scale_search [1] and rotation_search [0] unless --scale-search and
--rotation-search say otherwise); the network is imhn.IMHN at the reference's random initialisation, bf16 autocast,
channels-last (``imhn.Runner`` without a graph of its own: the frame graph records its forward).  Modes:
  * per_call:  predict + group + keypoints per frame, each frame finished before the next;
  * stream:    submit then result per frame (slots=2): the latency of one frame from submit to result;
  * pipelined: frame k+1 submitted before frame k's result is read (slots=2): the stream's frame rate.
Every mode runs once over every frame first (warm-up: every shape captured).  Reports per mode frames/s over the sequence
(host clock around work that ends in a device synchronise), the median and 90th percentile per-frame latency from the
first call to the result, and, in a separate pass under torch.profiler, the kernel time of the sequence (memcpy and
memset excluded; listed apart).  The people of every mode are compared with per_call's.  The card's name and power
limit are read in the same run.

usage: python tools/bench_frames.py [--frames 48] [--rounds 3] [--scale-search 1] [--rotation-search 0]
                                   [--out profiles/frames.json]"""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=48)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--scale-search", type=float, nargs="+", default=[1.0])
    ap.add_argument("--rotation-search", type=float, nargs="+", default=[0.0])
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "frames.json"))
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    from improved_body_parts_b200 import dropin, imhn, skeleton
    if not torch.cuda.is_available():
        raise SystemExit("bench_frames needs a CUDA device")
    dropin.configure(device=0, limbs=dropin.LIMBS, input_stage="device")
    rng = np.random.default_rng(2031)
    frames = [rng.integers(0, 256, size=SHAPES[int(rng.integers(len(SHAPES)))] + (3,), dtype=np.uint8)
              for _ in range(a.frames)]
    params = dict(skeleton.default_params(), scale_search=a.scale_search, rotation_search=a.rotation_search)
    runner = imhn.Runner(imhn.IMHN().init_like_reference_(0), device="cuda:0", use_graph=False)

    def model(x):
        return [[runner(x)]]

    fs = dropin.FrameStream(model, params, MODEL_PARAMS_REF, slots=2)

    def per_call(lat):
        out = []
        for f in frames:
            t = time.perf_counter()
            heat, paf = dropin.predict(f, params, model, MODEL_PARAMS_REF)
            out.append(dropin.keypoints(*dropin.group(heat, paf, f.shape[0], params)[3:]))
            lat.append(time.perf_counter() - t)
        return out

    def stream(lat):
        out = []
        for f in frames:
            t = time.perf_counter()
            out.append(fs.result(fs.submit(f)))
            lat.append(time.perf_counter() - t)
        return out

    def pipelined(lat):
        out, pending = [], []
        for f in frames:
            pending.append((fs.submit(f), time.perf_counter()))
            if len(pending) == 2:
                tk, t = pending.pop(0)
                out.append(fs.result(tk))
                lat.append(time.perf_counter() - t)
        for tk, t in pending:
            out.append(fs.result(tk))
            lat.append(time.perf_counter() - t)
        return out

    modes = {"per_call": per_call, "stream": stream, "pipelined": pipelined}
    people = {m: fn([]) for m, fn in modes.items()}  # warm-up: every shape once per mode (the stream captures its graphs)
    same = {m: repr(people[m]) == repr(people["per_call"]) for m in modes}
    times = {m: [] for m in modes}
    lats = {m: [] for m in modes}
    for _ in range(a.rounds):
        for m, fn in modes.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            fn(lats[m])
            torch.cuda.synchronize()
            times[m].append(time.perf_counter() - t)
    kern = {}
    for m, fn in modes.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn([])
            torch.cuda.synchronize()
        k = c = 0.0
        for ev in prof.key_averages():
            if ev.device_type is not None and "CUDA" in str(ev.device_type) and ev.device_time_total > 0:
                if ev.key.startswith(("Memcpy", "Memset")):
                    c += ev.device_time_total / 1e3
                else:
                    k += ev.device_time_total / 1e3
        kern[m] = (k, c)
    name, pl = card()
    res = {"card": name, "power_limit": pl, "frames": a.frames, "rounds": a.rounds, "scale_search": a.scale_search,
           "rotation_search": a.rotation_search, "captures": fs.captures, "modes": {}}
    print(f"{name}, power limit {pl}; {a.frames} frames, IMHN bf16, boxsize 640, scale_search {a.scale_search}, "
          f"rotation_search {a.rotation_search}; {fs.captures} graphs captured")
    for m in modes:
        ts = sorted(times[m])
        med = ts[len(ts) // 2]
        lat = np.sort(np.asarray(lats[m])) * 1e3
        k, c = kern[m]
        res["modes"][m] = dict(frames_per_s=a.frames / med, spread=[a.frames / ts[-1], a.frames / ts[0]], wall_ms=med * 1e3,
                               kernel_ms=k, copy_ms=c, latency_ms_p50=float(np.percentile(lat, 50)),
                               latency_ms_p90=float(np.percentile(lat, 90)), people_equal_per_call=same[m])
        print(f"  {m:>9}: {a.frames / med:6.1f} frames/s (min {a.frames / ts[-1]:.1f}, max {a.frames / ts[0]:.1f}); wall "
              f"{med * 1e3:.1f} ms vs kernels {k:.1f} ms (+ copies {c:.1f} ms); latency p50 "
              f"{np.percentile(lat, 50):.2f} ms, p90 {np.percentile(lat, 90):.2f} ms; people == per_call: {same[m]}")
    fs.close()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
