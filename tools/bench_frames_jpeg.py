#!/usr/bin/env python
"""A single stream of JPEG frames through ``dropin.FrameStream``: decoded on the host with ``cv2.imdecode`` and submitted
as images, against the bytes submitted as they are and decoded inside each frame's CUDA graph (``spg_jpeg_decode_frame``),
alternated round by round in the same run.

Workload: --frames seeded ``synth.photo`` frames, shapes drawn from a fixed table of COCO val2017 sizes, encoded by
``cv2.imencode`` at quality 95, 4:2:0 (as most COCO files are), at the reference's settings (boxsize 640, max_downsample
64, scale_search [1], rotation_search [0], stride 4); the network is imhn.IMHN at the reference's random initialisation,
bf16 autocast, channels-last (``imhn.Runner`` without a graph of its own: the frame graph records its forward).  Each
frame's result is read before the next submit (slots=2).  Modes, each with a stream of its own:
  * cv2:      ``cv2.imdecode`` on the host, then ``submit(image)``;
  * jpeg:     ``submit(bytes)``, files without restart intervals (the subsequence decode);
  * jpeg_rst: ``submit(bytes)``, files with a restart interval per MCU row (one thread decodes each interval).
Every mode runs once over every frame first (warm-up: every shape and format captured).  Reports per mode frames/s over
the sequence (host clock around work that ends in a device synchronise; median and min-max over the rounds), the median
and 90th percentile per-frame latency from the submit (the cv2 mode: from the decode) to the result, and, in a separate
pass under torch.profiler, the decode kernels' time per frame.  The people of every mode are compared with cv2's.  The
card's name and power limit are read in the same run.

usage: python tools/bench_frames_jpeg.py [--frames 48] [--rounds 5] [--out profiles/frames_jpeg.json]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_frames import MODEL_PARAMS_REF, SHAPES, card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=48)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "frames_jpeg.json"))
    a = ap.parse_args()
    import cv2
    import torch
    from torch.profiler import ProfilerActivity, profile

    from improved_body_parts_b200 import dropin, imhn, skeleton, synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_frames_jpeg needs a CUDA device")
    dropin.configure(device=0, limbs=dropin.LIMBS, input_stage="device")
    rng = np.random.default_rng(2032)
    images = [synth.photo(int(rng.integers(1 << 30)), *SHAPES[int(rng.integers(len(SHAPES)))]) for _ in range(a.frames)]

    def encode(img, restart):
        ok, buf = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 95, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, 0x221111,
                                             cv2.IMWRITE_JPEG_RST_INTERVAL, restart])
        assert ok
        return buf.tobytes()

    plain = [encode(img, 0) for img in images]
    rst = [encode(img, -(-img.shape[1] // 16)) for img in images]  # 4:2:0: an MCU is 16 pixels wide
    params = dict(skeleton.default_params(), scale_search=[1.0], rotation_search=[0.0])
    runner = imhn.Runner(imhn.IMHN().init_like_reference_(0), device="cuda:0", use_graph=False)

    def model(x):
        return [[runner(x)]]

    streams = {m: dropin.FrameStream(model, params, MODEL_PARAMS_REF, slots=2) for m in ("cv2", "jpeg", "jpeg_rst")}

    def run(mode, files, lat):
        fs, out = streams[mode], []
        for data in files:
            t = time.perf_counter()
            frame = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR) if mode == "cv2" else data
            out.append(fs.result(fs.submit(frame)))
            lat.append(time.perf_counter() - t)
        return out

    modes = {"cv2": plain, "jpeg": plain, "jpeg_rst": rst}
    people = {m: run(m, files, []) for m, files in modes.items()}  # warm-up: every shape and format captured
    same = {m: repr(people[m]) == repr(people["cv2"]) for m in modes}
    times = {m: [] for m in modes}
    lats = {m: [] for m in modes}
    for _ in range(a.rounds):
        for m, files in modes.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            run(m, files, lats[m])
            torch.cuda.synchronize()
            times[m].append(time.perf_counter() - t)
    decode = {}
    for m, files in modes.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run(m, files, [])
            torch.cuda.synchronize()
        decode[m] = sum(ev.device_time_total for ev in prof.key_averages()
                        if ev.device_type is not None and "CUDA" in str(ev.device_type) and "jpeg_" in ev.key) / 1e3
    name, pl = card()
    sizes = np.asarray([len(d) for d in plain]) / 1e3
    res = {"card": name, "power_limit": pl, "host_cpus": os.cpu_count(), "frames": a.frames, "rounds": a.rounds,
           "file_kb_median": float(np.median(sizes)), "modes": {}}
    print(f"{name}, power limit {pl}, {os.cpu_count()} host CPUs; {a.frames} frames (median {np.median(sizes):.0f} kB), "
          f"IMHN bf16, boxsize 640, scale_search [1], rotation_search [0]; each result read before the next submit")
    for m in modes:
        fs = streams[m]
        ts = sorted(times[m])
        med = ts[len(ts) // 2]
        lat = np.sort(np.asarray(lats[m])) * 1e3
        res["modes"][m] = dict(frames_per_s=a.frames / med, spread=[a.frames / ts[-1], a.frames / ts[0]],
                               latency_ms_p50=float(np.percentile(lat, 50)), latency_ms_p90=float(np.percentile(lat, 90)),
                               decode_kernel_ms_per_frame=decode[m] / a.frames, captures=fs.captures,
                               host_decodes=fs.host_decodes, people_equal_cv2=same[m])
        print(f"  {m:>8}: {a.frames / med:6.1f} frames/s (min {a.frames / ts[-1]:.1f}, max {a.frames / ts[0]:.1f}); latency "
              f"p50 {np.percentile(lat, 50):.2f} ms, p90 {np.percentile(lat, 90):.2f} ms; decode kernels "
              f"{decode[m] / a.frames:.3f} ms/frame; {fs.captures} graphs, {fs.host_decodes} cv2 decodes; people == cv2: "
              f"{same[m]}")
        fs.close()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
