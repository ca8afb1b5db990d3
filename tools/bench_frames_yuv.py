#!/usr/bin/env python
"""A single stream of YUV frames through ``dropin.FrameStream``: converted on the host with ``cv2.cvtColor`` and
submitted as BGR images, against the planes submitted as ``dropin.YUVFrame`` and converted inside each frame's CUDA graph
(``spg_yuv_to_bgr``), alternated round by round in the same run.

Workload: --frames seeded ``synth.photo`` frames, shapes drawn from a fixed table of COCO val2017 sizes (odd sizes made
even by dropping a row or column, as 4:2:0 needs), turned into YUV planes by ``cv2.cvtColor(COLOR_BGR2YUV)`` with the
chroma taken at even rows and columns; at the reference's settings (boxsize 640, max_downsample 64, scale_search [1],
rotation_search [0], stride 4); the network is imhn.IMHN at the reference's random initialisation, bf16 autocast,
channels-last (``imhn.Runner`` without a graph of its own: the frame graph records its forward).  Each frame's result
is read before the next submit (slots=2).  Modes, each with a stream of its own:
  * cv2:           ``cv2.cvtColor`` of host NV12 planes, then ``submit(image)``;
  * nv12, i420, yuyv: ``submit(YUVFrame)`` of host planes (uploaded packed inside the graph);
  * cuda_nv12:     ``submit(YUVFrame)`` of NV12 planes already on the device (a hardware decoder's output);
  * cuda_nv12_cv2: the same device planes downloaded, ``cv2.cvtColor``, then ``submit(image)``.
Every mode runs once over every frame first (warm-up: every shape captured).  Reports per mode frames/s over the
sequence (host clock around work that ends in a device synchronise; median and min-max over the rounds), the median and
90th percentile per-frame latency from the conversion or submit to the result, in a separate pass under torch.profiler
the conversion kernel's time per frame, and the host-to-device bytes per frame the mode uploads (from the shapes).  Each
mode's people are compared with those of cv2's image of the same planes.  The card's name and power limit are read in
the same run.

usage: python tools/bench_frames_yuv.py [--frames 48] [--rounds 5] [--out profiles/frames_yuv.json]"""
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

CODES = {"nv12": "COLOR_YUV2BGR_NV12", "i420": "COLOR_YUV2BGR_I420", "yuyv": "COLOR_YUV2BGR_YUYV"}


def planes_of(cv2, img, fmt):
    """``fmt``'s planes of a BGR image: cv2's YUV, chroma at even rows and columns."""
    yuv = cv2.cvtColor(img, cv2.COLOR_BGR2YUV)
    Y, U, V = yuv[..., 0].copy(), yuv[..., 1], yuv[..., 2]
    H, W = Y.shape
    if fmt == "yuyv":
        p = np.empty((H, 2 * W), np.uint8)
        p[:, 0::4], p[:, 1::4], p[:, 2::4], p[:, 3::4] = Y[:, 0::2], U[:, 0::2], Y[:, 1::2], V[:, 0::2]
        return (p,)
    u, v = U[0::2, 0::2].copy(), V[0::2, 0::2].copy()
    if fmt == "nv12":
        uv = np.empty((H // 2, W), np.uint8)
        uv[:, 0::2], uv[:, 1::2] = u, v
        return Y, uv
    return Y, u, v


def cvt(cv2, fmt, planes):
    """``cv2.cvtColor`` on cv2's single-array layout of the planes."""
    if fmt == "yuyv":
        src = planes[0].reshape(planes[0].shape[0], -1, 2)
    else:
        src = np.concatenate([p.reshape(-1) for p in planes]).reshape(planes[0].shape[0] * 3 // 2, -1)
    return cv2.cvtColor(src, getattr(cv2, CODES[fmt]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=48)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "frames_yuv.json"))
    a = ap.parse_args()
    import cv2
    import torch
    from torch.profiler import ProfilerActivity, profile

    from improved_body_parts_b200 import dropin, imhn, skeleton, synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_frames_yuv needs a CUDA device")
    dropin.configure(device=0, limbs=dropin.LIMBS, input_stage="device")
    rng = np.random.default_rng(2033)
    images = []
    for _ in range(a.frames):
        H, W = SHAPES[int(rng.integers(len(SHAPES)))]
        images.append(synth.photo(int(rng.integers(1 << 30)), H - H % 2, W - W % 2))
    planes = {fmt: [planes_of(cv2, img, fmt) for img in images] for fmt in CODES}
    dev_nv12 = [tuple(torch.from_numpy(p).to("cuda:0") for p in pl) for pl in planes["nv12"]]
    params = dict(skeleton.default_params(), scale_search=[1.0], rotation_search=[0.0])
    runner = imhn.Runner(imhn.IMHN().init_like_reference_(0), device="cuda:0", use_graph=False)

    def model(x):
        return [[runner(x)]]

    modes = ("cv2", "nv12", "i420", "yuyv", "cuda_nv12", "cuda_nv12_cv2")
    streams = {m: dropin.FrameStream(model, params, MODEL_PARAMS_REF, slots=2) for m in modes + ("cv2_yuyv",)}

    def frame(mode, i):
        if mode == "cv2":
            return cvt(cv2, "nv12", planes["nv12"][i])
        if mode == "cv2_yuyv":
            return cvt(cv2, "yuyv", planes["yuyv"][i])
        if mode == "cuda_nv12":
            return dropin.YUVFrame("nv12", dev_nv12[i])
        if mode == "cuda_nv12_cv2":
            return cvt(cv2, "nv12", tuple(p.cpu().numpy() for p in dev_nv12[i]))
        return dropin.YUVFrame(mode, planes[mode][i])

    def run(mode, lat):
        fs, out = streams[mode], []
        for i in range(a.frames):
            t = time.perf_counter()
            out.append(fs.result(fs.submit(frame(mode, i))))
            lat.append(time.perf_counter() - t)
        return out

    people = {m: run(m, []) for m in modes + ("cv2_yuyv",)}  # warm-up: every shape captured
    same = {m: repr(people[m]) == repr(people["cv2_yuyv" if m == "yuyv" else "cv2"]) for m in modes}
    streams.pop("cv2_yuyv").close()
    times = {m: [] for m in modes}
    lats = {m: [] for m in modes}
    for _ in range(a.rounds):
        for m in modes:
            torch.cuda.synchronize()
            t = time.perf_counter()
            run(m, lats[m])
            torch.cuda.synchronize()
            times[m].append(time.perf_counter() - t)
    convert = {}
    for m in modes:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run(m, [])
            torch.cuda.synchronize()
        convert[m] = sum(ev.device_time_total for ev in prof.key_averages()
                         if ev.device_type is not None and "CUDA" in str(ev.device_type) and "yuv_to_bgr" in ev.key) / 1e3
    px = float(np.mean([img.shape[0] * img.shape[1] for img in images]))
    upload = {"cv2": 3 * px, "nv12": 1.5 * px, "i420": 1.5 * px, "yuyv": 2 * px, "cuda_nv12": 0.0, "cuda_nv12_cv2": 3 * px}
    name, pl = card()
    res = {"card": name, "power_limit": pl, "host_cpus": os.cpu_count(), "frames": a.frames, "rounds": a.rounds,
           "mean_pixels": px, "modes": {}}
    print(f"{name}, power limit {pl}, {os.cpu_count()} host CPUs; {a.frames} frames (mean {px / 1e3:.0f} kpixels), "
          f"IMHN bf16, boxsize 640, scale_search [1], rotation_search [0]; each result read before the next submit")
    for m in modes:
        fs = streams[m]
        ts = sorted(times[m])
        med = ts[len(ts) // 2]
        lat = np.sort(np.asarray(lats[m])) * 1e3
        res["modes"][m] = dict(frames_per_s=a.frames / med, spread=[a.frames / ts[-1], a.frames / ts[0]],
                               latency_ms_p50=float(np.percentile(lat, 50)), latency_ms_p90=float(np.percentile(lat, 90)),
                               convert_kernel_ms_per_frame=convert[m] / a.frames, upload_bytes_per_frame=upload[m],
                               captures=fs.captures, people_equal_cv2=same[m])
        print(f"  {m:>13}: {a.frames / med:6.1f} frames/s (min {a.frames / ts[-1]:.1f}, max {a.frames / ts[0]:.1f}); "
              f"latency p50 {np.percentile(lat, 50):.2f} ms, p90 {np.percentile(lat, 90):.2f} ms; yuv_to_bgr "
              f"{convert[m] / a.frames * 1e3:.1f} us/frame; upload {upload[m] / 1e6:.2f} MB/frame; {fs.captures} graphs; "
              f"people == cv2: {same[m]}")
        fs.close()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
