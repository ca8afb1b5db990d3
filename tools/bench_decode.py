#!/usr/bin/env python
"""The device JPEG decoder (``dropin.imread_many``) against ``cv2.imread`` on one host thread.

Workload: seeded COCO-like JPEGs -- ``synth.photo`` content at 10 shapes around 480 x 640 (the common val2017 sizes),
quality 95, 4:2:0, no restart markers -- written to a temporary directory and read in batches of 16 and 64 files; then
the same files with a restart interval of one MCU row (the interval path instead of the subsequence decode).

Reported per (variant, batch), with the card's name and power limit read in the same run:
  - cv2.imread: images/s on one host thread (file read and decode);
  - imread_many: images/s end to end (file read, parse, one pinned upload, one ragged decode, the status read that
    synchronises), median of --repeats timed batches after a warm-up, with the host parse alone timed apart;
  - per kernel: device time per batch from torch.profiler, in a separate pass;
  - the Huffman kernels' rate: entropy-coded bytes of the batch over their summed device time;
  - whether the timed batch's outputs equal cv2.imdecode of the same bytes, byte for byte.

usage: python tools/bench_decode.py [--batches 16,64] [--repeats 20] [--out profiles/bench_decode.json] [--lib PATH]
--lib loads another build of the library (the Makefile's jpeg_variants: other subsequence sizes).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [(480, 640), (427, 640), (640, 480), (640, 427), (425, 640), (500, 375), (375, 500), (512, 640), (640, 512),
          (480, 600)]
HUFFMAN = ("jpeg_sync_kernel", "jpeg_fixup_kernel", "jpeg_write_kernel", "jpeg_interval_kernel")


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else "unknown"


def write_files(directory, n, restart):
    import cv2

    from improved_body_parts_b200 import synth
    paths = []
    for k in range(n):
        h, w = SHAPES[k % len(SHAPES)]
        params = [cv2.IMWRITE_JPEG_QUALITY, 95, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420,
                  cv2.IMWRITE_JPEG_RST_INTERVAL, (w + 15) // 16 if restart else 0]
        ok, buf = cv2.imencode(".jpg", synth.photo(9000 + k, h, w), params)
        p = os.path.join(directory, f"{'rst' if restart else 'plain'}_{k:03d}.jpg")
        with open(p, "wb") as f:
            f.write(buf.tobytes())
        paths.append(p)
    return paths


def kernel_times(dropin, paths, calls=5):
    """Device time per batch of every kernel of the decode, from torch.profiler (its own pass)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            dropin.imread_many(paths)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.key.startswith("spg::jpeg_") or e.key.startswith("void spg::jpeg_") or "jpeg_" in e.key:
            name = next((k for k in e.key.replace("(", " ").split() if "jpeg_" in k), e.key).split("::")[-1]
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = e.cuda_time_total
            out[name] = out.get(name, 0.0) + t / calls / 1e3  # ms per batch
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="16,64")
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "bench_decode.json"))
    ap.add_argument("--lib", default=None)
    a = ap.parse_args()
    import cv2
    import torch

    from improved_body_parts_b200 import dropin, grouping
    if a.lib:
        grouping.LIB_PATH = os.path.abspath(a.lib)
    if not torch.cuda.is_available():
        raise SystemExit("bench_decode needs a CUDA device")
    batches = [int(b) for b in a.batches.split(",")]
    res = {"card": card(), "lib": os.path.basename(grouping.LIB_PATH), "host_cpus": os.cpu_count(), "runs": {}}
    print(f"card: {res['card']}; library: {res['lib']}", flush=True)
    dropin.configure(device=0)
    with tempfile.TemporaryDirectory() as d:
        for restart in (False, True):
            files = write_files(d, max(batches), restart)
            for n in batches:
                paths = files[:n]
                datas = [open(p, "rb").read() for p in paths]
                seg_bytes = 0
                for data in datas:
                    seg_bytes += int(grouping.jpeg_parse(data)["scan_length"])
                # cv2.imread on one thread
                cv2.setNumThreads(1)
                for p in paths:
                    cv2.imread(p)
                t = time.perf_counter()
                for p in paths:
                    cv2.imread(p)
                cv2_s = time.perf_counter() - t
                # host parse alone
                t = time.perf_counter()
                for data in datas:
                    grouping.jpeg_parse(data)
                parse_s = time.perf_counter() - t
                # imread_many end to end
                for _ in range(3):
                    imgs, host = dropin.imread_many(paths)
                times = []
                for _ in range(a.repeats):
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    imgs, host = dropin.imread_many(paths)
                    torch.cuda.synchronize()
                    times.append(time.perf_counter() - t)
                times.sort()
                med = times[len(times) // 2]
                identical = all(np.array_equal(img.cpu().numpy(), cv2.imdecode(np.frombuffer(data, np.uint8),
                                                                                 cv2.IMREAD_COLOR))
                                for img, data in zip(imgs, datas))
                kt = kernel_times(dropin, paths)
                huff_ms = sum(v for k, v in kt.items() if k in HUFFMAN)
                key = f"{'restart' if restart else 'plain'}_{n}"
                r = {"files": n, "file_bytes": sum(len(x) for x in datas), "entropy_bytes": seg_bytes,
                     "cv2_imread_images_per_s": n / cv2_s, "parse_ms": 1e3 * parse_s,
                     "imread_many_ms": {"median": 1e3 * med, "min": 1e3 * times[0], "max": 1e3 * times[-1]},
                     "imread_many_images_per_s": n / med, "host_fallbacks": host, "identical_to_cv2": identical,
                     "kernel_ms": kt, "kernels_ms_total": sum(kt.values()),
                     "huffman_GB_per_s": seg_bytes / (huff_ms * 1e-3) / 1e9 if huff_ms else None}
                res["runs"][key] = r
                print(f"{key}: cv2.imread {r['cv2_imread_images_per_s']:.0f} img/s on one thread; imread_many "
                      f"{r['imread_many_images_per_s']:.0f} img/s (median {1e3 * med:.2f} ms, min {1e3 * times[0]:.2f}, "
                      f"max {1e3 * times[-1]:.2f}); parse {1e3 * parse_s:.2f} ms; kernels {r['kernels_ms_total']:.3f} ms "
                      f"{ {k: round(v, 3) for k, v in kt.items()} }; Huffman {r['huffman_GB_per_s'] or 0:.2f} GB/s of "
                      f"{seg_bytes} entropy bytes; fallbacks {host}; identical to cv2.imdecode: {identical}", flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
