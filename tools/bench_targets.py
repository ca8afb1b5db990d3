"""Training-sample stage on one GPU: make_batch samples/s, per-kernel times and HBM shares, and the CPU rate.

Prints one JSON line.  256 seeded samples at the default 512 x 512 config (128 x 128 maps): COCO-like source sizes, 1-15
persons, random augmentations (tint off).  Kernel times are CUDA events around many launches of one kernel on the whole
batch; a kernel's algorithmic bytes are what it must write plus the source bytes it must read, over its time, as a share
of the H100 SXM's 3.35 TB/s.  The CPU rate is the single-process numpy port (tests/targets_port.py) on the same samples,
or the reference's own classes when --reference points at them.

Colour distortion: targets_tint_kernel's time over many launches tinting every source of the batch in place (6
algorithmic bytes per source pixel), make_batch(tint=True) samples/s with no sample tinted and with tint drawn at the
reference's tint_prob 0.2 (the two alternated, median of --iters each), and the CPU rate of distort_color on the same
sources (the reference's with --reference, else its cv2 calls restated).  Usage:
    python tools/bench_targets.py [--samples 256] [--iters 20] [--cpu-samples 16] [--reference DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")]

HBM = 3.35e12


def make_samples(n: int, seed: int = 0):
    from improved_body_parts_b200 import targets
    rng = np.random.default_rng(seed)
    random.seed(seed)
    cfg = targets.TargetConfig()
    sizes = [(480, 640), (640, 480), (427, 640), (640, 427), (375, 500), (500, 375), (612, 612)]
    samples, augs = [], []
    for i in range(n):
        h, w = sizes[int(rng.integers(0, len(sizes)))]
        P = int(rng.integers(1, 16))
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        mm = np.where(rng.random((h, w)) < 0.05, 0, 255).astype(np.uint8)
        ma = np.where(rng.random((h, w)) < 0.3, 255, 0).astype(np.uint8)
        j = np.zeros((P, 18, 3))
        c = rng.uniform([0, 0], [w, h], (P, 1, 2))
        j[:, :, 0:2] = c + rng.normal(0, 40, (P, 18, 2))
        j[:, :, 2] = rng.choice([0, 1, 2], (P, 18), p=[0.3, 0.55, 0.15])
        meta = {"objpos": [[float(c[0, 0, 0]), float(c[0, 0, 1])]], "scale_provided": [float(rng.uniform(0.3, 1.0))],
                "joints": j}
        aug = targets.AugmentSelection.random(cfg.transform_params)
        aug.tint = False
        samples.append((img, mm, ma, meta))
        augs.append(aug)
    return cfg, samples, augs


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, power = out.strip().splitlines()[0].split(", ")
        return name, power
    except Exception as e:  # reported, never guessed
        return f"unknown ({e})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--cpu-samples", type=int, default=16)
    ap.add_argument("--reference", default=None)
    a = ap.parse_args()
    import torch
    from improved_body_parts_b200 import grouping, targets
    if not torch.cuda.is_available():
        raise SystemExit("bench_targets needs a CUDA device")
    dev = torch.device("cuda:0")
    name, power = gpu_info()
    cfg, samples, augs = make_samples(a.samples)
    # end to end: host geometry, staging, uploads and both kernels
    for _ in range(2):
        targets.make_batch(samples, augs, cfg)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.iters):
        out = targets.make_batch(samples, augs, cfg)
    torch.cuda.synchronize()
    e2e = a.iters * a.samples / (time.perf_counter() - t0)
    # kernels alone: the records make_batch would pass, on resident sources
    params = targets.target_params(cfg)
    n, H, W, m = a.samples, cfg.width, cfg.height, cfg.width // cfg.stride
    srcs = [[torch.from_numpy(x).to(dev) for x in s[:3]] for s in samples]
    images = torch.empty((n, H, W, 3), device=dev)
    miss = torch.empty((n, m, m), device=dev)
    alls = torch.empty((n, m, m), device=dev)
    labels = torch.empty((n, 50, m, m), device=dev)
    ws, wj, joints = np.zeros(n, grouping.TARGET_SAMPLE), np.zeros(n, grouping.TARGET_JOINTS), []
    src_bytes = 0
    for i, ((img, mm, ma, meta), aug) in enumerate(zip(samples, augs)):
        M, _ = aug.affine(meta["objpos"][0], meta["scale_provided"][0], cfg)
        jt = torch.from_numpy(targets.transform_joints(meta["joints"], M, aug.flip, cfg).astype(np.float32)).to(dev)
        joints.append(jt)
        h, w = img.shape[:2]
        src_bytes += h * w * 5  # image and both masks, counted whole: the warp may read less of a large source
        s = srcs[i]
        ws[i] = (s[0].data_ptr(), s[1].data_ptr(), s[2].data_ptr(), 3 * w, w, h, w, M.reshape(6), images[i].data_ptr(),
                 miss[i].data_ptr(), alls[i].data_ptr())
        wj[i] = (jt.data_ptr(), jt.shape[0], 0, alls[i].data_ptr(), labels[i].data_ptr())
    g = targets._Device.grouper(cfg, 0)

    def timed(fn):
        for _ in range(3):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / a.iters * 1e-3

    t_warp = timed(lambda: g.targets_warp(params, ws))
    t_maps = timed(lambda: g.targets_maps(params, wj))
    warp_bytes = n * (H * W * 3 * 4 + 2 * m * m * 4) + src_bytes
    maps_bytes = n * (50 * m * m * 4 + m * m * 4) + sum(j.numel() * 4 for j in joints)
    # colour distortion: every source of the batch tinted in place, repeatedly (6 bytes per pixel: read and write BGR)
    drng = np.random.default_rng(1)
    tint_recs = targets.tint_records([(s[0].data_ptr(), 3 * s[0].shape[1], s[0].shape[0], s[0].shape[1]) for s in srcs],
                                     [tuple(int(v) for v in drng.integers(0, (21, 81, 61))) for _ in srcs],
                                     cfg.tint_row_block)
    t_tint = timed(lambda: g.targets_tint(tint_recs))
    tint_px = sum(s[0].shape[0] * s[0].shape[1] for s in srcs)
    # make_batch at the reference's tint_prob 0.2 and at 0, alternated so that both see the same host and device state
    trng = np.random.default_rng(2)
    augs_tint = []
    for aug in augs:
        t = targets.AugmentSelection(aug.flip, bool(trng.random() < cfg.transform_params.tint_prob), aug.degree, aug.crop,
                                     aug.scale)
        augs_tint.append(t)
    rates = {0.0: [], 0.2: []}
    for _ in range(a.iters):
        for prob, aa in ((0.0, augs), (0.2, augs_tint)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = targets.make_batch(samples, aa, cfg, tint=True)
            torch.cuda.synchronize()
            rates[prob].append(n / (time.perf_counter() - t0))
    # CPU: the numpy port (or the reference's classes) on the first samples, one process
    k = min(a.cpu_samples, n)
    t0 = time.perf_counter()
    if a.reference:
        import make_targets_golden as mg
        cfg_mod, tr, hm = mg.load_reference(a.reference)
        rc = cfg_mod.CanonicalConfig()
        T, Hm = tr.Transformer(rc), hm.Heatmapper(rc)
        for (img, mm, ma, meta), aug in zip(samples[:k], augs[:k]):
            ti, tm, ta, m2 = T.transform(img, mm, ma, {**meta, "joints": meta["joints"].copy()}, aug)
            Hm.create_heatmaps(m2["joints"].astype(np.float32), ta)
        cpu_what = "reference classes"
    else:
        import targets_port as tp
        from improved_body_parts_b200 import skeleton
        for (img, mm, ma, meta), aug in zip(samples[:k], augs[:k]):
            M, _ = aug.affine(meta["objpos"][0], meta["scale_provided"][0], cfg)
            jt = targets.transform_joints(meta["joints"], M, aug.flip, cfg).astype(np.float32)
            _, _, pma = tp.warp_sample(img, mm, ma, M, (H, W), cfg.stride)
            tp.label_maps(jt, pma, skeleton.LIMBS, 4, 9, 7, 0.015, 4, 14)
        cpu_what = "numpy port"
    cpu_rate = k / (time.perf_counter() - t0)
    # CPU colour distortion: the reference's Transformer.distort_color (or its cv2 calls restated, without --reference)
    # on the same sources, one process
    try:
        import cv2  # noqa: F401
        if a.reference:
            distort, dc_what = tr.Transformer.distort_color, "reference distort_color"
        else:
            def distort(img):
                hsv = cv2.cvtColor(img, cv2.COLOR_BGR2HSV).astype(np.int16)
                for ch, (hi, off, top) in enumerate(((20, 10, 179), (80, 20, 255), (60, 20, 255))):
                    hsv[:, :, ch] = np.maximum(np.minimum(hsv[:, :, ch] - off + np.random.randint(hi + 1), top), 0)
                return cv2.cvtColor(hsv.astype(np.uint8), cv2.COLOR_HSV2BGR)
            dc_what = "distort_color's cv2 calls"
        t0 = time.perf_counter()
        for s in samples[:k]:
            distort(s[0])
        dc_rate = round(k / (time.perf_counter() - t0), 1)
    except ImportError as e:
        dc_rate, dc_what = None, f"not measured ({e})"
    del out
    print(json.dumps({
        "gpu": name, "power_limit": power, "samples": n, "config": f"{W}x{H}, stride {cfg.stride}",
        "make_batch_samples_per_s": round(e2e, 1),
        "targets_warp_kernel_ms": round(t_warp * 1e3, 3), "targets_maps_kernel_ms": round(t_maps * 1e3, 3),
        "kernel_samples_per_s": round(n / (t_warp + t_maps), 1),
        "warp_hbm_share": round(warp_bytes / t_warp / HBM, 3), "maps_hbm_share": round(maps_bytes / t_maps / HBM, 3),
        "cpu_samples_per_s": round(cpu_rate, 2), "cpu": cpu_what, "cpu_samples": k,
        "targets_tint_kernel_ms": round(t_tint * 1e3, 3), "tint_hbm_share": round(6 * tint_px / t_tint / HBM, 3),
        "make_batch_samples_per_s_tint_prob_0": round(float(np.median(rates[0.0])), 1),
        "make_batch_samples_per_s_tint_prob_0.2": round(float(np.median(rates[0.2])), 1),
        "tinted_samples_at_0.2": sum(t.tint for t in augs_tint),
        "cpu_distort_color_per_s": dc_rate, "cpu_distort_color": dc_what}))


if __name__ == "__main__":
    main()
