#!/usr/bin/env python
"""Time keypoint evaluation (COCOeval's evaluate() + accumulate()) on the GPU against the numpy port on the CPU.

    python tools/bench_cocoeval.py [--images 500,5000] [--iters 50] [--json out.json]

Inputs are seeded ``person_keypoints_val2017``-shaped sets (synth.coco_keypoint_set): 5000 images as val2017 has, and
the 500 that ``validation()`` takes by default.  Per size it prints, in one JSON line:

- ``pack_ms``: the host packing of one evaluate() (annotations to the packed arrays), best of 3;
- ``kernels_ms``: the device work of spg_coco_evaluate + spg_coco_accumulate on uploaded inputs, CUDA events around
  ``--iters`` calls after a warm-up, per call;
- ``device_ms``: ``COCOeval.evaluate() + accumulate()`` end to end with a synchronise, median of 5 after a warm-up
  (packing, uploads, kernels, downloads);
- ``port_ms``: the numpy port's evaluate() + accumulate() on this host's CPU (one core; the core count is printed),
  and ``pycocotools_ms`` where pycocotools is installed.

The card's name and power limit are read in the same run.  Nothing is written unless --json is given.
"""
from __future__ import annotations

import argparse
import contextlib
import io
import json
import os
import platform
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return {"gpu": name, "power_limit_and_max_sm_clock": q}


def coco(ds):
    from improved_body_parts_b200 import cocoeval
    c = cocoeval.COCO()
    c.dataset = ds
    c.createIndex()
    return c


def bench(n, iters):
    import numpy as np
    import torch
    from improved_body_parts_b200 import cocoeval, synth
    from oracle import cocoeval_port as port

    ds, res = synth.coco_keypoint_set(2024 + n, n)
    gt = coco(ds)
    dt = gt.loadRes(res)
    out = {"images": n, "ground_truths": len(ds["annotations"]), "detections": len(res)}

    def device_once():
        e = cocoeval.COCOeval(gt, dt)
        e.evaluate()
        e.accumulate()
        torch.cuda.synchronize()
        return e

    e = device_once()  # warm-up: module load, the handle, the sort scratch
    times = []
    for _ in range(5):
        t = time.perf_counter()
        e = device_once()
        times.append((time.perf_counter() - t) * 1e3)
    out["device_ms"] = statistics.median(times)

    p = e._paramsEval
    gts = gt.loadAnns(gt.getAnnIds(imgIds=p.imgIds, catIds=p.catIds))
    dts = dt.loadAnns(dt.getAnnIds(imgIds=p.imgIds, catIds=p.catIds))
    pack = []
    for _ in range(3):
        t = time.perf_counter()
        cocoeval._Packed(gts, dts, p.imgIds, p.catIds, 17, 20)
        pack.append((time.perf_counter() - t) * 1e3)
    out["pack_ms"] = min(pack)

    dv = e._dev
    g, recs = dv["grouper"], dv["records"]
    T, R, K, A, M = e.eval["counts"]
    prec = torch.empty((T, R, K, A, M), dtype=torch.float64, device="cuda")
    rec = torch.empty((T, K, A, M), dtype=torch.float64, device="cuda")
    sc = torch.empty_like(prec)

    def kernels():
        g.coco_evaluate(*recs)
        g.coco_accumulate(*recs, prec.data_ptr(), rec.data_ptr(), sc.data_ptr())

    for _ in range(3):
        kernels()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        kernels()
    b.record()
    torch.cuda.synchronize()
    out["kernels_ms"] = a.elapsed_time(b) / iters
    out["kernels_match_end_to_end"] = bool(np.array_equal(prec.cpu().numpy(), e.eval["precision"]))

    with contextlib.redirect_stdout(io.StringIO()):
        t = time.perf_counter()
        r = port.COCOevalPort(gt, dt)
        r.evaluate()
        r.accumulate()
        out["port_ms"] = (time.perf_counter() - t) * 1e3
    out["port_equal"] = all(np.array_equal(r.eval[f].view(np.int64), e.eval[f].view(np.int64))
                            for f in ("precision", "recall", "scores"))
    try:
        from pycocotools.coco import COCO
        from pycocotools.cocoeval import COCOeval
    except ImportError:
        out["pycocotools_ms"] = "not installed"
    else:
        import copy
        pg = COCO()
        pg.dataset = copy.deepcopy(ds)
        pg.createIndex()
        with contextlib.redirect_stdout(io.StringIO()):
            pd = pg.loadRes(copy.deepcopy(res))
            t = time.perf_counter()
            pe = COCOeval(pg, pd, 'keypoints')
            pe.evaluate()
            pe.accumulate()
            out["pycocotools_ms"] = (time.perf_counter() - t) * 1e3
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--images", default="500,5000")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_cocoeval needs a CUDA device")
    import __graft_entry__ as ge
    ge.build()
    host = {"cpu": platform.processor() or platform.machine(), "cpu_count": os.cpu_count(),
            "cpus_usable": len(os.sched_getaffinity(0)), "port_threads": 1}
    rows = [bench(int(n), a.iters) for n in a.images.split(",")]
    result = {"card": card(), "host": host, "rows": rows}
    print(json.dumps(result))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
