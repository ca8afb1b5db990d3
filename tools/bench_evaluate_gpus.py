#!/usr/bin/env python
"""evaluate.py's validation end to end on G GPUs of one box: the launcher's sharded ``predict_many`` for G = 1, 2, 4, 8.

Workload: --images-per-gpu seeded random uint8 images per GPU (G x 64 by default: the work per GPU stays the same, so
linear scaling means G times the images/s of one GPU), shapes drawn from the COCO val2017 sizes of
tools/bench_predict_batch.py, written as PNG to a temporary directory.  The reference's utils/config (boxsize 640,
max_downsample 64, stride 4, scale_search [1], rotation_search [0]), --batch 16 --forward-batch 8, the host input stage
(the launcher's default).  The network is imhn.IMHN at the reference's random initialisation, bf16 autocast, no CUDA graph.

For each G this script starts ``torch.distributed.run --nproc-per-node G`` on itself.  Every rank joins the process
group as the launcher does (``run_evaluate_b200.init_ranks``), installs the batched ``predict_many`` on a stand-in
``evaluate`` module whose ``validation()`` calls it, and calls the launcher's ``validate``: rank 0 runs ``validation()``,
the other ranks serve their blocks.  One warm-up pass runs every image (every shape of every block) once; then
--repeats timed passes.  Reported per G: images/s (host clock on rank 0 around the whole ``validate`` call, which ends
after the gather of every rank's people), the slowest rank's block time as a share of that wall time, each rank's
block time and its time in ``cv2.imread``, and each card's name and power limit, read in the same run.  A G larger than
the number of visible devices is reported as not measured.

``--jpeg`` writes the images as JPEG instead (``synth.photo`` content at the same shapes, quality 95, 4:2:0: COCO
val2017 is JPEG).  ``--device-decode`` (with ``--jpeg``) installs the device input stage and compares the two ways
``predict_many`` reads the files in one run: ``cv2.imread`` per file and ``imread_many`` per group of --batch files,
alternated pass by pass after a warm-up of each; it reports both, with each rank's time in the file reading of each.

usage: python tools/bench_evaluate_gpus.py [--gpus 1,2,4,8] [--images-per-gpu 64] [--batch 16] [--forward-batch 8]
                                           [--repeats 3] [--jpeg [--device-decode]] [--out profiles/evaluate_gpus.json]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

#: the reference's utils/config, read as the launcher reads it
CONFIG = os.path.join(ROOT, "tests", "golden", "reference_utils_config.ini")


def write_images(directory, n, jpeg=False):
    import cv2

    from bench_predict_batch import SHAPES
    from improved_body_parts_b200 import synth
    rng = np.random.default_rng(2033)
    names = {}
    for k in range(n):
        iid = 100000 + k
        names[iid] = f"{iid:012d}.{'jpg' if jpeg else 'png'}"
        shape = SHAPES[int(rng.integers(len(SHAPES)))] + (3,)
        if jpeg:
            cv2.imwrite(os.path.join(directory, names[iid]), synth.photo(k, *shape[:2]),
                        [cv2.IMWRITE_JPEG_QUALITY, 95, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420])
        else:
            cv2.imwrite(os.path.join(directory, names[iid]), rng.integers(0, 256, size=shape, dtype=np.uint8))
    return names


def cards():
    out = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout
    return [line.strip() for line in out.splitlines() if line.strip()]


def worker(a):
    """One rank under torchrun: the warm-up and timed passes; rank 0 writes the result to --result."""
    import torch
    import torch.distributed as dist

    import run_evaluate_b200 as L
    from improved_body_parts_b200 import dropin, imhn, skeleton
    local = L.init_ranks()
    rank, world = dist.get_rank(), dist.get_world_size()
    names = {int(k): v for k, v in json.load(open(os.path.join(a.dir, "names.json"))).items()}
    ids = sorted(names)[:world * a.images_per_gpu]
    coco = types.SimpleNamespace(imgs={i: {"file_name": names[i]} for i in ids}, getImgIds=lambda: ids)
    params, model_params = skeleton.read_reference_ini(CONFIG)
    runner = imhn.Runner(imhn.IMHN().init_like_reference_(0), device=f"cuda:{local}", use_graph=False)
    mod = types.ModuleType("evaluate")
    mod.limbSeq = list(dropin.LIMBS)
    mod.posenet = lambda x: [[runner(x)]]
    mod.get_image_name = lambda c, image_id: c.imgs[image_id]["file_name"]
    mod.validation = lambda model: mod.predict_many(coco, a.dir, ids, params, model, model_params, 18, 30)
    dropin.configure(device=local)
    dropin.install(mod, device_predict=True, batch=a.batch, forward_batch=a.forward_batch,
                   **(dict(device_input=True, device_decode=True) if a.device_decode else {}))
    # the passes alternate the two decodes by switching the module's setting: configure() would also close the handles
    modes = ["host", "device"] if a.device_decode else [dropin._decode]

    import cv2
    clocks = {"block": 0.0, "imread": 0.0}
    block, imread, imread_many = dropin._predict_block, cv2.imread, dropin.imread_many

    def timed_block(*args, **kw):
        t = time.perf_counter()
        try:
            return block(*args, **kw)
        finally:
            torch.cuda.synchronize()
            clocks["block"] += time.perf_counter() - t

    def timed_imread(*args, **kw):
        t = time.perf_counter()
        try:
            return imread(*args, **kw)
        finally:
            clocks["imread"] += time.perf_counter() - t

    def timed_imread_many(*args, **kw):
        t = time.perf_counter()
        try:
            return imread_many(*args, **kw)
        finally:
            clocks["imread"] += time.perf_counter() - t

    dropin._predict_block, cv2.imread, dropin.imread_many = timed_block, timed_imread, timed_imread_many
    for mode in modes:  # warm-up: every image of every block once, with each decode
        dropin._decode = mode
        L.validate(mod)
    passes = {m: [] for m in modes}
    for _ in range(a.repeats):
        for mode in modes:
            dropin._decode = mode
            clocks.update(block=0.0, imread=0.0)
            dist.barrier()
            t = time.perf_counter()
            L.validate(mod)
            wall = time.perf_counter() - t
            per_rank = [None] * world if rank == 0 else None
            dist.gather_object(dict(clocks), per_rank, dst=0)
            if rank == 0:
                passes[mode].append(dict(wall_s=wall, images_per_s=len(ids) / wall, slowest_rank_share=max(
                    r["block"] for r in per_rank) / wall, block_s=[r["block"] for r in per_rank],
                    imread_s=[r["imread"] for r in per_rank]))
    if rank == 0:
        with open(a.result, "w") as f:
            json.dump(dict(images=len(ids), device=torch.cuda.get_device_name(local), passes=passes), f)
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", default="1,2,4,8")
    ap.add_argument("--images-per-gpu", type=int, default=64)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--forward-batch", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--jpeg", action="store_true", help="write the images as JPEG (quality 95, 4:2:0) instead of PNG")
    ap.add_argument("--device-decode", action="store_true",
                    help="alternate cv2.imread and the device decode (needs --jpeg), both with the device input stage")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "evaluate_gpus.json"))
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--dir", help=argparse.SUPPRESS)
    ap.add_argument("--result", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a)
    if a.device_decode and not a.jpeg:
        ap.error("--device-decode needs --jpeg")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_evaluate_gpus needs CUDA devices")
    n_dev = torch.cuda.device_count()
    gs = [int(g) for g in a.gpus.split(",")]
    res = {"cards": cards(), "host_cpus": os.cpu_count(), "images_per_gpu": a.images_per_gpu, "batch": a.batch,
           "forward_batch": a.forward_batch, "repeats": a.repeats, "jpeg": a.jpeg, "device_decode": a.device_decode,
           "runs": {}}
    print(f"cards: {res['cards']}; host CPUs: {res['host_cpus']}")
    with tempfile.TemporaryDirectory() as d:
        names = write_images(d, max([g for g in gs if g <= n_dev], default=0) * a.images_per_gpu, a.jpeg)
        with open(os.path.join(d, "names.json"), "w") as f:
            json.dump(names, f)
        for g in gs:
            if g > n_dev:
                res["runs"][str(g)] = f"not measured: {n_dev} visible CUDA device(s)"
                print(f"G={g}: not measured ({n_dev} visible CUDA device(s))")
                continue
            out = os.path.join(d, f"result_{g}.json")
            cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", f"--nproc-per-node={g}",
                   os.path.abspath(__file__), "--worker", "--dir", d, "--result", out, "--images-per-gpu",
                   str(a.images_per_gpu), "--batch", str(a.batch), "--forward-batch", str(a.forward_batch),
                   "--repeats", str(a.repeats)] + (["--device-decode"] if a.device_decode else [])
            subprocess.run(cmd, check=True, cwd=ROOT)
            r = json.load(open(out))
            r["median"] = {}
            for mode, passes in r["passes"].items():
                ps = sorted(passes, key=lambda p: p["images_per_s"])
                med = r["median"][mode] = ps[len(ps) // 2]
                print(f"G={g} {mode} decode: {r['images']} images, {med['images_per_s']:.1f} images/s (min "
                      f"{ps[0]['images_per_s']:.1f}, max {ps[-1]['images_per_s']:.1f}); slowest rank "
                      f"{100 * med['slowest_rank_share']:.1f} % of the wall time; block s per rank "
                      f"{[round(v, 3) for v in med['block_s']]}; file reading s per rank "
                      f"{[round(v, 3) for v in med['imread_s']]}", flush=True)
            if not a.device_decode:  # one decode: the passes list and the median pass, as without the comparison
                (mode, passes), = r["passes"].items()
                r["passes"], r["median"] = passes, r["median"][mode]
            res["runs"][str(g)] = r
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
