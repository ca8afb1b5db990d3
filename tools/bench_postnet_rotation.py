"""Cost of the rotation search in the post-network stage (spg_postnet_rotated), at the reference's default geometry.

A 480 x 640 image at boxsize 640 is scaled to 640 x 853 and padded to 640 x 896, so the network output is
[N, 2, 50, 160, 224] and the maps 480 x 640.  Runs rotation_search [0] (one postnet_kernel launch) against
[0, 30, -30] (postnet_kernel, then postnet_rot_kernel twice, float64 sums through memory), with float32 and float16
network outputs, N = 8.  Reports:
  - CUDA-event time per call and, from torch.profiler in a separate pass, per kernel, over --iters launches after warm-up;
  - the algorithmic bytes of each kernel (computed from the shapes) and their fraction of 3.35 TB/s (H100 SXM HBM3);
  - the card's name and power limit, read in the same run;
  - a bit-exact check of image 0 against oracle/postnet_rotation_port.py.
Prints one JSON line per run.

    python tools/bench_postnet_rotation.py [--iters 100] [--warmup 10]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_BPS = 3.35e12
N, h, w = 8, 160, 224
CROP, IMAGE = (640, 853), (480, 640)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def kernel_bytes(n_items, t, net_elem, paf_f32):
    """Bytes one launch must move: the 48 used channels of both outputs of the pair, the float64 sums of the earlier items
    (read), and this item's sums (float64) or, for the last item, the float32 keypoint maps and the body-part maps."""
    H, W = IMAGE
    b = N * 2 * 48 * h * w * net_elem
    if t > 0:
        b += N * 48 * H * W * 8
    last = t == n_items - 1
    b += N * 18 * H * W * (4 if last else 8)
    b += N * 30 * H * W * (4 if paf_f32 else 8)
    return b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    import torch

    from improved_body_parts_b200 import skeleton, synth
    from improved_body_parts_b200.grouping import Grouper
    from oracle import postnet_port as pp
    from oracle import postnet_rotation_port as pr
    from test_gpu_postnet import _network_like_output

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda:0")
    gpu = card()

    class E:
        pass
    e = E(); e.synth, e.skeleton = synth, skeleton
    base = _network_like_output(e, 2024, N, h, w, 6)
    g = Grouper(max_batch=N, max_h=IMAGE[0], max_w=IMAGE[1])
    try:
        for dtype in ("f32", "f16"):
            net = torch.from_numpy(base.astype(np.float16) if dtype == "f16" else base).to(dev)
            for angles in ([0], [0, 30, -30]):
                outs, crops = [net] * len(angles), [CROP] * len(angles)
                mats = [None if a == 0 else pr.rotation_matrices((4 * h, 4 * w), a)[1] for a in angles]
                paf_dtype = torch.float32 if len(angles) == 1 else torch.float64
                heat = torch.empty((N, 18) + IMAGE, dtype=torch.float32, device=dev)
                paf = torch.empty((N, 30) + IMAGE, dtype=paf_dtype, device=dev)

                def call():
                    g.postnet(outs, crops, IMAGE, heat_out=heat, paf_out=paf, rotations=mats)
                for _ in range(args.warmup):
                    call()
                torch.cuda.synchronize()
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                for _ in range(args.iters):
                    call()
                t1.record()
                torch.cuda.synchronize()
                call_ms = t0.elapsed_time(t1) / args.iters
                # per kernel: a separate, profiled pass
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(args.iters):
                        call()
                    torch.cuda.synchronize()
                per = {}
                for ev in prof.events():
                    if ev.device_type.name == "CUDA" and "postnet" in ev.name:
                        per.setdefault(ev.name, []).append(ev.device_time if hasattr(ev, "device_time") else ev.cuda_time)
                kernels = []
                for name, ts in sorted(per.items(), key=lambda kv: "rot" in kv[0]):
                    ms = float(np.mean(ts)) / 1e3
                    n_launch = len(ts) // args.iters
                    kernels.append(dict(kernel=name.split("(")[0], launches_per_call=n_launch, ms=round(ms, 4)))
                # algorithmic bytes and share of HBM bandwidth per launch in item order
                launches = []
                for t in range(len(mats)):
                    b = kernel_bytes(len(mats), t, 2 if dtype == "f16" else 4, paf_dtype == torch.float32)
                    launches.append(dict(item=t, angle=angles[t], bytes=b))
                for k in kernels:
                    rot = "rot" in k["kernel"]
                    bs = [x["bytes"] for x, M in zip(launches, mats) if (M is not None) == rot]
                    k["bytes_per_launch"] = int(np.mean(bs))
                    k["hbm_fraction"] = round(k["bytes_per_launch"] / (k["ms"] * 1e-3) / HBM_BPS, 3)
                # bit-exact check of image 0 against the port
                hm_ref, pf_ref = np.zeros(IMAGE + (18,)), np.zeros(IMAGE + (30,))
                pad = [0, 0, 4 * h - CROP[0], 4 * w - CROP[1]]
                src = base[0].astype(np.float16).astype(np.float32) if dtype == "f16" else base[0]
                for M in mats:
                    hm, pf = pr.post_network_item(src, 4, (4 * h, 4 * w), pad, IMAGE, 30, 48, skeleton.FLIP_PAF_ORD,
                                                  skeleton.FLIP_HEAT_ORD[:18], rotate_matrix=M)
                    hm_ref, pf_ref = pp.accumulate(hm_ref, hm, len(mats)), pp.accumulate(pf_ref, pf, len(mats))
                exact = bool(np.array_equal(heat[0].cpu().numpy(), hm_ref.transpose(2, 0, 1).astype(np.float32)) and
                             np.array_equal(paf[0].cpu().numpy().astype(np.float64), pf_ref.transpose(2, 0, 1)))
                print(json.dumps(dict(card=gpu, net=f"[{N},2,50,{h},{w}] {dtype}", image=IMAGE, crop=CROP,
                                      rotation_search=angles, iters=args.iters, call_ms=round(call_ms, 4), kernels=kernels,
                                      bit_exact_image0=exact)), flush=True)
    finally:
        g.close()


if __name__ == "__main__":
    main()
