"""Measure the fused training loss (csrc/loss.cuh) against the reference's torch-op loss (oracle/loss_port.py on CUDA).

    python tools/bench_loss.py [--reps 50]

Per configuration (B in {4, 16}, 128 x 128 maps, nstack 4, float32 and bfloat16 predictions) one JSON line: the fused
forward and backward kernel times and the port's forward + backward time (CUDA events; the fused kernels around a CUDA
graph of `reps` calls, so host overhead is not counted, the port's eager torch ops around `reps` steps), the algorithmic bytes (predictions read twice, gradients written once, labels
and mask read twice) over the fused kernel time as a fraction of 3.35 TB/s, each path's peak-memory delta over one eager
step, whether the outputs agree (gradients bit for bit; loss within 1e-5), and the card's name and power limit read in
the same call.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from improved_body_parts_b200 import grouping, loss as L, targets  # noqa: E402
from oracle import loss_port  # noqa: E402

HBM = 3.35e12
SW = [0.1, 0.2, 0.4, 1.6, 6.4]


def power_limit() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def graph_time(fn, reps: int) -> float:
    """Milliseconds per call of `fn`, from a CUDA graph of `reps` calls (after eager warm-up)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        for _ in range(reps):
            fn()
    g.replay()
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        b.synchronize()
        best = min(best, a.elapsed_time(b) / reps)
    return best


def eager_time(fn, reps: int) -> float:
    """Milliseconds per call of `fn` run eagerly `reps` times between two CUDA events (best of 3)."""
    fn()
    best = float("inf")
    for _ in range(3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        b.synchronize()
        best = min(best, a.elapsed_time(b) / reps)
    return best


def peak_delta(fn) -> int:
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def run(B: int, dtype: torch.dtype, reps: int) -> dict:
    dev = torch.device("cuda", torch.cuda.current_device())
    H = W = 128
    C, ns = 50, 4
    gen = torch.Generator(device=dev).manual_seed(B)
    mask = (torch.randint(0, 256, (B, 1, H, W), generator=gen, device=dev).float() / 255).contiguous()
    labels = torch.rand(B, C, H, W, generator=gen, device=dev) * (torch.rand(B, C, H, W, generator=gen, device=dev) < 0.3)
    preds = [[(torch.rand(B, C, H >> j, W >> j, generator=gen, device=dev) * 1.5 - 0.25).to(dtype).requires_grad_()
              for j in range(5)] for _ in range(ns)]
    flat = [p for s in preds for p in s]
    opt = argparse.Namespace(nstack=ns, batch_size=B, multi_task_weight=0.1, keypoint_task_weight=3, scale_weight=SW,
                             nstack_weight=[1] * ns)
    cfg = argparse.Namespace(heat_start=30, bkg_start=48, offset_start=50)
    crit = L.MultiTaskLoss(opt, cfg)

    def port():
        f = [[p.float() for p in s] for s in preds]
        return loss_port.port_loss(f, mask, labels, nstack=ns, scale_weight=SW, nstack_weight=[1] * ns, batch_size=B,
                                   heat_start=30, bkg_start=48, multi_task_weight=0.1, keypoint_task_weight=3).loss

    # outputs compared in the same run
    fused_loss = crit(preds, (mask, labels))
    ga = torch.autograd.grad(fused_loss, flat)
    port_loss = port()
    gb = torch.autograd.grad(port_loss, flat)
    same = all(bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all()) for a, b in zip(ga, gb))
    loss_ok = abs(float(fused_loss.detach()) - float(port_loss.detach())) <= 1e-5 * abs(float(port_loss.detach()))
    del fused_loss, port_loss, ga, gb  # no autograd graph of these outlives the comparison

    # the two kernels alone, through the library with prebuilt records
    g = targets._Device.for_device(dev.index)
    params = crit._params((B, C, H, W))
    grads = [torch.empty_like(p) for p in flat]
    recs = L._records(flat, grads)
    sums = torch.empty(5, ns, device=dev)
    out = torch.empty((), device=dev)
    one = torch.ones((), device=dev)
    dt = L._DTYPES[dtype]
    t_fwd = graph_time(lambda: g.loss_forward(params, mask.data_ptr(), labels.data_ptr(), recs, dt, sums.data_ptr(),
                                              out.data_ptr()), reps)
    t_bwd = graph_time(lambda: g.loss_backward(params, mask.data_ptr(), labels.data_ptr(), recs, dt, one.data_ptr()), reps)
    t_port = eager_time(lambda: torch.autograd.grad(port(), flat), reps)

    mem_fused = peak_delta(lambda: torch.autograd.grad(crit(preds, (mask, labels)), flat))
    mem_port = peak_delta(lambda: torch.autograd.grad(port(), flat))
    esz = torch.finfo(dtype).bits // 8
    pred_elems = sum(p.numel() for p in flat)
    target_bytes = (labels.numel() + mask.numel()) * 4
    bytes_ = 3 * pred_elems * esz + 2 * target_bytes
    t_kern = (t_fwd + t_bwd) * 1e-3
    return {"B": B, "maps": [H, W], "nstack": ns, "dtype": str(dtype).replace("torch.", ""),
            "fused_forward_ms": round(t_fwd, 4), "fused_backward_ms": round(t_bwd, 4),
            "port_forward_backward_ms": round(t_port, 4), "speedup": round(t_port / (t_fwd + t_bwd), 2),
            "algorithmic_bytes": bytes_, "hbm_fraction": round(bytes_ / t_kern / HBM, 3),
            "peak_mem_delta_fused_mb": round(mem_fused / 2 ** 20, 1), "peak_mem_delta_port_mb": round(mem_port / 2 ** 20, 1),
            "gradients_bit_identical": same, "loss_within_1e-5": loss_ok,
            "gpu": torch.cuda.get_device_name(dev), "power_limit": power_limit()}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    for dtype in (torch.float32, torch.bfloat16):
        for B in (4, 16):
            print(json.dumps(run(B, dtype, a.reps)), flush=True)


if __name__ == "__main__":
    main()
