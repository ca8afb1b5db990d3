"""Regenerate tests/golden/loss/: the reference's own ``MultiTaskLoss`` (models/loss_model.py) and
``MultiTaskLossParallel`` (models/loss_model_parallel.py), loaded unmodified (they import only torch) and run on CPU.
Usage: python tests/golden/make_loss_golden.py REFERENCE_ROOT

Each case's inputs are regenerated from its seed by ``make_inputs`` (numpy PCG64), so a file holds only what the
reference made of them: the loss, the per-stack sums it prints (captured from its ``print``) and the gradient of every
prediction after ``loss.backward(grad_output)``.  The inputs cover the 0.01 label threshold (0.01f and both neighbours),
``k / 255`` masks with 2 x 2 checkerboards whose resized values are exactly 0.5, ``s = 1`` on labels >= 0.01 and tiny
``s`` below, ``opt.batch_size`` != B, ``grad_output`` 3 and 65536, nstack 2 and 4 with non-unit stack weights, a NaN
prediction, and both losses (the L2 one with predictions carrying two channels past ``offset_start``).
"""
from __future__ import annotations

import importlib.util
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "loss")

SCALE_WEIGHT = [0.1, 0.2, 0.4, 1.6, 6.4]
CASES = [  # name, mode, seed, B, C, H, W, nstack, nstack_weight, opt.batch_size, grad_output, NaN prediction
    dict(name="focal_c50_ns2", mode="focal", seed=11, B=3, C=50, H=16, W=16, nstack=2, nstack_weight=[1, 2.5],
         batch_size=5, grad_output=3.0, nan=False),
    dict(name="focal_c12_ns4", mode="focal", seed=12, B=3, C=12, H=16, W=32, nstack=4, nstack_weight=[0.5, 1, 1, 3],
         batch_size=3, grad_output=65536.0, nan=False),
    dict(name="focal_c12_nan", mode="focal", seed=13, B=3, C=12, H=16, W=16, nstack=2, nstack_weight=[1, 1],
         batch_size=4, grad_output=1.0, nan=True),
    dict(name="l2_c12_ns2", mode="l2", seed=14, B=3, C=12, H=16, W=16, nstack=2, nstack_weight=[2, 1],
         batch_size=4, grad_output=3.0, nan=False),
    dict(name="l2_c12_ns4", mode="l2", seed=15, B=3, C=12, H=32, W=16, nstack=4, nstack_weight=[1, 1, 0.25, 2],
         batch_size=3, grad_output=65536.0, nan=False),
]


def channel_layout(C: int):
    """(heat_start, bkg_start) of a C-channel layout: the reference's 30 / 48 of 50, else proportionally."""
    return (30, 48) if C == 50 else (C // 3, C - 2)


def make_inputs(case):
    """``(preds [nstack][5] float32 arrays, mask_miss [B,1,H,W], labels [B,C,H,W])`` of a case, from its seed."""
    rng = np.random.Generator(np.random.PCG64(case["seed"]))
    B, C, H, W, ns = case["B"], case["C"], case["H"], case["W"], case["nstack"]
    labels = rng.random((B, C, H, W), dtype=np.float32)
    labels[rng.random(labels.shape) < 0.5] = 0
    f = np.float32(0.01)
    specials = np.array([np.nextafter(f, np.float32(0)), f, np.nextafter(f, np.float32(1))], np.float32)
    idx = rng.choice(labels.size, labels.size // 8, replace=False)
    labels.flat[idx] = specials[rng.integers(0, 3, idx.size)]
    mask = rng.integers(0, 256, (B, 1, H, W)).astype(np.float32) / np.float32(255)
    mask[0, 0, :8, :8] = (np.add.outer(np.arange(8), np.arange(8)) % 2).astype(np.float32)  # resized: exactly 0.5
    mask[1, 0, 4:12, :] = np.float32(128) / np.float32(255)
    cp = C + 2 if case["mode"] == "l2" else C
    preds = []
    for k in range(ns):
        stack = []
        for j in range(5):
            p = rng.uniform(-0.25, 1.25, (B, cp, H >> j, W >> j)).astype(np.float32)
            stack.append(p)
        preds.append(stack)
    s0 = preds[0][0][:, :C]
    pos = (labels >= f) & (rng.random(labels.shape) < 0.3)
    s0[pos] = 1.0
    neg = (labels < f) & (rng.random(labels.shape) < 0.3)
    tiny = np.array([2.0 ** -26, -2.0 ** -27, 3e-8, 2.0 ** -24], np.float32)
    s0[neg] = tiny[rng.integers(0, 4, int(neg.sum()))]
    if case["nan"]:
        preds[ns - 1][1][1, 3, 2, 5] = np.nan
    return preds, mask, labels


class _Opt:
    def __init__(self, case):
        self.nstack = case["nstack"]
        self.batch_size = case["batch_size"]
        self.multi_task_weight = 0.1
        self.keypoint_task_weight = 3
        self.scale_weight = list(SCALE_WEIGHT)
        self.nstack_weight = list(case["nstack_weight"])


class _Config:
    def __init__(self, case):
        self.heat_start, self.bkg_start = channel_layout(case["C"])
        self.offset_start = case["C"]


def _load(root: str, rel: str, name: str):
    spec = importlib.util.spec_from_file_location(name, os.path.join(root, rel))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main(root: str) -> None:
    import torch

    focal_mod = _load(root, "models/loss_model.py", "ref_loss_model")
    l2_mod = _load(root, "models/loss_model_parallel.py", "ref_loss_model_parallel")
    os.makedirs(OUT, exist_ok=True)
    manifest = {"source": ["models/loss_model.py:MultiTaskLoss", "models/loss_model_parallel.py:MultiTaskLossParallel"],
                "torch": torch.__version__, "device": "cpu", "scale_weight": SCALE_WEIGHT,
                "multi_task_weight": 0.1, "keypoint_task_weight": 3, "cases": []}
    for case in CASES:
        mod = focal_mod if case["mode"] == "focal" else l2_mod
        printed = []
        mod.print = lambda *a, **k: printed.append(np.array(a[-1], np.float32))  # the per-stack sums it prints
        cls = mod.MultiTaskLoss if case["mode"] == "focal" else mod.MultiTaskLossParallel
        crit = cls(_Opt(case), _Config(case))
        preds, mask, labels = make_inputs(case)
        tp = [[torch.from_numpy(p).requires_grad_() for p in stack] for stack in preds]
        loss = crit(tp, [torch.from_numpy(mask), torch.from_numpy(labels)])
        loss.backward(torch.tensor(case["grad_output"], dtype=torch.float32))
        out = {"loss": loss.detach().numpy().astype(np.float32), "stack_sums": np.stack(printed)}
        for k, stack in enumerate(tp):
            for j, p in enumerate(stack):
                out[f"grad_{k}_{j}"] = p.grad.numpy()
        np.savez_compressed(os.path.join(OUT, case["name"] + ".npz"), **out)
        manifest["cases"].append(dict(case, heat_start=_Config(case).heat_start, bkg_start=_Config(case).bkg_start,
                                      loss=float(out["loss"])))
        print(case["name"], float(out["loss"]), out["stack_sums"].shape, file=sys.stderr)
    with open(os.path.join(OUT, "MANIFEST.json"), "w") as f:
        json.dump(manifest, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__.split("\n")[2])
    main(sys.argv[1])
