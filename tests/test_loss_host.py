"""CPU: the training loss's host layer -- ValueError for malformed shapes, scale ratios, dtypes and devices before
anything reaches the library, and the numpy records against include/spgroup.h."""
import os
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from improved_body_parts_b200 import grouping
from improved_body_parts_b200.loss import MultiTaskLoss, MultiTaskLossParallel, loss_params

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPT = SimpleNamespace(nstack=2, batch_size=2, multi_task_weight=0.1, keypoint_task_weight=3,
                      scale_weight=[0.1, 0.2, 0.4, 1.6, 6.4], nstack_weight=[1, 1])
CFG = SimpleNamespace(heat_start=30, bkg_start=48, offset_start=50)


def preds(B=2, C=50, H=32, W=48, nstack=2, dtype=torch.float32):
    return [[torch.zeros(B, C, H >> j, W >> j, dtype=dtype) for j in range(5)] for _ in range(nstack)]


def targets(B=2, C=50, H=32, W=48):
    return torch.zeros(B, 1, H, W), torch.zeros(B, C, H, W)


def test_well_formed_cpu_input_is_refused_for_its_device_only():
    with pytest.raises(ValueError, match="CUDA devices only"):
        MultiTaskLoss(OPT, CFG)(preds(), targets())
    with pytest.raises(ValueError, match="CUDA devices only"):
        MultiTaskLossParallel(OPT, CFG)(preds(C=52), targets())


@pytest.mark.parametrize("make, match", [
    (lambda: (preds(), (torch.zeros(2, 1, 32, 48), torch.zeros(2, 50, 32, 48, dtype=torch.float64))), "labels must be a float32"),
    (lambda: (preds(), (torch.zeros(2, 2, 32, 48), torch.zeros(2, 50, 32, 48))), "mask_miss must be"),
    (lambda: (preds(), (torch.zeros(2, 32, 48), torch.zeros(2, 50, 32, 48))), "mask_miss must be a float32"),
    (lambda: (preds(H=24), targets(H=24)), "multiples of 16"),
    (lambda: (preds(nstack=1), targets()), "pred_tuple has 1 stacks"),
    (lambda: ([p[:4] for p in preds()], targets()), "stack 0 has 4 scales"),
    (lambda: (preds(dtype=torch.float64), targets()), "float32, bfloat16 or float16"),
    (lambda: ([[p.half() if k else p for p in s] for k, s in enumerate(preds())], targets()), "the other predictions"),
    (lambda: ([[p if j != 2 else torch.zeros(2, 50, 9, 12) for j, p in enumerate(s)] for s in preds()], targets()),
     r"scale 2 of the 32x48"),
    (lambda: ([[p if j != 1 else torch.zeros(3, 50, 16, 24) for j, p in enumerate(s)] for s in preds()], targets()),
     r"pred_tuple\[0\]\[1\] must be \[2, 50"),
    (lambda: ([[p if j != 0 else torch.zeros(2, 51, 32, 48) for j, p in enumerate(s)] for s in preds()], targets()),
     r"pred_tuple\[0\]\[0\] must be"),
    (lambda: ([[p.to("meta") if j == 4 else p for j, p in enumerate(s)] for s in preds()], targets()), "is on meta"),
])
def test_malformed_input_raises_value_error(make, match):
    pt, tt = make()
    with pytest.raises(ValueError, match=match):
        MultiTaskLoss(OPT, CFG)(pt, tt)


def test_parallel_loss_needs_offset_start_channels():
    with pytest.raises(ValueError, match=r"must be \[2, >= 50"):
        MultiTaskLossParallel(OPT, CFG)(preds(C=40), targets())
    with pytest.raises(ValueError, match="labels have 52 channels"):
        MultiTaskLossParallel(OPT, CFG)(preds(C=52), targets(C=52))


def test_weights_and_channel_layout_are_checked():
    with pytest.raises(ValueError, match="nstack_weight has 3 entries"):
        loss_params(grouping.LOSS_FOCAL, 2, (2, 50, 32, 48), nstack_weight=[1, 1, 1], scale_weight=OPT.scale_weight)
    with pytest.raises(ValueError, match="scale_weight has 4 entries"):
        loss_params(grouping.LOSS_FOCAL, 2, (2, 50, 32, 48), nstack_weight=[1, 1], scale_weight=[1, 1, 1, 1])
    with pytest.raises(ValueError, match="heat_start 30 / bkg_start 60"):
        MultiTaskLoss(OPT, SimpleNamespace(heat_start=30, bkg_start=60, offset_start=50))._params((2, 50, 32, 48))
    with pytest.raises(ValueError, match="nstack 9 outside"):
        MultiTaskLoss(SimpleNamespace(**dict(vars(OPT), nstack=9, nstack_weight=[1] * 9)), CFG)(preds(nstack=9), targets())


def test_params_record_takes_python_sums():
    p = loss_params(grouping.LOSS_FOCAL, 2, (3, 50, 32, 48), heat_start=30, bkg_start=48, multi_task_weight=0.1,
                    keypoint_task_weight=3, nstack_weight=[1, 2.5], scale_weight=OPT.scale_weight, batch_size=5)
    assert p["scale_weight_sum"][0] == sum(OPT.scale_weight) and p["nstack_weight_sum"][0] == 3.5
    assert (p["batch"][0], p["channels"][0], p["height"][0], p["width"][0]) == (3, 50, 32, 48)
    assert list(p["nstack_weight"][0]) == [1, 2.5, 0, 0, 0, 0, 0, 0] and p["batch_divisor"][0] == 5


def test_loss_records_match_the_header(tmp_path):
    """LOSS_PARAMS and LOSS_PRED against spg_loss_params / spg_loss_pred: sizeof and every field's offset."""
    lines = []
    for name, dt in (("spg_loss_params", grouping.LOSS_PARAMS), ("spg_loss_pred", grouping.LOSS_PRED)):
        fields = list(dt.names)
        args = ", ".join([f"sizeof({name})"] + [f"offsetof({name}, {f})" for f in fields])
        lines.append(f'printf("{name}{" %zu" * (1 + len(fields))}\\n", {args});')
    probe, exe = tmp_path / "probe.c", tmp_path / "probe"
    probe.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "spgroup.h"\nint main(void){\n' + "\n".join(lines) +
                     "\nreturn 0;}\n")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(probe), "-o", str(exe)])
    got = {n: [int(v) for v in vals] for n, *vals in (l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())}
    for name, dt in (("spg_loss_params", grouping.LOSS_PARAMS), ("spg_loss_pred", grouping.LOSS_PRED)):
        assert got[name] == [dt.itemsize] + [dt.fields[f][1] for f in dt.names], name
    src = open(os.path.join(ROOT, "include", "spgroup.h")).read()
    assert "SPG_BF16 = 4" in src and grouping.BF16 == 4
    assert "SPG_LOSS_FOCAL = 0" in src and "SPG_LOSS_L2 = 1" in src and (grouping.LOSS_FOCAL, grouping.LOSS_L2) == (0, 1)
