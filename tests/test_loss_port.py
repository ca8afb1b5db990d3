"""CPU: oracle/loss_port.py equals the reference's own MultiTaskLoss / MultiTaskLossParallel (tests/golden/loss/, made by
tests/golden/make_loss_golden.py): the loss and the printed per-stack sums bit for bit, every gradient as values."""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "loss")
sys.path[:0] = [os.path.join(HERE, "golden"), os.path.dirname(HERE)]

import make_loss_golden as mlg  # noqa: E402
from oracle import loss_port  # noqa: E402

CASES = json.load(open(os.path.join(GOLDEN, "MANIFEST.json")))["cases"]


def run_port(case, device="cpu"):
    """The port on a golden case's regenerated inputs: (result, prediction tensors) after backward(grad_output)."""
    preds, mask, labels = mlg.make_inputs(case)
    tp = [[torch.from_numpy(p).to(device).requires_grad_() for p in stack] for stack in preds]
    hs, bs = mlg.channel_layout(case["C"])
    r = loss_port.port_loss(tp, torch.from_numpy(mask).to(device), torch.from_numpy(labels).to(device),
                            nstack=case["nstack"], scale_weight=mlg.SCALE_WEIGHT, nstack_weight=case["nstack_weight"],
                            batch_size=case["batch_size"], focal=case["mode"] == "focal", heat_start=hs, bkg_start=bs,
                            multi_task_weight=0.1, keypoint_task_weight=3, offset_start=case["C"])
    r.loss.backward(torch.tensor(case["grad_output"], dtype=torch.float32, device=device))
    return r, tp


def same_values(a, b) -> bool:
    """Equal as values: +0 == -0, NaN where NaN."""
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_port_equals_the_reference(case):
    g = np.load(os.path.join(GOLDEN, case["name"] + ".npz"))
    r, tp = run_port(case)
    assert np.asarray(r.loss.detach()).tobytes() == g["loss"].tobytes()
    assert np.stack([s.numpy() for s in r.stack_sums]).tobytes() == g["stack_sums"].tobytes()
    for k, stack in enumerate(tp):
        for j, p in enumerate(stack):
            assert same_values(p.grad.numpy(), g[f"grad_{k}_{j}"]), (k, j)


def test_goldens_cover_the_issue_cases():
    names = {c["name"]: c for c in CASES}
    assert {c["mode"] for c in CASES} == {"focal", "l2"}
    assert any(c["batch_size"] != c["B"] for c in CASES)
    assert {3.0, 65536.0} <= {c["grad_output"] for c in CASES}
    assert {2, 4} <= {c["nstack"] for c in CASES}
    assert any(c["nan"] for c in CASES)
    assert math.isnan(float(np.load(os.path.join(GOLDEN, "focal_c12_nan.npz"))["loss"]))
    preds, mask, labels = mlg.make_inputs(names["focal_c50_ns2"])
    f = np.float32(0.01)
    for v in (np.nextafter(f, np.float32(0)), f, np.nextafter(f, np.float32(1))):
        assert (labels == v).any()
    m1 = torch.nn.functional.interpolate(torch.from_numpy(mask), size=(8, 8), mode="bilinear")
    assert (m1 == 0.5).any()


def test_exact_sums_of_the_terms_are_close_to_the_printed_ones():
    """The terms the port returns add up (math.fsum) to its per-stack sums within float32 summation error."""
    r, _ = run_port(CASES[0])
    for j in range(5):
        for k in range(CASES[0]["nstack"]):
            exact = math.fsum(r.terms[j][k].double().reshape(-1).tolist())
            assert abs(float(r.stack_sums[j][k]) - exact) <= 1e-5 * abs(exact) + 1e-30
