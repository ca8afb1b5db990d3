"""Torch port of the reference's two training losses, for checking ``improved_body_parts_b200.loss``.

TEST INFRASTRUCTURE ONLY.  Restated from the formulas of ``models/loss_model.py:MultiTaskLoss`` (focal L2, gamma 1,
alpha = beta = 0) and ``models/loss_model_parallel.py:MultiTaskLossParallel`` (plain L2), with the same torch operations
in the same order so that it carries whichever device's arithmetic its tensors are on: on CPU it equals the reference
class bit for bit (tests/golden/loss/), on CUDA it is what the reference computes on the GPU it trains on.  Gradients
come from autograd.  ``port_loss`` also returns the elementwise terms, so that a test can form exact per-(scale, stack)
sums, and ``combine`` is its last step alone, to be applied to another implementation's per-stack sums.
"""
from __future__ import annotations

from typing import List, NamedTuple

import torch
import torch.nn.functional as F


class PortResult(NamedTuple):
    loss: torch.Tensor                # 0-dim, differentiable
    stack_sums: List[torch.Tensor]    # per scale: [nstack], what the reference prints
    terms: List[torch.Tensor]         # per scale: [nstack, B, C, h, w], detached


def scale_targets(mask_miss, labels, size, focal: bool):
    """One scale's ground truth: the pooled labels and the resized mask (thresholded at 0.5 for the focal loss)."""
    gt = F.adaptive_avg_pool2d(labels, output_size=size)
    m = F.interpolate(mask_miss, size=size, mode="bilinear")
    if focal:
        m[m < 0.5] = 0
    return gt, m


def combine(stack_sums, nstack_weight, scale_weight, batch_size=1, focal=True):
    """The reference's loss from its per-stack sums (``stack_sums[j][k]``, one 0-dim or ``[nstack]`` tensor per scale, or
    a ``[5, nstack]`` tensor): the stacks weighted and summed per scale, the scales weighted and summed, each sum with
    Python's ``sum()`` and each division by a Python number, in that order.  ``focal``: divided by ``batch_size``."""
    per_scale = []
    for j in range(5):
        weighted = [stack_sums[j][k] * nstack_weight[k] for k in range(len(nstack_weight))]
        per_scale.append(sum(weighted) / sum(nstack_weight) * scale_weight[j])
    loss = sum(per_scale) / sum(scale_weight)
    if focal:
        loss = loss / batch_size
    return loss


def port_loss(pred_tuple, mask_miss, labels, *, nstack, scale_weight, nstack_weight, batch_size=1, focal=True,
              heat_start=0, bkg_start=0, multi_task_weight=0.1, keypoint_task_weight=1, offset_start=None):
    """The reference's loss of ``pred_tuple[k][j]`` (k < nstack, j < 5) against ``(mask_miss, labels)``.  ``focal``:
    MultiTaskLoss (divided by ``batch_size``); else MultiTaskLossParallel (channels ``:offset_start``, no division)."""
    per_stack_sums, sums, terms = [], [], []
    for j in range(5):
        s = torch.cat([pred_tuple[k][j][None, ...] for k in range(nstack)], dim=0)
        if not focal:
            s = s[:, :, :offset_start]
        gt, m = scale_targets(mask_miss, labels, s.shape[-2:], focal)
        gt, m = gt[None, ...], m[None, ...]
        if focal:
            w = m.expand_as(gt).clone()
            w[:, :, -2, :, :] *= multi_task_weight
            w[:, :, heat_start:bkg_start, :, :] *= keypoint_task_weight
            st = torch.where(torch.ge(gt, 0.01), s, 1 - s)
            out = (s - gt) ** 2 * torch.abs(1. - st) * w
        else:
            out = (s - gt) ** 2 * m
        per_stack = out.sum(dim=(1, 2, 3, 4))
        per_stack_sums.append(per_stack)
        sums.append(per_stack.detach())
        terms.append(out.detach())
    return PortResult(combine(per_stack_sums, nstack_weight, scale_weight, batch_size, focal), sums, terms)
