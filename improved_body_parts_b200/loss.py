"""The training loss on the device: the reference's ``MultiTaskLoss`` and ``MultiTaskLossParallel``.

The reference trains with ``models/loss_model.py:MultiTaskLoss`` (``train.py``, ``train_distributed*.py``) and
``models/loss_model_parallel.py:MultiTaskLossParallel`` (``train_parallel.py``).  Both build each scale's ground truth
from the full-size targets (``adaptive_avg_pool2d`` of the labels, a bilinear resize of ``mask_miss``) and sum a masked
(focal) L2 over ``[nstack, B, 50, h, w]`` tensors with about ten elementwise torch ops, and autograd keeps four such
tensors per scale for the backward.  Here both directions are one CUDA kernel each (csrc/loss.cuh) through
``spg_loss_forward`` / ``spg_loss_backward``, wrapped in a ``torch.autograd.Function``:

- ``MultiTaskLoss(opt, config)`` and ``MultiTaskLossParallel(opt, config)`` keep the reference's constructors and
  ``forward(pred_tuple, target_tuple)``; ``target_tuple`` is ``(mask_miss [B, 1, H, W], labels [B, C, H, W])``, i.e.
  ``targets.make_batch(...)[1:]``, taken without a copy.
- Gradients equal autograd of the reference on CUDA torch bit for bit; the loss is combined from float64-accumulated
  per-stack sums, which are kept on the device as ``last_stack_losses [5, nstack]`` instead of being printed (a print
  would synchronise the host every step).
- Predictions may be float32, bfloat16 or float16.  A low-precision prediction is taken as the reference applied to
  ``pred.float()``, autograd included: the float32 gradient is rounded once to the prediction's dtype.  That is not what
  the reference computes under apex O1, where ``where`` and ``abs`` run in float16.
- A prediction whose columns are not contiguous is made ``.contiguous()`` first (autograd carries the gradient through
  the copy); any batch, channel and row strides are read in place.

Malformed shapes, dtypes and devices raise ``ValueError``.  The handle is the per-device one ``targets`` caches; there
is no CPU path.  Each forward takes its own ticket and partial sums from torch's allocator on the current stream, so
losses may run concurrently on different streams and a forward captured in a CUDA graph needs no warm-up call.
"""
from __future__ import annotations

from typing import Sequence

import numpy as np
import torch
from torch import nn

from . import grouping, targets

SCALES = 5
MAX_STACKS = 8
_DTYPES = {torch.float32: grouping.F32, torch.bfloat16: grouping.BF16, torch.float16: grouping.F16}


def _target(t, name: str, shape_hint: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or t.dim() != 4:
        raise ValueError(f"{name} must be a float32 tensor {shape_hint}, got "
                         f"{getattr(t, 'dtype', type(t))} {tuple(getattr(t, 'shape', ()))}")
    return t


def _check(pred_tuple, mask_miss, labels, nstack: int, focal: bool, channels: int):
    """The checked targets and the ``nstack x 5`` predictions (columns made contiguous), or ``ValueError``."""
    mask_miss = _target(mask_miss, "mask_miss", "[B, 1, H, W]")
    labels = _target(labels, "labels", "[B, C, H, W]")
    B, C, H, W = labels.shape
    if tuple(mask_miss.shape) != (B, 1, H, W):
        raise ValueError(f"mask_miss must be [{B}, 1, {H}, {W}] to match labels, got {tuple(mask_miss.shape)}")
    if mask_miss.device != labels.device:
        raise ValueError(f"mask_miss is on {mask_miss.device}, labels on {labels.device}")
    if H < 16 or W < 16 or H % 16 or W % 16:
        raise ValueError(f"the targets' {H}x{W} maps must be multiples of 16 (five scales, each half the last)")
    if C != channels:
        raise ValueError(f"labels have {C} channels; the loss reads {channels}")
    if not 1 <= nstack <= MAX_STACKS:
        raise ValueError(f"nstack {nstack} outside [1, {MAX_STACKS}]")
    if len(pred_tuple) < nstack:
        raise ValueError(f"pred_tuple has {len(pred_tuple)} stacks; nstack is {nstack}")
    preds, dtype = [], None
    for k in range(nstack):
        if len(pred_tuple[k]) < SCALES:
            raise ValueError(f"stack {k} has {len(pred_tuple[k])} scales; the loss needs {SCALES}")
        for j in range(SCALES):
            p = pred_tuple[k][j]
            name = f"pred_tuple[{k}][{j}]"
            if not isinstance(p, torch.Tensor) or p.dtype not in _DTYPES:
                raise ValueError(f"{name} must be a float32, bfloat16 or float16 tensor, got {getattr(p, 'dtype', type(p))}")
            if p.device != labels.device:
                raise ValueError(f"{name} is on {p.device}; the targets are on {labels.device}")
            dtype = p.dtype if dtype is None else dtype
            if p.dtype != dtype:
                raise ValueError(f"{name} is {p.dtype}; the other predictions are {dtype}")
            want = (B, C, H >> j, W >> j)
            if p.dim() != 4 or p.shape[0] != B or p.shape[2:] != want[2:] or \
                    (p.shape[1] != C if focal else p.shape[1] < C):
                raise ValueError(f"{name} must be [{B}, {C if focal else f'>= {C}'}, {H >> j}, {W >> j}] (scale {j} of "
                                 f"the {H}x{W} targets), got {tuple(p.shape)}")
            preds.append(p if p.stride(-1) == 1 or p.shape[-1] == 1 else p.contiguous())
    if not labels.is_cuda:
        raise ValueError(f"the loss runs on CUDA devices only; the targets are on {labels.device}")
    aligned = [t if t.is_contiguous() and t.data_ptr() % 16 == 0 else t.clone(memory_format=torch.contiguous_format)
               for t in (mask_miss, labels)]
    return aligned[0], aligned[1], preds


def _records(preds: Sequence[torch.Tensor], grads=None) -> np.ndarray:
    r = np.zeros(len(preds), grouping.LOSS_PRED)
    for i, p in enumerate(preds):
        g = grads[i] if grads is not None else None
        r[i] = (p.data_ptr(), 0 if g is None else g.data_ptr(), p.stride(0), p.stride(1), p.stride(2),
                *((0, 0, 0) if g is None else (g.stride(0), g.stride(1), g.stride(2))))
    return r


class _FusedLoss(torch.autograd.Function):
    """``(loss, stack_sums)`` of ``preds`` (flat, ``k * 5 + j``); ``stack_sums`` is not differentiable."""

    @staticmethod
    def forward(ctx, params, mask_miss, labels, *preds):
        dev = labels.device
        g = targets._Device.for_device(dev.index)
        sums = torch.empty((SCALES, int(params["nstack"][0])), dtype=torch.float32, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        # the call's own ticket and partial sums, from torch's allocator on the current stream (the graph's pool while
        # capturing): no buffer is shared with another call, another stream or a captured graph
        ticket = torch.zeros((), dtype=torch.int32, device=dev)
        partials = torch.empty(g.loss_workspace_bytes(params) // 8, dtype=torch.float64, device=dev)
        g.loss_forward(params, mask_miss.data_ptr(), labels.data_ptr(), _records(preds), _DTYPES[preds[0].dtype],
                       sums.data_ptr(), loss.data_ptr(), ticket.data_ptr(), partials.data_ptr())
        ctx.params = params
        ctx.save_for_backward(mask_miss, labels, *preds)
        ctx.mark_non_differentiable(sums)
        return loss, sums

    @staticmethod
    def backward(ctx, grad_loss, _grad_sums):
        mask_miss, labels, *preds = ctx.saved_tensors
        C = labels.shape[1]
        grads = []
        for p in preds:
            gp = torch.empty(p.shape, dtype=p.dtype, device=p.device)
            if p.shape[1] > C:  # channels the loss does not read
                gp[:, C:].zero_()
            grads.append(gp)
        go = grad_loss.reshape(()).to(torch.float32).contiguous()
        g = targets._Device.for_device(labels.device.index)
        g.loss_backward(ctx.params, mask_miss.data_ptr(), labels.data_ptr(), _records(preds, grads),
                        _DTYPES[preds[0].dtype], go.data_ptr())
        return (None, None, None, *grads)


def loss_params(mode: int, nstack: int, labels_shape, *, heat_start: int = 0, bkg_start: int = 0,
                multi_task_weight: float = 1.0, keypoint_task_weight: float = 1.0, nstack_weight=None,
                scale_weight=None, batch_size: float = 1) -> np.ndarray:
    """The ``LOSS_PARAMS`` record: the weights as given, their sums as Python sums them."""
    B, C, H, W = (int(v) for v in labels_shape)
    nstack_weight = list(nstack_weight)
    scale_weight = list(scale_weight)
    if len(nstack_weight) != nstack:
        raise ValueError(f"nstack_weight has {len(nstack_weight)} entries; nstack is {nstack}")
    if len(scale_weight) < SCALES:
        raise ValueError(f"scale_weight has {len(scale_weight)} entries; the loss has {SCALES} scales")
    p = np.zeros(1, grouping.LOSS_PARAMS)
    p["mode"], p["nstack"], p["batch"], p["channels"], p["height"], p["width"] = mode, nstack, B, C, H, W
    p["heat_start"], p["bkg_start"] = heat_start, bkg_start
    p["multi_task_weight"], p["keypoint_task_weight"] = multi_task_weight, keypoint_task_weight
    p["nstack_weight"][0, :nstack] = nstack_weight
    p["scale_weight"][0] = scale_weight[:SCALES]
    p["batch_divisor"] = batch_size
    p["scale_weight_sum"], p["nstack_weight_sum"] = sum(scale_weight), sum(nstack_weight)
    return p


class MultiTaskLoss(nn.Module):
    """The reference's ``MultiTaskLoss``: the focal L2 of every stack and scale, weighted, over ``opt.batch_size``."""

    def __init__(self, opt, config, heatmap_weight=1, offset_weight=1, **kwargs):
        super().__init__()
        self.nstack = opt.nstack
        self.batch_size = opt.batch_size
        self.offset_start = config.offset_start
        self.heat_start = config.heat_start
        self.bkg_start = config.bkg_start
        self.multi_task_weight = opt.multi_task_weight
        self.keypoint_task_weight = opt.keypoint_task_weight
        self.scale_weight = opt.scale_weight
        self.nstack_weight = opt.nstack_weight
        self.heatmap_weight = heatmap_weight
        self.offset_weight = offset_weight
        #: ``[5, nstack]`` float32 on the device after each forward: the per-stack sums the reference prints per scale
        self.last_stack_losses = None

    def _params(self, labels_shape) -> np.ndarray:
        if not 0 <= self.heat_start <= self.bkg_start <= labels_shape[1]:
            raise ValueError(f"heat_start {self.heat_start} / bkg_start {self.bkg_start} outside the {labels_shape[1]} "
                             "label channels")
        if labels_shape[1] < 2:
            raise ValueError("the focal loss weights channel C - 2: labels need at least 2 channels")
        return loss_params(grouping.LOSS_FOCAL, self.nstack, labels_shape, heat_start=self.heat_start,
                           bkg_start=self.bkg_start, multi_task_weight=self.multi_task_weight,
                           keypoint_task_weight=self.keypoint_task_weight, nstack_weight=self.nstack_weight,
                           scale_weight=self.scale_weight, batch_size=self.batch_size)

    def _run(self, pred_tuple, target_tuple, focal: bool, channels=None):
        mask_miss, labels = target_tuple[0], target_tuple[1]
        C = channels if channels is not None else (labels.shape[1] if isinstance(labels, torch.Tensor) and labels.dim() == 4 else 0)
        mask_miss, labels, preds = _check(pred_tuple, mask_miss, labels, self.nstack, focal, C)
        loss, sums = _FusedLoss.apply(self._params(tuple(labels.shape)), mask_miss, labels, *preds)
        self.last_stack_losses = sums
        return loss

    def forward(self, pred_tuple, target_tuple):
        """``pred_tuple[k][j]``: stack k's ``[B, C, H >> j, W >> j]`` prediction; ``target_tuple``: ``(mask_miss
        [B, 1, H, W], labels [B, C, H, W])``.  Returns the 0-dim float32 loss."""
        return self._run(pred_tuple, target_tuple, True)


class MultiTaskLossParallel(MultiTaskLoss):
    """The reference's ``MultiTaskLossParallel``: the plain L2 of channels ``0..offset_start-1`` against the raw bilinear
    mask, weighted, not divided by the batch size (its training script does that)."""

    def __init__(self, opt, config, heatmap_weight=1, offset_weight=1, **kwargs):
        nn.Module.__init__(self)
        self.nstack = opt.nstack
        self.batch_size = opt.batch_size
        self.offset_start = config.offset_start
        self.multi_task_weight = opt.multi_task_weight
        self.scale_weight = opt.scale_weight
        self.nstack_weight = opt.nstack_weight
        self.heatmap_weight = heatmap_weight
        self.offset_weight = offset_weight
        self.last_stack_losses = None

    def _params(self, labels_shape) -> np.ndarray:
        return loss_params(grouping.LOSS_L2, self.nstack, labels_shape, nstack_weight=self.nstack_weight,
                           scale_weight=self.scale_weight, batch_size=1)

    def forward(self, pred_tuple, target_tuple):
        """As ``MultiTaskLoss.forward``; predictions may carry channels past ``offset_start`` (their gradient is 0)."""
        return self._run(pred_tuple, target_tuple, False, self.offset_start)
