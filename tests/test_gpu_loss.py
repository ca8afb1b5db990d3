"""GPU: the fused training loss (csrc/loss.cuh through improved_body_parts_b200.loss) against oracle/loss_port.py run
with CUDA torch: every prediction's gradient bit for bit as values, the per-stack sums within 1 float32 ULP of the exact
sum of the port's terms, the loss within 1e-5, repeatable bits, CUDA-graph capture, and one IMHN training step."""
import math
import os
import random
import sys
from types import SimpleNamespace

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.join(HERE, "golden"), os.path.dirname(HERE)]

pytestmark = pytest.mark.gpu

SW = [0.1, 0.2, 0.4, 1.6, 6.4]


def _opt(nstack, batch_size, nw=None):
    return SimpleNamespace(nstack=nstack, batch_size=batch_size, multi_task_weight=0.1, keypoint_task_weight=3,
                           scale_weight=list(SW), nstack_weight=list(nw or [1] * nstack))


CFG = SimpleNamespace(heat_start=30, bkg_start=48, offset_start=50)


def _same(a, b) -> bool:
    import torch
    return a.shape == b.shape and bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all())


def _synthetic_targets(B, H, W, seed, dev):
    """k/255 masks with checkerboard blocks (every resized value there is exactly 0.5) and labels with 0.01f and its
    neighbours."""
    import torch
    rng = np.random.default_rng(seed)
    labels = rng.random((B, 50, H, W), dtype=np.float32)
    labels[rng.random(labels.shape) < 0.5] = 0
    f = np.float32(0.01)
    sp = np.array([np.nextafter(f, np.float32(0)), f, np.nextafter(f, np.float32(1))], np.float32)
    idx = rng.choice(labels.size, labels.size // 10, replace=False)
    labels.flat[idx] = sp[rng.integers(0, 3, idx.size)]
    mask = rng.integers(0, 256, (B, 1, H, W)).astype(np.float32) / np.float32(255)
    mask[:, 0, :32, :32] = (np.add.outer(np.arange(32), np.arange(32)) % 2).astype(np.float32)[:H, :W]
    mask[:, 0, 40:56, :] = np.float32(128) / np.float32(255)
    return torch.from_numpy(mask).to(dev), torch.from_numpy(labels).to(dev)


def _make_batch_targets(B, seed, size=512):
    """(mask_miss, labels) of make_batch on the golden targets' sources with random joints and augmentations."""
    import targets_port as tp
    from improved_body_parts_b200 import targets
    rng = np.random.default_rng(seed)
    random.seed(seed)
    cfg = targets.TargetConfig(size, size)
    paths = tp.golden_paths()
    samples, augs = [], []
    for i in range(B):
        z = tp.load_case(paths[i % len(paths)])
        img, mm, ma = z["img"], z["mask_miss_src"], z["mask_all_src"]
        h, w = img.shape[:2]
        P = int(rng.integers(1, 8))
        j = np.zeros((P, 18, 3))
        j[:, :, 0:2] = rng.uniform([0, 0], [w, h], (P, 18, 2))
        j[:, :, 2] = rng.choice([0, 1, 2], (P, 18), p=[0.3, 0.6, 0.1])
        meta = {"objpos": [[w / 2, h / 2]], "scale_provided": [float(rng.uniform(0.3, 1.0))], "joints": j}
        aug = targets.AugmentSelection.random(cfg.transform_params)
        aug.tint = False
        samples.append((img, mm, ma, meta))
        augs.append(aug)
    _, miss, labels = targets.make_batch(samples, augs, cfg)
    return miss, labels


def _preds(B, C, H, W, nstack, seed, dev, labels=None, view=None):
    """pred_tuple[k][j] float32 leaves (or views of leaves: view="strided" / "transposed") and the leaves."""
    import torch
    g = torch.Generator(device=dev).manual_seed(seed)
    out, leaves = [], []
    for k in range(nstack):
        stack = []
        for j in range(5):
            h, w = H >> j, W >> j
            if view == "strided" and j % 2 == 0:
                base = (torch.rand(B, C + 3, h, w + 5, generator=g, device=dev) * 1.5 - 0.25).requires_grad_()
                p = base[:, 1:C + 1, :, 2:2 + w]
            elif view == "transposed" and j == 1:
                base = (torch.rand(B, C, w, h, generator=g, device=dev) * 1.5 - 0.25).requires_grad_()
                p = base.transpose(2, 3)
            else:
                base = (torch.rand(B, C, h, w, generator=g, device=dev) * 1.5 - 0.25)
                if j == 0 and k == 0 and labels is not None:  # s = 1 on labels >= 0.01, tiny s below
                    sel = torch.rand(base[:, :labels.shape[1]].shape, generator=g, device=dev) < 0.3
                    lab = labels.to(dev)
                    v = base[:, :labels.shape[1]]
                    v[sel & (lab >= 0.01)] = 1.0
                    v[sel & (lab < 0.01)] = 2.0 ** -26
                base.requires_grad_()
                p = base
            stack.append(p)
            leaves.append(base)
        out.append(stack)
    return out, leaves


def _clone(leaves, pred_tuple, dtype=None):
    """The same predictions as new leaves (float32 copies of low-precision ones when dtype is given)."""
    mapping = {}
    new = []
    for L in leaves:
        c = L.detach().float().clone() if dtype is not None else L.detach().clone()
        c.requires_grad_()
        mapping[id(L)] = c
        new.append(c)
    out = []
    for stack in pred_tuple:
        row = []
        for p in stack:
            base = p if p._base is None else p._base
            c = mapping[id(base)]
            row.append(c if p._base is None else c.as_strided(p.shape, p.stride(), p.storage_offset()))
        out.append(row)
    return out, new


def _port(pred_tuple, mask, labels, opt, focal, cfg=CFG):
    from oracle import loss_port
    return loss_port.port_loss(pred_tuple, mask, labels, nstack=opt.nstack, scale_weight=opt.scale_weight,
                               nstack_weight=opt.nstack_weight, batch_size=opt.batch_size, focal=focal,
                               heat_start=cfg.heat_start, bkg_start=cfg.bkg_start, multi_task_weight=opt.multi_task_weight,
                               keypoint_task_weight=opt.keypoint_task_weight, offset_start=cfg.offset_start)


def _criterion(opt, focal, cfg=CFG):
    from improved_body_parts_b200.loss import MultiTaskLoss, MultiTaskLossParallel
    return (MultiTaskLoss if focal else MultiTaskLossParallel)(opt, cfg)


def _ulps(a: float, b: float) -> int:
    fa, fb = np.array([a], np.float32).view(np.int32)[0], np.array([b], np.float32).view(np.int32)[0]
    return abs(int(fa) - int(fb))


def _check_case(dev, pred_tuple, leaves, mask, labels, opt, focal, go, exact_sums=False, cfg=CFG):
    import torch
    crit = _criterion(opt, focal, cfg)
    loss = crit(pred_tuple, (mask, labels))
    loss.backward(torch.tensor(go, device=dev))
    sums = crit.last_stack_losses.cpu()
    pt, pleaves = _clone(leaves, pred_tuple)
    r = _port(pt, mask, labels, opt, focal, cfg)
    r.loss.backward(torch.tensor(go, device=dev))
    for i, (a, b) in enumerate(zip(leaves, pleaves)):
        assert _same(a.grad, b.grad), f"gradient of leaf {i} differs"
    for j in range(5):
        for k in range(opt.nstack):
            t = r.terms[j][k]
            exact = math.fsum(t.double().cpu().reshape(-1).tolist()) if exact_sums else float(t.double().sum())
            assert _ulps(float(sums[j, k]), float(np.float32(exact))) <= 1, (j, k, float(sums[j, k]), exact)
    lv, rv = float(loss.detach()), float(r.loss.detach())
    assert abs(lv - rv) <= 1e-5 * abs(rv), (lv, rv)
    return loss, sums


@pytest.mark.parametrize("B, go, focal", [(4, 1.0, True), (16, 3.0, True), (4, 65536.0, False), (16, 1.0, False)])
def test_make_batch_targets_128(cuda_device, B, go, focal):
    mask, labels = _make_batch_targets(B, 100 + B)
    opt = _opt(4, B, [1, 1, 0.5, 2])
    pt, leaves = _preds(B, 50 if focal else 52, 128, 128, 4, B, cuda_device, labels)
    _check_case(cuda_device, pt, leaves, mask, labels, opt, focal, go)


@pytest.mark.parametrize("go, focal, view", [(65536.0, True, None), (3.0, True, "strided"), (1.0, False, "transposed"),
                                             (3.0, False, "strided")])
def test_crafted_targets_96x160(cuda_device, go, focal, view):
    mask, labels = _synthetic_targets(3, 96, 160, 7, cuda_device)
    opt = _opt(2, 5, [1, 2.5])
    pt, leaves = _preds(3, 50 if focal else 52, 96, 160, 2, 9, cuda_device, labels, view)
    _check_case(cuda_device, pt, leaves, mask, labels, opt, focal, go, exact_sums=view is None)


@pytest.mark.parametrize("dtype", ["bfloat16", "float16"])
def test_low_precision_predictions(cuda_device, dtype):
    import torch
    dt = getattr(torch, dtype)
    mask, labels = _synthetic_targets(2, 64, 96, 3, cuda_device)
    opt = _opt(2, 3)
    pt32, _ = _preds(2, 50, 64, 96, 2, 4, cuda_device, labels)
    lp = [[p.detach().to(dt).requires_grad_() for p in s] for s in pt32]
    crit = _criterion(opt, True)
    loss = crit(lp, (mask, labels))
    loss.backward(torch.tensor(3.0, device=cuda_device))
    ref = [[p.detach().float().requires_grad_() for p in s] for s in lp]
    r = _port(ref, mask, labels, opt, True)
    r.loss.backward(torch.tensor(3.0, device=cuda_device))
    for s, rs in zip(lp, ref):
        for p, q in zip(s, rs):
            assert p.grad.dtype == dt and _same(p.grad, q.grad.to(dt))
    assert abs(float(loss.detach()) - float(r.loss.detach())) <= 1e-5 * abs(float(r.loss.detach()))


def test_nan_prediction_matches_the_port(cuda_device):
    import torch
    mask, labels = _synthetic_targets(2, 32, 48, 5, cuda_device)
    opt = _opt(2, 2)
    pt, leaves = _preds(2, 50, 32, 48, 2, 6, cuda_device)
    with torch.no_grad():
        leaves[6][1, 3, 2, 5] = float("nan")
    crit = _criterion(opt, True)
    loss = crit(pt, (mask, labels))
    loss.backward()
    pt2, leaves2 = _clone(leaves, pt)
    r = _port(pt2, mask, labels, opt, True)
    r.loss.backward()
    assert math.isnan(float(loss.detach())) and math.isnan(float(r.loss.detach()))
    for a, b in zip(leaves, leaves2):
        assert _same(a.grad, b.grad)
    assert bool(torch.isnan(leaves[6].grad).any())


def test_repeatable_bits_and_another_stream(cuda_device):
    import torch
    mask, labels = _synthetic_targets(4, 128, 128, 8, cuda_device)
    opt = _opt(4, 4)
    pt, leaves = _preds(4, 50, 128, 128, 4, 8, cuda_device, labels)
    crit = _criterion(opt, True)

    def step():
        for L in leaves:
            L.grad = None
        loss = crit(pt, (mask, labels))
        loss.backward(torch.tensor(3.0, device=cuda_device))
        return loss.detach().clone(), crit.last_stack_losses.clone(), [L.grad.clone() for L in leaves]

    a = step()
    b = step()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        c = step()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for other in (b, c):
        assert torch.equal(a[0].view(torch.int32), other[0].view(torch.int32))
        assert torch.equal(a[1].view(torch.int32), other[1].view(torch.int32))
        for x, y in zip(a[2], other[2]):
            assert torch.equal(x.view(torch.int32), y.view(torch.int32))


def test_forward_and_backward_capture_in_a_cuda_graph(cuda_device):
    import torch
    mask, labels = _synthetic_targets(2, 64, 64, 12, cuda_device)
    opt = _opt(2, 2)
    pt, leaves = _preds(2, 50, 64, 64, 2, 12, cuda_device, labels)
    crit = _criterion(opt, True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):  # the eager bits to compare with (test_gpu_loss_space.py captures without this call)
        loss = crit(pt, (mask, labels))
        loss.backward()
        eager = [L.grad.clone() for L in leaves]
        eager_loss = loss.detach().clone()
    del loss
    for L in leaves:
        L.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        static_loss = crit(pt, (mask, labels))
        static_loss.backward()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static_loss.view(torch.int32), eager_loss.view(torch.int32))
    for L, e in zip(leaves, eager):
        assert torch.equal(L.grad.view(torch.int32), e.view(torch.int32))


def test_one_training_step_with_imhn(cuda_device):
    """make_batch -> IMHN(...).train().forward_all -> MultiTaskLoss -> backward: the parameter gradients agree with the
    same step through the port's loss to a relative L2 distance of 1e-4 (only cuDNN's backward order differs)."""
    import torch
    from improved_body_parts_b200 import imhn, targets
    random.seed(3)
    cfg = targets.TargetConfig(256, 256)
    rng = np.random.default_rng(3)
    samples, augs = [], []
    for i in range(2):
        img = rng.integers(0, 256, (300, 400, 3), dtype=np.uint8)
        mm = np.where(rng.random((300, 400)) < 0.1, 0, 255).astype(np.uint8)
        ma = np.where(rng.random((300, 400)) < 0.3, 255, 0).astype(np.uint8)
        j = np.zeros((3, 18, 3))
        j[:, :, 0:2] = rng.uniform([0, 0], [400, 300], (3, 18, 2))
        samples.append((img, mm, ma, {"objpos": [[200.0, 150.0]], "scale_provided": [0.5], "joints": j}))
        augs.append(targets.AugmentSelection.unrandom())
    images, mask, labels = targets.make_batch(samples, augs, cfg)
    torch.manual_seed(0)
    model = imhn.IMHN(nstack=2).to(cuda_device).train()
    preds = model.forward_all(images)
    opt = _opt(2, 2)
    params = [p for p in model.parameters() if p.requires_grad]
    ga = torch.autograd.grad(_criterion(opt, True)(preds, (mask, labels)), params, retain_graph=True, allow_unused=True)
    gb = torch.autograd.grad(_port(preds, mask, labels, opt, True).loss, params, allow_unused=True)
    num = den = 0.0
    for a, b in zip(ga, gb):
        if a is None:
            assert b is None
            continue
        num += float((a.double() - b.double()).pow(2).sum())
        den += float(b.double().pow(2).sum())
    assert den > 0 and math.sqrt(num / den) <= 1e-4, math.sqrt(num / den)
