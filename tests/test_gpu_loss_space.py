"""GPU: the fused training loss across what it admits (tests/loss_cases.py): every stack count, channel layout, target
shape, dtype and access path, each against oracle/loss_port.py on CUDA torch four ways -- every gradient bit for bit,
every per-stack sum within 1 float32 ULP of the exact sum of the port's terms, the loss bit for bit as the port's
``combine`` of the kernel's own per-stack sums (also over 32 seeded draws), and the kernel spg_stage_kernel names.  Then
the backward's writes confined to ``[B, C, h, w]`` of strided gradients, the 16 x 16 targets' 1 x 1 scale, and the
forward's per-call workspace: interleaved grids, graph capture without a warm-up, an eager call between capture and
replay, two streams."""
import math
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE)]

from loss_cases import CASES, SW, LossCase  # noqa: E402
from test_gpu_loss import _clone, _preds, _same, _synthetic_targets, _ulps  # noqa: E402

pytestmark = pytest.mark.gpu

TAGS = {"float32": "float", "bfloat16": "bf16", "float16": "f16"}


def _targets(case: LossCase, dev):
    """_synthetic_targets with case.C label channels (two draws side by side past 50)."""
    import torch
    mask, labels = _synthetic_targets(case.B, case.H, case.W, case.seed, dev)
    if case.C > 50:
        labels = torch.cat([labels, _synthetic_targets(case.B, case.H, case.W, case.seed + 100, dev)[1][:, :case.C - 50]], 1)
    return mask, labels[:, :case.C].contiguous()


def _criterion(case: LossCase):
    from improved_body_parts_b200.loss import MultiTaskLoss, MultiTaskLossParallel
    opt = SimpleNamespace(nstack=case.nstack, batch_size=case.batch_size, multi_task_weight=0.1, keypoint_task_weight=3,
                          scale_weight=list(case.scale_weight), nstack_weight=list(case.nstack_weight))
    cfg = SimpleNamespace(heat_start=case.heat[0], bkg_start=case.heat[1], offset_start=case.C)
    return (MultiTaskLoss if case.focal else MultiTaskLossParallel)(opt, cfg)


def _sequential_mean(labels):
    """The kernel's pooled label at a 1 x 1 scale of 16 x 16 targets: the 256 values summed row-major in sequence in
    float32, then divided by 16 and by 16."""
    import torch
    x = labels.detach().cpu().numpy().reshape(labels.shape[0], labels.shape[1], -1)
    s = np.cumsum(x, axis=-1, dtype=np.float32)[..., -1]
    v = (s / np.float32(16)) / np.float32(16)
    return torch.from_numpy(v.astype(np.float32)).reshape(labels.shape[0], labels.shape[1], 1, 1).to(labels.device)


def _port(case: LossCase, pred_tuple, mask, labels, sequential_1x1=None):
    """The port on CUDA torch.  ``sequential_1x1`` (default: for 16 x 16 targets) takes the 1 x 1 scale's pooled label
    as the kernel forms it, DESIGN.md §4's one documented difference from CUDA torch's ``mean``."""
    from oracle import loss_port
    if sequential_1x1 is None:
        sequential_1x1 = case.H == case.W == 16
    plain = loss_port.scale_targets

    def targets_1x1(m, lab, size, focal):
        gt, mk = plain(m, lab, size, focal)
        return (_sequential_mean(lab), mk) if tuple(size) == (1, 1) else (gt, mk)

    loss_port.scale_targets = targets_1x1 if sequential_1x1 else plain
    try:
        return loss_port.port_loss(pred_tuple, mask, labels, nstack=case.nstack, scale_weight=case.scale_weight,
                                   nstack_weight=case.nstack_weight, batch_size=case.batch_size, focal=case.focal,
                                   heat_start=case.heat[0], bkg_start=case.heat[1], multi_task_weight=0.1,
                                   keypoint_task_weight=3, offset_start=case.C)
    finally:
        loss_port.scale_targets = plain


def _check(case: LossCase, dev, pred_tuple, leaves, mask, labels, dtype_name="float32"):
    """The four checks of one case; returns the loss, the per-stack sums and the leaves' gradients."""
    import torch
    from improved_body_parts_b200 import targets
    from oracle import loss_port
    g = targets._Device.for_device(dev.index)
    crit = _criterion(case)
    loss = crit(pred_tuple, (mask, labels))
    fwd_kernel = g.loss_kernel()
    loss.backward(torch.tensor(case.grad_output, device=dev))
    bwd_kernel = g.loss_kernel()
    sums = crit.last_stack_losses
    # 4. the dtype's kernels ran
    assert (fwd_kernel, bwd_kernel) == (f"loss_forward_kernel<{TAGS[dtype_name]}>", f"loss_backward_kernel<{TAGS[dtype_name]}>")
    # 1. every gradient bit for bit (as values, NaN by position): low precision as the float32 gradient rounded once
    low = dtype_name != "float32"
    pt, pleaves = _clone(leaves, pred_tuple, torch.float32 if low else None)
    r = _port(case, pt, mask, labels)
    r.loss.backward(torch.tensor(case.grad_output, device=dev))
    for i, (a, b) in enumerate(zip(leaves, pleaves)):
        assert a.grad.dtype == a.dtype and _same(a.grad, b.grad.to(a.dtype)), f"{case.name}: gradient of leaf {i} differs"
    # 2. every per-stack sum within 1 ULP of the exact sum of the port's terms
    host = sums.cpu()
    for j in range(5):
        for k in range(case.nstack):
            exact = math.fsum(r.terms[j][k].double().cpu().reshape(-1).tolist())
            assert _ulps(float(host[j, k]), float(np.float32(exact))) <= 1, (case.name, j, k, float(host[j, k]), exact)
    # 3. the loss is the reference's combination of the kernel's own sums, bit for bit, and close to the port's loss
    want = loss_port.combine(sums, case.nstack_weight, case.scale_weight, case.batch_size, case.focal)
    assert torch.equal(loss.detach().view(torch.int32), want.reshape(()).view(torch.int32)), \
        (case.name, float(loss), float(want))
    lv, rv = float(loss.detach()), float(r.loss.detach())
    assert abs(lv - rv) <= 1e-5 * abs(rv), (case.name, lv, rv)
    return loss.detach(), sums, [L.grad for L in leaves]


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_case(cuda_device, case):
    mask, labels = _targets(case, cuda_device)
    pt, leaves = _preds(case.B, case.pred_channels, case.H, case.W, case.nstack, case.seed, cuda_device, labels)
    _check(case, cuda_device, pt, leaves, mask, labels)


def test_combination_over_seeds(cuda_device):
    """The loss is combine() of the kernel's own per-stack sums, bit for bit, over many draws of 8 weighted stacks: a
    float32 combination in another order (inv_nw applied per stack, say) moves the loss's last bits in about a third of
    the draws."""
    import torch
    from oracle import loss_port
    for seed in range(32):
        case = LossCase(f"seed{seed}", seed % 2 == 0, [1.0, 0.1, 0.3, 2.5, 1.0, 0.0, 1.0, 0.3], SW, 1, 3, 16, 32,
                        (0, 1), 3, 1.0, 200 + seed, 0 if seed % 2 == 0 else 3)
        mask, labels = _targets(case, cuda_device)
        pt, _ = _preds(case.B, case.pred_channels, case.H, case.W, case.nstack, case.seed, cuda_device, labels)
        crit = _criterion(case)
        with torch.no_grad():
            loss = crit(pt, (mask, labels))
        want = loss_port.combine(crit.last_stack_losses, case.nstack_weight, case.scale_weight, case.batch_size,
                                 case.focal)
        assert torch.equal(loss.view(torch.int32), want.reshape(()).view(torch.int32)), (seed, float(loss), float(want))


# ---- dtype x access: vector and scalar accesses across the scales of one tensor, through strided views ---------------
VIEWS = ["contiguous", "column_offset", "row_stride", "batch_stride", "transposed"]


def _view_preds(case: LossCase, dev, dtype, view):
    """pred_tuple[k][j] of ``dtype`` as ``view`` of a leaf: contiguous; columns one element in; rows 2 elements longer
    (a row stride that is not a multiple of 4); an odd batch stride; a transposed copy (columns not contiguous)."""
    import torch
    gen = torch.Generator(device=dev).manual_seed(case.seed)
    B, C = case.B, case.pred_channels
    out, leaves = [], []
    for k in range(case.nstack):
        stack = []
        for j in range(5):
            h, w = case.H >> j, case.W >> j
            vals = (torch.rand(B, C, h, w, generator=gen, device=dev) * 1.5 - 0.25).to(dtype)
            if view == "contiguous":
                base = vals
                take = lambda t: t  # noqa: E731
            elif view == "column_offset":
                base = torch.zeros(B, C, h, w + 1, dtype=dtype, device=dev)
                base[..., 1:] = vals
                take = lambda t: t[..., 1:]  # noqa: E731
            elif view == "row_stride":
                base = torch.zeros(B, C, h, w + 2, dtype=dtype, device=dev)
                base[..., :w] = vals
                take = lambda t, w=w: t[..., :w]  # noqa: E731
            elif view == "batch_stride":
                n = C * h * w + 1
                base = torch.zeros(B * n, dtype=dtype, device=dev)
                take = lambda t, s=(B, C, h, w), st=(n, h * w, w, 1): t.as_strided(s, st)  # noqa: E731
                take(base).copy_(vals)
            else:
                base = vals.transpose(2, 3).contiguous()
                take = lambda t: t.transpose(2, 3)  # noqa: E731
            base.requires_grad_()
            p = take(base)
            assert torch.equal(p.detach(), vals)
            stack.append(p)
            leaves.append(base)
        out.append(stack)
    return out, leaves


@pytest.mark.parametrize("view", VIEWS)
@pytest.mark.parametrize("dtype_name", ["float32", "bfloat16", "float16"])
def test_dtype_and_access(cuda_device, dtype_name, view):
    import torch
    W = 48 if dtype_name == "float32" else 80  # scales 0-2 may take vector accesses, 3-4 (w = 6, 3 or 10, 5) may not
    case = LossCase(f"{dtype_name}_{view}", True, [1.0, 0.3, 2.5], SW, 2, 12, 32, W, (3, 9), 3, 3.0, 21)
    mask, labels = _targets(case, cuda_device)
    pt, leaves = _view_preds(case, cuda_device, getattr(torch, dtype_name), view)
    _check(case, cuda_device, pt, leaves, mask, labels, dtype_name)


# ---- the backward writes [B, C, h, w] of each gradient and nothing else ------------------------------------------------
@pytest.mark.parametrize("layout", ["vector", "scalar"])
@pytest.mark.parametrize("dtype_name", ["float32", "bfloat16"])
@pytest.mark.parametrize("forward_first", [False, True])
def test_backward_writes_only_its_gradients(cuda_device, dtype_name, layout, forward_first):
    """spg_loss_backward into views of sentinel-filled buffers with a batch, channels, rows and columns around them
    (16-byte aligned strides for ``vector``, odd ones for ``scalar``); the predictions carry 2 channels past C."""
    import torch
    from improved_body_parts_b200 import loss as L, targets
    dev = cuda_device
    dt = getattr(torch, dtype_name)
    case = LossCase("confined", True, [1.0, 2.5], SW, 2, 6, 32, 80, (1, 4), 2, 3.0, 31)
    B, C = case.B, case.C
    mask, labels = _targets(case, dev)
    gen = torch.Generator(device=dev).manual_seed(case.seed)
    pt, leaves, grads, bufs, regions = [], [], [], [], []
    pad = 4 if layout == "vector" else 1
    for k in range(case.nstack):
        row = []
        for j in range(5):
            h, w = case.H >> j, case.W >> j
            base = (torch.rand(B, C + 2, h, w, generator=gen, device=dev) * 1.5 - 0.25).to(dt).requires_grad_()
            row.append(base[:, :C])
            leaves.append(base)
            buf = torch.full((B + 1, C + 3, h + 2, w + pad + 4), -7.0, dtype=dt, device=dev)
            region = (slice(1, None), slice(1, C + 1), slice(1, h + 1), slice(pad, pad + w))
            bufs.append(buf)
            regions.append(region)
            grads.append(buf[region])
        pt.append(row)
    flat = [p for s in pt for p in s]
    before = [b.clone() for b in bufs]
    g = targets._Device.for_device(dev.index)
    params = _criterion(case)._params(tuple(labels.shape))
    if forward_first:
        sums = torch.empty(5, case.nstack, device=dev)
        out = torch.empty((), device=dev)
        ticket = torch.zeros((), dtype=torch.int32, device=dev)
        partials = torch.empty(g.loss_workspace_bytes(params) // 8, dtype=torch.float64, device=dev)
        g.loss_forward(params, mask.data_ptr(), labels.data_ptr(), L._records(flat), L._DTYPES[dt], sums.data_ptr(),
                       out.data_ptr(), ticket.data_ptr(), partials.data_ptr())
        assert int(ticket) == 0  # left as it was found
    go = torch.tensor(case.grad_output, device=dev)
    g.loss_backward(params, mask.data_ptr(), labels.data_ptr(), L._records(flat, grads), L._DTYPES[dt], go.data_ptr())
    torch.cuda.synchronize()
    assert g.loss_kernel() == f"loss_backward_kernel<{TAGS[dtype_name]}>"
    rt, rleaves = _clone(leaves, pt, torch.float32)
    r = _port(case, rt, mask, labels)
    r.loss.backward(go)
    bits = torch.int32 if dt == torch.float32 else torch.int16
    for i, (buf, b0, region, rl) in enumerate(zip(bufs, before, regions, rleaves)):
        outside = torch.ones(buf.shape, dtype=torch.bool, device=dev)
        outside[region] = False
        assert torch.equal(buf.view(bits)[outside], b0.view(bits)[outside]), f"prediction {i}: a write outside [B, C, h, w]"
        assert _same(buf[region], rl.grad[:, :C].to(dt)), f"prediction {i}: gradient differs from the port"


# ---- 16 x 16 targets: the 1 x 1 scale ----------------------------------------------------------------------------------
def test_16x16_targets_differ_from_cuda_torch_only_in_the_documented_label(cuda_device):
    """At a 1 x 1 coarsest scale CUDA torch's adaptive_avg_pool2d is ``mean``, whose reduction order is its own; the
    kernel sums the 256 labels row-major in sequence (DESIGN.md §4).  Exactly that differs: every gradient of scales 0-3
    equals the unmodified port, every gradient of scale 4 equals the port given the sequential label, and the two labels
    are within the float32 summation bound of each other.  The loss stays within 1e-5 of CUDA torch's."""
    import torch
    import torch.nn.functional as F
    case = LossCase("ns4_c50_16x16_b8", True, [1.0, 0.3, 2.5, 0.1], SW, 8, 50, 16, 16, (30, 48), 8, 3.0, 41)
    dev = cuda_device
    mask, labels = _targets(case, dev)
    pt, leaves = _preds(case.B, case.C, 16, 16, case.nstack, case.seed, dev, labels)
    loss, _, _ = _check(case, dev, pt, leaves, mask, labels)  # against the port with the sequential 1 x 1 label
    qt, qleaves = _clone(leaves, pt)
    r = _port(case, qt, mask, labels, sequential_1x1=False)
    r.loss.backward(torch.tensor(case.grad_output, device=dev))
    differ = 0
    for i, (a, b) in enumerate(zip(leaves, qleaves)):
        if i % 5 < 4:
            assert _same(a.grad, b.grad), f"leaf {i} (scale {i % 5}) differs from CUDA torch"
        else:
            differ += int((a.grad != b.grad).sum())
    torch_label = F.adaptive_avg_pool2d(labels, (1, 1)).double().cpu()
    seq_label = _sequential_mean(labels).double().cpu()
    exact = labels.double().cpu().sum(dim=(2, 3), keepdim=True) / 256
    bound = 2 * 255 * 2.0 ** -24 * exact  # two orders of 256 non-negative float32 terms, each within 255 u of the sum
    assert bool(((torch_label - seq_label).abs() <= bound).all())
    ulps = (torch_label.float().view(torch.int32).long() - seq_label.float().view(torch.int32).long()).abs()
    assert abs(float(loss) - float(r.loss.detach())) <= 1e-5 * abs(float(r.loss.detach()))
    print(f"16x16: {int((ulps > 0).sum())} of {ulps.numel()} pooled labels differ from CUDA torch's mean, at most "
          f"{int(ulps.max())} ULP; {differ} scale-4 gradient elements differ")


# ---- the forward's workspace: one per call ----------------------------------------------------------------------------
SMALL = LossCase("small", True, [1.0, 0.3], SW, 2, 12, 32, 48, (3, 9), 2, 1.0, 51)
LARGE = LossCase("large", True, [1.0, 0.1, 0.3, 2.5, 1.0, 0.0, 1.0], SW, 4, 50, 64, 96, (30, 48), 4, 1.0, 52)
LARGEST = LossCase("largest", False, [1.0] * 8, SW, 8, 50, 128, 128, (0, 0), 8, 1.0, 53, 3)
# the largest grid of this file: 16 x 57 x 8 CTAs x 40 (scale, stack) sums
CAPTURED = LossCase("captured", True, [1.0, 0.1, 0.3, 2.5, 1.0, 1.0, 0.0, 1.0], SW, 16, 57, 128, 128, (1, 56), 16, 1.0, 54)


def _inputs(case, dev):
    mask, labels = _targets(case, dev)
    pt, leaves = _preds(case.B, case.pred_channels, case.H, case.W, case.nstack, case.seed, dev, labels)
    return pt, leaves, mask, labels


def _step(case, inputs):
    """One eager forward + backward (grad_output 1) on fresh copies of the leaves: (loss, sums, gradients) as bits."""
    import torch
    pt, leaves, mask, labels = inputs
    qt, qleaves = _clone(leaves, pt)
    crit = _criterion(case)
    loss = crit(qt, (mask, labels))
    loss.backward()
    return [t.detach().clone() for t in [loss, crit.last_stack_losses] + [L.grad for L in qleaves]]


def _same_bits(a, b) -> bool:
    import torch
    return len(a) == len(b) and all(x.dtype == y.dtype and torch.equal(x.view(torch.int32), y.view(torch.int32))
                                    for x, y in zip(a, b))


def test_interleaved_grids_and_stack_counts(cuda_device):
    cases = [SMALL, LARGE, LARGEST]
    inputs = [_inputs(c, cuda_device) for c in cases]
    first = [_step(c, i) for c, i in zip(cases, inputs)]
    for order in ([2, 0, 1], [0, 2, 0, 1, 1]):
        for n in order:
            assert _same_bits(_step(cases[n], inputs[n]), first[n]), cases[n].name


def _capture(case, inputs, stream):
    """A CUDA graph of one forward + backward on fresh copies of the leaves: (graph, its outputs)."""
    import torch
    pt, leaves, mask, labels = inputs
    qt, qleaves = _clone(leaves, pt)
    crit = _criterion(case)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        loss = crit(qt, (mask, labels))
        loss.backward()
    return graph, [loss, crit.last_stack_losses] + [L.grad for L in qleaves]


def test_capture_without_a_warm_up(cuda_device):
    """The first forward of a grid larger than any before it, captured: its workspace comes from the graph's pool."""
    import torch
    small, large = _inputs(SMALL, cuda_device), _inputs(CAPTURED, cuda_device)
    _step(SMALL, small)  # the handle exists and the kernels are loaded; nothing of CAPTURED's size has run
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph, outs = _capture(CAPTURED, large, side)
    graph.replay()
    torch.cuda.synchronize()
    assert _same_bits([t.clone() for t in outs], _step(CAPTURED, large))


def test_eager_call_between_capture_and_replay(cuda_device):
    """Capture a small grid, run a larger one eagerly, replay: the graph keeps its own workspace."""
    import torch
    small, large = _inputs(SMALL, cuda_device), _inputs(LARGEST, cuda_device)
    want = _step(SMALL, small)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph, outs = _capture(SMALL, small, side)
    big = _step(LARGEST, large)
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert _same_bits([t.clone() for t in outs], want)
    assert _same_bits(_step(LARGEST, large), big)


def test_two_streams_without_a_wait(cuda_device):
    """Forwards issued on two streams with nothing ordering them: each equals its eager bits."""
    import torch
    cases = [SMALL, LARGE, LARGE, SMALL]
    inputs = {c.name: _inputs(c, cuda_device) for c in (SMALL, LARGE)}
    want = {c.name: _step(c, inputs[c.name])[:2] for c in (SMALL, LARGE)}
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for s in streams:
        s.wait_stream(torch.cuda.current_stream())
    got = []
    with torch.no_grad():
        for rep in range(3):
            for i, c in enumerate(cases):
                pt, _, mask, labels = inputs[c.name]
                with torch.cuda.stream(streams[i % 2]):
                    crit = _criterion(c)
                    got.append((c.name, crit(pt, (mask, labels)), crit.last_stack_losses))
    for s in streams:
        torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    for name, loss, sums in got:
        assert _same_bits([loss, sums], want[name]), name
