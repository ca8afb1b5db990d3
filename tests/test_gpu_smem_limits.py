"""GPU: every launch plan that sizes shared memory by the shape or the capacities, at the device's per-block limit.

A block's dynamic shared memory plus its kernel's static ``__shared__`` arrays must fit the opt-in limit; a plan that
checks the dynamic part alone admits a band of shapes just under the limit that can never launch.  These tests step
plane sizes, widths and capacities through that band for each such plan: the limb scorer's plane ring and staged plane,
the keypoint NMS's bands, the fused matcher-assembler and the training loss.  Every call either runs and equals its
reference bit for bit (float tolerance 0), or fails with the library's own shared-memory error before any launch --
never a CUDA error -- and the handle stays usable for the next call.

The shapes are where the H100's opt-in limit (232 448 B) falls for the sizes in csrc/; the sweeps themselves only
assume that plans change monotonically with the plane size, so they stay meaningful if those sizes move.
"""
import os

import numpy as np
import pytest

from test_gpu_loss import _check_case, _criterion, _opt, _preds
from test_gpu_parity import _assert_same

pytestmark = pytest.mark.gpu

PERSONS = 4


@pytest.fixture(scope="module")
def env(cuda_device):
    import torch
    from improved_body_parts_b200 import grouping, skeleton, synth
    from oracle import spg_oracle as so

    class Env:
        pass

    e = Env()
    e.torch, e.grouping, e.skeleton, e.synth, e.so, e.dev = torch, grouping, skeleton, synth, so, cuda_device
    e.params = skeleton.default_params()
    # the normal call that shows a handle is still usable after a call near (or past) a limit
    e.heat128, e.paf128 = synth.make_batch(128128, 2, 128, 128, 6)
    e.ref128 = so.group_batch(e.heat128, e.paf128, skeleton.LIMBS, 128, e.params)
    return e


def _smem_error(e) -> bool:
    """The library's own refusal: SPG_E_INVALID (-1) naming shared memory."""
    return "failed (-1)" in str(e) and "shared memory" in str(e)


def _batch(env, seed, n, H, W, f64):
    heat, paf = env.synth.make_batch(seed, n, H, W, PERSONS, edge=True)
    if f64 == "f64":
        paf = paf.astype(np.float64) * (1.0 + 2.0 ** -29) + 2.0 ** -41
    ref = env.so.group_batch(heat, paf.astype(np.float64) if f64 == "f32_as_f64" else paf, env.skeleton.LIMBS, H, env.params)
    assert (ref.status == 0).all(), ref.status
    return heat, paf, ref


def _grouper(env, n, H, W, **cfg):
    return env.grouping.Grouper(max_batch=max(n, 2), max_h=max(H, 128), max_w=max(W, 128), **cfg)


def _assert_matches(ref, r, n, what):
    assert (r.status[:n] == 0).all(), f"{what}: status {r.status[:n]}"
    for i in range(n):
        _assert_same(ref.as_reference_structures(i), r.as_reference_structures(i), f"{what} image {i}")


def _still_usable(env, g):
    t = env.torch
    g.group_device(t.from_numpy(env.heat128).to(env.dev), t.from_numpy(env.paf128).to(env.dev), 128, env.params)
    _assert_matches(env.ref128, g.fetch(2), 2, "the next call on the same handle")


# ---- limb scoring: persistent plane ring -> staged plane -> sampled through L2 ------------------------------------------
RANK = {"persistent": 0, "staged": 1, "sampled": 2}


def _score_plan(name: str) -> str:
    if "persist" in name:
        return "persistent"
    return "staged" if ",true" in name else "sampled"


# (paf dtype, max_peaks_per_part, shapes).  Each sweep crosses the last bytes under one plan's limit: the persistent
# scorer's three-plane ring (float32 planes of 66 448 .. 66 560 B at any capP <= 64: 128x130, 104x160, 80x208) and the
# staged scorer's one plane with its capP-sized tables (float32 146x384, 226x248, 196x286 at capP 64; 184x308 at 32;
# 176x310 at 128; float64 146x192).  146x383 and 146x385 are the unaligned neighbours, sampled whatever their size.
SCORE_SWEEPS = {
    "ring_f32_H128": ("f32", 64, [(128, w) for w in range(120, 137)]),
    "ring_f32_same_plane": ("f32", 64, [(128, 128), (128, 129), (104, 160), (80, 208), (130, 128), (128, 131)]),
    "ring_f32_as_f64": ("f32_as_f64", 64, [(128, 128), (128, 129), (128, 130), (128, 131)]),
    "staged_f32_cap64": ("f32", 64, [(145, 384), (226, 248), (196, 286), (146, 383), (146, 384), (146, 385), (147, 384)]),
    "staged_f32_cap32": ("f32", 32, [(184, 300), (184, 304), (184, 308), (184, 312)]),
    "staged_f32_cap128": ("f32", 128, [(176, 302), (176, 306), (176, 310), (176, 314)]),
    "staged_f64": ("f64", 64, [(64, 128), (64, 130), (145, 192), (146, 192), (147, 192)]),
}


def _maps_on_device(env, heat, paf):
    return env.torch.from_numpy(heat).to(env.dev), env.torch.from_numpy(paf).to(env.dev)


@pytest.mark.parametrize("sweep", list(SCORE_SWEEPS))
def test_limb_score_plans_across_their_limits(env, sweep):
    dtype, capP, shapes = SCORE_SWEEPS[sweep]
    esz = 8 if dtype == "f64" else 4
    n = 3
    plans = []
    for j, (H, W) in enumerate(shapes):
        heat, paf, ref = _batch(env, 9100 + 37 * j, n, H, W, dtype)
        with _grouper(env, n, H, W, max_peaks_per_part=capP) as g:
            hd, pd = _maps_on_device(env, heat, paf)
            g.group_device(hd, pd, H, env.params, paf_as_f64=dtype == "f32_as_f64")
            r = g.fetch(n)
            plan = _score_plan(g.stage_kernels()[1])
            _assert_matches(ref, r, n, f"{H}x{W} {dtype} capP {capP} ({g.stage_kernels()[1]})")
            _still_usable(env, g)
        if (H * W * esz) % 16:
            assert plan == "sampled", f"{H}x{W}: an unaligned plane is sampled, not {plan}"
        else:
            plans.append((H * W, plan, (H, W)))
    # along growing planes the scorer only ever moves to a plan that needs less shared memory
    plans.sort(key=lambda p: p[0])
    ranks = [RANK[p[1]] for p in plans]
    assert ranks == sorted(ranks), [(s, p) for _, p, s in plans]
    assert len(set(ranks)) == 2, f"the sweep should cross one plan limit: {[(s, p) for _, p, s in plans]}"


@pytest.mark.parametrize("sweep", list(SCORE_SWEEPS))
def test_limb_score_plans_in_ragged_calls(env, sweep):
    """The same shapes through spg_group_ragged, each in one call with a 128x128 image: the ragged staged launch takes
    the largest shared memory any of its images needs."""
    dtype, capP, shapes = SCORE_SWEEPS[sweep]
    t = env.torch
    h0, p0, ref0 = _batch(env, 5150, 1, 128, 128, dtype)
    for j, (H, W) in enumerate(shapes):
        heat, paf, ref = _batch(env, 9100 + 37 * j, 1, H, W, dtype)
        maps = [(t.from_numpy(h0[0]).to(env.dev), t.from_numpy(p0[0]).to(env.dev)),
                (t.from_numpy(heat[0]).to(env.dev), t.from_numpy(paf[0]).to(env.dev))]
        with _grouper(env, 2, H, W, max_peaks_per_part=capP) as g:
            g.group_ragged(maps, [128.0, float(H)], env.params, paf_as_f64=dtype == "f32_as_f64")
            r = g.fetch(2)
            what = f"ragged {H}x{W} {dtype} capP {capP}"
            assert (r.status[:2] == 0).all(), f"{what}: status {r.status[:2]}"
            _assert_same(ref0.as_reference_structures(0), r.as_reference_structures(0), f"{what}: the 128x128 image")
            _assert_same(ref.as_reference_structures(0), r.as_reference_structures(1), f"{what}: the {H}x{W} image")
            _still_usable(env, g)


# ---- keypoint NMS: the band kernel's three band buffers at widths where they reach the limit ---------------------------
# At capP 96 the three bands of an image of 32 rows need exactly the opt-in limit, 232 448 B, at widths 3 126 .. 3 128,
# and more from 3 129 on.  Whole-batch calls plan the band kernel for widths that are not multiples of 4 (the persistent
# and banded forms need 16-byte rows); ragged calls plan it for every image.
NMS_WIDTHS = list(range(3118, 3139))


@pytest.mark.parametrize("ragged", [False, True], ids=["batch", "ragged"])
def test_nms_band_plan_across_its_limit(env, ragged):
    H, capP, n = 32, 96, 2
    t = env.torch
    outcomes = []
    for W in NMS_WIDTHS:
        heat, paf, ref = _batch(env, 3100 + W, n, H, W, "f32")
        with _grouper(env, n, H, W, max_peaks_per_part=capP) as g:
            try:
                if ragged:
                    maps = [(t.from_numpy(heat[i]).to(env.dev), t.from_numpy(paf[i]).to(env.dev)) for i in range(n)]
                    g.group_ragged(maps, [float(H)] * n, env.params)
                else:
                    g.group_device(*_maps_on_device(env, heat, paf), H, env.params)
                _assert_matches(ref, g.fetch(n), n, f"{H}x{W} ({g.stage_kernels()[0]})")
                outcomes.append((W, "ran"))
            except env.grouping.GroupingError as e:
                assert _smem_error(e), f"{H}x{W}: {e}"
                outcomes.append((W, "refused"))
            _still_usable(env, g)
    # the widths the band kernel plans (whole-batch calls give 16-byte rows to the persistent and banded forms): once one
    # is refused every wider one is, and the sweep crosses that limit
    ran = [o == "ran" for W, o in outcomes if ragged or W % 4]
    assert ran == sorted(ran, reverse=True) and ran[0] and not ran[-1], outcomes


# ---- the fused matcher-assembler: its matcher scratch grows with the warps, its person table with capR -----------------
# With 15 matcher warps (SPG_MA_WARPS is clamped to 15) and capP 128, the fused kernel needs 231 824 / 232 144 / 232 512 B
# dynamic at capR 47 / 48 / 49; past its room the call runs the matcher and the assembler back to back.
def test_match_assemble_plan_across_its_limit(env):
    t = env.torch
    heat, paf, ref = _batch(env, 4747, 4, 128, 128, "f32")
    hd, pd = _maps_on_device(env, heat, paf)
    fused = []
    for capR in (46, 47, 48, 49, 50):
        os.environ["SPG_MA_WARPS"] = "15"
        try:
            g = _grouper(env, 4, 128, 128, max_peaks_per_part=128, max_person_rows=capR)
        finally:
            os.environ.pop("SPG_MA_WARPS", None)
        with g:
            g.group_device(hd, pd, 128, env.params)
            r = g.fetch(4)
            names = g.stage_kernels()
            assert names[2:] in (("match_assemble_kernel", ""), ("limb_match_kernel", "assemble_kernel")), names
            _assert_matches(ref, r, 4, f"capR {capR} ({names[2]})")
            fused.append(names[2] == "match_assemble_kernel")
            _still_usable(env, g)
    assert fused == sorted(fused, reverse=True), f"fused per capR 46..50: {fused}"
    assert fused[0] and not fused[-1], f"the sweep should cross the fused kernel's limit: {fused}"


# ---- the training loss: one CTA stages a band of 16 rows of both pyramids, so its shared memory grows with the width -----
def _loss_case(env, W, focal):
    """One sample of one band of 16 rows: k/255 masks (every bilinear tie at 0.5 included) and half-zero labels."""
    from types import SimpleNamespace
    torch, dev = env.torch, env.dev
    C = 2 if focal else 1
    rng = np.random.default_rng(W)
    labels = rng.random((1, C, 16, W), dtype=np.float32)
    labels[rng.random(labels.shape) < 0.5] = 0
    mask = rng.integers(0, 256, (1, 1, 16, W)).astype(np.float32) / np.float32(255)
    mask, labels = torch.from_numpy(mask).to(dev), torch.from_numpy(labels).to(dev)
    opt = _opt(1, 1)
    cfg = SimpleNamespace(heat_start=0, bkg_start=1, offset_start=C)
    pt, leaves = _preds(1, C, 16, W, 1, W + 1, dev, labels)
    return pt, leaves, mask, labels, opt, cfg


def _loss_backward_alone(env, pt, mask, labels, opt, cfg, focal):
    """spg_loss_backward without a forward first (the autograd path would stop at the forward's refusal)."""
    from improved_body_parts_b200 import grouping, loss, targets
    torch = env.torch
    preds = [p for stack in pt for p in stack]
    grads = [torch.empty_like(p) for p in preds]
    go = torch.ones((), device=env.dev)
    params = _criterion(opt, focal, cfg)._params(tuple(labels.shape))
    targets._Device.for_device(env.dev.index).loss_backward(params, mask.data_ptr(), labels.data_ptr(),
                                                            loss._records(preds, grads), grouping.F32, go.data_ptr())
    torch.cuda.synchronize()


@pytest.mark.parametrize("focal", [True, False], ids=["focal", "l2"])
def test_loss_across_its_width_limit(env, focal):
    """W = 304 is the first width past the 48 KB default (the opt-in is in use), 1 344 fits, 1 376 needs more than the
    opt-in limit itself, and 1 360's 231 904 B fit the limit but not beside the forward kernel's static memory."""
    refused = {}
    for W in (304, 1344, 1360, 1376):
        pt, leaves, mask, labels, opt, cfg = _loss_case(env, W, focal)
        try:
            _check_case(env.dev, pt, leaves, mask, labels, opt, focal, 1.0, exact_sums=True, cfg=cfg)
            fwd = False
        except env.grouping.GroupingError as e:
            assert _smem_error(e), f"W {W} forward: {e}"
            fwd = True
        try:
            _loss_backward_alone(env, pt, mask, labels, opt, cfg, focal)
            bwd = False
        except env.grouping.GroupingError as e:
            assert _smem_error(e), f"W {W} backward: {e}"
            bwd = True
        assert fwd == bwd, f"W {W}: forward {'refused' if fwd else 'ran'}, backward {'refused' if bwd else 'ran'}"
        refused[W] = fwd
        # the per-device handle the loss uses takes the next call
        pt, leaves, mask, labels, opt, cfg = _loss_case(env, 64, focal)
        _check_case(env.dev, pt, leaves, mask, labels, opt, focal, 1.0, exact_sums=True, cfg=cfg)
    assert not refused[304] and not refused[1344] and refused[1376], refused
