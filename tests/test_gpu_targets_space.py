"""GPU: spg_targets_warp / spg_targets_maps across what they admit through the C ABI (tests/targets_cases.py): every
case against the port bit for bit and its warp against cv2; the mask area resize against cv2 directly at every stride
1-64 and a few up to 512, on boxes holding the exact ties and the sums where cv2's float32 product is not the correctly
rounded quotient; and the largest stride whose box sums fit an int."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE)]

import targets_cases as tc  # noqa: E402
import targets_port as tp  # noqa: E402
from improved_body_parts_b200 import grouping, skeleton, targets  # noqa: E402

pytestmark = pytest.mark.gpu


def _grouper(limbs, K):
    return targets._Device.grouper(SimpleNamespace(limbs_conn=limbs, num_parts=K), 0)


def _params(stride, out_hw, gsize=0, sigma=9.0, paf_sigma=7.0, limb_thre=0.015, paf_thre=4.0, borders=tc.DEFAULT_BORDERS):
    p = np.zeros(1, grouping.TARGET_PARAMS)
    p["stride"], p["gaussian_size"], p["out_h"], p["out_w"] = stride, gsize, out_hw[0], out_hw[1]
    p["sigma"], p["paf_sigma"], p["limb_gaussian_thre"], p["paf_thre"] = sigma, paf_sigma, limb_thre, paf_thre
    p["border_image"], p["border_mask_miss"], p["border_mask_all"] = borders
    return p


def _pitched(dev, a, pad, rng):
    """``a`` ([h, w] or [h, w, 3] uint8) on the device in rows of ``row bytes + pad``, the padding filled with noise."""
    import torch
    h = a.shape[0]
    row = a[0].size
    buf = rng.integers(0, 256, (h, row + pad), dtype=np.uint8)
    buf[:, :row] = a.reshape(h, row)
    return torch.from_numpy(buf).to(dev), row + pad


def _warp(g, dev, params, samples, out_hw, stride, rng, pad=(0, 0)):
    """Images and both masks of ``samples`` (per sample ``(img, mask_miss, mask_all, M)``) from one spg_targets_warp
    call, with rows padded by ``pad`` bytes; also the source tensors, kept alive for spg_targets_maps."""
    import torch
    H, W = out_hw
    mh, mw = H // stride, W // stride
    rec = np.zeros(len(samples), grouping.TARGET_SAMPLE)
    keep, outs = [], []
    for i, (img, mm, ma, M) in enumerate(samples):
        (si, ps), (sm, pm), (sa, _) = _pitched(dev, img, pad[0], rng), _pitched(dev, mm, pad[1], rng), _pitched(dev, ma, pad[1], rng)
        o = (torch.full((H, W, 3), -1.0, device=dev), torch.full((mh, mw), -1.0, device=dev),
             torch.full((mh, mw), -1.0, device=dev))
        h, w = mm.shape
        rec[i] = (si.data_ptr(), sm.data_ptr(), sa.data_ptr(), ps, pm, h, w, np.asarray(M, np.float64).reshape(6),
                  o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr())
        keep.append((si, sm, sa))
        outs.append(o)
    g.targets_warp(params, rec)
    assert (g._lib.spg_stage_kernel(g._h, 6) or b"").decode() == "targets_warp_kernel"
    return outs, keep


def _same_bits_or_nan(a, b) -> bool:
    """Equal bit for bit, except that a NaN matches any NaN (numpy and CUDA give NaNs different sign and payload)."""
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a.view(np.int32)[~na], b.view(np.int32)[~nb])


def _cv2_sample(cv2, img, mm, ma, M, out_hw, stride, borders):
    H, W = out_hw
    t = tp.lut()
    wi = cv2.warpAffine(img, M, (W, H), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=borders[0])
    r = []
    for m, b in ((mm, borders[1]), (ma, borders[2])):
        wm = cv2.warpAffine(m, M, (W, H), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=b)
        r.append(t[cv2.resize(wm, (W // stride, H // stride), interpolation=cv2.INTER_AREA)])
    return t[wi], r[0], r[1]


@pytest.mark.parametrize("case", tc.CASES, ids=lambda c: c.name)
def test_case(cuda_device, case):
    """Both kernels against the port bit for bit (NaN against NaN) at the case's stride, output shape, parameters,
    borders, row pitches and limb table, with the joints of targets_cases.joints_of; the warp against cv2."""
    import torch
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(case.seed + 1000)
    g = _grouper(case.limbs, case.K)
    params = _params(case.stride, case.out_hw, case.gaussian_size, case.sigma, case.paf_sigma, case.limb_thre,
                     case.paf_thre, case.borders)
    data = tc.inputs(case)
    outs, keep = _warp(g, cuda_device, params, [d[:4] for d in data], case.out_hw, case.stride, rng, case.pad)
    L, K = len(case.limbs), case.K
    mh, mw = case.map_hw
    labels, joints = [], []
    rec = np.zeros(len(data), grouping.TARGET_JOINTS)
    for i, d in enumerate(data):
        j = torch.from_numpy(np.ascontiguousarray(d[4])).to(cuda_device)
        lab = torch.full((L + K + 2, mh, mw), -1.0, device=cuda_device)
        rec[i] = (j.data_ptr() if len(d[4]) else 0, len(d[4]), 0, outs[i][2].data_ptr(), lab.data_ptr())
        joints.append(j)
        labels.append(lab)
    g.targets_maps(params, rec)
    assert (g._lib.spg_stage_kernel(g._h, 6) or b"").decode() == "targets_maps_kernel"
    for i, (img, mm, ma, M, jn) in enumerate(data):
        im, km, ka = (t.cpu().numpy() for t in outs[i])
        pim, pmm, pma = tp.warp_sample(img, mm, ma, M, case.out_hw, case.stride, case.borders)
        assert np.array_equal(im, pim) and np.array_equal(km, pmm) and np.array_equal(ka, pma), i
        cim, cmm, cma = _cv2_sample(cv2, img, mm, ma, M, case.out_hw, case.stride, case.borders)
        assert np.array_equal(im, cim) and np.array_equal(km, cmm) and np.array_equal(ka, cma), i
        with np.errstate(all="ignore"):  # float32 overflow of the +-FLT_MAX limbs' lengths, as in the kernel
            plab = tp.label_maps(jn, pma, case.limbs, case.stride, case.sigma, case.paf_sigma, case.limb_thre,
                                 case.paf_thre, case.gaussian_size, exp="rounded")
        lab = labels[i].cpu().numpy()
        for c in range(L + K + 2):
            assert _same_bits_or_nan(lab[c], plab[c]), (i, c)
        # a joint with a non-finite coordinate draws no keypoint (its limbs are pinned by the port: empty for a NaN end)
        assert not np.isnan(lab[L:]).any()


FACTORS = list(range(1, 65)) + [165, 256, 331, 512]


@pytest.mark.parametrize("f", FACTORS)
def test_masks_against_cv2_at_every_stride(cuda_device, f):
    """Stride f in one call of two samples: identity warps of area_probe masks (exact ties and cv2's critical sums), so
    each map pixel is cv2.resize of one probe box; and a rotated, mirrored warp of random masks at a non-square output
    against cv2.warpAffine then cv2.resize."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(f)
    probe, sums = tc.area_probe(f, budget=1 << 20)
    other = 255 - probe[::-1]  # box sums 255 f^2 - s: the ties stay ties
    h, w = probe.shape
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    eye = np.array([[1.0, 0, 0], [0, 1.0, 0]])
    # the rotated sample shares the call's output shape: the probe's
    sh, sw = max(h // 3, 1), max(w // 2, 1)
    rimg = rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8)
    rm = [np.where(rng.random((sh, sw)) < 0.5, 0, 255).astype(np.uint8) for _ in range(2)]
    rm[1][rng.random((sh, sw)) < 0.2] = 77
    a = np.deg2rad(rng.uniform(-40, 40))
    s = 0.9 * max(h, w) / max(sh, sw)
    R = np.array([[-s * np.cos(a), -s * np.sin(a), 0.0], [-s * np.sin(a), s * np.cos(a), 0.0]])
    R[:, 2] = np.array([w / 2, h / 2]) - R[:, :2] @ np.array([sw / 2, sh / 2])
    borders = ((124, 127, 127), 255, 0)
    params = _params(f, (h, w), borders=borders)
    g = _grouper(skeleton.LIMBS, 18)
    outs, _ = _warp(g, cuda_device, params, [(img, probe, other, eye), (rimg, rm[0], rm[1], R)], (h, w), f, rng, (3, 1))
    t = tp.lut()
    im, km, ka = (o.cpu().numpy() for o in outs[0])
    assert np.array_equal(im, t[img])
    want = cv2.resize(probe, (w // f, h // f), interpolation=cv2.INTER_AREA)
    assert np.array_equal(km, t[want]) and np.array_equal(ka, t[cv2.resize(other, (w // f, h // f), interpolation=cv2.INTER_AREA)])
    if f == 2 or f in (22, 34, 44, 62, 165, 331):  # the probe holds sums a correctly rounded quotient gets wrong
        box = probe.reshape(h // f, f, w // f, f).astype(np.int64).sum(axis=(1, 3))
        assert (np.rint(box / (f * f)) != want).any()
    got = [o.cpu().numpy() for o in outs[1]]
    exp = _cv2_sample(cv2, rimg, rm[0], rm[1], R, (h, w), f, borders)
    for a_, b_ in zip(got, exp):
        assert np.array_equal(a_, b_)


def test_largest_stride_is_2901(cuda_device):
    """255 * 2901^2 fits an int and 255 * 2902^2 does not: 2901 is admitted (one 1 x 1 map through spg_targets_maps; no
    warp is run at that stride: 8.4 M taps per thread), 2902 is refused by both calls, naming the stride, before any
    launch.  Every buffer fits its 1 x 1 map, so that a library admitting 2902 fails the test and nothing else."""
    import torch
    g = _grouper(skeleton.LIMBS, 18)
    mask = torch.ones((1, 1), device=cuda_device)
    lab = torch.full((50, 1, 1), -1.0, device=cuda_device)
    ws = np.zeros(0, grouping.TARGET_SAMPLE)
    wj = np.zeros(1, grouping.TARGET_JOINTS)
    wj[0] = (0, 0, 0, mask.data_ptr(), lab.data_ptr())
    ok = _params(2901, (2901, 2901))
    before = g.launch_count
    g.targets_warp(ok, ws)
    g.targets_maps(ok, wj)
    torch.cuda.synchronize()
    assert g.launch_count == before + 1
    assert lab[48].item() == 1.0 and (lab[:48] == 0).all() and lab[49].item() == 0
    bad = _params(2902, (2902, 2902))
    before = g.launch_count
    with pytest.raises(grouping.GroupingError, match="stride 2902"):
        g.targets_warp(bad, ws)  # no sample: a library that admitted the stride would launch nothing
    with pytest.raises(grouping.GroupingError, match="stride 2902"):
        g.targets_maps(bad, wj)
    assert g.launch_count == before
