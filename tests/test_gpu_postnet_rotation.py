"""GPU: the rotation search of the post-network stage (spg_postnet_rotated, postnet_rot_kernel -- evaluate.py:107-158 with
angle != 0) against its CPU checker oracle/postnet_rotation_port.py, which tests/test_postnet_rotation_port.py pins to cv2.

The warp is OpenCV's fixed-point algorithm and the resizes the port's float32 operations, so the bar is BIT-IDENTICAL maps."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env(cuda_device):
    import torch
    from improved_body_parts_b200 import grouping, skeleton, synth
    from oracle import postnet_port as pp
    from oracle import postnet_rotation_port as pr
    from oracle import spg_oracle as so

    class Env:
        pass

    e = Env()
    e.torch, e.grouping, e.skeleton, e.synth, e.pp, e.pr, e.so, e.dev = torch, grouping, skeleton, synth, pp, pr, so, cuda_device
    e.Grouper = grouping.Grouper
    return e


def _net(env, seed, n, h, w, persons=4):
    from test_gpu_postnet import _network_like_output
    return _network_like_output(env, seed, n, h, w, persons)


def _reverse(env, hw, angle):
    """rotate_matrix_reverse of an item whose network output is h x w (padded input 4h x 4w), None for angle 0."""
    return None if angle == 0 else env.pr.rotation_matrices((4 * hw[0], 4 * hw[1]), angle)[1]


def _port_maps(env, outs, crops, image_hw, mats):
    """The checker: every item through postnet_rotation_port, float64 sums over the items (:160-161)."""
    sk = env.skeleton
    N = outs[0].shape[0]
    H, W = image_hw
    heat_avg, paf_avg = np.zeros((N, H, W, 18)), np.zeros((N, H, W, 30))
    for o, (ch, cw), M in zip(outs, crops, mats):
        h, w = o.shape[3:]
        padded = (4 * h, 4 * w)
        pad = [0, 0, padded[0] - ch, padded[1] - cw]
        for i in range(N):
            hm, pf = env.pr.post_network_item(o[i].astype(np.float32), 4, padded, pad, (H, W), 30, 48, sk.FLIP_PAF_ORD,
                                              sk.FLIP_HEAT_ORD[:18], rotate_matrix=M)
            heat_avg[i] = env.pp.accumulate(heat_avg[i], hm, len(outs))
            paf_avg[i] = env.pp.accumulate(paf_avg[i], pf, len(outs))
    return heat_avg.transpose(0, 3, 1, 2), paf_avg.transpose(0, 3, 1, 2)


def _same(a, b):
    """Bit-identical, except that a NaN equals any NaN (the device's and the host's NaN payloads differ)."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.dtype != b.dtype or a.shape != b.shape or not np.array_equal(np.isnan(a), np.isnan(b)):
        return False
    keep = ~np.isnan(a)
    return np.array_equal(a[keep].view(np.uint8), b[keep].view(np.uint8))


CASES = {
    # name: (network sizes per item, crops per item, image size, angle per item)
    "a45_square": ([(32, 32)], [(128, 128)], (128, 128), [45]),
    "a90_non_square": ([(24, 40)], [(96, 160)], (96, 160), [90]),           # centre quirk: (rows / 2, cols / 2)
    "a180_640_style_crop": ([(32, 48)], [(120, 180)], (96, 144), [180]),    # crop smaller than the padded grid, image smaller
    "a0.5_odd_sizes": ([(19, 23)], [(70, 89)], (131, 167), [0.5]),         # not multiples of 4, image larger than the crop
    "am30_tall": ([(40, 18)], [(157, 70)], (120, 53), [-30]),
    "scales2_angles3": ([(16, 20)] * 3 + [(24, 30)] * 3, [(64, 77)] * 3 + [(96, 116)] * 3, (80, 96), [0, 30, -30] * 2),
}


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("net_dtype", ["f32", "f16"])
def test_rotated_maps_are_the_checkers_maps(env, name, net_dtype):
    t = env.torch
    sizes, crops, image_hw, angles = CASES[name]
    if net_dtype == "f16" and name not in ("a45_square", "scales2_angles3"):
        pytest.skip("f16 input is covered on two geometries")
    N = 2
    outs = [_net(env, 700 + 11 * k, N, h, w) for k, (h, w) in enumerate(sizes)]
    if net_dtype == "f16":
        outs = [o.astype(np.float16) for o in outs]
    mats = [_reverse(env, hw, a) for hw, a in zip(sizes, angles)]
    ref_heat, ref_paf = _port_maps(env, outs, crops, image_hw, mats)
    g = env.Grouper(max_batch=N, max_h=image_hw[0], max_w=image_hw[1])
    try:
        dev_outs = [t.from_numpy(o).to(env.dev) for o in outs]
        heat, paf = g.postnet(dev_outs, crops, image_hw, paf_dtype=t.float64, rotations=mats)
        last = g.postnet_kernel()
        assert _same(heat.cpu().numpy(), ref_heat.astype(np.float32)), "keypoint maps differ from the checker"
        assert _same(paf.cpu().numpy(), ref_paf), "body-part maps differ from the checker"
        if len(sizes) == 1:  # a single rotated item: float32 planes hold the same values
            heat2, paf2 = g.postnet(dev_outs, crops, image_hw, rotations=mats)
            assert paf2.dtype == t.float32 and _same(paf2.cpu().numpy().astype(np.float64), ref_paf)
            assert _same(heat2.cpu().numpy(), heat.cpu().numpy())
    finally:
        g.close()
    assert last == ("postnet_rot_kernel" if mats[-1] is not None else "postnet_kernel")
    assert np.abs(ref_heat).max() > 0.3 and np.abs(ref_paf).max() > 0.3


def test_strided_network_output_with_three_images(env):
    t = env.torch
    sizes, crops, image_hw = [(24, 28)], [(90, 100)], (90, 100)
    out = _net(env, 77, 3, 24, 28)
    mats = [_reverse(env, sizes[0], 13)]
    big = t.zeros((3, 2, 64, 24, 28), device=env.dev)
    big[:, :, 7:57] = t.from_numpy(out).to(env.dev)
    ref_heat, ref_paf = _port_maps(env, [out], crops, image_hw, mats)
    g = env.Grouper(max_batch=3, max_h=90, max_w=100)
    try:
        heat, paf = g.postnet([big[:, :, 7:57]], crops, image_hw, paf_dtype=t.float64, rotations=mats)
        assert _same(heat.cpu().numpy(), ref_heat.astype(np.float32)) and _same(paf.cpu().numpy(), ref_paf)
    finally:
        g.close()


def test_nan_scrub_after_the_warp(env):
    """NaN in the network output spreads through the resize and the warp (0 * NaN); nan_scrub zeroes what the sums hold."""
    t = env.torch
    sizes, crops, image_hw = [(16, 16), (16, 16)], [(60, 62), (60, 62)], (75, 70)
    outs = [_net(env, 78 + k, 1, 16, 16, 2) for k in range(2)]
    outs[0][0, 0, 3, 5, 5] = np.nan
    outs[1][0, 1, 35, 2, 9] = np.nan
    mats = [_reverse(env, s, a) for s, a in zip(sizes, (30, 0))]
    ref_heat, ref_paf = _port_maps(env, outs, crops, image_hw, mats)
    g = env.Grouper(max_batch=1, max_h=image_hw[0], max_w=image_hw[1])
    try:
        d = [t.from_numpy(o).to(env.dev) for o in outs]
        h0, p0 = g.postnet(d, crops, image_hw, rotations=mats)
        h1, p1 = g.postnet(d, crops, image_hw, rotations=mats, nan_scrub=True)
    finally:
        g.close()
    assert _same(h0.cpu().numpy(), ref_heat.astype(np.float32)) and _same(p0.cpu().numpy(), ref_paf)
    assert t.isnan(h0).any() and t.isnan(p0).any() and not t.isnan(h1).any() and not t.isnan(p1).any()
    keep = ~t.isnan(p0)  # where an item was NaN, the scrubbed sum holds the other item's part
    assert t.equal(p0[keep], p1[keep]) and t.equal(h0[~t.isnan(h0)], h1[~t.isnan(h0)])


class _PlainEntry:
    """Routes Grouper.postnet's call to spg_postnet (the entry point without a rotation array)."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, k):
        return getattr(self._lib, k)

    def spg_postnet_rotated(self, h, desc, rot, *rest):
        assert rot is None
        return self._lib.spg_postnet(h, desc, *rest)


@pytest.mark.parametrize("name", ["identity_odd", "padded_ratio_1.25", "three_scales"])
def test_no_rotated_item_is_spg_postnet(env, name):
    """rot = NULL and every apply = 0 run exactly what spg_postnet runs: same bytes, same kernel."""
    from test_gpu_postnet import CASES as PLAIN
    t = env.torch
    sizes, crops, image_hw = PLAIN[name]
    outs = [t.from_numpy(_net(env, 600 + k, 2, h, w)).to(env.dev) for k, (h, w) in enumerate(sizes)]
    g = env.Grouper(max_batch=2, max_h=image_hw[0], max_w=image_hw[1])
    got = []
    try:
        lib = g._lib
        g._lib = _PlainEntry(lib)
        try:
            got.append(g.postnet(outs, crops, image_hw) + (g.postnet_kernel(),))
        finally:
            g._lib = lib
        got.append(g.postnet(outs, crops, image_hw) + (g.postnet_kernel(),))
        got.append(g.postnet(outs, crops, image_hw, rotations=[None] * len(outs)) + (g.postnet_kernel(),))
    finally:
        g.close()
    (h0, p0, k0) = got[0]
    for h, p, k in got[1:]:
        assert k == k0 and _same(h.cpu().numpy(), h0.cpu().numpy()) and _same(p.cpu().numpy(), p0.cpu().numpy())


def test_rotated_maps_then_grouping_equal_the_checkers_pipeline(env):
    from test_gpu_parity import _assert_same
    t = env.torch
    n, h, w = 3, 32, 40
    from test_gpu_postnet import _network_like_output
    out = _network_like_output(env, 950, n, h, w, 6, noise=0.004)
    image_hw = (4 * h, 4 * w)
    mats = [_reverse(env, (h, w), 7.5)]
    ref_heat, ref_paf = _port_maps(env, [out], [image_hw], image_hw, mats)
    params = env.skeleton.default_params()
    o = env.so.group_batch(ref_heat.astype(np.float32), np.ascontiguousarray(ref_paf), env.skeleton.LIMBS, image_hw[0], params)
    g = env.Grouper(max_batch=n, max_h=image_hw[0], max_w=image_hw[1], max_peaks_per_part=128, max_person_rows=128)
    try:
        heat, paf = g.postnet([t.from_numpy(out).to(env.dev)], [image_hw], image_hw, rotations=mats)
        assert paf.dtype == t.float32
        g.group_device(heat, paf, image_hw[0], params, paf_as_f64=True)
        r = g.fetch()
    finally:
        g.close()
    assert (r.status == 0).all() and (o.status == 0).all() and r.n_persons.sum() >= n
    for i in range(n):
        _assert_same(o.as_reference_structures(i), r.as_reference_structures(i), f"image {i}")


def test_device_predict_with_scale_and_rotation_search(env):
    """dropin.predict over product(scale_search, rotation_search): the inputs it hands the network are cv2's rotated padded
    images and their mirrors, and the maps are the checker's accumulation of whatever the network answered per item."""
    import cv2
    from parity import diff_structures

    from improved_body_parts_b200 import dropin
    t, sk = env.torch, env.skeleton
    rng = np.random.default_rng(5)
    image = rng.integers(0, 255, size=(150, 210, 3), dtype=np.uint8)
    params = dict(sk.default_params(), scale_search=[1.0, 0.75], rotation_search=[0.0, 30.0, -30.0])
    model_params = dict(boxsize=160, stride=4, max_downsample=64, padValue=128)
    seen, answers, items = [], [], []
    for scale in (x * 160 / 150 for x in params["scale_search"]):
        resized = cv2.resize(image, (0, 0), fx=scale, fy=scale, interpolation=cv2.INTER_CUBIC)
        padded, pad = dropin.pad_right_down_corner(resized, 64, 128)
        for angle in params["rotation_search"]:
            items.append((resized.shape[:2], padded, pad, angle))

    def model(x):
        seen.append(x.cpu().numpy())
        h, w = x.shape[1] // 4, x.shape[2] // 4
        answers.append(_net(env, 1000 + len(answers), 1, h, w, 5)[0])
        return [[t.from_numpy(answers[-1]).to(x.device)]]

    dropin.configure(limbs=sk.LIMBS)
    heatmap, paf = dropin.predict(image, params, model, model_params, 20, 30, "synthetic")
    assert len(seen) == 6
    heat_avg, paf_avg = np.zeros((150, 210, 18)), np.zeros((150, 210, 30))
    for x, out, (crop, padded, pad, angle) in zip(seen, answers, items):
        inp = np.float32(padded / 255)
        M = None
        if angle != 0:
            rot, M = env.pr.rotation_matrices(inp.shape[:2], angle)
            inp = cv2.warpAffine(inp, rot, (0, 0))
        assert np.array_equal(x[0], inp) and np.array_equal(x[1], inp[:, ::-1, :])
        hm, pf = env.pr.post_network_item(out, 4, padded.shape[:2], pad, image.shape[:2], 30, 48, sk.FLIP_PAF_ORD,
                                          sk.FLIP_HEAT_ORD[:18], rotate_matrix=M)
        heat_avg, paf_avg = env.pp.accumulate(heat_avg, hm, 6), env.pp.accumulate(paf_avg, pf, 6)
    assert not paf.as_f64 and paf.tensor.dtype == t.float64
    assert np.array_equal(heatmap.numpy(), heat_avg.astype(np.float32).astype(np.float64)) and np.array_equal(paf.numpy(), paf_avg)
    all_peaks = dropin.find_peaks(heatmap, params)
    connection_all, special_k = dropin.find_connections(all_peaks, paf, image.shape[0], params)
    subset, candidate = dropin.find_people(connection_all, special_k, all_peaks, params)
    o = env.so.group_batch(np.ascontiguousarray(heat_avg.transpose(2, 0, 1)[None]).astype(np.float32),
                           np.ascontiguousarray(paf_avg.transpose(2, 0, 1)[None]), sk.LIMBS, image.shape[0], params)
    d = diff_structures(o.as_reference_structures(0), (all_peaks, connection_all, special_k, subset, candidate), float_tol=0.0)
    assert not d, "\n".join(d)


class _Tamper(_PlainEntry):
    """Sets apply = 2 in the rotation array Grouper.postnet passes."""

    def spg_postnet_rotated(self, h, desc, rot, *rest):
        rot[0].apply = 2
        return self._lib.spg_postnet_rotated(h, desc, rot, *rest)


def test_invalid_rotations_are_rejected(env):
    t = env.torch
    out = [t.from_numpy(_net(env, 5, 1, 16, 16)).to(env.dev)]
    M = _reverse(env, (16, 16), 30)
    g = env.Grouper(max_batch=1, max_h=64, max_w=64)
    try:
        bad = M.copy()
        bad[1, 2] = np.inf
        with pytest.raises(env.grouping.GroupingError, match=r"\(-1\).*not finite"):
            g.postnet(out, [(64, 64)], (64, 64), rotations=[bad])
        with pytest.raises(env.grouping.GroupingError, match=r"\(-1\).*stride 4"):
            g.postnet(out, [(32, 32)], (32, 32), stride=2, rotations=[M])
        lib = g._lib
        g._lib = _Tamper(lib)
        try:
            with pytest.raises(env.grouping.GroupingError, match=r"\(-1\).*apply must be 0 or 1"):
                g.postnet(out, [(64, 64)], (64, 64), rotations=[M])
        finally:
            g._lib = lib
        g.postnet(out, [(64, 64)], (64, 64), rotations=[M])  # the handle still works
    finally:
        g.close()
