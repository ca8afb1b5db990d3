"""GPU: the post-network stage on network outputs holding NaN, +inf and -inf, against its CPU checker.

evaluate.py does not scrub its maps; demo_image.py zeroes NaN in the averaged maps (nan_scrub) and keeps the infinities.
Every kernel family -- the x4 identity, the four-phase, the generic-stride and the rotated kernel, and their ragged
forms -- on such outputs in float32 and float16, with nan_scrub off and on, against oracle/postnet_port.py and
oracle/postnet_rotation_port.py (which tests/test_postnet_port.py and tests/test_postnet_rotation_port.py pin to cv2 on
non-finite inputs): finite values bit-identical, NaN at the same positions, infinities equal.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env(cuda_device):
    import torch
    from improved_body_parts_b200 import skeleton, synth
    from improved_body_parts_b200.grouping import Grouper
    from oracle import postnet_port as pp
    from oracle import postnet_rotation_port as pr

    class Env:
        pass

    e = Env()
    e.torch, e.skeleton, e.synth, e.Grouper, e.pp, e.pr, e.dev = torch, skeleton, synth, Grouper, pp, pr, cuda_device
    return e


def _dirty_output(env, seed, n, h, w):
    """[n, 2, 50, h, w] float32 network output with NaN / +inf / -inf in body-part and keypoint channels of both halves."""
    from test_gpu_postnet import _network_like_output
    out = _network_like_output(env, seed, n, h, w, 3)
    rng = np.random.default_rng(seed)
    vals = np.array([np.nan, np.inf, -np.inf], np.float32)
    for i in range(n):
        for half in (0, 1):
            for c in list(rng.choice(30, 4, replace=False)) + list(30 + rng.choice(18, 4, replace=False)):
                y, x = int(rng.integers(h)), int(rng.integers(w))
                out[i, half, c, y, x] = vals[(c + y + half) % 3]
    return out


def _port(env, outs, crops, image_hw, stride, mats, nan_scrub):
    """The checker's maps (heat float32, paf float64): the items' maps through the ports, float64 sums over the items;
    nan_scrub zeroes NaN in the sums after every item (demo_image.py:176-180, inside the scale loop)."""
    sk = env.skeleton
    N = outs[0].shape[0]
    H, W = image_hw
    heat_avg, paf_avg = np.zeros((N, H, W, 18)), np.zeros((N, H, W, 30))
    for o, (ch, cw), M in zip(outs, crops, mats):
        h, w = o.shape[3:]
        padded = (stride * h, stride * w)
        pad = [0, 0, padded[0] - ch, padded[1] - cw]
        for i in range(N):
            args = (o[i].astype(np.float32), stride, padded, pad, (H, W), 30, 48, sk.FLIP_PAF_ORD, sk.FLIP_HEAT_ORD[:18])
            hm, pf = env.pr.post_network_item(*args, rotate_matrix=M) if stride == 4 else env.pp.post_network_scale(*args)
            heat_avg[i] = env.pp.accumulate(heat_avg[i], hm, len(outs))
            paf_avg[i] = env.pp.accumulate(paf_avg[i], pf, len(outs))
            if nan_scrub:
                heat_avg[i][np.isnan(heat_avg[i])] = 0
                paf_avg[i][np.isnan(paf_avg[i])] = 0
    return heat_avg.transpose(0, 3, 1, 2).astype(np.float32), paf_avg.transpose(0, 3, 1, 2)


def _same(got, want, what):
    """Finite values bit-identical, NaN at the same positions, infinities equal."""
    got, want = np.ascontiguousarray(got), np.ascontiguousarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape, what
    assert np.array_equal(np.isnan(got), np.isnan(want)), f"{what}: NaN positions differ"
    keep = ~np.isnan(want)
    assert np.array_equal(got[keep].view(np.uint8), want[keep].view(np.uint8)), f"{what}: values differ"


CASES = {
    # name: (network sizes per item, crops, image size, stride, angle per item, kernel)
    "ident": ([(32, 40)], [(128, 160)], (128, 160), 4, [0], "postnet_x4_ident_kernel"),
    "four_phase": ([(32, 48)], [(120, 180)], (96, 144), 4, [0], "postnet_kernel"),
    "three_scales": ([(16, 16), (32, 32), (64, 64)], [(64, 64), (128, 128), (250, 250)], (125, 125), 4, [0, 0, 0],
                     "postnet_kernel"),
    "generic_stride2": ([(40, 48)], [(76, 90)], (61, 77), 2, [0], "postnet_generic_kernel"),
    "rotated": ([(32, 32)], [(128, 128)], (128, 128), 4, [45], "postnet_rot_kernel"),
}


@pytest.mark.parametrize("nan_scrub", [False, True], ids=["no_scrub", "scrub"])
@pytest.mark.parametrize("net_dtype", ["f32", "f16"])
@pytest.mark.parametrize("name", list(CASES))
def test_nonfinite_network_outputs_through_each_kernel(env, name, net_dtype, nan_scrub):
    t = env.torch
    sizes, crops, image_hw, stride, angles, kernel = CASES[name]
    outs = [_dirty_output(env, 40 + 13 * k, 2, h, w) for k, (h, w) in enumerate(sizes)]
    if net_dtype == "f16":
        outs = [o.astype(np.float16) for o in outs]
    mats = [None if a == 0 else env.pr.rotation_matrices((4 * h, 4 * w), a)[1] for (h, w), a in zip(sizes, angles)]
    ref_heat, ref_paf = _port(env, outs, crops, image_hw, stride, mats, nan_scrub)
    g = env.Grouper(max_batch=2, max_h=image_hw[0], max_w=image_hw[1])
    try:
        heat, paf = g.postnet([t.from_numpy(o).to(env.dev) for o in outs], crops, image_hw, stride=stride,
                              paf_dtype=t.float64, nan_scrub=nan_scrub,
                              rotations=mats if any(m is not None for m in mats) else None)
        assert g.postnet_kernel() == kernel
        _same(heat.cpu().numpy(), ref_heat, f"{name}: keypoint maps")
        _same(paf.cpu().numpy(), ref_paf, f"{name}: body-part maps")
    finally:
        g.close()
    for m in (ref_heat, ref_paf):  # the maps really hold what the test is about
        assert np.isinf(m).any() and np.isfinite(m).any()
        assert np.isnan(m).any() != nan_scrub


RAGGED = {
    # name: (per image (network size, crop, image size), angle, kernel)
    "ident_ragged": ([((32, 40), (128, 160), (128, 160)), ((19, 23), (75, 90), (75, 90))], 0,
                     "postnet_x4_ident_ragged_kernel"),
    "four_phase_ragged": ([((32, 48), (120, 180), (96, 144)), ((16, 32), (60, 110), (100, 183))], 0,
                          "postnet_ragged_kernel"),
    "rotated_ragged": ([((32, 32), (128, 128), (128, 128)), ((24, 40), (96, 160), (96, 160))], 30,
                       "postnet_rot_ragged_kernel"),
}


@pytest.mark.parametrize("nan_scrub", [False, True], ids=["no_scrub", "scrub"])
@pytest.mark.parametrize("net_dtype", ["f32", "f16"])
@pytest.mark.parametrize("name", list(RAGGED))
def test_nonfinite_network_outputs_through_the_ragged_kernels(env, name, net_dtype, nan_scrub):
    t = env.torch
    images, angle, kernel = RAGGED[name]
    outs = [_dirty_output(env, 90 + 7 * i, 1, *hw) for i, (hw, _, _) in enumerate(images)]
    if net_dtype == "f16":
        outs = [o.astype(np.float16) for o in outs]
    mats = [None if angle == 0 else env.pr.rotation_matrices((4 * hw[0], 4 * hw[1]), angle)[1] for hw, _, _ in images]
    g = env.Grouper(max_batch=len(images), max_h=256, max_w=256)
    try:
        dev = [t.from_numpy(o[0]).to(env.dev) for o in outs]
        if angle == 0:
            got = g.postnet_ragged([(d, crop, ihw) for d, (_, crop, ihw) in zip(dev, images)], paf_dtype=t.float64,
                                   nan_scrub=nan_scrub)
        else:
            got = g.postnet_ragged_items([([(d, crop, m)], ihw) for d, (_, crop, ihw), m in zip(dev, images, mats)],
                                         paf_dtype=t.float64, nan_scrub=nan_scrub)
        assert g.postnet_kernel() == kernel
        for i, (hw, crop, ihw) in enumerate(images):
            ref_heat, ref_paf = _port(env, [outs[i]], [crop], ihw, 4, [mats[i]], nan_scrub)
            _same(got[i][0].cpu().numpy(), ref_heat, f"{name} image {i}: keypoint maps")
            _same(got[i][1].cpu().numpy(), ref_paf, f"{name} image {i}: body-part maps")
    finally:
        g.close()


def test_nonfinite_network_outputs_through_the_items_ragged_kernel(env):
    """Two scales per image: postnet_items_ragged_kernel, float64 sums over the items."""
    t = env.torch
    images = [([(16, 20), (24, 30)], [(64, 77), (96, 116)], (80, 96)), ([(12, 16), (20, 24)], [(45, 60), (78, 94)], (60, 75))]
    outs = [[_dirty_output(env, 300 + 11 * i + k, 1, *hw) for k, hw in enumerate(sizes)] for i, (sizes, _, _) in
            enumerate(images)]
    g = env.Grouper(max_batch=2, max_h=128, max_w=128)
    try:
        got = g.postnet_ragged_items([([(t.from_numpy(o[0]).to(env.dev), c, None) for o, c in zip(outs[i], crops)], ihw)
                                      for i, (_, crops, ihw) in enumerate(images)])
        assert g.postnet_kernel() == "postnet_items_ragged_kernel"
        for i, (_, crops, ihw) in enumerate(images):
            ref_heat, ref_paf = _port(env, outs[i], crops, ihw, 4, [None, None], False)
            _same(got[i][0].cpu().numpy(), ref_heat, f"image {i}: keypoint maps")
            _same(got[i][1].cpu().numpy(), ref_paf, f"image {i}: body-part maps")
    finally:
        g.close()


@pytest.mark.parametrize("variant", ["evaluate", "demo"])
@pytest.mark.parametrize("case", ["heat_nan", "heat_pinf", "heat_ninf", "paf_nan_inf"])
def test_predict_then_grouping_raises_where_the_checker_raises(env, variant, case):
    """dropin.predict with a stand-in network whose answer holds a non-finite value, then the drop-in grouping stages.
    The checker runs on the port's maps of the same answer (NaN zeroed for the demo variant, whose scrub keeps the
    infinities): where it stops with a non-finite end point find_connections raises GroupingError naming NONFINITE,
    elsewhere the structures are the checker's, bit for bit."""
    from parity import diff_structures

    from improved_body_parts_b200 import dropin
    from improved_body_parts_b200.grouping import GroupingError
    from oracle import spg_oracle as so
    from test_gpu_postnet import _network_like_output
    t, sk = env.torch, env.skeleton
    image = np.random.default_rng(3).integers(0, 255, size=(64, 64, 3), dtype=np.uint8)
    params = dict(sk.default_params(), scale_search=[1.0], rotation_search=[0.0])
    model_params = dict(boxsize=64, stride=4, max_downsample=64, padValue=128)
    answers = []

    def model(x):
        h, w = x.shape[1] // 4, x.shape[2] // 4
        out = _network_like_output(env, 61, 1, h, w, 3)[0]
        if case.startswith("heat_"):
            # every keypoint channel, so that every limb has both end-point lists non-empty
            out[0, 30:48, h // 2, w // 2] = {"heat_nan": np.nan, "heat_pinf": np.inf, "heat_ninf": -np.inf}[case]
        else:
            out[0, 5, h // 2, w // 3] = np.nan
            out[1, 7, h // 3, w // 2] = np.inf
            out[0, 9, h // 2, w // 2] = -np.inf
        answers.append((out, x.shape[1:3]))
        return [[t.from_numpy(out).to(x.device)]]

    dropin.configure(limbs=sk.LIMBS, variant=variant)
    try:
        heatmap, paf = dropin.predict(image, params, model, model_params, 20, 30, "synthetic")
        (out, padded), = answers
        pad = [0, 0, padded[0] - 64, padded[1] - 64]
        hm, pf = env.pr.post_network_item(out, 4, tuple(padded), pad, (64, 64), 30, 48, sk.FLIP_PAF_ORD,
                                          sk.FLIP_HEAT_ORD[:18], rotate_matrix=None)
        heat_avg, paf_avg = env.pp.accumulate(np.zeros((64, 64, 18)), hm, 1), env.pp.accumulate(np.zeros((64, 64, 30)), pf, 1)
        if variant == "demo":
            heat_avg[np.isnan(heat_avg)] = 0
            paf_avg[np.isnan(paf_avg)] = 0
        assert np.array_equal(heatmap.numpy(), heat_avg.astype(np.float32).astype(np.float64), equal_nan=True)
        assert np.array_equal(paf.numpy(), paf_avg, equal_nan=True)
        check_params = dict(params, crit1_strict=1, refresh_len_check=1, min_parts=4) if variant == "demo" else params
        o = so.group_batch(np.ascontiguousarray(heat_avg.transpose(2, 0, 1)[None]).astype(np.float32),
                           np.ascontiguousarray(paf_avg.transpose(2, 0, 1)[None]), sk.LIMBS, 64, check_params,
                           cap_peaks=8192)  # a NaN blob in every part: 18 x ~256 peaks
        all_peaks = dropin.find_peaks(heatmap, params)
        if o.status[0] == so.ERR_NONFINITE:
            with pytest.raises(GroupingError, match="NONFINITE"):
                dropin.find_connections(all_peaks, paf, 64, params)
            assert not (case == "heat_nan" and variant == "demo"), "the demo's scrub removes the NaN"
            assert case != "paf_nan_inf", "non-finite body-part samples never raise"
            return
        assert o.status[0] == 0
        conns, special = dropin.find_connections(all_peaks, paf, 64, params)
        subset, candidate = dropin.find_people(conns, special, all_peaks, params)
        d = diff_structures(o.as_reference_structures(0), (all_peaks, conns, special, subset, candidate), float_tol=0.0)
        assert not d, "\n".join(d)
    finally:
        dropin.configure(variant="evaluate")
    # reached only without a raise: an interior NaN keypoint raises unless the demo scrubs it
    assert not (case == "heat_nan" and variant == "evaluate")
