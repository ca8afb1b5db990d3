"""CPU: the numpy port of the training-sample stage (tests/targets_port.py) against the reference's goldens and cv2."""
import os

import numpy as np
import pytest

import targets_port as tp

CASES = tp.golden_paths()


def _ulp(a, b):
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


def _avx512_dispatch() -> bool:
    feats = getattr(np._core._multiarray_umath, "__cpu_features__", {})
    return bool(feats.get("AVX512_SKX"))


def test_goldens_exist_and_cover_the_cases():
    names = {os.path.basename(p)[:-4] for p in CASES}
    assert {"p0_unrandom", "p1_rot_scale", "p5_flip", "p15_random", "p100_crowd", "p5_far_coincident", "src_1x1",
            "masks_255_0", "masks_0_255", "d512_p5", "d512_p15_flip"} <= names


@pytest.mark.parametrize("path", CASES, ids=lambda p: os.path.basename(p)[:-4])
def test_port_rounded_exp_within_the_contract(path):
    """exp="rounded" (the kernel's arithmetic): image, masks and channel 48 bit-exact; body parts within 1 ULP (numpy's
    float32 ``** 2`` of the limb length); keypoints and channel 49 within 5 ULP with the same zero pattern."""
    z = tp.load_case(path)
    im, mm, ma, lab = tp.port_case(z, "rounded")
    assert np.array_equal(im, z["image"]) and np.array_equal(mm, z["mask_miss"]) and np.array_equal(ma, z["mask_all"])
    ref = z["labels"]
    assert np.array_equal(lab[48], ref[48])
    assert _ulp(lab[:30], ref[:30]).max() <= 1
    for c in list(range(30, 48)) + [49]:
        assert np.array_equal(lab[c] == 0, ref[c] == 0), c
        assert _ulp(lab[c], ref[c]).max() <= 5, c


@pytest.mark.parametrize("path", CASES, ids=lambda p: os.path.basename(p)[:-4])
def test_port_numpy_exp_is_bit_exact(path):
    if not _avx512_dispatch():
        pytest.skip("the goldens were made where numpy dispatches float32 exp to AVX512_SKX; this host does not, and "
                    "numpy's float32 exp differs between its dispatch paths")
    z = tp.load_case(path)
    im, mm, ma, lab = tp.port_case(z, "numpy")
    assert np.array_equal(lab, z["labels"])


SIZES = [(480, 640), (640, 427), (1, 1), (37, 53)]


@pytest.mark.parametrize("hw", SIZES)
@pytest.mark.parametrize("kind", ["random", "binary"])
def test_uint8_warp_and_area_resize_match_cv2(hw, kind):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(hash((hw, kind)) % 2**32)
    h, w = hw
    for t in range(4):
        if kind == "random":
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            m = rng.integers(0, 256, (h, w), dtype=np.uint8)
        else:
            img = (rng.integers(0, 2, (h, w, 3)) * 255).astype(np.uint8)
            m = (rng.integers(0, 2, (h, w)) * 255).astype(np.uint8)
        ang, sc = rng.uniform(-40, 40), rng.uniform(0.3, 2.5)
        A, B = np.cos(np.deg2rad(ang)) * sc, np.sin(np.deg2rad(ang)) * sc
        f = -1.0 if t % 2 else 1.0
        M = np.array([[f * A, f * B, rng.uniform(-300, 400)], [-B, A, rng.uniform(-300, 400)]])
        got = tp.warp_affine_u8(img, M, (256, 256), (124, 127, 127))
        want = cv2.warpAffine(img, M, (256, 256), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT,
                              borderValue=(124, 127, 127))
        assert np.array_equal(got, want)
        for border in (0, 255):
            wm = tp.warp_affine_u8(m, M, (256, 256), border)
            assert np.array_equal(wm, cv2.warpAffine(m, M, (256, 256), flags=cv2.INTER_LINEAR,
                                                     borderMode=cv2.BORDER_CONSTANT, borderValue=border))
            assert np.array_equal(tp.resize_area_int(wm, 4), cv2.resize(wm, (64, 64), interpolation=cv2.INTER_AREA))


def test_erode_matches_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(5)
    for shape in ((64, 64), (1, 1), (2, 7), (128, 128)):
        m = rng.integers(0, 256, shape).astype(np.float32) / 255.
        assert np.array_equal(tp.erode3(m), cv2.erode(m, np.ones((3, 3), np.uint8)))
