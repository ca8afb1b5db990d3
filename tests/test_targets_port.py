"""CPU: the numpy port of the training-sample stage (tests/targets_port.py) against the reference's goldens and cv2."""
import os

import numpy as np
import pytest

import targets_cases as tc
import targets_port as tp

CASES = tp.golden_paths()
SPACE = tp.golden_paths("targets_space")


def _ulp(a, b):
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


def _avx512_dispatch() -> bool:
    feats = getattr(np._core._multiarray_umath, "__cpu_features__", {})
    return bool(feats.get("AVX512_SKX"))


def test_goldens_exist_and_cover_the_cases():
    names = {os.path.basename(p)[:-4] for p in CASES}
    assert {"p0_unrandom", "p1_rot_scale", "p5_flip", "p15_random", "p100_crowd", "p5_far_coincident", "src_1x1",
            "masks_255_0", "masks_0_255", "d512_p5", "d512_p15_flip"} <= names
    space = [tp.case_params(dict(np.load(p))) for p in SPACE]
    assert {c["stride"] for c in space} >= {1, 2, 3, 5, 6, 8}
    assert {len(c["limbs"]) for c in space} >= {5, 24, 30}
    assert len({c["gsize"] for c in space}) >= 5 and len({c["paf_thre"] for c in space}) >= 5
    assert {int(np.load(p)["size"]) for p in SPACE} >= {48, 64, 96, 128, 160, 255, 368}


@pytest.mark.parametrize("path", CASES + SPACE, ids=lambda p: os.path.basename(p)[:-4])
def test_port_rounded_exp_within_the_contract(path):
    """exp="rounded" (the kernel's arithmetic): image, masks and channel L+K bit-exact; body parts within 1 ULP (numpy's
    float32 ``** 2`` of the limb length); keypoints and channel L+K+1 within 5 ULP with the same zero pattern."""
    z = tp.load_case(path)
    im, mm, ma, lab = tp.port_case(z, "rounded")
    assert np.array_equal(im, z["image"]) and np.array_equal(mm, z["mask_miss"]) and np.array_equal(ma, z["mask_all"])
    ref = z["labels"]
    L = len(tp.case_params(z)["limbs"])
    assert lab.shape == ref.shape == (L + 20,) + mm.shape
    assert np.array_equal(lab[L + 18], ref[L + 18])
    assert _ulp(lab[:L], ref[:L]).max(initial=0) <= 1
    for c in list(range(L, L + 18)) + [L + 19]:
        assert np.array_equal(lab[c] == 0, ref[c] == 0), c
        assert _ulp(lab[c], ref[c]).max() <= 5, c


@pytest.mark.parametrize("path", CASES + SPACE, ids=lambda p: os.path.basename(p)[:-4])
def test_port_numpy_exp_is_bit_exact(path):
    if not _avx512_dispatch():
        pytest.skip("the goldens were made where numpy dispatches float32 exp to AVX512_SKX; this host does not, and "
                    "numpy's float32 exp differs between its dispatch paths")
    z = tp.load_case(path)
    im, mm, ma, lab = tp.port_case(z, "numpy")
    assert np.array_equal(lab, z["labels"])


SIZES = [(480, 640), (640, 427), (1, 1), (37, 53)]


# output (rows, columns) of the warp with a factor dividing both, and the masks' border values
OUTPUTS = [((256, 256), 4, (0, 255)), ((96, 160), 2, (3, 250)), ((255, 255), 3, (128, 127)), ((40, 88), 8, (1, 254))]


@pytest.mark.parametrize("hw", SIZES)
@pytest.mark.parametrize("kind", ["random", "binary"])
def test_uint8_warp_and_area_resize_match_cv2(hw, kind):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng([SIZES.index(hw), len(kind)])
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
        for (oh, ow), f, borders in OUTPUTS:
            bi = (124, 127, 127) if f == 4 else tuple(int(v) for v in rng.integers(0, 256, 3))
            got = tp.warp_affine_u8(img, M, (ow, oh), bi)
            want = cv2.warpAffine(img, M, (ow, oh), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT,
                                  borderValue=bi)
            assert np.array_equal(got, want)
            for border in borders:
                wm = tp.warp_affine_u8(m, M, (ow, oh), border)
                assert np.array_equal(wm, cv2.warpAffine(m, M, (ow, oh), flags=cv2.INTER_LINEAR,
                                                         borderMode=cv2.BORDER_CONSTANT, borderValue=border))
                assert np.array_equal(tp.resize_area_int(wm, f),
                                      cv2.resize(wm, (ow // f, oh // f), interpolation=cv2.INTER_AREA))


FACTORS = list(range(1, 65)) + [165, 256, 257, 331, 512]


@pytest.mark.parametrize("f", FACTORS)
def test_uint8_area_resize_matches_cv2_at_every_factor(f):
    """Boxes holding the exact ties (q + 1/2) f^2, every sum where cv2's float32 product differs from the correctly
    rounded quotient (f = 22, 34, 44, 62, 165, 331 here), the extremes and seeded sums; then random and binary masks."""
    cv2 = pytest.importorskip("cv2")
    m, sums = tc.area_probe(f)
    want = cv2.resize(m, (m.shape[1] // f, m.shape[0] // f), interpolation=cv2.INTER_AREA)
    assert np.array_equal(tp.resize_area_int(m, f), want)
    box = m.reshape(m.shape[0] // f, f, -1, f).astype(np.int64).sum(axis=(1, 3)).reshape(-1)
    assert np.array_equal(box[:len(sums)], sums)
    if f == 2 or f in (22, 34, 44, 62, 165, 331):  # the probe reaches what a correctly rounded quotient gets wrong
        assert (np.rint(box / (f * f)) != want.reshape(-1)).any()
    rng = np.random.default_rng(f)
    for kind in ("random", "binary"):
        r = rng.integers(0, 256 if kind == "random" else 2, (3 * f, 5 * f)).astype(np.uint8) * (1 if kind == "random" else 255)
        assert np.array_equal(tp.resize_area_int(r, f), cv2.resize(r, (5, 3), interpolation=cv2.INTER_AREA))


def test_erode_matches_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(5)
    for shape in ((64, 64), (1, 1), (2, 7), (128, 128)):
        m = rng.integers(0, 256, shape).astype(np.float32) / 255.
        assert np.array_equal(tp.erode3(m), cv2.erode(m, np.ones((3, 3), np.uint8)))
