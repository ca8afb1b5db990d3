"""CPU: the rotation search's warp (oracle/postnet_rotation_port.py) against OpenCV.

``cv2.warpAffine`` on float32 maps is OpenCV's generic fixed-point warp, which the port restates: the bar is BIT-IDENTICAL
maps (compared as uint32, so NaN payloads and signed zeros count), NaN and inf included.  The item chain
(evaluate.py:143-158: resize, warp, crop, resize) is checked against the reference's lines written out with cv2.
"""
import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from improved_body_parts_b200 import skeleton
from oracle import postnet_port as pp
from oracle import postnet_rotation_port as pr

GRIDS = [(640, 896), (256, 256), (257, 131), (131, 257)]
ANGLES = [-45, -30, -7.5, 0.5, 13, 30, 90, 180]


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _maps(seed, shape, specials=True):
    rng = np.random.default_rng(seed)
    m = rng.standard_normal(shape).astype(np.float32)
    if specials:
        flat = m.reshape(-1)
        for v in (np.nan, np.inf, -np.inf):
            flat[rng.integers(0, flat.size, 40)] = v
    return m


@pytest.mark.parametrize("channels", [18, 30])
@pytest.mark.parametrize("grid", GRIDS, ids=[f"{h}x{w}" for h, w in GRIDS])
@pytest.mark.parametrize("angle", ANGLES)
def test_warp_is_cv2_bit_for_bit(channels, grid, angle):
    if grid == (640, 896) and channels == 30 and angle not in (-30, 90):
        pytest.skip("the full-size grid with 30 channels is run at two angles")
    src = _maps(int(angle * 10) + 2000 + channels, grid + (channels,))
    M = cv2.getRotationMatrix2D((grid[0] / 2, grid[1] / 2), angle, 1)  # evaluate.py:114: (rows / 2, cols / 2)
    ref = cv2.warpAffine(src, M, (0, 0))
    got = pr.warp_affine_linear(src, M)
    assert got.shape == ref.shape and got.dtype == np.float32
    assert np.array_equal(_bits(got), _bits(ref))
    assert np.isnan(got).any() and np.isfinite(got).mean() > 0.5


def test_warp_of_a_far_translation_is_all_border():
    src = _maps(7, (131, 257, 18))
    M = np.array([[1.0, 0.0, 5000.0], [0.0, 1.0, -3000.0]])
    ref, got = cv2.warpAffine(src, M, (0, 0)), pr.warp_affine_linear(src, M)
    assert np.array_equal(_bits(got), _bits(ref)) and not got.any()


def test_inversion_follows_opencv():
    M = cv2.getRotationMatrix2D((131 / 2, 257 / 2), 13, 1)
    assert np.allclose(pr.invert_affine(M).reshape(2, 3), cv2.invertAffineTransform(M), rtol=0, atol=1e-12)


def _reference_item(out_pair, stride, padded, pad, image_hw, M, resize):
    """evaluate.py:128-158 for one item with angle != 0, written out with cv2.warpAffine (and ``resize`` for cv2.resize)."""
    paf_avg, heat_avg = pp.flip_ensemble(out_pair, 30, 48, skeleton.FLIP_PAF_ORD, skeleton.FLIP_HEAT_ORD[:18])
    res = []
    for m in (heat_avg, paf_avg):
        up = resize(np.ascontiguousarray(m, np.float32), stride)
        up = cv2.warpAffine(up, M, (0, 0))
        up = up[pad[0]:padded[0] - pad[2], pad[1]:padded[1] - pad[3], :]
        res.append(resize(np.ascontiguousarray(up), (image_hw[1], image_hw[0])))
    return res


def _cv2_resize(a, arg):
    if isinstance(arg, tuple):
        return cv2.resize(a, arg, interpolation=cv2.INTER_CUBIC)
    return cv2.resize(a, (0, 0), fx=arg, fy=arg, interpolation=cv2.INTER_CUBIC)


def _port_resize(a, arg):
    return pp.resize_cubic(a, arg) if isinstance(arg, tuple) else pp.resize_cubic(a, None, fx=arg, fy=arg)


@pytest.mark.parametrize("hw,crop,image,angle", [((32, 48), (120, 180), (96, 144), 30), ((40, 24), (157, 90), (131, 77), -45),
                                                 ((16, 16), (64, 64), (64, 64), 90)])
def test_item_chain_places_the_warp_between_the_resizes(hw, crop, image, angle):
    rng = np.random.default_rng(11)
    out = rng.random((2, 50, hw[0], hw[1]), dtype=np.float32)
    padded = (4 * hw[0], 4 * hw[1])
    pad = [0, 0, padded[0] - crop[0], padded[1] - crop[1]]
    _, M_rev = pr.rotation_matrices(padded, angle)
    got = pr.post_network_item(out, 4, padded, pad, image, 30, 48, skeleton.FLIP_PAF_ORD, skeleton.FLIP_HEAT_ORD[:18],
                               rotate_matrix=M_rev)
    ref_cv = _reference_item(out, 4, padded, pad, image, M_rev, _cv2_resize)
    ref_port = _reference_item(out, 4, padded, pad, image, M_rev, _port_resize)
    for g, c, p in zip(got, ref_cv, ref_port):
        assert g.shape == image + (g.shape[2],)
        assert np.abs(g - c).max() <= 1e-4  # cv2.resize is IPP here: the tolerance of tests/test_postnet_port.py
        assert np.array_equal(_bits(g), _bits(p))  # with the port's resize: bit for bit, so the warp sits where the reference has it
    # without a matrix the item is postnet_port.post_network_scale itself
    plain = pr.post_network_item(out, 4, padded, pad, image, 30, 48, skeleton.FLIP_PAF_ORD, skeleton.FLIP_HEAT_ORD[:18])
    base = pp.post_network_scale(out, 4, padded, pad, image, 30, 48, skeleton.FLIP_PAF_ORD, skeleton.FLIP_HEAT_ORD[:18])
    assert all(np.array_equal(_bits(a), _bits(b)) for a, b in zip(plain, base))
