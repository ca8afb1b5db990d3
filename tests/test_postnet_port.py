"""CPU: oracle/postnet_port.py (groundwork for SURVEY §8 f-1, the reference's post-network stage) against OpenCV.

The reference's maps come out of ``cv2.resize(..., INTER_CUBIC)`` (evaluate.py:143-158).  In its environment that is
Intel IPP's routine, which OpenCV's own generic path does not reproduce bit for bit; the port follows the generic path.
Pinned here: (a) the port equals OpenCV's generic path to float rounding (IPP switched off), (b) it stays inside the
1e-4 float tolerance of ``north_star`` against whatever ``cv2.resize`` does by default on this host, (c) the stage's
plumbing (flip ensemble, crop, second resize, f64 average) equals the reference's lines run with ``cv2`` itself.
"""
import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from improved_body_parts_b200 import skeleton
from oracle import postnet_port as pp

CASES = [((32, 40, 5), dict(fx=4, fy=4)), ((128, 128, 18), dict(fx=4, fy=4)), ((46, 63, 3), dict(dsize=(640, 427))),
         ((512, 512, 4), dict(dsize=(427, 640))), ((100, 80), dict(dsize=(31, 57))), ((7, 9, 2), dict(fx=4, fy=4))]


def _cv(src, kw):
    if "dsize" in kw:
        return cv2.resize(src, kw["dsize"], interpolation=cv2.INTER_CUBIC)
    return cv2.resize(src, (0, 0), fx=kw["fx"], fy=kw["fy"], interpolation=cv2.INTER_CUBIC)


def _port(src, kw):
    return pp.resize_cubic(src, kw.get("dsize"), fx=kw.get("fx", 0.0), fy=kw.get("fy", 0.0))


@pytest.fixture
def no_ipp():
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    yield
    cv2.ipp.setUseIPP(was)


@pytest.mark.parametrize("shape,kw", CASES)
def test_resize_equals_opencv_generic_path_to_rounding(no_ipp, shape, kw):
    src = np.random.default_rng(5).random(shape, dtype=np.float32)
    ref, got = _cv(src, kw), _port(src, kw)
    assert ref.shape == got.shape and got.dtype == np.float32
    assert np.abs(ref - got).max() <= 5e-7  # values in [0, 1): an ulp or two (FMA contraction in OpenCV's SIMD rows)
    assert (ref == got).mean() > 0.5


@pytest.mark.parametrize("shape,kw", CASES)
def test_resize_within_north_star_tolerance_of_default_cv2(shape, kw):
    src = np.random.default_rng(6).random(shape, dtype=np.float32)
    assert np.abs(_cv(src, kw) - _port(src, kw)).max() <= 1e-4  # measured: 2.4e-7 for x4, up to 2.8e-5 for arbitrary sizes (IPP)


def test_cubic_weights_sum_to_one_and_interpolate():
    fx = np.linspace(0, 1, 33, dtype=np.float32)
    c = pp.cubic_coeffs(fx)
    assert np.allclose(c.sum(-1), 1.0, atol=1e-6)
    assert np.allclose(c[0], [0, 1, 0, 0], atol=1e-7)
    flat = np.full((9, 11), 0.37, np.float32)
    assert np.allclose(pp.resize_cubic(flat, None, fx=4, fy=4), 0.37, atol=1e-6)


def test_post_network_stage_equals_the_reference_lines_with_cv2():
    """evaluate.py:126-161 written out with cv2 itself vs the port, one scale, angle 0, on a synthetic network output."""
    rng = np.random.default_rng(7)
    n_paf, n_heat = skeleton.NUM_LIMBS, skeleton.NUM_PARTS + 2
    n_layers = n_paf + n_heat
    stride, h, w = 4, 48, 64                                # network output 48 x 64 -> padded input 192 x 256
    padded_shape, pad, image_shape = (192, 256), [0, 0, 7, 12], (370, 488)
    out = rng.random((2, n_layers, h, w), dtype=np.float32)

    # --- the reference's lines (:128-161), cv2 doing the resizes
    blob, blob_flip = out[0].transpose(1, 2, 0), out[1].transpose(1, 2, 0)
    b0, b1 = blob[:, :, :n_paf], blob[:, :, n_paf:n_layers]
    f0, f1 = blob_flip[:, :, :n_paf], blob_flip[:, :, n_paf:n_layers]
    b0_avg = (b0 + f0[:, ::-1, :][:, :, list(skeleton.FLIP_PAF_ORD)]) / 2
    b1_avg = (b1 + f1[:, ::-1, :][:, :, list(skeleton.FLIP_HEAT_ORD)]) / 2
    heat = cv2.resize(b1_avg, (0, 0), fx=stride, fy=stride, interpolation=cv2.INTER_CUBIC)
    heat = heat[pad[0]:padded_shape[0] - pad[2], pad[1]:padded_shape[1] - pad[3], :]
    heat = cv2.resize(heat, (image_shape[1], image_shape[0]), interpolation=cv2.INTER_CUBIC)
    paf = cv2.resize(b0_avg, (0, 0), fx=stride, fy=stride, interpolation=cv2.INTER_CUBIC)
    paf = paf[pad[0]:padded_shape[0] - pad[2], pad[1]:padded_shape[1] - pad[3], :]
    paf = cv2.resize(paf, (image_shape[1], image_shape[0]), interpolation=cv2.INTER_CUBIC)
    heat_avg = np.zeros((image_shape[0], image_shape[1], n_heat)) + heat / 1
    paf_avg = np.zeros((image_shape[0], image_shape[1], n_paf)) + paf / 1

    got_heat, got_paf = pp.post_network_scale(out, stride, padded_shape, pad, image_shape, n_paf, n_layers,
                                              skeleton.FLIP_PAF_ORD, skeleton.FLIP_HEAT_ORD)
    assert got_heat.shape == heat.shape and got_paf.shape == paf.shape
    assert np.abs(pp.accumulate(np.zeros_like(heat_avg), got_heat, 1) - heat_avg).max() <= 1e-4
    assert np.abs(pp.accumulate(np.zeros_like(paf_avg), got_paf, 1) - paf_avg).max() <= 1e-4
    # and with the same resize routine on both sides the plumbing is exact
    same_heat, same_paf = pp.post_network_scale(out, stride, padded_shape, pad, image_shape, n_paf, n_layers,
                                                skeleton.FLIP_PAF_ORD, skeleton.FLIP_HEAT_ORD,
                                                resize=lambda m, dsize, fx=0.0, fy=0.0: _cv(m, dict(dsize=dsize) if dsize else dict(fx=fx, fy=fy)))
    assert np.array_equal(same_heat, heat) and np.array_equal(same_paf, paf)


def test_three_instruction_division_of_the_multi_scale_kernel_is_exact():
    """csrc/postnet.cuh::div_by_scales replaces `map / n_scales` (evaluate.py:160-161) by a multiply and two FMAs; the
    tool checks it against the correctly rounded quotient for every float32 significand (here: n = 3, one binade)."""
    import importlib.util
    import os
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "check_div_by_scales.py")
    spec = importlib.util.spec_from_file_location("check_div_by_scales", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert mod.check(3, binades=(127,), sample=300) == 0


@pytest.mark.parametrize("shape,kw", CASES)
def test_resize_on_nonfinite_maps_equals_opencv_generic_path(no_ipp, shape, kw):
    """NaN, +inf and -inf in the source (a network output the reference does not scrub): the port and cv2 (IPP off)
    agree on where NaN lands (inf * a tap weight of either sign, inf - inf), on every infinity, and to rounding on the
    finite values."""
    rng = np.random.default_rng(8)
    src = rng.random(shape, dtype=np.float32)
    flat = src.reshape(-1)
    pos = rng.choice(flat.size, size=max(3, flat.size // 200), replace=False)
    flat[pos] = np.array([np.nan, np.inf, -np.inf], np.float32)[np.arange(pos.size) % 3]
    ref, got = _cv(src, kw), _port(src, kw)
    assert ref.shape == got.shape
    assert np.array_equal(np.isnan(ref), np.isnan(got))
    assert np.array_equal(np.isposinf(ref), np.isposinf(got)) and np.array_equal(np.isneginf(ref), np.isneginf(got))
    fin = np.isfinite(ref)
    assert np.isnan(got).any() and np.isinf(got).any() and fin.any()
    assert np.abs(ref[fin] - got[fin]).max() <= 5e-7


def test_same_size_resize_is_a_copy_as_in_opencv(no_ipp):
    """cv2.resize to the source's own size copies the source (resize.cpp's dsize == ssize shortcut): an infinity stays
    one pixel, where the [0, 1, 0, 0] taps would make NaN of its neighbours (inf * 0)."""
    src = np.random.default_rng(9).random((9, 11, 3), dtype=np.float32)
    src[4, 5, 0], src[2, 3, 1], src[6, 6, 2] = np.inf, -np.inf, np.nan
    ref, got = cv2.resize(src, (11, 9), interpolation=cv2.INTER_CUBIC), _port(src, dict(dsize=(11, 9)))
    assert np.array_equal(ref, src, equal_nan=True) and np.array_equal(got.view(np.uint32), src.view(np.uint32))
