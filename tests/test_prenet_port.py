"""CPU: the input side of predict() (oracle/prenet_port.py) against OpenCV.

``cv2.resize`` of uint8 images with IPP switched off is OpenCV's generic path, which the port restates: the bar is
BIT-IDENTICAL images.  With IPP on (what the reference's wheels run) every pixel is within 1 LSB.  The item chain
(evaluate.py:94-121: clamp, resize, pad, / 255, warp, mirror) is checked against the reference's lines written out
with cv2.
"""
import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from oracle import prenet_port as pn


@pytest.fixture
def generic_path():
    """OpenCV's generic resize (IPP off) for the test, the previous setting restored afterwards."""
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    yield
    cv2.ipp.setUseIPP(was)


def _image(kind, h, w, seed):
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "blurred":
        return cv2.GaussianBlur(rng.integers(0, 256, (h, w, 3), dtype=np.uint8), (7, 7), 2.0)
    board = (np.indices((h, w)).sum(0) % 2 * 255).astype(np.uint8)  # 0/255 checkerboard: the overshoot saturates
    return np.repeat(board[:, :, None], 3, axis=2)


KINDS = ["random", "blurred", "checker"]
SIZES = [(480, 640, 640 / 480), (427, 640, 1.499), (375, 500, 3.41), (60, 50, 0.61), (33, 35, 0.37), (100, 90, 1.0),
         (1, 1, 3.0), (2, 3, 2.5), (41, 37, 1.0001)]
# every residue of dst_w * 3 mod 32: where the vector body of the vertical pass ends and the scalar tail begins
RESIDUES = [(24, w, 1.37) for w in range(20, 72)]


def _cases():
    return [(k, h, w, fx) for k in KINDS for h, w, fx in SIZES + RESIDUES]


def test_residue_sweep_covers_every_tail_length():
    got = {pn.resized_size(h, w, fx)[1] * 3 % 32 for h, w, fx in RESIDUES}
    assert got == set(range(32))


@pytest.mark.parametrize("kind", KINDS)
def test_resize_is_cv2_generic_path_bit_for_bit(kind, generic_path):
    for i, (h, w, fx) in enumerate(SIZES + RESIDUES):
        img = _image(kind, h, w, 100 + i)
        ref = cv2.resize(img, (0, 0), fx=fx, fy=fx, interpolation=cv2.INTER_CUBIC)
        got = pn.resize_cubic_u8(img, fx)
        assert got.shape == ref.shape and got.dtype == np.uint8, (h, w, fx)
        assert np.array_equal(got, ref), (kind, h, w, fx, int((got != ref).sum()))


def test_tail_elements_take_the_integer_path(generic_path):
    """Elements where the float and integer vertical passes disagree: cv2 follows the float one in the 8-lane body and
    the integer one in the tail -- a lane count of 4 or 16 mispredicts some of them."""
    rng = np.random.default_rng(2)
    seen = {"body": 0, "tail": 0}
    for _ in range(400):
        h, w, fx = int(rng.integers(50, 200)), int(rng.integers(2, 20)), float(rng.uniform(0.5, 3.5))
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        ref = cv2.resize(img, (0, 0), fx=fx, fy=fx, interpolation=cv2.INTER_CUBIC)
        if ref.shape[:2] == (h, w):
            continue
        got = pn.resize_cubic_u8(img, fx)
        assert np.array_equal(got, ref)
        lanes = pn.VEC_LANES
        try:
            pn.VEC_LANES = 1
            body = pn.resize_cubic_u8(img, fx).reshape(ref.shape[0], -1)
            pn.VEC_LANES = 1 << 30
            tail = pn.resize_cubic_u8(img, fx).reshape(ref.shape[0], -1)
        finally:
            pn.VEC_LANES = lanes
        n_body = ref.shape[1] * 3 // lanes * lanes
        for _, xc in np.argwhere(body != tail):
            seen["body" if xc < n_body else "tail"] += 1
    assert seen["body"] > 0 and seen["tail"] > 0, seen


def test_resize_is_within_one_lsb_of_ipp():
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(True)
    try:
        n_diff = n_all = 0
        for i, (kind, h, w, fx) in enumerate(_cases()):
            img = _image(kind, h, w, 100 + i)
            ref = cv2.resize(img, (0, 0), fx=fx, fy=fx, interpolation=cv2.INTER_CUBIC).astype(np.int16)
            got = pn.resize_cubic_u8(img, fx).astype(np.int16)
            assert np.abs(got - ref).max() <= 1, (kind, h, w, fx)
            n_diff += int((got != ref).sum())
            n_all += got.size
    finally:
        cv2.ipp.setUseIPP(was)
    print(f"generic path vs IPP: {n_diff} of {n_all} values differ by 1 LSB ({n_diff / n_all:.4%})")


def test_unit_scale_is_a_copy_and_empty_sizes_raise():
    img = _image("random", 17, 23, 5)
    assert np.array_equal(pn.resize_cubic_u8(img, 1.0), img)
    with pytest.raises(ValueError):
        pn.resize_cubic_u8(img, 0.01)


def _reference_item(image, scale, angle, md, pv):
    """evaluate.py:94-121 written out with cv2 (generic resize path under the fixture)."""
    if scale * image.shape[0] > 2600 or scale * image.shape[1] > 3800:
        scale = min(2600 / image.shape[0], 3800 / image.shape[1])
    image_to_test = cv2.resize(image, (0, 0), fx=scale, fy=scale, interpolation=cv2.INTER_CUBIC)
    h, w = image_to_test.shape[:2]
    pad = [0, 0, 0 if h % md == 0 else md - h % md, 0 if w % md == 0 else md - w % md]
    padded = np.pad(image_to_test, ((0, pad[2]), (0, pad[3]), (0, 0)), constant_values=pv)
    input_img = np.float32(padded / 255)
    reverse = None
    if angle != 0:
        centre = (input_img.shape[0] / 2, input_img.shape[1] / 2)
        rotate_matrix = cv2.getRotationMatrix2D(centre, angle, 1)
        reverse = cv2.getRotationMatrix2D(centre, -angle, 1)
        input_img = cv2.warpAffine(input_img, rotate_matrix, (0, 0))
    swap = input_img[:, ::-1, :].copy()
    return np.concatenate((input_img[None, ...], swap[None, ...]), axis=0), image_to_test.shape[:2], pad, reverse


ITEMS = [((120, 160), 1.37, a) for a in (0, 0.5, 30, -30, 90, 180)] + \
        [((90, 200), 1.0, 30), ((200, 90), 0.8, -30), ((90, 200), 1.0, 0),  # non-square: the centre's x / y swap
         ((40, 1400), 3.0, 0), ((1200, 30), 3.0, 30)]  # the 2600 / 3800 clamp


@pytest.mark.parametrize("shape,scale,angle", ITEMS)
def test_prenet_item_is_the_reference_bit_for_bit(shape, scale, angle, generic_path):
    img = _image("blurred", shape[0], shape[1], 7)
    got = pn.prenet_item(img, scale, angle, 8, 128)
    ref = _reference_item(img, scale, angle, 8, 128)
    assert got[0].dtype == np.float32 and got[0].shape == ref[0].shape
    assert np.array_equal(got[0].view(np.uint32), ref[0].view(np.uint32))
    assert tuple(got[1]) == tuple(ref[1]) and list(got[2]) == list(ref[2])
    assert (got[3] is None) == (ref[3] is None)
    if ref[3] is not None:
        assert np.array_equal(got[3], ref[3])
    if shape == (40, 1400):
        assert got[1][1] == 3800  # clamped


def test_pad_value_goes_through_the_table():
    img = _image("random", 9, 13, 3)
    pair, crop, pad, _ = pn.prenet_item(img, 1.0, 0, 8, 200)
    assert crop == (9, 13) and pad == [0, 0, 7, 3]
    assert (pair[0, 9:, :, :] == np.float32(200 / 255)).all() and (pair[0, :, 13:, :] == np.float32(200 / 255)).all()
    assert np.array_equal(pair[1], pair[0, :, ::-1, :])
