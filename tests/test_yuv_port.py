"""CPU: ``oracle/yuv_port.py`` -- the numpy restatement of cv2.cvtColor's YUV -> BGR conversions -- against cv2 itself,
on every (Y, U, V) triple and on seeded frames at the widths where OpenCV's vector loops leave a scalar tail."""
import numpy as np
import pytest

from oracle import yuv_port as yp

cv2 = pytest.importorskip("cv2")


def _cv2(fmt, planes):
    return cv2.cvtColor(yp.cv2_layout(fmt, planes), yp.cv2_code(fmt))


@pytest.mark.parametrize("fmt", yp.FORMATS)
def test_every_triple_equals_cv2(fmt):
    planes = yp.every_triple(fmt)
    got = yp.convert(fmt, planes)
    assert got.shape == (4096, 4096, 3)
    assert np.array_equal(got, _cv2(fmt, planes))


def test_every_triple_holds_each_triple_once():
    y, uv = yp.every_triple("nv12")
    Y = y.reshape(2048, 2, 2048, 2).transpose(0, 2, 1, 3).reshape(-1, 4).astype(np.int64)
    U, V = uv[:, 0::2].reshape(-1, 1).astype(np.int64), uv[:, 1::2].reshape(-1, 1).astype(np.int64)
    keys = np.sort((Y + (U << 8) + (V << 16)).reshape(-1))
    assert np.array_equal(keys, np.arange(1 << 24))


# widths around OpenCV's 16- and 32-pixel vector blocks and their tails; I420 heights whose H/2 is odd (the U and V
# planes then end in the middle of a row of cv2's [H*3/2, W] layout)
@pytest.mark.parametrize("fmt", yp.FORMATS)
@pytest.mark.parametrize("W", [2, 6, 14, 30, 34, 62, 66, 642])
@pytest.mark.parametrize("H", [2, 6, 10, 480])
def test_seeded_frames_equal_cv2(fmt, H, W):
    rng = np.random.default_rng(H * 10007 + W * 31 + yp.FORMATS.index(fmt))
    planes = yp.random_planes(rng, fmt, H, W)
    assert np.array_equal(yp.convert(fmt, planes), _cv2(fmt, planes))


def test_extremes_saturate_as_cv2_does():
    for fmt in yp.FORMATS:
        for y, u, v in [(0, 0, 0), (255, 255, 255), (16, 128, 128), (235, 240, 16), (255, 0, 255), (0, 255, 0)]:
            planes = tuple(np.full(s, val, np.uint8) for s, val in zip(yp.plane_shapes(fmt, 4, 8), (y, u, v)))
            if fmt == "nv12":
                planes[1][:, 1::2] = v
            elif fmt == "yuyv":
                planes[0][:, 1::4], planes[0][:, 3::4] = u, v
            assert np.array_equal(yp.convert(fmt, planes), _cv2(fmt, planes)), (fmt, y, u, v)
