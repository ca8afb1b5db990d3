"""CPU: oracle/jpeg_port.py, the numpy restatement of cv2's JPEG decode, against the goldens (cv2.imdecode's bytes) and
against cv2.imdecode on seeded encodings made at test time; every refused file classified with its reason."""
import json
import os

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

import make_jpeg_golden as mjg  # noqa: E402
from oracle import jpeg_port as jp  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg")
MANIFEST = json.load(open(os.path.join(GOLDEN, "MANIFEST.json")))["cases"]


def _file(name: str) -> bytes:
    with open(os.path.join(GOLDEN, name + ".jpg"), "rb") as f:
        return f.read()


@pytest.fixture(scope="module")
def decoded():
    return dict(np.load(os.path.join(GOLDEN, "decoded.npz")))


@pytest.mark.parametrize("name", sorted(MANIFEST))
def test_golden_status(name):
    assert jp.REASONS[jp.classify(_file(name))] == MANIFEST[name]["status"]


@pytest.mark.parametrize("name", sorted(n for n, c in MANIFEST.items() if c["status"] in ("ok", "range")))
def test_golden_decode(name, decoded):
    """Every file the port decodes equals cv2's decode, the out-of-range ones included (they decode with libjpeg's C
    arithmetic, which is what the port restates; the device leaves them to cv2)."""
    got = jp.decode(_file(name))
    if MANIFEST[name]["status"] == "ok":
        assert np.array_equal(got, decoded[name]), name
    else:
        assert got.shape == decoded[name].shape


def test_golden_refusals_are_the_expected_ones():
    refused = {n: c["status"] for n, c in MANIFEST.items() if c["status"] != "ok"}
    assert refused == {"samp_411": "sampling", "progressive": "process", "truncated": "truncated",
                       "garbage_scan": "range", "short_scan": "corrupt", "dqt16_x8_range": "range",
                       "fill_before_stuffing": "malformed"}


@pytest.mark.parametrize("shape", [(480, 640), (427, 640)])
@pytest.mark.parametrize("sampling", ["444", "422", "420", "440"])
@pytest.mark.parametrize("restart", [0, 4])
def test_coco_sized_against_cv2(shape, sampling, restart):
    data = mjg.encode(mjg.content(100 + len(sampling) + restart, *shape), sampling, 95, restart=restart)
    want = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)
    assert jp.classify(data) == jp.OK
    assert np.array_equal(jp.decode(data), want)


def test_stages_are_consistent():
    """The exposed stages compose to decode(): header -> coefficients -> planes -> BGR -> orientation."""
    data = _file("exif6_MM")
    h = jp.parse(data)
    assert (h.frame_height, h.frame_width, h.orientation, h.height, h.width) == (9, 13, 6, 13, 9)
    co = jp.coefficients(data, h)
    assert [c.shape for c in co] == [(2, 2, 64), (1, 1, 64), (1, 1, 64)]
    pl = jp.planes(h, co)
    assert [p.shape for p in pl] == [(16, 16), (8, 8), (8, 8)]
    assert np.array_equal(jp.orient(jp.bgr(h, pl), h.orientation), jp.decode(data))


def test_huffman_table_checks():
    bits = np.zeros(17, np.int32)
    bits[1] = 2  # two 1-bit codes: the second is all ones
    with pytest.raises(jp.Refused) as e:
        jp.build_huffman(bits, np.arange(2, dtype=np.uint8))
    assert e.value.status == jp.TABLES
    bits = np.zeros(17, np.int32)
    bits[16] = 257
    with pytest.raises(jp.Refused):
        jp.build_huffman(bits, np.zeros(257, np.uint8))
