"""CPU: JPEG frames in ``dropin.FrameStream`` before they touch a device -- the C declarations of the frame decode,
the checks ``_admit`` makes for ``submit``, the tick key the host parser gives the goldens, and the routing of the files
the parser refuses to ``cv2.imdecode`` (the device path stubbed)."""
import ctypes
import json
import os
import re

import frames_stub
import numpy as np
import pytest

from improved_body_parts_b200 import dropin, grouping

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "spgroup.h")
GOLDEN = os.path.join(ROOT, "tests", "golden", "jpeg")
MANIFEST = json.load(open(os.path.join(GOLDEN, "MANIFEST.json")))["cases"]
cv2 = pytest.importorskip("cv2")


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return grouping.load_library()


def _golden(name):
    with open(os.path.join(GOLDEN, name + ".jpg"), "rb") as f:
        return f.read()


@pytest.mark.parametrize("name,params", [
    ("spg_jpeg_decode_frame", ["spg_handle *h", "const spg_jpeg_record *device_record", "const spg_jpeg_record *format",
                               "int64_t max_scan_bytes", "void *stream"]),
    ("spg_jpeg_reserve_frame", ["spg_handle *h", "const spg_jpeg_record *format", "int64_t max_scan_bytes",
                                "int32_t *moved"])])
def test_frame_decode_is_declared_and_bound(name, params):
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(rf"int\s+{name}\s*\(([^)]*)\)\s*;", src)
    assert m, f"{name} is not declared"
    assert [" ".join(p.split()) for p in m.group(1).split(",")] == params
    restype, argtypes = grouping._PROTOTYPES[name]
    assert restype is ctypes.c_int and len(argtypes) == len(params)
    assert int(re.search(r"#define SPG_ABI_VERSION (\d+)", src).group(1)) == grouping.ABI_VERSION == 3


def test_frame_decode_without_a_handle_is_invalid(lib):
    fmt = np.zeros(1, grouping.JPEG_RECORD)
    fmt[0] = grouping.jpeg_parse(_golden("samp_420"))
    moved = ctypes.c_int32(7)
    assert lib.spg_jpeg_reserve_frame(None, fmt.ctypes.data, 1 << 16, ctypes.byref(moved)) == -1
    assert lib.spg_jpeg_decode_frame(None, None, None, 1 << 16, None) == -1


def _admit(frames, input_stage="device"):
    return dropin._admit(frames, [0] * len(frames), input_stage=input_stage, device=0, n_streams=None)


@pytest.mark.parametrize("frame,match", [(b"", "empty"), (bytearray(), "empty"), (12, "uint8 BGR"),
                                         ("frame.jpg", "uint8 BGR"), (np.zeros((4, 4), np.uint8), "uint8 BGR"),
                                         (b"not a jpeg", "imdecode")])
def test_submit_arguments(lib, frame, match):
    with pytest.raises(ValueError, match=match):
        _admit([frame])
    fs = frames_stub.stream()
    with pytest.raises(ValueError, match=match):
        fs.submit(frame)
    assert fs.launched == [] and fs.host_decodes == 0


def test_the_format_key_of_the_goldens(lib):
    keys = {}
    for name, case in MANIFEST.items():
        rec = grouping.jpeg_parse(_golden(name))
        if case["status"] not in ("ok", "corrupt", "range"):
            assert int(rec["status"]) != grouping.JPEG_OK, name
            continue
        assert int(rec["status"]) == grouping.JPEG_OK, name
        key = {k: int(rec[k]) for k in dropin.JPEG_FORMAT}
        h, w = (key["frame_width"], key["frame_height"]) if key["orientation"] >= 5 else \
            (key["frame_height"], key["frame_width"])
        assert [h, w, 3] == case["cv2_shape"] == [int(rec["height"]), int(rec["width"]), 3], name
        (f,), _, _ = _admit([_golden(name)])
        assert f.key == (h, w, "jpeg", tuple(key.values())), name
        keys[name] = key
    assert keys["grey"]["n_components"] == 1 and (keys["grey"]["h_samp"], keys["grey"]["v_samp"]) == (1, 1)
    for name, hv in (("samp_444", (1, 1)), ("samp_422", (2, 1)), ("samp_440", (1, 2)), ("samp_420", (2, 2))):
        assert keys[name]["n_components"] == 3 and (keys[name]["h_samp"], keys[name]["v_samp"]) == hv, name
    assert all(keys[n]["restart_interval"] > 0 for n in ("rst1", "rst2_444", "rst3", "rst7"))
    assert keys["samp_420"]["restart_interval"] == 0
    for o in range(1, 9):
        assert keys[f"exif{o}_II"]["orientation"] == keys[f"exif{o}_MM"]["orientation"] == o
    assert keys["exif_9_ignored"]["orientation"] == 1
    # the formats of the files that differ only in their tables or the segments in front of the scan are one
    assert keys["q1"] == keys["q50"] == keys["q100"]
    assert keys["exif1_II"] == keys["exif_9_ignored"]


def test_admit_routes_refused_files_to_cv2(lib):
    prog = cv2.imencode(".jpg", np.full((16, 24, 3), 90, np.uint8), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()
    refused = [_golden("progressive"), _golden("samp_411"), _golden("fill_before_stuffing"), prog]
    parsed = [_golden("samp_420"), memoryview(_golden("rst3")), bytearray(_golden("exif6_MM"))]
    for data in refused:
        (f,), _, decodes = _admit([data])
        want = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)
        assert decodes == 1 and f.rec is None and f.key == want.shape[:2] + ("image", None)  # keyed as a cv2 image
        assert np.array_equal(f.data, want) and f.decoded is f.data
    for data in parsed:
        (f,), _, decodes = _admit([data])
        assert decodes == 0 and f.rec is not None and int(f.rec["status"]) == grouping.JPEG_OK
        assert f.key.source == "jpeg" and f.decoded is None
        assert f.data.dtype == np.uint8 and f.data.tobytes() == bytes(data)
    fs = frames_stub.stream()
    for k, data in enumerate(refused + parsed):
        fs.submit(data)
        _, frames, _ = fs.launched[-1]
        assert len(frames) == 1  # submit poses a tick of one frame
        assert fs.host_decodes == min(k + 1, len(refused))


def test_admit_decodes_jpeg_with_cv2_at_the_host_input_stage(lib):
    data = _golden("samp_420")
    (f,), _, decodes = _admit([data], "host")
    want = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)
    assert decodes == 1 and f.rec is None and f.key == want.shape[:2] + ("image", None)
    assert np.array_equal(f.data, want)
    fs = frames_stub.stream("host")
    fs.submit(data)
    assert len(fs.launched[-1][1]) == 1 and fs.host_decodes == 1
