"""CPU: YUV frames before they touch a device -- ``spg_yuv_to_bgr``'s declaration and member record against the real
header, its refusal without a handle, ``dropin.YUVFrame``'s checks, and the tick key ``_admit`` forms for YUV
frames."""
import ctypes
import os
import re
import subprocess

import frames_stub
import numpy as np
import pytest

from improved_body_parts_b200 import dropin, grouping
from oracle import yuv_port as yp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "spgroup.h")
GOLDEN = os.path.join(ROOT, "tests", "golden", "jpeg")
cv2 = pytest.importorskip("cv2")
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return grouping.load_library()


def test_call_is_declared_and_bound():
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"int\s+spg_yuv_to_bgr\s*\(([^)]*)\)\s*;", src)
    assert m, "spg_yuv_to_bgr is not declared"
    assert [" ".join(p.split()) for p in m.group(1).split(",")] == [
        "spg_handle *h", "const spg_yuv_member *members", "int32_t n", "void *stream"]
    restype, argtypes = grouping._PROTOTYPES["spg_yuv_to_bgr"]
    assert restype is ctypes.c_int and len(argtypes) == 4
    assert "spg_yuv_to_bgr" in grouping.EXPORTS
    assert re.search(r"#define SPG_ABI_VERSION 3\b", src)  # an additive change


def test_member_record_is_the_header_struct(tmp_path):
    """``YUV_MEMBER`` against ``spg_yuv_member`` of the real header: sizeof, the offset of every field and the format
    codes."""
    dt = grouping.YUV_MEMBER
    fields = ["format", "height", "width", "reserved", "planes", "pitches", "out", "out_pitch"]
    assert list(dt.names) == fields
    args = ", ".join(["(int)sizeof(spg_yuv_member)"] + [f"(int)offsetof(spg_yuv_member, {f})" for f in fields] +
                     ["SPG_YUV_NV12", "SPG_YUV_I420", "SPG_YUV_YUYV"])
    probe, exe = tmp_path / "probe.c", tmp_path / "probe"
    probe.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "spgroup.h"\nint main(void){\nprintf("' +
                     " %d" * (4 + len(fields)) + '\\n", ' + args + ");\nreturn 0;}\n")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(probe), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert got[:-3] == [dt.itemsize] + [dt.fields[f][1] for f in fields]
    assert got[:-3] == [80, 0, 4, 8, 12, 16, 40, 64, 72]
    assert got[-3:] == [grouping.YUV_NV12, grouping.YUV_I420, grouping.YUV_YUYV]


def test_call_without_a_handle_is_invalid(lib):
    members = np.zeros(1, grouping.YUV_MEMBER)
    assert lib.spg_yuv_to_bgr(None, members.ctypes.data, 1, None) == -1


def _planes(fmt, H, W, seed=0):
    return yp.random_planes(np.random.default_rng(seed), fmt, H, W)


@pytest.mark.parametrize("fmt", yp.FORMATS)
def test_frame_takes_its_planes_and_converts_as_cv2(fmt):
    planes = _planes(fmt, 6, 10)
    f = dropin.YUVFrame(fmt, planes)
    assert (f.format, f.height, f.width, f.device) == (fmt, 6, 10, None)
    want = cv2.cvtColor(yp.cv2_layout(fmt, planes), yp.cv2_code(fmt))
    assert np.array_equal(f.to_bgr(), want)
    # pitched rows: views of wider buffers, as a decoder's surface hands them out
    pitched = []
    for p in planes:
        buf = np.zeros((p.shape[0], p.shape[1] + 6), np.uint8)
        buf[:, :p.shape[1]] = p
        pitched.append(buf[:, :p.shape[1]])
    g = dropin.YUVFrame(fmt, pitched)
    assert np.array_equal(g.to_bgr(), want)
    # CPU tensors are taken as numpy arrays
    assert np.array_equal(dropin.YUVFrame(fmt, [torch.from_numpy(p) for p in planes]).to_bgr(), want)


def test_frame_checks():
    y, uv = _planes("nv12", 4, 6)
    with pytest.raises(ValueError, match="format"):
        dropin.YUVFrame("nv21", (y, uv))
    with pytest.raises(ValueError, match="format"):
        dropin.YUVFrame("NV12", (y, uv))
    with pytest.raises(ValueError, match="plane"):  # plane count
        dropin.YUVFrame("nv12", (y,))
    with pytest.raises(ValueError, match="plane"):
        dropin.YUVFrame("i420", (y, uv))
    with pytest.raises(ValueError, match="plane"):
        dropin.YUVFrame("yuyv", (y, uv))
    with pytest.raises(ValueError, match="uint8"):  # dtype
        dropin.YUVFrame("nv12", (y.astype(np.uint16), uv))
    with pytest.raises(ValueError, match="uint8"):
        dropin.YUVFrame("nv12", (y, uv.astype(np.float32)))
    with pytest.raises(ValueError, match="uint8"):  # not 2-D
        dropin.YUVFrame("nv12", (y[..., None], uv))
    with pytest.raises(ValueError, match="uint8"):
        dropin.YUVFrame("nv12", (y.tolist(), uv))
    with pytest.raises(ValueError, match="planes of a 4x6 nv12"):  # plane shape
        dropin.YUVFrame("nv12", (y, uv[:, :4]))
    with pytest.raises(ValueError, match="planes of a 4x6 nv12"):
        dropin.YUVFrame("nv12", (y, np.zeros((4, 6), np.uint8)))
    yi, u, v = _planes("i420", 4, 6)
    with pytest.raises(ValueError, match="planes of a 4x6 i420"):
        dropin.YUVFrame("i420", (yi, u, v[:, :2]))
    with pytest.raises(ValueError, match="planes of a 4x6 i420"):
        dropin.YUVFrame("i420", (yi, uv, v))
    with pytest.raises(ValueError, match="even"):  # odd sizes: cv2 refuses them
        dropin.YUVFrame("nv12", (np.zeros((5, 6), np.uint8), np.zeros((2, 6), np.uint8)))
    with pytest.raises(ValueError, match="even"):
        dropin.YUVFrame("i420", (np.zeros((4, 7), np.uint8), np.zeros((2, 3), np.uint8), np.zeros((2, 3), np.uint8)))
    with pytest.raises(ValueError, match="even"):
        dropin.YUVFrame("yuyv", (np.zeros((4, 6), np.uint8),))  # 3 pixels per row
    dropin.YUVFrame("yuyv", (np.zeros((5, 8), np.uint8),))  # an odd height is fine for 4:2:2
    with pytest.raises(ValueError, match="empty"):
        dropin.YUVFrame("yuyv", (np.zeros((0, 8), np.uint8),))
    with pytest.raises(ValueError, match="stride"):  # non-unit column stride
        dropin.YUVFrame("nv12", (np.zeros((4, 12), np.uint8)[:, ::2], uv))
    with pytest.raises(ValueError, match="stride"):
        dropin.YUVFrame("nv12", (np.asfortranarray(np.zeros((4, 6), np.uint8)), uv))
    with pytest.raises(ValueError, match="stride"):  # rows that overlap
        dropin.YUVFrame("yuyv", (np.lib.stride_tricks.as_strided(np.zeros(64, np.uint8), (4, 8), (4, 1)),))


def _admit(frames, input_stage="device"):
    return dropin._admit(frames, [0] * len(frames), input_stage=input_stage, device=0, n_streams=None)


def _cuda_frame(fmt, H, W, device=0):
    """A YUVFrame whose planes claim to be CUDA tensors on ``device`` (built without a device: its device is all the
    tick key reads)."""
    f = dropin.YUVFrame(fmt, _planes(fmt, H, W))
    f.device = device
    return f


def test_admit_keys_yuv_frames(lib):
    with open(os.path.join(GOLDEN, "samp_420.jpg"), "rb") as fh:
        jpeg = fh.read()
    rec = grouping.jpeg_parse(jpeg)
    host = dropin.YUVFrame("nv12", _planes("nv12", 6, 10))
    cuda = _cuda_frame("nv12", 6, 10)
    img = np.zeros((6, 10, 3), np.uint8)
    frames, _, decodes = _admit([host, cuda, img, jpeg, dropin.YUVFrame("yuyv", _planes("yuyv", 5, 10))])
    keys = tuple(f.key for f in frames)
    assert [k[:2] for k in keys] == [(6, 10), (6, 10), (6, 10), (int(rec["height"]), int(rec["width"])), (5, 10)]
    k_host, k_cuda, k_img, k_jpeg, k_yuyv = keys
    assert k_host != k_cuda  # host and CUDA planes: two keys
    assert k_host == (6, 10, "yuv", "nv12") and k_cuda == (6, 10, "yuv_cuda", "nv12")
    assert k_yuyv == (5, 10, "yuv", "yuyv")
    # neither is taken for a JPEG frame, an image or each other's format
    assert k_jpeg.source == "jpeg" and k_img == (6, 10, "image", None)
    for k in (k_host, k_cuda):
        assert k not in (k_img, k_jpeg)
    assert frames[0].data is host and frames[0].rec is None and frames[1].data is cuda and decodes == 0
    # the same frames again form the same key; another format or another side forms another
    again, _, _ = _admit([dropin.YUVFrame("nv12", _planes("nv12", 6, 10, seed=1)), _cuda_frame("nv12", 6, 10), img, jpeg,
                          dropin.YUVFrame("yuyv", _planes("yuyv", 5, 10, seed=2))])
    assert tuple(f.key for f in again) == keys
    (i420,), _, _ = _admit([dropin.YUVFrame("i420", _planes("i420", 6, 10))])
    assert i420.key == (6, 10, "yuv", "i420")
    assert len({(i420.key,), (k_host,), (k_cuda,)}) == 3
    # every layout, on the host and on the device
    for fmt in yp.FORMATS:
        got, _, _ = _admit([dropin.YUVFrame(fmt, _planes(fmt, 6, 10)), _cuda_frame(fmt, 6, 10)])
        assert [f.key for f in got] == [(6, 10, "yuv", fmt), (6, 10, "yuv_cuda", fmt)]
    # submit and submit_many pose the same key
    fs = frames_stub.stream()
    fs.submit(host)
    fs.submit_many([host])
    assert frames_stub.keys(fs.launched[0][1]) == frames_stub.keys(fs.launched[1][1]) == ((6, 10, "yuv", "nv12"),)


def test_yuv_frames_on_another_device_or_host_stage(lib):
    with pytest.raises(ValueError, match="cuda:0"):
        _admit([_cuda_frame("nv12", 6, 10, device=1)])
    with pytest.raises(ValueError, match="host frames"):
        _admit([_cuda_frame("nv12", 6, 10)], "host")
    fs = frames_stub.stream()
    with pytest.raises(ValueError, match="cuda:0"):
        fs.submit(_cuda_frame("nv12", 6, 10, device=1))
    assert fs.launched == []


@pytest.mark.parametrize("fmt", yp.FORMATS)
def test_admit_converts_yuv_with_cv2_at_the_host_input_stage(lib, fmt):
    planes = _planes(fmt, 6, 10)
    (f,), _, decodes = _admit([dropin.YUVFrame(fmt, planes)], "host")
    want = cv2.cvtColor(yp.cv2_layout(fmt, planes), yp.cv2_code(fmt))
    assert f.key == (6, 10, "image", None)  # posed as an image
    assert np.array_equal(f.data, want) and f.decoded is f.data  # and kept for detail's image
    assert decodes == 0  # which counts JPEG frames only
    fs = frames_stub.stream("host")
    assert fs.submit(dropin.YUVFrame(fmt, planes)) == 0 and fs.host_decodes == 0
    assert frames_stub.keys(fs.launched[-1][1]) == ((6, 10, "image", None),)
