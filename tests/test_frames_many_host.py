"""CPU: ``FrameStream.submit_many`` before it touches a device -- the C declarations of the tick calls, their refusal
without a handle, ``submit_many``'s argument checks, the tick key it forms, ``submit`` as a tick of one frame and the
routing of refused JPEG files to ``cv2.imdecode`` (the device path stubbed)."""
import ctypes
import os
import re

import frames_stub
import numpy as np
import pytest

from improved_body_parts_b200 import dropin, grouping

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "spgroup.h")
GOLDEN = os.path.join(ROOT, "tests", "golden", "jpeg")
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
    ("spg_jpeg_decode_frames", ["spg_handle *h", "const spg_jpeg_record *device_records", "const spg_jpeg_record *formats",
                                "const int64_t *capacities", "int32_t n", "void *stream"]),
    ("spg_jpeg_reserve_frames", ["spg_handle *h", "const spg_jpeg_record *formats", "const int64_t *capacities",
                                 "int32_t n", "int32_t *moved"]),
    ("spg_reserve_frames", ["spg_handle *h", "int32_t max_downsample", "const spg_prenet_member *members",
                            "int32_t n_images", "int32_t n_items", "int32_t *moved"])])
def test_tick_calls_are_declared_and_bound(name, params):
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(rf"int\s+{name}\s*\(([^)]*)\)\s*;", src)
    assert m, f"{name} is not declared"
    assert [" ".join(p.split()) for p in m.group(1).split(",")] == params
    restype, argtypes = grouping._PROTOTYPES[name]
    assert restype is ctypes.c_int and len(argtypes) == len(params)


def test_tick_calls_without_a_handle_are_invalid(lib):
    fmt = np.zeros(1, grouping.JPEG_RECORD)
    fmt[0] = grouping.jpeg_parse(_golden("samp_420"))
    caps = np.array([1 << 16], np.int64)
    moved = ctypes.c_int32(7)
    assert lib.spg_jpeg_reserve_frames(None, fmt.ctypes.data, caps.ctypes.data, 1, ctypes.byref(moved)) == -1
    assert lib.spg_jpeg_decode_frames(None, None, fmt.ctypes.data, caps.ctypes.data, 1, None) == -1
    members = np.zeros(1, grouping.PRENET_MEMBER)
    assert lib.spg_reserve_frames(None, 32, members.ctypes.data, 1, 1, ctypes.byref(moved)) == -1


def test_submit_many_arguments(lib):
    with pytest.raises(ValueError, match="at least one"):
        frames_stub.stream().submit_many([])
    with pytest.raises(ValueError, match="input_stage"):
        frames_stub.stream("host").submit_many([np.zeros((8, 8, 3), np.uint8)])
    fs = frames_stub.stream()
    with pytest.raises(ValueError, match="uint8 BGR"):  # one bad frame refuses the whole tick before it is staged
        fs.submit_many([np.zeros((8, 8, 3), np.uint8), np.zeros((4, 4), np.uint8)])
    with pytest.raises(ValueError, match="empty"):
        fs.submit_many([b""])
    with pytest.raises(ValueError, match="uint8 BGR"):  # a refused file cv2 decoded before the bad frame is not counted
        fs.submit_many([_golden("progressive"), np.zeros((4, 4), np.uint8)])
    assert fs.launched == [] and fs._next == 0 and fs.host_decodes == 0


def test_admitted_keys_tickets_and_slots_through_the_one_launcher(lib):
    fs = frames_stub.stream()
    jpeg = _golden("samp_420")
    rec = grouping.jpeg_parse(jpeg)
    img = np.zeros((30, 40, 3), np.uint8)
    prog = _golden("progressive")
    tickets = fs.submit_many([img, jpeg, prog])
    assert tickets == [0, 1, 2]
    slot, frames, streams = fs.launched[-1]
    decoded = cv2.imdecode(np.frombuffer(prog, np.uint8), cv2.IMREAD_COLOR)
    assert slot == 0 and streams == [0, 0, 0]
    assert frames_stub.keys(frames) == (
        (30, 40, "image", None),
        (int(rec["height"]), int(rec["width"]), "jpeg", tuple(int(rec[k]) for k in dropin.JPEG_FORMAT)),
        decoded.shape[:2] + ("image", None))
    assert frames[1].rec is not None and frames[1].data.tobytes() == jpeg  # the parser's file goes up as bytes
    assert frames[2].rec is None and np.array_equal(frames[2].data, decoded)  # the refused one as cv2's image
    assert fs.host_decodes == 1
    assert fs._busy[0][0] == tickets
    assert fs.submit_many([img]) == [3] and fs.launched[-1][0] == 1  # the next tick takes the next slot


def test_submit_and_a_one_frame_submit_many_share_a_key(lib):
    fs = frames_stub.stream()
    img = np.zeros((30, 40, 3), np.uint8)
    jpeg = _golden("samp_420")
    assert fs.submit(img) == 0 and fs.submit_many([img]) == [1]
    assert fs.submit_many([jpeg]) == [2] and fs.submit(jpeg) == 3
    assert [slot for slot, _, _ in fs.launched] == [0, 1, 0, 1]  # one counter: each call takes the next slot
    keys = [frames_stub.keys(frames) for _, frames, _ in fs.launched]
    assert keys[0] == keys[1] == ((30, 40, "image", None),)  # the same key
    assert keys[2] == keys[3] and len(keys[3]) == 1
    assert fs._busy[1][0] == [3]


def _admit(frames, input_stage="device"):
    return dropin._admit(frames, [0] * len(frames), input_stage=input_stage, device=0, n_streams=None)


def test_admit_keys_host_images_of_either_array_type(lib):
    import torch
    img = np.arange(30 * 40 * 3, dtype=np.uint8).reshape(30, 40, 3)
    for frame in (img, img[:, ::-1], torch.from_numpy(img)):  # numpy, a strided view, a CPU tensor
        (f,), _, decodes = _admit([frame])
        assert f.key == (30, 40, "image", None) and decodes == 0 and f.rec is None and f.decoded is None
        assert f.data.flags["C_CONTIGUOUS"] and np.array_equal(f.data, np.asarray(frame))


@pytest.mark.gpu
def test_admit_keys_a_cuda_image(lib, cuda_device):
    import torch
    img = torch.zeros((30, 40, 3), dtype=torch.uint8, device=cuda_device)
    (f,), _, decodes = _admit([img])
    assert f.key == (30, 40, "cuda", None) and f.data is img and decodes == 0
    with pytest.raises(ValueError, match="host frames"):
        _admit([img], "host")
    with pytest.raises(ValueError, match="uint8 tensor"):
        _admit([img.float()])
