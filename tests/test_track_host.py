"""CPU: ``FrameStream`` tracking before it touches a device -- ``TrackParams`` and stream-index checks, ``ids=True``
without tracking, ``spg_track_frames``'s declaration and its refusal without a handle, and (the launch stubbed) the
stream indices passed to the tick apart from its key, with -1 for the second pose of a flagged JPEG frame."""
import ctypes
import os
import re
import types

import frames_stub
import numpy as np
import pytest

from improved_body_parts_b200 import dropin, grouping, wire

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
cv2 = pytest.importorskip("cv2")


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return grouping.load_library()


def test_track_frames_is_declared_and_bound():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "spgroup.h")).read(), flags=re.S)
    m = re.search(r"int\s+spg_track_frames\s*\(([^)]*)\)\s*;", src)
    assert [" ".join(p.split()) for p in m.group(1).split(",")] == [
        "spg_handle *h", "const spg_track_frame *frames", "int32_t n", "spg_track_table *tables", "int32_t n_tables",
        "double oks_threshold", "int32_t max_age", "void *stream"]
    assert grouping.TRACK.itemsize == 296 and grouping.TRACK_TABLE.itemsize == 16 + 128 * 296
    assert grouping.TRACK_FRAME.itemsize == 40


def test_track_frames_without_a_handle_is_invalid(lib):
    f = np.zeros(1, grouping.TRACK_FRAME)
    assert lib.spg_track_frames(None, f.ctypes.data, 1, None, 1, 0.5, 30, None) == -1


@pytest.mark.parametrize("kw,match", [
    (dict(streams=0), "streams"), (dict(streams=1.0), "int"), (dict(streams=True), "int"), (dict(max_age=-1), "max_age"),
    (dict(max_age=2.5), "int"), (dict(oks_threshold=1.5), "oks_threshold"), (dict(oks_threshold=-0.1), "oks_threshold"),
    (dict(oks_threshold=float("nan")), "oks_threshold"), (dict(oks_threshold="0.5"), "oks_threshold")])
def test_track_params_are_checked(kw, match):
    with pytest.raises(ValueError, match=match):
        dropin.TrackParams(**kw)


def test_track_params_defaults():
    assert dropin.TrackParams() == dropin.TrackParams(streams=1, oks_threshold=0.5, max_age=30)
    dropin.TrackParams(streams=np.int64(4), oks_threshold=1, max_age=0)


def test_streams_need_tracking():
    fs = frames_stub.stream()
    with pytest.raises(ValueError, match="need tracking"):
        fs.submit(np.zeros((8, 8, 3), np.uint8), stream=1)
    with pytest.raises(ValueError, match="need tracking"):
        fs.submit_many([np.zeros((8, 8, 3), np.uint8)] * 2, streams=[0, 1])
    fs.submit(np.zeros((8, 8, 3), np.uint8), stream=0)
    fs.submit_many([np.zeros((8, 8, 3), np.uint8)] * 2, streams=[0, 0])
    assert [s for _, _, s in fs.launched] == [[0], [0, 0]]  # without tracking every stream index is 0


@pytest.mark.parametrize("streams,match", [([0, 3], "outside"), ([-1, 0], "outside"), ([0], "2 frames but 1"),
                                           ([0, 1.0], "int"), ([0, True], "int")])
def test_stream_indices_are_checked_before_anything_is_staged(streams, match):
    fs = frames_stub.stream(track=dropin.TrackParams(streams=3))
    with pytest.raises(ValueError, match=match):
        fs.submit_many([np.zeros((8, 8, 3), np.uint8), b"not a jpeg"], streams=streams)
    assert fs.launched == [] and fs.host_decodes == 0 and fs._next == 0
    if match != "2 frames but 1":
        with pytest.raises(ValueError, match=match):
            dropin._admit([np.zeros((8, 8, 3), np.uint8), b"not a jpeg"], streams, input_stage="device", device=0,
                          n_streams=3)


def test_stream_indices_reach_the_launcher_outside_the_key():
    fs = frames_stub.stream(track=dropin.TrackParams(streams=4))
    frames = [np.zeros((8, 8, 3), np.uint8), np.zeros((8, 16, 3), np.uint8)]
    fs.submit_many(frames, streams=[2, 3])
    fs.submit_many(frames, streams=[1, 1])
    fs.submit_many(frames)
    fs.submit(frames[0], stream=3)
    fs.submit(frames[0])
    keys = [frames_stub.keys(f) for _, f, _ in fs.launched]
    assert keys[0] == keys[1] == keys[2] and keys[3] == keys[4]
    assert [s for _, _, s in fs.launched] == [[2, 3], [1, 1], [0, 0], [3], [0]]
    _, streams, _ = dropin._admit(frames, [np.int64(2), 3], input_stage="device", device=0, n_streams=4)
    assert streams == [2, 3] and all(type(s) is int for s in streams)


def test_ids_need_tracking():
    fs = frames_stub.stream()
    fs._done = {0: ([], np.zeros(8, np.uint8), None)}
    with pytest.raises(ValueError, match="tracking"):
        fs.result(0, ids=True)
    assert fs.result(0) == []


def _golden_jpeg():
    with open(os.path.join(ROOT, "tests", "golden", "jpeg", "samp_420.jpg"), "rb") as f:
        return np.frombuffer(f.read(), np.uint8)


def test_flagged_jpeg_frame_is_posed_again_with_stream_minus_one():
    """_finish of a tick whose JPEG frame the device flagged: the frame is decoded with cv2 from the slot's bytes and
    posed again as a tick of one host image with stream -1 (its tracking step ran in the tick, as unobserved); its
    people get id -1."""
    import torch
    data = _golden_jpeg()
    rec_bytes = wire.record_bytes(17, dropin.CAP_ROWS)
    fs = frames_stub.stream(track=dropin.TrackParams(streams=2), slots=1)
    fs._g = types.SimpleNamespace(J=17, capR=dropin.CAP_ROWS)

    again_rec = np.zeros(1, wire.record_dtype(17, dropin.CAP_ROWS))
    again_rec[0]["n_persons"] = 2

    def launch(slot, frames, streams):
        fs.launched.append((slot, frames, streams))
        again = types.SimpleNamespace(rec_host=torch.from_numpy(again_rec.view(np.uint8).reshape(1, -1).copy()),
                                      heat=[torch.zeros(1)], paf=[torch.zeros(1)])
        return again, types.SimpleNamespace(synchronize=lambda: None)

    fs._launch = launch
    first = np.zeros(1, wire.record_dtype(17, dropin.CAP_ROWS))
    first[0]["n_persons"] = 1
    (frame,), _, _ = dropin._admit([data.tobytes()], [1], input_stage="device", device=0, n_streams=2)
    assert frame.key.source == "jpeg"
    tk = types.SimpleNamespace(
        rec_host=torch.from_numpy(first.view(np.uint8).reshape(1, -1).copy()), track=np.zeros(1, grouping.TRACK_FRAME),
        ids_host=torch.full((1, dropin.CAP_ROWS), 5, dtype=torch.int64), jpeg=[0], yuv=[],
        status_host=torch.tensor([grouping.JPEG_CORRUPT], dtype=torch.int32), up_host=torch.from_numpy(data.copy()),
        at={0: 0}, heat=[torch.zeros(1)], paf=[torch.zeros(1)], keys=(frame.key,), as_f64=True, held=[], images=[None])
    assert first.itemsize == rec_bytes
    fs._busy[0] = ([0], tk, types.SimpleNamespace(synchronize=lambda: None), [frame])
    dropin.FrameStream._finish(fs, 0)
    (_, (again,), streams), = fs.launched
    decoded = cv2.imdecode(data, cv2.IMREAD_COLOR)
    assert streams == [-1] and again.key == decoded.shape[:2] + ("image", None)
    assert np.array_equal(again.data, decoded) and again.decoded is again.data
    assert fs.host_decodes == 1
    people, _, ids = fs._done[0]
    assert len(people) == 2 and ids == [-1, -1]
