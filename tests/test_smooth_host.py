"""CPU: ``FrameStream`` smoothing before it touches a device -- the dtypes and declaration of ``spg_smooth_frames`` and
its refusal without a handle, ``SmoothParams`` and frame-time checks (no ticket on error), the times that reach the
launcher, ``smooth`` without ``track`` and ``smoothed=True`` without ``smooth``, and how smoothed people are formed."""
import os
import re

import frames_stub
import numpy as np
import pytest

from improved_body_parts_b200 import dropin, grouping, wire

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IMG = np.zeros((8, 8, 3), np.uint8)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return grouping.load_library()


def test_smooth_frames_is_declared_and_the_dtypes_are_pinned():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "spgroup.h")).read(), flags=re.S)
    m = re.search(r"int\s+spg_smooth_frames\s*\(([^)]*)\)\s*;", src)
    assert [" ".join(p.split()) for p in m.group(1).split(",")] == [
        "spg_handle *h", "const spg_smooth_frame *frames", "int32_t n", "spg_smooth_table *tables", "int32_t n_tables",
        "double min_cutoff", "double beta", "double d_cutoff", "void *stream"]
    assert grouping.SMOOTH_SLOT.itemsize == 704 and grouping.SMOOTH_SLOT.fields["joint"][1] == 24
    assert grouping.SMOOTH_TABLE.itemsize == 16 + 128 * 704 and grouping.SMOOTH_TABLE.fields["slots"][1] == 16
    assert grouping.SMOOTH_FRAME.itemsize == 40
    assert [grouping.SMOOTH_FRAME.fields[f][1] for f in ("record", "stream", "ids", "time", "xy")] == [0, 8, 16, 24, 32]


def test_smooth_frames_without_a_handle_is_invalid(lib):
    f = np.zeros(1, grouping.SMOOTH_FRAME)
    assert lib.spg_smooth_frames(None, f.ctypes.data, 1, None, 1, 1.0, 1.0, 1.0, None) == -1


@pytest.mark.parametrize("kw,match", [
    (dict(min_cutoff=0.0), "min_cutoff"), (dict(min_cutoff=-1.0), "min_cutoff"), (dict(min_cutoff=float("inf")), "min_cutoff"),
    (dict(d_cutoff=0), "d_cutoff"), (dict(d_cutoff=float("nan")), "d_cutoff"), (dict(beta=-0.1), "beta"),
    (dict(beta=float("nan")), "beta"), (dict(beta=True), "beta"), (dict(rate=0.0), "rate"), (dict(rate="30"), "rate")])
def test_smooth_params_are_checked(kw, match):
    with pytest.raises(ValueError, match=match):
        dropin.SmoothParams(**kw)


def test_smooth_params_defaults():
    assert dropin.SmoothParams() == dropin.SmoothParams(min_cutoff=1.0, beta=1.0, d_cutoff=1.0, rate=30.0)
    dropin.SmoothParams(min_cutoff=np.float32(0.5), beta=0, d_cutoff=np.int64(2), rate=60)


def test_smooth_needs_track():
    with pytest.raises(ValueError, match="needs track"):
        dropin.FrameStream(None, {}, {"stride": 4}, smooth=dropin.SmoothParams())
    with pytest.raises(ValueError, match="SmoothParams"):
        dropin.FrameStream(None, {}, {"stride": 4}, track=dropin.TrackParams(), smooth=dict(beta=1.0))


def _smoothing(streams=2, rate=30.0):
    fs = frames_stub.stream(track=dropin.TrackParams(streams=streams))
    fs._smooth, fs._times, fs._smoothed = dropin.SmoothParams(rate=rate), [None] * streams, {}
    return fs


def _times(fs):
    return [[f.t for f in frames] for _, frames, _ in fs.launched]


def test_missing_times_follow_the_rate_per_stream():
    fs = _smoothing(rate=25.0)
    fs.submit(IMG)
    fs.submit(IMG)
    fs.submit(IMG, stream=1, t=10.0)
    fs.submit_many([IMG] * 3, streams=[0, 1, 0], times=[None, None, 5.0])
    fs.submit(IMG, t=5.5)
    assert _times(fs) == [[0.0], [0.04], [10.0], [0.08, 10.04, 5.0], [5.5]]
    assert fs._times == [5.5, 10.04]


@pytest.mark.parametrize("times,match", [
    ([1.5, float("nan")], "finite"), ([1.5, float("inf")], "finite"), ([True, None], "finite"), (["1", None], "finite"),
    ([2.0, 2.0], "not later"), ([2.0, 1.5], "not later"), ([0.5, None], "not later"), ([1.0], "2 frames but 1 times")])
def test_times_are_checked_before_anything_is_staged(times, match):
    fs = _smoothing()
    fs.submit(IMG, t=1.0)
    with pytest.raises(ValueError, match=match):
        fs.submit_many([IMG, b"not a jpeg"], times=times)
    assert len(fs.launched) == 1 and fs._next == 1 and fs.host_decodes == 0 and fs._times == [1.0, None]
    with pytest.raises(ValueError, match="not later"):
        fs.submit(IMG, t=1.0)
    assert fs._next == 1
    fs.submit_many([IMG, IMG], streams=[0, 1], times=[1.25, 1.0])  # streams keep their own clocks
    assert _times(fs)[-1] == [1.25, 1.0]


def test_times_need_smoothing():
    for fs in (frames_stub.stream(), frames_stub.stream(track=dropin.TrackParams())):
        with pytest.raises(ValueError, match="needs smoothing"):
            fs.submit(IMG, t=0.0)
        with pytest.raises(ValueError, match="needs smoothing"):
            fs.submit_many([IMG], times=[0.0])
        fs.submit_many([IMG], times=[None])
        assert _times(fs) == [[None]]


def test_smoothed_needs_smoothing():
    fs = frames_stub.stream(track=dropin.TrackParams())
    fs._done = {0: ([], np.zeros(8, np.uint8), [])}
    with pytest.raises(ValueError, match="smoothing"):
        fs.result(0, smoothed=True)
    assert fs.result(0, ids=True) == ([], [])


def test_smoothed_people_replace_present_joints_only():
    rec = np.zeros(1, wire.record_dtype(17, 4))[0]
    rec["n_persons"] = 2
    rec["rows"]["xy"][:2] = np.arange(2 * 17 * 2).reshape(2, 17, 2) + 0.5
    rec["rows"]["present"][:2] = [0b101, (1 << 17) - 1]
    rec["rows"]["score"][:2] = [0.25, 0.75]
    xy = -np.arange(4 * 17 * 2, dtype=np.float64).reshape(4, 17, 2)
    people = wire.people_of(rec)
    got = dropin._smoothed_people(people, rec, xy)
    assert [s for _, s in got] == [0.25, 0.75]
    assert got[0][0][0] == (xy[0, 0, 0], xy[0, 0, 1]) and got[0][0][2] == (xy[0, 2, 0], xy[0, 2, 1])
    assert got[0][0][1] == (0, 0) and type(got[0][0][1][0]) is int
    assert got[1][0] == [tuple(v) for v in xy[1]] and all(type(v) is np.float64 for pt in got[1][0] for v in pt)


def test_smoothed_result_and_raw_result():
    fs = _smoothing()
    people = [([(np.float64(1.0), np.float64(2.0))] + [(0, 0)] * 16, np.float64(0.5))]
    smoothed = [([(np.float64(1.5), np.float64(2.5))] + [(0, 0)] * 16, np.float64(0.5))]
    for tk in (0, 1):
        fs._done[tk] = (people, np.zeros(8, np.uint8), [3])
        fs._smoothed[tk] = smoothed
    assert fs.result(0, ids=True, smoothed=True) == (smoothed, [3])
    assert fs.result(1) == people and fs._smoothed == {}
