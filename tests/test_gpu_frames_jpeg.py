"""GPU: ``dropin.FrameStream`` fed JPEG bytes -- the decode recorded into each format's CUDA graph
(``spg_jpeg_decode_frame``) -- against the same stream fed ``cv2.imdecode`` of the bytes: results, maps and records equal,
the decoded frame byte for byte cv2's and ``spg_jpeg_decode_ragged``'s, one capture per slot and format, capacity growth,
the files left to cv2 and the library's refusal to grow inside a capture.  Inputs are ``cv2.imencode`` of seeded
``synth.photo`` images and the goldens under tests/golden/jpeg."""
import json
import os
import types

import numpy as np
import pytest

import make_jpeg_golden as mjg
from frames_reference import MODEL_PARAMS, StandIn, _live, _typed

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg")
MANIFEST = json.load(open(os.path.join(GOLDEN, "MANIFEST.json")))["cases"]
SEARCHES = {"1 scale": [1.0], "2 scales": [1.0, 0.5]}


@pytest.fixture()
def env(cuda_device):
    import torch
    from improved_body_parts_b200 import dropin, grouping, skeleton, synth, wire

    dropin.configure(device=0, limbs=dropin.LIMBS)
    yield types.SimpleNamespace(torch=torch, dropin=dropin, grouping=grouping, skeleton=skeleton, synth=synth, wire=wire,
                                dev=cuda_device)
    dropin.configure(input_stage="host", variant="evaluate")


def _golden(name):
    with open(os.path.join(GOLDEN, name + ".jpg"), "rb") as f:
        return f.read()


def _params(env, scales=(1.0,)):
    return dict(env.skeleton.default_params(), scale_search=list(scales), rotation_search=[0.0])


def _one_format(n=12, h=120, w=160):
    """``n`` JPEGs of one format (h x w, 4:2:0, no restart interval) that differ in content, quality (tables), Huffman
    tables (optimised), scan length around the first's and the length of a COM segment in front of the scan."""
    out = []
    for k in range(n):
        img = mjg.content(100 + k, h, w)
        data = mjg.encode(img, "420", quality=(75, 95, 40, 90, 60, 98)[k % 6], optimize=k % 3 == 1)
        if k % 4 == 2:
            data = mjg.insert_segment(data, 0xFE, bytes(range(256)) * (1 + k))  # the scan starts further on
        out.append(data)
    return out


def _assert_same(env, got, want, what):
    assert _typed(got.people) == _typed(want.people), f"{what}: people"
    assert _live(env, got.record) == _live(env, want.record), f"{what}: wire record"
    for a, b, name in ((got.heat, want.heat, "heat"), (got.paf, want.paf, "paf")):
        x, y = a.tensor.cpu().numpy(), b.tensor.cpu().numpy()
        assert a.as_f64 == b.as_f64 and x.dtype == y.dtype and np.array_equal(x, y, equal_nan=True), f"{what}: {name}"


def _decode(data):
    return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)


def _ragged(env, data):
    """spg_jpeg_decode_ragged of one file the parser accepts: (decode status, image)."""
    t, g = env.torch, env.grouping
    rec = g.jpeg_parse(data)
    assert int(rec["status"]) == g.JPEG_OK
    buf = t.from_numpy(np.frombuffer(data, np.uint8).copy()).to(env.dev)
    out = t.empty((int(rec["height"]), int(rec["width"]), 3), dtype=t.uint8, device=env.dev)
    st = t.full((1,), -1, dtype=t.int32, device=env.dev)
    arr = np.zeros(1, g.JPEG_RECORD)
    arr[0] = rec
    arr[0]["data"], arr[0]["out"], arr[0]["decode_status"] = buf.data_ptr(), out.data_ptr(), st.data_ptr()
    env.dropin._grouper().jpeg_decode(arr)
    return int(st.cpu()[0]), out.cpu().numpy()


def _pair(env, files, params, model=None, slots=2, check_image=True):
    """Every file through a stream of bytes and a stream of cv2.imdecode's frames: equal results; returns the bytes
    stream's counters (captures, host_decodes)."""
    model = model or StandIn(env.torch, env.synth)
    d = env.dropin
    with d.FrameStream(model, params, MODEL_PARAMS, slots=slots) as fs, \
            d.FrameStream(model, params, MODEL_PARAMS, slots=slots) as ref:
        for k, data in enumerate(files):
            got = fs.result(fs.submit(data), detail=True)
            want = ref.result(ref.submit(_decode(data)), detail=True)
            _assert_same(env, got, want, f"frame {k}")
            if check_image:
                assert got.image.dtype == np.uint8 and np.array_equal(got.image, _decode(data)), f"frame {k}: image"
        return fs.captures, fs.host_decodes


@pytest.mark.parametrize("search", list(SEARCHES))
def test_jpeg_frames_equal_the_cv2_path(env, search):
    files = _one_format()
    lengths = [env.grouping.jpeg_parse(f)["scan_length"] for f in files]
    assert min(lengths[1:]) < lengths[0] < max(lengths[1:])  # shorter and longer scans than the captured frame's
    assert len({env.grouping.jpeg_parse(f)["scan_offset"] for f in files}) > 1
    captures, host = _pair(env, files, _params(env, SEARCHES[search]))
    assert captures == 2  # one graph per slot for the one format: every later frame replayed it
    assert host == 0


def _formats():
    out = []
    for s, row in (("grey", 16), ("444", 16), ("422", 8), ("420", 8), ("440", 16)):  # row: MCUs per row, 122 wide
        img = mjg.content(7, 90, 122, grey=s == "grey")
        for rst in (0, 3, row):  # none, short intervals, one per MCU row
            out.append((f"{s} rst{rst}", mjg.encode(img, "420" if s == "grey" else s, quality=90, restart=rst)))
    out += [(n, _golden(n)) for n in MANIFEST if n.startswith("exif") and n.endswith("_II")]
    return out


def test_decode_is_bit_identical_to_cv2_and_ragged(env):
    files = _formats()
    with env.dropin.FrameStream(StandIn(env.torch, env.synth), _params(env), MODEL_PARAMS, slots=1) as fs:
        for name, data in files:
            for _ in range(2):  # the format's first frame runs call by call, the second replays its graph
                got = fs.result(fs.submit(data), detail=True)
                status, ragged = _ragged(env, data)
                assert status == 0, name
                assert np.array_equal(got.image, _decode(data)), name
                assert np.array_equal(got.image, ragged), name
        assert fs.host_decodes == 0
        assert fs.captures == len(files)


def test_a_longer_frame_grows_the_capacity(env):
    img = mjg.content(21, 480, 640)
    small = mjg.encode(img, "420", quality=30)
    small2 = mjg.encode(mjg.content(22, 480, 640), "420", quality=40)
    large = mjg.encode(img, "420", quality=100)
    assert len(small) < 1 << 16 < len(large) and len(small2) < 1 << 16
    captures, host = _pair(env, [small, small2, large, large, small], _params(env), slots=1)
    assert captures == 2  # the first frame's capture, and the one after the growth
    assert host == 0


def test_files_the_device_does_not_take_go_to_cv2(env):
    prog = mjg.encode(mjg.content(31, 120, 160), "420", quality=80, progressive=True)
    refused = [_golden("progressive"), _golden("samp_411"), _golden("fill_before_stuffing"), prog]
    flagged = [_golden(n) for n in MANIFEST if MANIFEST[n]["status"] in ("corrupt", "range")]
    assert len(flagged) >= 3
    for data in refused:
        assert int(env.grouping.jpeg_parse(data)["status"]) != 0
    for data in flagged:
        assert _ragged(env, data)[0] != 0
    files = [refused[0], flagged[0], refused[1], flagged[1], refused[2], flagged[2], refused[3]] + flagged[3:]
    captures, host = _pair(env, files, _params(env))
    assert host == len(files)
    with env.dropin.FrameStream(StandIn(env.torch, env.synth), _params(env), MODEL_PARAMS) as fs:
        with pytest.raises(ValueError, match="imdecode"):
            fs.submit(_golden("truncated"))  # refused by the parser, and cv2 cannot decode it either
        with pytest.raises(ValueError, match="empty"):
            fs.submit(b"")


def test_host_input_stage_decodes_with_cv2(env):
    files = _one_format(4)
    model = StandIn(env.torch, env.synth)
    d = env.dropin
    with d.FrameStream(model, _params(env), MODEL_PARAMS, input_stage="host") as fs, \
            d.FrameStream(model, _params(env), MODEL_PARAMS, input_stage="host") as ref:
        for k, data in enumerate(files):
            got = fs.result(fs.submit(bytearray(data)), detail=True)
            _assert_same(env, got, ref.result(ref.submit(_decode(data)), detail=True), f"frame {k}")
            assert np.array_equal(got.image, _decode(data))
        assert fs.host_decodes == len(files)


def test_mixed_input_kinds(env):
    t = env.torch
    files = _one_format(6)
    model = StandIn(t, env.synth)
    d = env.dropin
    with d.FrameStream(model, _params(env), MODEL_PARAMS, slots=2) as fs, \
            d.FrameStream(model, _params(env), MODEL_PARAMS, slots=2) as ref:
        tickets, wants = [], []
        for k, data in enumerate(files * 2):
            img = _decode(data)
            frame = (memoryview(data), img, t.from_numpy(img).to(env.dev))[k % 3]
            tickets.append(fs.submit(frame))
            wants.append(ref.result(ref.submit(img)))
            if k % 2:  # two frames in flight, then both read
                assert [_typed(fs.result(tk)) for tk in tickets] == [_typed(w) for w in wants]
                tickets, wants = [], []
        assert fs.host_decodes == 0


def test_crowded_jpeg_frame_takes_the_capacity_free_tier(env):
    import glob

    from conftest import ROOT
    from golden_io import load_case

    t, sk = env.torch, env.skeleton
    case = load_case(sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "crowd", "*.npz")))[0])
    h, w = case["heat"].shape[1:]
    net = np.zeros((2, 50, h, w), np.float32)
    net[0, :30], net[0, 30:48] = case["paf"], case["heat"]
    perm = list(sk.FLIP_PAF_ORD[:30]) + [30 + c for c in sk.FLIP_HEAT_ORD[:20]]
    net[1] = net[0][perm][:, :, ::-1]
    model = StandIn(t, env.synth, {(h, w): t.from_numpy(net).to(env.dev)})
    params = dict(case["params"], scale_search=[1.0], rotation_search=[0.0])
    model_params = dict(MODEL_PARAMS, boxsize=4 * h)
    d = env.dropin
    with d.FrameStream(model, params, model_params, slots=1) as fs, \
            d.FrameStream(model, params, model_params, slots=1) as ref:
        for k in range(3):
            data = mjg.encode(mjg.content(40 + k, 4 * h, 4 * w), "420", quality=85)
            got = fs.result(fs.submit(data), detail=True)
            want = ref.result(ref.submit(_decode(data)), detail=True)
            status = int(env.wire.as_records(got.record, 17, d.CAP_ROWS)[0]["status"])
            assert status & d.CAPACITY_BITS, f"frame {k}: status {status:#x}"
            assert _typed(got.people) == _typed(want.people) and len(got.people) > 0, f"frame {k}"
        assert fs.host_decodes == 0 and fs.captures == 1


def test_a_captured_decode_that_would_grow_is_refused(env):
    """spg_jpeg_decode_frame inside a capture without spg_jpeg_reserve_frame returns SPG_E_CAPTURE before enqueueing
    anything, and the capture, the stream and the handle stay usable; after the reserve the captured decode replays
    bit-identical to cv2."""
    t, g = env.torch, env.grouping
    data = mjg.encode(mjg.content(50, 96, 128), "420", quality=90)
    rec = g.jpeg_parse(data)
    grouper = env.dropin._new_grouper(1)
    try:
        cap = 1 << 16
        buf = t.zeros(cap, dtype=t.uint8, device=env.dev)
        buf[:len(data)] = t.from_numpy(np.frombuffer(data, np.uint8).copy()).to(env.dev)
        out = t.zeros((96, 128, 3), dtype=t.uint8, device=env.dev)
        st = t.full((1,), -1, dtype=t.int32, device=env.dev)
        fmt = np.zeros(1, g.JPEG_RECORD)
        fmt[0] = rec
        fmt[0]["data"], fmt[0]["out"], fmt[0]["decode_status"] = buf.data_ptr(), out.data_ptr(), st.data_ptr()
        drec = t.from_numpy(np.frombuffer(fmt.tobytes(), np.uint8).copy()).to(env.dev)
        marker = t.zeros(1, device=env.dev)
        stream = t.cuda.Stream()
        graph = t.cuda.CUDAGraph()
        with t.cuda.graph(graph, stream=stream):
            marker.add_(1)
            with pytest.raises(g.GroupingError, match=rf"\({g.E_CAPTURE}\).*reserve"):
                grouper.jpeg_decode_frame(drec.data_ptr(), fmt, cap)
        graph.replay()
        t.cuda.synchronize()
        assert float(marker) == 1.0 and int(st.cpu()[0]) == -1
        assert grouper.jpeg_reserve_frame(fmt, cap)
        assert not grouper.jpeg_reserve_frame(fmt, cap)  # already reserved: nothing moves
        graph = t.cuda.CUDAGraph()
        with t.cuda.graph(graph, stream=stream):
            grouper.jpeg_decode_frame(drec.data_ptr(), fmt, cap)
        graph.replay()
        t.cuda.synchronize()
        assert int(st.cpu()[0]) == 0 and np.array_equal(out.cpu().numpy(), _decode(data))
        # a frame whose scan exceeds the capacity decodes nothing and is flagged
        small = fmt.copy()
        small[0]["scan_length"] = cap + 1
        drec.copy_(t.from_numpy(np.frombuffer(small.tobytes(), np.uint8).copy()).to(env.dev))
        graph.replay()
        t.cuda.synchronize()
        assert int(st.cpu()[0]) == g.JPEG_CORRUPT
    finally:
        grouper.close()
