"""GPU: ``dropin.FrameStream.submit_many`` -- a tick of frames through one CUDA graph (``spg_jpeg_decode_frames``,
``spg_prenet_ragged``, one forward per input size, ``spg_postnet_ragged_items``, ``spg_group_ragged``) -- against
``dropin.predict`` + ``dropin.group`` of each frame (of ``cv2.imdecode``'s image for JPEG bytes): people by value and
type, wire records, maps and decoded images equal.  ``submit`` and a one-frame ``submit_many`` share one graph.  Then
the C calls under it: the ragged calls recorded after ``spg_reserve_frames`` equal the same calls made one by one,
refuse to grow inside a capture, and ``spg_jpeg_decode_frames`` equals ``spg_jpeg_decode_ragged`` and ``cv2.imdecode``.
The reference and the stand-in network, whose output for a sample does not depend on its batch, are
frames_reference.py's."""
import glob
import os
import types

import numpy as np
import pytest

import make_jpeg_golden as mjg
from frames_reference import MODEL_PARAMS, StandIn, _live, _reference, _typed

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg")
SEARCHES = {"1 item": ([1.0], [0.0]), "2 scales": ([1.0, 0.5], [0.0]), "3 angles": ([1.0], [0.0, 30.0, -30.0])}
SHAPES = [(120, 160), (160, 120), (90, 120), (120, 160)]


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


def _params(env, search="1 item"):
    scales, angles = SEARCHES[search]
    return dict(env.skeleton.default_params(), scale_search=scales, rotation_search=angles)


def _decode(data):
    return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)


def _frames(env, k, shapes, seed):
    """k frames cycling through shapes and the three kinds: numpy, CUDA, JPEG bytes (4:2:0, some with restarts)."""
    rng = np.random.default_rng(seed)
    out = []
    for j in range(k):
        H, W = shapes[j % len(shapes)]
        img = mjg.content(int(rng.integers(1 << 20)), H, W)
        kind = j % 3
        if kind == 0:
            out.append(img)
        elif kind == 1:
            out.append(env.torch.from_numpy(img).to(env.dev))
        else:
            out.append(mjg.encode(img, "420", quality=90, restart=3 if j % 2 else 0))
    return out


def _assert_same(env, got, want, what):
    assert _typed(got.people) == _typed(want.people), f"{what}: people"
    status = int(env.wire.as_records(want.record, 17, env.dropin.CAP_ROWS)[0]["status"])
    if status & env.dropin.CAPACITY_BITS:  # past the capacities the bounded record is unspecified but for its status
        assert int(env.wire.as_records(got.record, 17, env.dropin.CAP_ROWS)[0]["status"]) == status, f"{what}: status"
    else:
        assert _live(env, got.record) == _live(env, want.record), f"{what}: wire record"
    for a, b, name in ((got.heat, want.heat, "heat"), (got.paf, want.paf, "paf")):
        x, y = a.tensor.cpu().numpy(), b.tensor.cpu().numpy()
        assert a.as_f64 == b.as_f64 and x.dtype == y.dtype and np.array_equal(x, y, equal_nan=True), f"{what}: {name}"
    if want.image is not None:
        assert got.image is not None and np.array_equal(got.image, want.image), f"{what}: image"


def _want(env, frame, params, model, model_params=MODEL_PARAMS):
    """The reference's FrameResult for ``frame``: predict + group of the frame (of cv2.imdecode's image for JPEG
    bytes)."""
    image = _decode(frame) if isinstance(frame, bytes) else None
    heat, paf, people, record = _reference(env, frame if image is None else image, params, model,
                                           model_params=model_params)
    return env.dropin.FrameResult(people, record, heat, paf, image)


def _compare(env, ticks, params, model=None, slots=2, model_params=MODEL_PARAMS):
    """Every tick through submit_many, every frame through the reference: equal results.  Returns the tick stream and
    the number of persons seen."""
    model = model or StandIn(env.torch, env.synth)
    fs = env.dropin.FrameStream(model, params, model_params, slots=slots)
    persons = 0
    for n, frames in enumerate(ticks):
        tickets = fs.submit_many(frames)
        assert len(tickets) == len(frames) and len(set(tickets)) == len(frames)
        for j, (tk, frame) in enumerate(zip(tickets, frames)):
            got = fs.result(tk, detail=True)
            _assert_same(env, got, _want(env, frame, params, model, model_params), f"tick {n} frame {j}")
            persons += len(got.people)
    return fs, persons


@pytest.mark.parametrize("search", list(SEARCHES))
@pytest.mark.parametrize("k,shapes", [(1, SHAPES), (3, SHAPES), (16, SHAPES), (3, SHAPES[:1]), (16, SHAPES[:1])],
                         ids=["1 mixed", "3 mixed", "16 mixed", "3 one shape", "16 one shape"])
def test_ticks_equal_submit(env, search, k, shapes):
    frames = _frames(env, k, shapes, 11)
    again = _frames(env, k, shapes, 12)  # the same key: a replay of the tick's graph
    fs, persons = _compare(env, [frames, again, _frames(env, k, shapes, 13)], _params(env, search), slots=2)
    try:
        assert fs.captures == 2  # one per slot for the one tick key
        assert fs.host_decodes == 0
    finally:
        fs.close()
    assert persons > 0


def _formats():
    out = []
    for s in ("grey", "444", "422", "420", "440"):
        img = mjg.content(7, 90, 122, grey=s == "grey")
        for rst in (0, 3):
            out.append(mjg.encode(img, "420" if s == "grey" else s, quality=90, restart=rst))
    return out


def test_every_sampling_and_kind_in_one_tick(env):
    t = env.torch
    files = _formats()
    imgs = [mjg.content(60, 96, 128), mjg.content(61, 120, 160)]
    tick = files + [imgs[0], t.from_numpy(imgs[1]).to(env.dev)]
    fs, _ = _compare(env, [tick, tick], _params(env), slots=1)
    try:
        assert fs.captures == 1 and fs.host_decodes == 0
    finally:
        fs.close()


def test_refused_flagged_and_crowded_frames_in_one_tick(env):
    import json

    from conftest import ROOT
    from golden_io import load_case

    t, sk = env.torch, env.skeleton
    manifest = json.load(open(os.path.join(GOLDEN, "MANIFEST.json")))["cases"]
    case = load_case(sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "crowd", "*.npz")))[0])
    h, w = case["heat"].shape[1:]
    net = np.zeros((2, 50, h, w), np.float32)
    net[0, :30], net[0, 30:48] = case["paf"], case["heat"]
    perm = list(sk.FLIP_PAF_ORD[:30]) + [30 + c for c in sk.FLIP_HEAT_ORD[:20]]
    net[1] = net[0][perm][:, :, ::-1]
    model = StandIn(t, env.synth, {(h, w): t.from_numpy(net).to(env.dev)})
    params = dict(case["params"], scale_search=[1.0], rotation_search=[0.0])
    model_params = dict(MODEL_PARAMS, boxsize=4 * h)
    refused = [_golden("progressive"), _golden("samp_411")]
    flagged = [_golden(n) for n in manifest if manifest[n]["status"] in ("corrupt", "range")][:2]
    crowd = mjg.encode(mjg.content(40, 4 * h, 4 * w), "420", quality=85)
    plain = mjg.encode(mjg.content(41, 96, 128), "420", quality=85)
    tick = [refused[0], flagged[0], crowd, plain, refused[1], flagged[1]]
    fs = None
    try:
        fs, _ = _compare(env, [tick, tick], params, model=model, slots=1, model_params=model_params)
        assert fs.host_decodes == 2 * (len(refused) + len(flagged))
        tickets = fs.submit_many([crowd])
        status = int(env.wire.as_records(fs.result(tickets[0], detail=True).record, 17, env.dropin.CAP_ROWS)[0]["status"])
        assert status & env.dropin.CAPACITY_BITS
    finally:
        if fs is not None:
            fs.close()


def test_k_rises_and_an_older_key_returns(env):
    """A larger tick replaces the ticks' handle; a key seen before it then runs on the new handle.  Its call-by-call run
    must reserve the new handle's scratch first (and drop the graphs a moved buffer invalidates), or graphs captured
    since would replay a freed buffer.  Rotation search and two scales: the grid, the float64 sums and the JPEG
    scratch all take part."""
    large = mjg.encode(mjg.content(90, 480, 640), "420", quality=100)
    small = [mjg.encode(mjg.content(91 + k, 120, 160), "420", quality=90) for k in range(2)]
    assert len(large) > 1 << 16
    params = dict(_params(env), scale_search=[1.0, 0.5], rotation_search=[0.0, 30.0])
    ticks = [[large], small, [large], small, [large], small]
    fs, persons = _compare(env, ticks, params, slots=1)
    try:
        # [large] captured; [small, small] on the new handle; [large] again: reserved on the new handle, whose JPEG
        # scratch grows, which drops the small key's graph; [small, small] captured again; then both replay
        assert fs.captures == 4 and fs.host_decodes == 0
    finally:
        fs.close()
    assert persons > 0


def test_slot_reuse_with_unread_tickets(env):
    params = _params(env, "2 scales")
    model = StandIn(env.torch, env.synth)
    d = env.dropin
    ticks = [_frames(env, 3, SHAPES, 20 + n) for n in range(5)]
    with d.FrameStream(model, params, MODEL_PARAMS, slots=2) as fs:
        tickets = [fs.submit_many(tick) for tick in ticks]  # every slot reused with its tickets unread
        for tick, tks in zip(ticks, tickets):
            for frame, tk in zip(tick, tks):
                assert _typed(fs.result(tk)) == _typed(_want(env, frame, params, model).people)
        last = fs.submit_many(ticks[0])
        fs.submit_many(ticks[1])
        fs.submit_many(ticks[2])  # the slot of `last` now holds a later tick
        with pytest.raises(ValueError, match="later frame"):
            fs.result(last[0], detail=True)


def test_a_longer_jpeg_member_captures_again(env):
    img = mjg.content(21, 480, 640)
    small = mjg.encode(img, "420", quality=30)
    large = mjg.encode(img, "420", quality=100)
    other = mjg.encode(mjg.content(22, 120, 160), "420", quality=50)
    assert len(small) < 1 << 16 < len(large)
    fs, _ = _compare(env, [[small, other], [small, other], [large, other], [small, other]], _params(env), slots=1)
    try:
        assert fs.captures == 2 and fs.host_decodes == 0
    finally:
        fs.close()


@pytest.mark.parametrize("search", ["1 item", "3 angles"])
def test_submit_and_a_one_frame_tick_share_a_graph(env, search):
    """submit(a) and submit_many([a]) form one tick key: in one slot they share one graph, and with a rotation search
    (three items of one input size) the one-frame tick forwards each item alone, as predict and submit do."""
    params = _params(env, search)
    model = StandIn(env.torch, env.synth)
    a = mjg.content(30, 120, 160)
    want = _want(env, a, params, model)
    with env.dropin.FrameStream(model, params, MODEL_PARAMS, slots=1) as fs:
        got = [fs.result(fs.submit(a), detail=True), fs.result(fs.submit_many([a])[0], detail=True),
               fs.result(fs.submit(a), detail=True)]
        assert fs.captures == 1
    for n, g in enumerate(got):
        _assert_same(env, g, want, f"call {n}")


def test_submit_many_arguments(env):
    with env.dropin.FrameStream(StandIn(env.torch, env.synth), _params(env), MODEL_PARAMS) as fs:
        with pytest.raises(ValueError, match="at least one"):
            fs.submit_many([])
        with pytest.raises(ValueError, match="uint8 BGR"):
            fs.submit_many([np.zeros((4, 4), np.uint8)])
    with env.dropin.FrameStream(StandIn(env.torch, env.synth), _params(env), MODEL_PARAMS, input_stage="host") as fs:
        with pytest.raises(ValueError, match="input_stage"):
            fs.submit_many([np.zeros((8, 8, 3), np.uint8)])


# ---- the C calls under a tick ------------------------------------------------------------------------------------------
def _tick_calls(env, g, images, search, stream, rec, maps=None):
    """prenet_ragged -> stand-in forward per input size -> postnet_ragged_items (into ``maps`` when given) ->
    group_ragged with wire output."""
    t, d = env.torch, env.dropin
    params = _params(env, search)
    plan, buckets = d.plan_items([im.shape[:2] for im in images], params, MODEL_PARAMS)
    model = _tick_calls.model
    entries = [[None] * len(plan[0]) for _ in images]
    maps = maps or [(t.empty((1, 18, im.shape[0], im.shape[1]), dtype=t.float32, device=env.dev),
                     t.empty((1, 30, im.shape[0], im.shape[1]), dtype=t.float32 if len(plan[0]) == 1 else t.float64,
                             device=env.dev)) for im in images]
    with t.cuda.stream(stream):
        for (Hp, Wp), ms in buckets.items():
            x = _tick_calls.inputs.setdefault((len(ms), Hp, Wp), t.empty((2 * len(ms), Hp, Wp, 3), device=env.dev))
            pairs = g.prenet_ragged([(images[i], plan[i][tt][0], plan[i][tt][2]) for i, tt in ms], max_downsample=32,
                                    pad_value=128, out=[x[2 * k:2 * k + 2] for k in range(len(ms))])
            out = model(x)[-1][0]
            for k, (i, tt) in enumerate(ms):
                entries[i][tt] = (out[2 * k:2 * k + 2], pairs[k][1], pairs[k][2])
        g.postnet_ragged_items([(e, im.shape[:2]) for e, im in zip(entries, images)], outs=maps)
        g.set_wire_output(rec.data_ptr())
        try:
            g.group_ragged(maps, [im.shape[0] for im in images], d._params(params), paf_as_f64=len(plan[0]) == 1)
        finally:
            g.set_wire_output(None)
    return maps


def test_ragged_calls_recorded_after_reserve_frames(env):
    search = "3 angles"  # rotated items: both the scratch grid and the float64 sums must be reserved
    t, gm, d = env.torch, env.grouping, env.dropin
    images = [t.from_numpy(mjg.content(70 + k, *s)).to(env.dev) for k, s in enumerate(SHAPES[:3])]
    _tick_calls.model, _tick_calls.inputs = StandIn(t, env.synth), {}
    params = _params(env, search)
    plan, _ = d.plan_items([im.shape[:2] for im in images], params, MODEL_PARAMS)
    members = [(im.shape[0], im.shape[1], it[0], it[2]) for im, items in zip(images, plan) for it in items]
    g = d._new_grouper(len(images))
    try:
        stream = t.cuda.Stream()
        rec = t.zeros((len(images), g.wire_record_bytes()), dtype=t.uint8, device=env.dev)
        eager = [m.clone() for pair in _tick_calls(env, g, images, search, stream, rec) for m in pair]  # warm-up too
        stream.synchronize()
        eager_rec = rec.cpu().numpy()
        # a fresh handle: without the reserve a captured call that would grow returns SPG_E_CAPTURE, enqueues nothing
        g.close()
        g = d._new_grouper(len(images))
        marker = t.zeros(1, device=env.dev)
        graph = t.cuda.CUDAGraph()
        with t.cuda.graph(graph, stream=stream):
            marker.add_(1)
            with pytest.raises(gm.GroupingError, match=rf"\({gm.E_CAPTURE}\).*rotated items"):
                _tick_calls(env, g, images, search, stream, rec)
        graph.replay()
        t.cuda.synchronize()
        assert float(marker) == 1.0
        # the grid grown by an eager prenet_ragged, the float64 sums not: postnet_ragged_items refuses in the capture
        # and writes nothing, and the capture stays usable
        with t.cuda.stream(stream):
            g.prenet_ragged([(images[i], items[tt][0], items[tt][2]) for i, items in enumerate(plan)
                             for tt in range(len(items))], max_downsample=32, pad_value=128)
        stream.synchronize()
        sentinel = [(t.full_like(h, float("nan")), t.full_like(p, float("nan"))) for h, p in
                    zip(eager[0::2], eager[1::2])]
        graph = t.cuda.CUDAGraph()
        with t.cuda.graph(graph, stream=stream):
            marker.add_(1)
            with pytest.raises(gm.GroupingError, match=rf"\({gm.E_CAPTURE}\).*keypoint sums"):
                _tick_calls(env, g, images, search, stream, rec, maps=sentinel)
        graph.replay()
        t.cuda.synchronize()
        assert float(marker) == 2.0
        assert all(bool(m.isnan().all()) for pair in sentinel for m in pair)
        # group_ragged allocates nothing: captured on a handle never reserved, it replays to the eager records
        g3 = d._new_grouper(len(images))
        try:
            rec3 = t.zeros_like(rec)
            graph = t.cuda.CUDAGraph()
            with t.cuda.graph(graph, stream=stream):
                g3.set_wire_output(rec3.data_ptr())
                try:
                    g3.group_ragged(list(zip(eager[0::2], eager[1::2])), [im.shape[0] for im in images],
                                    d._params(params), paf_as_f64=False)
                finally:
                    g3.set_wire_output(None)
            graph.replay()
            t.cuda.synchronize()
            assert np.array_equal(rec3.cpu().numpy(), eager_rec)
        finally:
            g3.close()
        assert g.reserve_frames(members, len(plan[0]), max_downsample=32)
        assert not g.reserve_frames(members, len(plan[0]), max_downsample=32)
        rec.zero_()
        graph = t.cuda.CUDAGraph()
        with t.cuda.graph(graph, stream=stream):
            maps = _tick_calls(env, g, images, search, stream, rec)
        graph.replay()
        t.cuda.synchronize()
        got = [m for pair in maps for m in pair]
        assert all(np.array_equal(a.cpu().numpy(), b.cpu().numpy(), equal_nan=True) for a, b in zip(got, eager))
        assert np.array_equal(rec.cpu().numpy(), eager_rec)
        with pytest.raises(gm.GroupingError, match="max_batch"):
            g.reserve_frames(members * 2, len(plan[0]), max_downsample=32)
    finally:
        g.close()


def _decode_setup(env, files, caps):
    t, g = env.torch, env.grouping
    recs = [g.jpeg_parse(f) for f in files]
    assert all(int(r["status"]) == g.JPEG_OK for r in recs)
    bufs = [t.zeros(c, dtype=t.uint8, device=env.dev) for c in caps]
    for b, f in zip(bufs, files):
        n = min(len(f), b.numel())
        b[:n] = t.from_numpy(np.frombuffer(f, np.uint8)[:n].copy()).to(env.dev)
    outs = [t.zeros((int(r["height"]), int(r["width"]), 3), dtype=t.uint8, device=env.dev) for r in recs]
    st = t.full((len(files),), -1, dtype=t.int32, device=env.dev)
    fmt = np.zeros(len(files), g.JPEG_RECORD)
    for i, r in enumerate(recs):
        fmt[i] = r
        fmt[i]["data"], fmt[i]["out"], fmt[i]["decode_status"] = bufs[i].data_ptr(), outs[i].data_ptr(), st.data_ptr() + 4 * i
    drec = t.from_numpy(np.frombuffer(fmt.tobytes(), np.uint8).copy()).to(env.dev)
    return fmt, drec, outs, st, bufs  # the caller keeps bufs alive: the records point into them


def test_decode_frames_equals_ragged_and_cv2(env):
    t = env.torch
    files = _formats() + [_golden(n) for n in ("exif6_MM", "dqt16", "rst3")]
    caps = [(1 << 16) + 4096 * (i % 3) for i in range(len(files))]
    fmt, drec, outs, st, bufs = _decode_setup(env, files, caps)
    g = env.dropin._new_grouper(1)
    try:
        assert g.jpeg_reserve_frames(fmt, caps)
        stream = t.cuda.Stream()
        graph = t.cuda.CUDAGraph()
        with t.cuda.graph(graph, stream=stream):
            g.jpeg_decode_frames(drec.data_ptr(), fmt, caps)
        graph.replay()
        t.cuda.synchronize()
        assert st.cpu().tolist() == [0] * len(files)
        ragged = np.zeros(len(files), env.grouping.JPEG_RECORD)
        routs = [t.zeros_like(o) for o in outs]
        rst = t.full((len(files),), -1, dtype=t.int32, device=env.dev)
        ragged[:] = fmt
        for i in range(len(files)):
            ragged[i]["out"], ragged[i]["decode_status"] = routs[i].data_ptr(), rst.data_ptr() + 4 * i
        g.jpeg_decode(ragged)
        t.cuda.synchronize()
        assert rst.cpu().tolist() == [0] * len(files)
        for i, f in enumerate(files):
            assert np.array_equal(outs[i].cpu().numpy(), _decode(f)), i
            assert np.array_equal(outs[i].cpu().numpy(), routs[i].cpu().numpy()), i
    finally:
        g.close()


def test_a_member_past_its_capacity_is_flagged_alone(env):
    t = env.torch
    big = mjg.encode(mjg.content(80, 480, 640), "420", quality=100)
    files = [_formats()[3], big, _formats()[1]]
    caps = [1 << 16, 1 << 16, 1 << 16]
    assert env.grouping.jpeg_parse(big)["scan_length"] > caps[1]
    fmt, drec, outs, st, bufs = _decode_setup(env, files, caps)
    g = env.dropin._new_grouper(1)
    try:
        g.jpeg_reserve_frames(fmt, caps)
        g.jpeg_decode_frames(drec.data_ptr(), fmt, caps)
        t.cuda.synchronize()
        assert st.cpu().tolist() == [0, env.grouping.JPEG_CORRUPT, 0]
        assert np.array_equal(outs[0].cpu().numpy(), _decode(files[0]))
        assert np.array_equal(outs[2].cpu().numpy(), _decode(files[2]))
    finally:
        g.close()
