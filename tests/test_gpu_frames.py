"""GPU: ``dropin.FrameStream`` -- predict() + group() per frame replayed from one CUDA graph per slot and frame shape --
against ``dropin.predict`` followed by ``dropin.group`` on the same frames, and the library's refusal to grow a scratch
buffer inside a capture (``SPG_E_CAPTURE``).  The reference and the stand-in network are frames_reference.py's."""
import types

import numpy as np
import pytest

from frames_reference import MODEL_PARAMS, StandIn, _live, _reference, _typed

pytestmark = pytest.mark.gpu

SEARCHES = {"1 item": ([1.0], [0.0]), "2 scales": ([1.0, 0.5], [0.0]), "3 angles": ([1.0], [0.0, 30.0, -30.0])}
# three shapes, each seen again in the slot that captured it (slot = ticket % 2): replays of A and B in both slots' graphs
SHAPES = [(120, 160), (160, 120), (120, 160), (160, 120), (90, 120), (90, 120), (120, 160), (160, 120)]


@pytest.fixture()
def env(cuda_device):
    import torch
    from improved_body_parts_b200 import dropin, skeleton, synth, wire

    dropin.configure(device=0, limbs=dropin.LIMBS)
    yield types.SimpleNamespace(torch=torch, dropin=dropin, skeleton=skeleton, synth=synth, wire=wire, dev=cuda_device)
    dropin.configure(input_stage="host", variant="evaluate")


def _frames(seed, shapes=SHAPES):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, size=(H, W, 3), dtype=np.uint8) for H, W in shapes]


def _assert_frame(env, got, want, what):
    heat, paf, people, record = want
    assert _typed(got.people) == _typed(people), f"{what}: people"
    assert _live(env, got.record) == _live(env, record), f"{what}: wire record"
    for a, b, name in ((got.heat, heat, "heat"), (got.paf, paf, "paf")):
        x, y = a.tensor.cpu().numpy(), b.tensor.cpu().numpy()
        assert a.as_f64 == b.as_f64 and x.dtype == y.dtype and np.array_equal(x, y, equal_nan=True), f"{what}: {name}"


@pytest.mark.parametrize("search", list(SEARCHES))
@pytest.mark.parametrize("stage", ["device", "host"])
def test_frames_equal_predict_and_group(env, search, stage):
    scales, angles = SEARCHES[search]
    params = dict(env.skeleton.default_params(), scale_search=scales, rotation_search=angles)
    model = StandIn(env.torch, env.synth)
    persons = 0
    with env.dropin.FrameStream(model, params, MODEL_PARAMS, slots=2, input_stage=stage) as fs:
        for k, frame in enumerate(_frames(7)):
            got = fs.result(fs.submit(frame), detail=True)
            _assert_frame(env, got, _reference(env, frame, params, model, stage), f"frame {k} {frame.shape[:2]}")
            persons += len(got.people)
        # slot 0 saw two shapes and slot 1 two: one graph each, and every later frame of a shape replayed its graph
        assert fs.captures == 4
    assert persons > 0


def test_cuda_frames(env):
    t = env.torch
    params = dict(env.skeleton.default_params(), scale_search=[1.0, 0.5], rotation_search=[0.0, 30.0])
    model = StandIn(t, env.synth)
    frames = _frames(8, SHAPES[:4])
    with env.dropin.FrameStream(model, params, MODEL_PARAMS, slots=2) as fs:
        for k, frame in enumerate(frames):
            got = fs.result(fs.submit(t.from_numpy(frame).to(env.dev)), detail=True)
            _assert_frame(env, got, _reference(env, frame, params, model), f"frame {k}")
        assert fs.captures == 2


def test_more_frames_in_flight_than_slots(env):
    params = dict(env.skeleton.default_params(), scale_search=[1.0], rotation_search=[0.0])
    model = StandIn(env.torch, env.synth)
    frames = _frames(9) * 2
    want = [_reference(env, f, params, model)[2] for f in frames]
    with env.dropin.FrameStream(model, params, MODEL_PARAMS, slots=2) as fs:
        tickets = [fs.submit(f) for f in frames[:5]]  # three frames finished by later submits, two in flight
        got = {tk: fs.result(tk) for tk in reversed(tickets)}
        tickets += [fs.submit(f) for f in frames[5:]]
        got.update({tk: fs.result(tk) for tk in tickets[5:]})
        with pytest.raises(ValueError, match="unread"):
            fs.result(tickets[0])
    assert [_typed(got[tk]) for tk in tickets] == [_typed(w) for w in want]


def test_crowded_frame_takes_the_capacity_free_tier(env):
    """The golden crowd's maps as the network's answer for a 256 x 256 frame (its mirror the flipped, channel-permuted
    copy, so the flip ensemble gives them back at x4): the record says the frame is past the capacities and the people
    come from the tier, equal to dropin.group's."""
    import glob
    import os

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
    frames = _frames(10, [(4 * h, 4 * w)] * 3)
    with env.dropin.FrameStream(model, params, model_params, slots=1) as fs:
        for k, frame in enumerate(frames):
            got = fs.result(fs.submit(frame), detail=True)
            want = _reference(env, frame, params, model, model_params=model_params)
            status = int(env.wire.as_records(got.record, 17, env.dropin.CAP_ROWS)[0]["status"])
            assert status & env.dropin.CAPACITY_BITS, f"frame {k}: status {status:#x}"
            assert _typed(got.people) == _typed(want[2]), f"frame {k}"
            assert len(got.people) > 0


def test_demo_variant(env):
    d = env.dropin
    d.configure(variant="demo")
    params = dict(env.skeleton.default_params(), scale_search=[1.0, 0.5, 1.5], rotation_search=[0.0, 30.0])
    model = StandIn(env.torch, env.synth)
    with d.FrameStream(model, params, MODEL_PARAMS, slots=2) as fs:
        for k, frame in enumerate(_frames(11, SHAPES[:4])):
            got = fs.result(fs.submit(frame), detail=True)
            _assert_frame(env, got, _reference(env, frame, params, model), f"frame {k}")


def test_imhn_network_output_replayed_equals_eager(env):
    """imhn.IMHN (bf16 autocast, as imhn.Runner runs it without a graph of its own) inside the frame graph: the replayed
    frames' maps -- the network's output through the deterministic post-network stage -- equal the eager predict's."""
    from improved_body_parts_b200 import imhn
    runner = imhn.Runner(imhn.IMHN(nstack=1).init_like_reference_(0), device=env.dev, use_graph=False)

    def model(x):
        return [[runner(x)]]

    params = dict(env.skeleton.default_params(), scale_search=[1.0], rotation_search=[0.0])
    model_params = dict(MODEL_PARAMS, boxsize=128, max_downsample=64)  # the hourglass halves its input six times
    frames = _frames(12, [(128, 120)] * 3)
    with env.dropin.FrameStream(model, params, model_params, slots=1) as fs:
        for k, frame in enumerate(frames):
            got = fs.result(fs.submit(frame), detail=True)
            _assert_frame(env, got, _reference(env, frame, params, model, model_params=model_params), f"frame {k}")
        assert fs.captures == 1
        assert float(got.paf.tensor.abs().max()) > 0  # the network's output reached the maps


def test_a_captured_call_that_would_grow_is_refused(env):
    """spg_prenet with a rotated item needs the handle's scratch grid: inside a capture without spg_reserve_frame it
    returns SPG_E_CAPTURE before enqueueing anything, and the capture, the stream and the handle stay usable."""
    t, d = env.torch, env.dropin
    from improved_body_parts_b200 import grouping
    g = d._new_grouper(1)
    try:
        img = t.from_numpy(_frames(13, [(90, 120)])[0]).to(env.dev)
        kw = dict(max_downsample=32, pad_value=128)
        outs = [t.zeros((2, 96, 128, 3), dtype=t.float32, device=env.dev)]
        marker = t.zeros(1, device=env.dev)
        stream = t.cuda.Stream()
        graph = t.cuda.CUDAGraph()
        with t.cuda.graph(graph, stream=stream):
            marker.add_(1)
            with pytest.raises(grouping.GroupingError, match=rf"\({grouping.E_CAPTURE}\).*spg_reserve_frame"):
                g.prenet(img, [1.0], [30.0], out=outs, **kw)
        graph.replay()
        t.cuda.synchronize()
        assert float(marker) == 1.0
        assert g.reserve_frame(90, 120, [1.0], [30.0], max_downsample=32)
        assert not g.reserve_frame(90, 120, [1.0], [30.0], max_downsample=32)  # already reserved: nothing moves
        want = g.prenet(img, [1.0], [30.0], **kw)[0][0]
        graph = t.cuda.CUDAGraph()
        with t.cuda.graph(graph, stream=stream):
            g.prenet(img, [1.0], [30.0], out=outs, **kw)
        graph.replay()
        t.cuda.synchronize()
        assert t.equal(outs[0], want)
    finally:
        g.close()
