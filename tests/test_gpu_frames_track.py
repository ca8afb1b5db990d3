"""GPU: ``dropin.FrameStream(track=...)`` -- ``spg_track_frames`` recorded into each tick's graph -- against the port
(oracle/track_port.py) run on the same tickets' people in ticket order, per stream.  The frames are seeded pictures of
a few shapes; the stand-in network (frames_reference.py) answers each shape with its own people, so a stream that
changes shape sees its tracks go unmatched, age and drop, and new ones start."""
import glob
import os
import types

import numpy as np
import pytest

from frames_reference import MODEL_PARAMS, StandIn, _typed
from oracle import track_port as tp

pytestmark = pytest.mark.gpu

SHAPES = [(120, 160), (120, 160), (120, 160), (160, 120), (120, 160), (120, 160), (90, 120), (90, 120), (120, 160)]


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


def _params(env):
    return dict(env.skeleton.default_params(), scale_search=[1.0], rotation_search=[0.0])


def _port_ids(port, stream, people, record):
    status = int(np.asarray(record).view(np.uint32)[1])
    return port.step_people(stream, people, observed=status == 0)


def test_one_stream_equals_the_port(env):
    d = env.dropin
    track = d.TrackParams(oks_threshold=0.5, max_age=2)
    port = tp.Tracker(1, 0.5, 2)
    with d.FrameStream(StandIn(env.torch, env.synth), _params(env), MODEL_PARAMS, slots=2, track=track) as fs:
        seen = set()
        for frame in _frames(1):
            tk = fs.submit(frame)
            got, ids = fs.result(tk, detail=True, ids=True)
            assert ids == _port_ids(port, 0, got.people, got.record), f"ticket {tk}"
            assert len(ids) == len(got.people) > 0
            seen.update(ids)
        assert fs.captures == len({(k % 2, shape) for k, shape in enumerate(SHAPES)})  # later ticks replay graphs
    assert len(seen) > len(got.people)  # the shape changed: new tracks started


def test_submit_many_of_one_stream_equals_submits(env):
    d = env.dropin
    frames = _frames(2)
    out = []
    for many in (False, True):
        with d.FrameStream(StandIn(env.torch, env.synth), _params(env), MODEL_PARAMS, slots=2,
                           track=d.TrackParams(max_age=1)) as fs:
            if many:
                tickets = [t for k in range(0, len(frames), 3) for t in fs.submit_many(frames[k:k + 3])]
            else:
                tickets = [fs.submit(f) for f in frames]
            out.append([fs.result(t, ids=True) for t in tickets])
    assert [_typed(p) for p, _ in out[0]] == [_typed(p) for p, _ in out[1]]
    assert [i for _, i in out[0]] == [i for _, i in out[1]]


def test_interleaved_cameras_are_tracked_independently(env):
    d = env.dropin
    frames = _frames(3, SHAPES * 2)
    streams = [k % 3 for k in range(len(frames))]
    port = tp.Tracker(3, 0.4, 3)
    with d.FrameStream(StandIn(env.torch, env.synth), _params(env), MODEL_PARAMS, slots=3,
                       track=d.TrackParams(streams=3, oks_threshold=0.4, max_age=3)) as fs:
        tickets = []
        for k in range(0, len(frames), 6):
            tickets += fs.submit_many(frames[k:k + 6], streams=streams[k:k + 6])
        for tk, s in zip(tickets, streams):
            got, ids = fs.result(tk, detail=True, ids=True)
            assert ids == _port_ids(port, s, got.people, got.record), f"ticket {tk} (stream {s})"
    assert port.next_id[0] > 0 and port.next_id[1] > 0 and port.next_id[2] > 0


def test_replayed_graph_equals_the_warm_up(env):
    """The first tick of a key runs call by call; the same frames again replay its graph: the same ids, continued."""
    d = env.dropin
    frames = _frames(4, [(120, 160)] * 4)
    port = tp.Tracker(1, 0.5, 30)
    with d.FrameStream(StandIn(env.torch, env.synth), _params(env), MODEL_PARAMS, slots=1, track=d.TrackParams()) as fs:
        for rnd in range(3):
            got = [fs.result(t, detail=True, ids=True) for t in fs.submit_many(frames)]
            for r, ids in got:
                assert ids == _port_ids(port, 0, r.people, r.record), f"round {rnd}"
        assert fs.captures == 1


def test_crowded_frame_gets_minus_one_and_ages_its_stream(env):
    """The golden crowd's maps for one shape (as test_gpu_frames.py's crowded frame): its record has a capacity bit,
    its people come from the capacity-free tier with id -1, and its stream's tracks age as for an unobserved frame."""
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
    shapes = [(4 * h - 32, 4 * w)] * 2 + [(4 * h, 4 * w)] + [(4 * h - 32, 4 * w)] * 2
    port = tp.Tracker(1, 0.5, 30)
    with env.dropin.FrameStream(model, params, model_params, slots=1, track=env.dropin.TrackParams()) as fs:
        for k, frame in enumerate(_frames(5, shapes)):
            got, ids = fs.result(fs.submit(frame), detail=True, ids=True)
            status = int(env.wire.as_records(got.record, 17, env.dropin.CAP_ROWS)[0]["status"])
            assert bool(status & env.dropin.CAPACITY_BITS) == (k == 2), f"frame {k}: status {status:#x}"
            assert ids == _port_ids(port, 0, got.people, got.record), f"frame {k}"
            if k == 2:
                assert len(ids) > 0 and set(ids) == {-1}
                table = fs._tables.cpu().numpy().view(env.dropin.TRACK_TABLE).reshape(-1)[0]
                assert sorted(table["tracks"]["age"][table["tracks"]["live"] != 0]) == \
                    sorted(tr.age for tr in port.slots[0] if tr is not None)
                assert min(tr.age for tr in port.slots[0] if tr is not None) == 1


def test_without_tracking_nothing_changes(env):
    """track=None: the same captures and results as a stream with tracking, whose only extra launch is the tracking
    call in each warm-up run and capture; ids=True is refused."""
    d = env.dropin
    frames = _frames(6)
    out, launches = [], []
    for track in (None, d.TrackParams()):
        with d.FrameStream(StandIn(env.torch, env.synth), _params(env), MODEL_PARAMS, slots=2, track=track) as fs:
            people = [fs.result(fs.submit(f), detail=True) for f in frames]
            out.append((fs.captures, [_typed(r.people) for r in people], [bytes(r.record) for r in people]))
            launches.append(fs._g.launch_count)
            if track is None:
                with pytest.raises(ValueError, match="tracking"):
                    fs.result(fs.submit(frames[0]), ids=True)
                with pytest.raises(ValueError, match="tracking"):
                    fs.submit(frames[0], stream=1)
    assert out[0] == out[1]
    assert launches[1] - launches[0] == 2 * out[0][0]
