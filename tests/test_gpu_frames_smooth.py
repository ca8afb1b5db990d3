"""GPU: ``dropin.FrameStream(track=..., smooth=...)`` -- ``spg_smooth_frames`` recorded into each tick's graph after the
tracking -- against the tracking port and the smoothing port (oracle/track_port.py, oracle/smooth_port.py) run on the
same tickets' records in submit order, per stream, with single-frame and K-frame ticks, several streams and two slots
in flight.  Without ``smooth`` the ids, people, captures and launches are those of tracking alone."""
import types

import numpy as np
import pytest

from frames_reference import MODEL_PARAMS, StandIn, _typed
from oracle import smooth_port as sp
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


class Ports:
    """The tracking and smoothing ports, stepped ticket by ticket in submit order."""

    def __init__(self, env, streams, track, smooth):
        self.env = env
        self.track = tp.Tracker(streams, track.oks_threshold, track.max_age)
        self.smooth = sp.Smoother(streams, smooth.min_cutoff, smooth.beta, smooth.d_cutoff)

    def check(self, got, ids, stream, t, what):
        """``got``: ``result(ticket, detail=True, ids=True, smoothed=True)``'s FrameResult, whose record is raw."""
        d = self.env.dropin
        rec = self.env.wire.as_records(got.record, 17, d.CAP_ROWS)[0]
        raw = self.env.wire.people_of(rec)
        want_ids = self.track.step_record(stream, rec)
        assert ids == want_ids, f"{what}: ids"
        xy = self.smooth.step_record(stream, rec, want_ids, t)
        want = d._smoothed_people(raw, rec, xy)
        assert _typed(got.people) == _typed(want), f"{what}: smoothed people"
        return raw, want


def test_one_stream_of_single_frame_ticks(env):
    d = env.dropin
    track, smooth = d.TrackParams(oks_threshold=0.5, max_age=2), d.SmoothParams(min_cutoff=0.5, beta=2.0, rate=25.0)
    ports = Ports(env, 1, track, smooth)
    moved = 0
    with d.FrameStream(StandIn(env.torch, env.synth), _params(env), MODEL_PARAMS, slots=2, track=track,
                       smooth=smooth) as fs:
        frames = _frames(1)
        tickets = [fs.submit(f) for f in frames[:2]]  # two slots in flight: each result read one submit later
        t = 0.0
        for k, tk in enumerate(tickets):  # a frame without a time comes 1 / rate after its stream's previous one
            got, ids = fs.result(tk, detail=True, ids=True, smoothed=True)
            if k + 2 < len(frames):
                tickets.append(fs.submit(frames[k + 2]))
            raw, smoothed = ports.check(got, ids, 0, t, f"ticket {tk}")
            t += 1.0 / 25.0
            assert len(ids) > 0
            moved += _typed(raw) != _typed(smoothed)
        assert len(tickets) == len(frames)
        assert fs.captures == len({(k % 2, shape) for k, shape in enumerate(SHAPES)})
    assert moved > 0  # continued tracks were filtered


def test_k_frame_ticks_of_several_streams(env):
    d = env.dropin
    frames = _frames(3, SHAPES * 2)
    streams = [k % 3 for k in range(len(frames))]
    rng = np.random.default_rng(4)
    clock, times = [0.0] * 3, []
    for s in streams:
        clock[s] += float(rng.uniform(0.01, 0.2))
        times.append(clock[s])
    track, smooth = d.TrackParams(streams=3, oks_threshold=0.4, max_age=3), d.SmoothParams(beta=0.5)
    ports = Ports(env, 3, track, smooth)
    with d.FrameStream(StandIn(env.torch, env.synth), _params(env), MODEL_PARAMS, slots=2, track=track,
                       smooth=smooth) as fs:
        tickets = []
        for k in range(0, len(frames), 6):  # two ticks in flight before the first read
            tickets += fs.submit_many(frames[k:k + 6], streams=streams[k:k + 6], times=times[k:k + 6])
        for tk, s, t in zip(tickets, streams, times):
            got, ids = fs.result(tk, detail=True, ids=True, smoothed=True)
            ports.check(got, ids, s, t, f"ticket {tk} (stream {s})")
    assert all(c > 0 for c in ports.smooth.clock)


def test_replayed_graph_continues_the_filters(env):
    d = env.dropin
    frames = _frames(5, [(120, 160)] * 3)
    track, smooth = d.TrackParams(), d.SmoothParams()
    ports = Ports(env, 1, track, smooth)
    with d.FrameStream(StandIn(env.torch, env.synth), _params(env), MODEL_PARAMS, slots=1, track=track,
                       smooth=smooth) as fs:
        t = 0.0
        for rnd in range(3):
            for k, tk in enumerate(fs.submit_many(frames)):
                got, ids = fs.result(tk, detail=True, ids=True, smoothed=True)
                ports.check(got, ids, 0, t, f"round {rnd}, frame {k}")
                t += 1.0 / 30.0
        assert fs.captures == 1


def test_smoothing_changes_nothing_else(env):
    """track + smooth against track alone on the same frames: the same ids, raw people, records and captures; the only
    extra launch is the smoothing call in each warm-up run and capture."""
    d = env.dropin
    frames = _frames(6)
    out, launches = [], []
    for smooth in (None, d.SmoothParams()):
        with d.FrameStream(StandIn(env.torch, env.synth), _params(env), MODEL_PARAMS, slots=2, track=d.TrackParams(),
                           smooth=smooth) as fs:
            got = [fs.result(fs.submit(f), detail=True, ids=True) for f in frames]
            out.append((fs.captures, [_typed(r.people) for r, _ in got], [bytes(r.record) for r, _ in got],
                        [i for _, i in got]))
            launches.append(fs._g.launch_count)
            if smooth is None:
                with pytest.raises(ValueError, match="smoothing"):
                    fs.result(fs.submit(frames[0]), smoothed=True)
                with pytest.raises(ValueError, match="smoothing"):
                    fs.submit(frames[0], t=1.0)
    assert out[0] == out[1]
    assert launches[1] - launches[0] == 2 * out[0][0]
