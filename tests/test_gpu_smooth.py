"""GPU: ``spg_smooth_frames`` called directly on seeded wire records, ids and times, against the port
(oracle/smooth_port.py) after every call: every output coordinate and every table field equal bit for bit (float64
compared as integers).  The cases cover several streams and several frames of one stream per call, skipped frames and
id -1, new, absent and non-finite joints, irregular (also equal and decreasing) times, eviction past 128 ids, repeated
ids, and a call recorded into a CUDA graph and replayed with new contents."""
import types

import numpy as np
import pytest

from oracle import smooth_port as sp

pytestmark = pytest.mark.gpu

BASE = np.array([[20, 10], [18, 8], [22, 8], [15, 9], [25, 9], [10, 25], [30, 25], [8, 45], [32, 45], [6, 60], [34, 60],
                 [14, 60], [26, 60], [13, 80], [27, 80], [12, 100], [28, 100]], np.float64)
SENTINEL = -12345.5


@pytest.fixture(scope="module")
def env(cuda_device):
    import torch
    from improved_body_parts_b200 import dropin, grouping, wire

    g = dropin._new_grouper(1, 0)
    yield types.SimpleNamespace(torch=torch, grouping=grouping, wire=wire, g=g, dev=cuda_device)
    g.close()


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


class Run:
    """Device tables for ``streams`` streams and the port beside them."""

    def __init__(self, env, streams, min_cutoff=1.0, beta=1.0, d_cutoff=1.0):
        t = env.torch
        self.env, self.rows, self.params = env, env.g.capR, (min_cutoff, beta, d_cutoff)
        self.tables = t.zeros((streams, env.grouping.SMOOTH_TABLE.itemsize), dtype=t.uint8, device=env.dev)
        self.port = sp.Smoother(streams, min_cutoff, beta, d_cutoff)

    def buffers(self, n):
        """Device inputs and outputs for a call of n frames, and its SMOOTH_FRAME array."""
        env, t = self.env, self.env.torch
        b = types.SimpleNamespace(
            rec=t.zeros((n, env.g.wire_record_bytes()), dtype=t.uint8, device=env.dev),
            streams=t.zeros(n, dtype=t.int32, device=env.dev), ids=t.zeros((n, self.rows), dtype=t.int64, device=env.dev),
            times=t.zeros(n, dtype=t.float64, device=env.dev),
            xy=t.full((n, self.rows, 17, 2), SENTINEL, dtype=t.float64, device=env.dev))
        b.frames = np.zeros(n, env.grouping.SMOOTH_FRAME)
        for j in range(n):
            f = b.frames[j]
            f["record"], f["stream"] = b.rec[j].data_ptr(), b.streams.data_ptr() + 4 * j
            f["ids"], f["time"], f["xy"] = b.ids[j].data_ptr(), b.times.data_ptr() + 8 * j, b.xy[j].data_ptr()
        return b

    def fill(self, b, frames):
        """frames: [(stream, record, ids, time)] into the buffers (the output back to the sentinel)."""
        t = self.env.torch
        recs = np.stack([r for _, r, _, _ in frames])
        b.rec.copy_(t.from_numpy(recs.view(np.uint8).reshape(len(frames), -1).copy()))
        b.streams.copy_(t.tensor([s for s, _, _, _ in frames], dtype=t.int32))
        ids = np.full((len(frames), self.rows), -9, np.int64)
        for j, (_, _, i, _) in enumerate(frames):
            ids[j, :len(i)] = i
        b.ids.copy_(t.from_numpy(ids))
        b.times.copy_(t.tensor([tm for _, _, _, tm in frames], dtype=t.float64))
        b.xy.fill_(SENTINEL)

    def call(self, frames):
        b = self.buffers(len(frames))
        self.fill(b, frames)
        self.env.g.smooth_frames(b.frames, self.tables.data_ptr(), self.tables.shape[0], *self.params)
        self.check(b, frames)

    def check(self, b, frames):
        got = b.xy.cpu().numpy()
        for j, (s, rec, ids, tm) in enumerate(frames):
            n = int(rec["n_persons"])
            if s < 0:
                want = np.array(rec["rows"]["xy"][:n], np.float64)
            else:
                want = self.port.step_record(s, rec, ids, tm)
            assert np.array_equal(_bits(got[j, :n]), _bits(want)), f"frame {j} (stream {s}): smoothed joints"
            assert (got[j, n:] == SENTINEL).all(), f"frame {j}: rows past n_persons written"
        self.check_tables()

    def check_tables(self):
        got = self.tables.cpu().numpy().view(self.env.grouping.SMOOTH_TABLE).reshape(-1)
        for s, table in enumerate(self.port.slots):
            assert int(got[s]["clock"]) == self.port.clock[s], f"stream {s}: clock"
            for k, sl in enumerate(table):
                d = got[s]["slots"][k]
                if sl is None:
                    assert not d.tobytes().strip(b"\0"), f"stream {s} slot {k}: an unclaimed slot is zero"
                    continue
                assert (int(d["live"]), int(d["id"]), int(d["last"]), int(d["mask"])) == (1, sl.id, sl.last, sl.mask), \
                    f"stream {s} slot {k}"
                assert np.array_equal(_bits(d["joint"]), _bits(sl.joint)), f"stream {s} slot {k}: joint state"


class World:
    """``M`` people with fixed ids, each drifting a few pixels per frame; a frame shows some of them in a shuffled row
    order with joint noise, missing joints and, at ``nan`` rate, NaN or infinite coordinates."""

    def __init__(self, seed, M=60, first_id=0):
        self.rng = np.random.default_rng(seed)
        self.centre = self.rng.uniform(0, 2000, (M, 2))
        self.scale = self.rng.uniform(0.5, 3.0, M)
        self.vel = self.rng.normal(0, 3.0, (M, 2))
        self.ids = np.arange(first_id, first_id + M)
        self.M, self.k = M, 0

    def frame(self, n, nan=0.0, untracked=0.0, missing=0.15):
        r = self.rng
        pick = r.choice(self.M, n, replace=False)
        xy = BASE[None] * self.scale[pick, None, None] + self.centre[pick, None] + self.k * self.vel[pick, None]
        xy = xy + r.normal(0, 1.0, xy.shape)
        present = ((r.random((n, 17)) >= missing) @ (1 << np.arange(17))).astype(np.uint64)
        if nan:
            bad = r.random((n, 17, 2)) < nan
            xy[bad] = r.choice([np.nan, np.inf, -np.inf], int(bad.sum()))
        ids = [int(i) if r.random() >= untracked else -1 for i in self.ids[pick]]
        self.k += 1
        return xy, present, ids


def _record(env, xy, present, status=0):
    rec = np.zeros(1, env.wire.record_dtype(17, env.g.capR))[0]
    rec["n_persons"], rec["status"] = len(present), status
    rec["rows"]["xy"][:len(present)] = xy
    rec["rows"]["present"][:len(present)] = present
    rec["rows"]["score"][:len(present)] = 0.5
    return rec


def _frame(env, w, s, n, t, **kw):
    xy, present, ids = w.frame(n, **kw)
    return (s, _record(env, xy, present), ids, t)


@pytest.mark.parametrize("persons", [0, 1, 10, 30, 128])
def test_one_stream_frame_by_frame(env, persons):
    run, w = Run(env, 1), World(persons, M=max(persons, 1) + 20)
    for k in range(10):
        run.call([_frame(env, w, 0, persons if k % 3 else max(0, persons - 3), k / 30.0)])


@pytest.mark.parametrize("params", [(1.0, 0.0, 1.0), (0.05, 3.0, 0.3), (7.0, 0.007, 9.0)])
def test_several_streams_and_frames_per_call(env, params):
    """Interleaved streams, several frames of some in one call, streams absent from some calls, irregular times."""
    S = 6
    run, rng = Run(env, S, *params), np.random.default_rng(3)
    worlds = [World(10 + s, M=40, first_id=1000 * s) for s in range(S)]
    clock = [0.0] * S
    for _ in range(6):
        frames = []
        for s in rng.integers(0, S, 2 * S):
            clock[s] += float(rng.choice([1 / 30, 1 / 60, rng.uniform(0.001, 0.5)]))
            frames.append(_frame(env, worlds[s], int(s), int(rng.integers(0, 30)), clock[s]))
        run.call(frames)


def test_skipped_frames_and_untracked_people(env):
    run, w = Run(env, 2), World(21, M=50)
    for k in range(8):
        run.call([_frame(env, w, 0, 20, k * 0.04, untracked=0.3), _frame(env, w, -1, 12, 99.0),
                  _frame(env, w, 1, 25, k * 0.03 + 1.0, untracked=0.1), _frame(env, w, -1, 0, 0.0)])


def test_new_absent_and_nonfinite_joints(env):
    run, w = Run(env, 2), World(23, M=70)
    for k in range(10):
        run.call([_frame(env, w, s, 40, k / 25.0, nan=0.08, missing=0.4) for s in (0, 1)])


def test_irregular_equal_and_decreasing_times(env):
    """dt not positive and finite restarts a joint: equal, earlier, NaN and infinite times."""
    run, w = Run(env, 1), World(29, M=20)
    for t in [0.0, 0.01, 0.01, 0.5, 0.2, 0.21, float("nan"), 0.3, float("inf"), 0.4, 0.4000001, 3.0]:
        run.call([_frame(env, w, 0, 15, t)])


def test_eviction_past_128_ids(env):
    """128 people per frame from a crowd of 400 ids: slots fill, and each frame's new ids evict the least recently used
    slots, ties to the lowest index."""
    run, w = Run(env, 1), World(31, M=400)
    for k in range(12):
        run.call([_frame(env, w, 0, 128, k / 30.0, untracked=0.05)])


def test_repeated_ids(env):
    """A direct caller's repeated id: the first row keeps the slot, the others are passed through raw."""
    run, w = Run(env, 1), World(37, M=10)
    for k in range(5):
        xy, present, ids = w.frame(10)
        ids = [ids[0], ids[1], ids[0], ids[2], ids[1], ids[3], ids[3], ids[4], ids[0], ids[5]]
        run.call([(0, _record(env, xy, present), ids, k / 30.0)])


def test_graph_replay_with_new_contents(env):
    """One call recorded into a CUDA graph over fixed buffers, replayed with new records, ids, streams and times."""
    t = env.torch
    run = Run(env, 3)
    worlds = [World(40 + s, M=30, first_id=100 * s) for s in range(3)]
    b = run.buffers(4)
    stream = t.cuda.Stream()
    layouts = [[0, 1, 2, 0], [2, 2, -1, 1], [1, 0, 0, 0], [0, 1, 2, 0]]
    clock = [0.0] * 3

    def frames(order):
        out = []
        for s in order:
            if s >= 0:
                clock[s] += 0.04
            out.append(_frame(env, worlds[max(s, 0)], s, 20, clock[s] if s >= 0 else 0.0))
        return out

    first = frames(layouts[0])
    run.fill(b, first)
    t.cuda.synchronize()
    graph = t.cuda.CUDAGraph()
    with t.cuda.graph(graph, stream=stream):
        env.g.smooth_frames(b.frames, run.tables.data_ptr(), 3, *run.params)
    graph.replay()
    t.cuda.synchronize()
    run.check(b, first)
    for order in layouts[1:]:
        nxt = frames(order)
        run.fill(b, nxt)
        t.cuda.synchronize()
        graph.replay()
        t.cuda.synchronize()
        run.check(b, nxt)


def test_invalid_calls_are_refused(env):
    from improved_body_parts_b200.grouping import GroupingError
    run = Run(env, 1)
    f = np.zeros(1, env.grouping.SMOOTH_FRAME)
    tb = run.tables.data_ptr()
    with pytest.raises(GroupingError, match="NULL"):
        env.g.smooth_frames(f, tb, 1, 1.0, 1.0, 1.0)
    b = run.buffers(1)
    bad = b.frames.copy()
    bad[0]["time"] += 4
    with pytest.raises(GroupingError, match="aligned"):
        env.g.smooth_frames(bad, tb, 1, 1.0, 1.0, 1.0)
    for args, match in [((0.0, 1.0, 1.0), "min_cutoff"), ((float("nan"), 1.0, 1.0), "min_cutoff"),
                        ((1.0, -1.0, 1.0), "beta"), ((1.0, float("inf"), 1.0), "beta"), ((1.0, 1.0, 0.0), "d_cutoff")]:
        with pytest.raises(GroupingError, match=match):
            env.g.smooth_frames(b.frames, tb, 1, *args)
    with pytest.raises(GroupingError, match="n_tables"):
        env.g.smooth_frames(b.frames, tb, 0, 1.0, 1.0, 1.0)
    t = env.torch
    t.cuda.synchronize()
    assert not run.tables.cpu().numpy().any()  # nothing ran
