"""GPU: ``spg_track_frames`` called directly on seeded random wire records and tables, against the port
(oracle/track_port.py) after every call: every id, age, stored pose and id counter equal, every OKS within 4 ULP.  The
seeded data has no OKS within 1e-12 of the threshold and no two within 1e-12 of each other unless equal, so equal ids
are a claim about the matching order, not luck."""
import types

import numpy as np
import pytest

from oracle import track_port as tp

pytestmark = pytest.mark.gpu

BASE = np.array([[20, 10], [18, 8], [22, 8], [15, 9], [25, 9], [10, 25], [30, 25], [8, 45], [32, 45], [6, 60], [34, 60],
                 [14, 60], [26, 60], [13, 80], [27, 80], [12, 100], [28, 100]], np.float64)


@pytest.fixture(scope="module")
def env(cuda_device):
    import torch
    from improved_body_parts_b200 import dropin, grouping, wire

    g = dropin._new_grouper(1, 0)
    yield types.SimpleNamespace(torch=torch, grouping=grouping, wire=wire, g=g, dev=cuda_device)
    g.close()


class Run:
    """Device tables for ``streams`` streams and the port beside them."""

    def __init__(self, env, streams, thr=0.5, max_age=30):
        t = env.torch
        self.env, self.thr, self.max_age = env, thr, max_age
        self.rows = env.g.capR
        self.tables = t.zeros((streams, env.grouping.TRACK_TABLE.itemsize), dtype=t.uint8, device=env.dev)
        self.port = tp.Tracker(streams, thr, max_age)

    def call(self, frames):
        """frames: [(stream, record, jpeg_status or None)]; one spg_track_frames call, then the port frame by frame."""
        env, t, n = self.env, self.env.torch, len(frames)
        recs = np.stack([r for _, r, _ in frames])
        rec_dev = t.from_numpy(recs.view(np.uint8).reshape(n, -1).copy()).to(env.dev)
        streams = t.tensor([s for s, _, _ in frames], dtype=t.int32, device=env.dev)
        jst = t.tensor([j or 0 for _, _, j in frames], dtype=t.int32, device=env.dev)
        ids = t.full((n, self.rows), -7, dtype=t.int64, device=env.dev)
        oks = t.full((n, tp.SLOTS, self.rows), np.nan, dtype=t.float64, device=env.dev)
        f = np.zeros(n, env.grouping.TRACK_FRAME)
        for j, (_, _, js) in enumerate(frames):
            f[j]["record"] = rec_dev[j].data_ptr()
            f[j]["stream"] = streams.data_ptr() + 4 * j
            f[j]["jpeg_status"] = jst.data_ptr() + 4 * j if js is not None else 0
            f[j]["ids"] = ids[j].data_ptr()
            f[j]["oks"] = oks[j].data_ptr()
        env.g.track_frames(f, self.tables.data_ptr(), self.tables.shape[0], self.thr, self.max_age)
        ids, oks = ids.cpu().numpy(), oks.cpu().numpy()
        for j, (s, rec, js) in enumerate(frames):
            np_ = int(rec["n_persons"])
            if s < 0:
                assert (ids[j, :np_] == -1).all(), f"frame {j}: a skipped frame's people get -1"
                continue
            live = [k for k, tr in enumerate(self.port.slots[s]) if tr is not None]
            want = self.port.step_record(s, rec, js or 0)
            assert ids[j, :np_].tolist() == want, f"frame {j} (stream {s}): ids"
            assert (ids[j, np_:] == -7).all(), f"frame {j}: ids past n_persons written"
            observed = int(rec["status"]) == 0 and not js
            if observed:
                self._check_oks(oks[j], live, np_, f"frame {j}")
        self.check_tables()

    def _check_oks(self, got, live, np_, what):
        want = self.port.last_oks
        vals = []
        for k in live:
            for p in range(np_):
                a, b = got[k, p], want[(k, p)]
                if np.isnan(b):
                    assert np.isnan(a), f"{what}: OKS ({k}, {p})"
                    continue
                assert abs(a - b) <= 4 * np.spacing(abs(b)), f"{what}: OKS ({k}, {p}) {a!r} vs {b!r}"
                vals.append(b)
        v = np.array(vals)
        assert not (np.abs(v - self.thr) <= 1e-12).any(), f"{what}: an OKS within 1e-12 of the threshold"
        u = np.unique(v[v >= self.thr - 1e-12])
        assert not (np.diff(u) <= 1e-12).any(), f"{what}: two OKS within 1e-12 of each other"

    def check_tables(self):
        got = self.tables.cpu().numpy().view(self.env.grouping.TRACK_TABLE).reshape(-1)
        for s, table in enumerate(self.port.slots):
            assert int(got[s]["next_id"]) == self.port.next_id[s], f"stream {s}: next id"
            for k, tr in enumerate(table):
                d = got[s]["tracks"][k]
                assert bool(d["live"]) == (tr is not None), f"stream {s} slot {k}: live"
                if tr is None:
                    continue
                assert (int(d["id"]), int(d["age"]), int(d["present"])) == (tr.id, tr.age, tr.present), (s, k)
                assert np.array_equal(d["xy"], tr.xy, equal_nan=True), f"stream {s} slot {k}: pose"


class World:
    """``M`` skeletons far apart, each drifting a few pixels per frame; a frame shows some of them with joint noise,
    missing joints and, at ``nan`` rate, NaN or infinite coordinates."""

    def __init__(self, seed, M=300):
        self.rng = np.random.default_rng(seed)
        self.centre = self.rng.uniform(0, 40000, (M, 2))
        self.scale = self.rng.uniform(0.5, 2.0, M)
        self.vel = self.rng.normal(0, 2.0, (M, 2))
        self.M, self.t = M, 0

    def people(self, n, nan=0.0):
        r = self.rng
        pick = r.choice(self.M, n, replace=False)
        xy = BASE[None] * self.scale[pick, None, None] + self.centre[pick, None] + self.t * self.vel[pick, None]
        xy = xy + r.normal(0, 1.5, xy.shape)
        present = (r.random((n, 17)) < 0.85) @ (1 << np.arange(17))
        if nan:
            bad = r.random((n, 17, 2)) < nan
            xy[bad] = r.choice([np.nan, np.inf, -np.inf], int(bad.sum()))
        self.t += 1
        return xy, present.astype(np.uint64)


def _record(env, xy, present, status=0):
    rec = np.zeros(1, env.wire.record_dtype(17, env.g.capR))[0]
    rec["n_persons"], rec["status"] = len(present), status
    rec["rows"]["xy"][:len(present)] = xy
    rec["rows"]["present"][:len(present)] = present
    rec["rows"]["score"][:len(present)] = 0.5
    return rec


@pytest.mark.parametrize("persons", [0, 1, 10, 30, 128])
def test_one_stream_frame_by_frame(env, persons):
    run, w = Run(env, 1), World(persons)
    for k in range(8):
        n = persons if k % 3 else max(0, persons - 3)
        run.call([(0, _record(env, *w.people(n)), None)])


def test_full_tables_evict_and_drop(env):
    """128 persons per frame from a crowd of 300: the table fills, unmatched tracks age, drop at max_age and are
    evicted by new persons."""
    run, w = Run(env, 1, max_age=3), World(5)
    for _ in range(12):
        run.call([(0, _record(env, *w.people(128)), None)])


def test_several_frames_of_one_stream_in_one_call(env):
    run, w = Run(env, 1), World(11, M=60)
    for _ in range(4):
        run.call([(0, _record(env, *w.people(int(w.rng.integers(0, 50)))), None) for _ in range(5)])


@pytest.mark.parametrize("streams", [8, 64])
def test_many_streams_in_one_call(env, streams):
    """Interleaved streams, several frames of some in one call, streams absent from some calls."""
    run = Run(env, streams, thr=0.3)
    worlds = [World(100 + s, M=40) for s in range(streams)]
    rng = np.random.default_rng(streams)
    for _ in range(5):
        order = rng.integers(0, streams, 2 * streams)
        run.call([(int(s), _record(env, *worlds[s].people(int(rng.integers(0, 30)))), None) for s in order])


def test_nonfinite_coordinates(env):
    run, w = Run(env, 2), World(23, M=80)
    for _ in range(6):
        run.call([(s, _record(env, *w.people(40, nan=0.08)), None) for s in (0, 1)])


def test_unobserved_and_skipped_frames(env):
    """Status bits and flagged JPEG statuses age the tracks and give -1; a skipped frame changes nothing."""
    run, w = Run(env, 2, max_age=2), World(31, M=50)
    for k in range(8):
        frames = []
        for s in (0, 1):
            xy, pr = w.people(20)
            frames.append((s, _record(env, xy, pr, status=[0, 4, 0, 0x20][k % 4]), [None, None, 11, 0][(k + s) % 4]))
        frames.append((-1, _record(env, *w.people(5)), None))
        run.call(frames)


def test_exact_ties(env):
    """Identical tracks and identical persons: OKS exactly 1.0 on every side, taken by the lower id and row."""
    run, w = Run(env, 1), World(41, M=10)
    xy, pr = w.people(3)
    twice = np.concatenate([xy, xy]), np.concatenate([pr, pr])
    run.call([(0, _record(env, *twice), None)])       # tracks 0..5, pairwise identical
    run.call([(0, _record(env, xy, pr), None)])       # each person: two tracks at OKS 1.0
    run.call([(0, _record(env, *twice), None)])       # each track: two persons at OKS 1.0
    got = run.tables.cpu().numpy().view(env.grouping.TRACK_TABLE).reshape(-1)[0]
    assert int(got["next_id"]) == 6


def test_invalid_calls_are_refused(env):
    from improved_body_parts_b200.grouping import GroupingError
    run = Run(env, 1)
    f = np.zeros(1, env.grouping.TRACK_FRAME)
    with pytest.raises(GroupingError, match="NULL"):
        env.g.track_frames(f, run.tables.data_ptr(), 1, 0.5, 3)
    with pytest.raises(GroupingError, match="finite"):
        env.g.track_frames(f[:0], run.tables.data_ptr(), 1, float("nan"), 3)
    with pytest.raises(GroupingError, match="max_age"):
        env.g.track_frames(f[:0], run.tables.data_ptr(), 1, 0.5, -1)
