#!/usr/bin/env python
"""What tracking costs: ``spg_track_frames`` alone, and ``FrameStream``'s time per frame with and without it.

1. Kernel: CUDA-event time of one ``spg_track_frames`` call over a grid of streams x persons (1 / 8 / 64 streams, one
   frame each; 10 / 30 / 128 persons per frame), each stream's table holding as many live tracks as the frame has
   persons (a warm-up call fills it).  The persons are seeded skeletons far apart, each jittered by a pixel or two per
   call, so every person continues its track: the steady state of a video.  --calls calls per timed window, median of
   --rounds windows.
2. FrameStream: ``submit`` per frame (slots=2, each result read one submit later) of --frames seeded 480 x 640 uint8
   frames at the reference's settings (boxsize 640, max_downsample 64, scale_search [1], rotation_search [0]) with
   imhn.IMHN at the reference's random initialisation, track=None and track=TrackParams() alternated round by round in
   one process; wall time per frame, median and min-max over --rounds rounds.

The card's name and power limit are read in the same run.

usage: python tools/bench_track.py [--calls 200] [--rounds 5] [--frames 64] [--out profiles/track.json]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_frames import MODEL_PARAMS_REF, card  # noqa: E402

BASE = np.array([[20, 10], [18, 8], [22, 8], [15, 9], [25, 9], [10, 25], [30, 25], [8, 45], [32, 45], [6, 60], [34, 60],
                 [14, 60], [26, 60], [13, 80], [27, 80], [12, 100], [28, 100]], np.float64)


def kernel_grid(calls: int, rounds: int) -> list:
    import torch

    from improved_body_parts_b200 import dropin, grouping, wire
    g = dropin._new_grouper(1, 0)
    rng = np.random.default_rng(5)
    dt = wire.record_dtype(17, g.capR)
    out = []
    for S in (1, 8, 64):
        for P in (10, 30, 128):
            centre = rng.uniform(0, 40000, (S, P, 1, 2))
            recs = np.zeros(S, dt)
            recs["n_persons"] = P
            recs["rows"]["present"][:, :P] = (1 << 17) - 1

            def fill():
                recs["rows"]["xy"][:, :P] = BASE[None, None] + centre + rng.normal(0, 1.0, (S, P, 17, 2))
                return torch.from_numpy(recs.view(np.uint8).reshape(S, -1).copy()).cuda()
            variants = [fill() for _ in range(4)]  # records moved by a pixel or two from call to call
            streams = torch.arange(S, dtype=torch.int32, device="cuda")
            ids = torch.empty((S, g.capR), dtype=torch.int64, device="cuda")
            tables = torch.zeros((S, grouping.TRACK_TABLE.itemsize), dtype=torch.uint8, device="cuda")
            frames = []
            for v in variants:
                f = np.zeros(S, grouping.TRACK_FRAME)
                for s in range(S):
                    f[s]["record"], f[s]["stream"] = v[s].data_ptr(), streams.data_ptr() + 4 * s
                    f[s]["ids"] = ids[s].data_ptr()
                frames.append(f)
            for k in range(8):  # fills the tables; every later call continues every track
                g.track_frames(frames[k % 4], tables.data_ptr(), S, 0.5, 30)
            torch.cuda.synchronize()
            live = tables.cpu().numpy().view(grouping.TRACK_TABLE).reshape(-1)["tracks"]["live"].sum(axis=1)
            assert (live == P).all(), live
            times = []
            for _ in range(rounds):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for k in range(calls):
                    g.track_frames(frames[k % 4], tables.data_ptr(), S, 0.5, 30)
                b.record()
                b.synchronize()
                times.append(a.elapsed_time(b) * 1e3 / calls)
            assert int(tables.cpu().numpy().view(grouping.TRACK_TABLE).reshape(-1)["next_id"].max()) == P  # no track was lost
            out.append(dict(streams=S, persons=P, tracks=P, us_per_call=float(np.median(times)),
                            us_min=float(min(times)), us_max=float(max(times))))
            print(f"streams {S:3d} persons/tracks {P:3d}: {out[-1]['us_per_call']:8.2f} us per call "
                  f"({out[-1]['us_min']:.2f}-{out[-1]['us_max']:.2f})", flush=True)
    g.close()
    return out


def frame_stream(n_frames: int, rounds: int) -> dict:
    import torch

    from improved_body_parts_b200 import dropin, imhn, skeleton
    dropin.configure(device=0, limbs=dropin.LIMBS, input_stage="device")
    rng = np.random.default_rng(2031)
    frames = [rng.integers(0, 256, size=(480, 640, 3), dtype=np.uint8) for _ in range(n_frames)]
    params = dict(skeleton.default_params(), scale_search=[1.0], rotation_search=[0.0])
    runner = imhn.Runner(imhn.IMHN().init_like_reference_(0), device="cuda:0", use_graph=False)

    def model(x):
        return [[runner(x)]]

    streams = {"off": dropin.FrameStream(model, params, MODEL_PARAMS_REF, slots=2),
               "on": dropin.FrameStream(model, params, MODEL_PARAMS_REF, slots=2, track=dropin.TrackParams())}

    def run(fs, ids):
        prev, people = None, []
        for f in frames:
            t = fs.submit(f)
            if prev is not None:
                people.append(fs.result(prev, ids=True)[0] if ids else fs.result(prev))
            prev = t
        people.append(fs.result(prev, ids=True)[0] if ids else fs.result(prev))
        return people

    for name, fs in streams.items():  # warm-up: both slots captured
        run(fs, name == "on")
    per = {"off": [], "on": []}
    same = True
    for _ in range(rounds):
        got = {}
        for name, fs in streams.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            got[name] = run(fs, name == "on")
            per[name].append((time.perf_counter() - t) * 1e3 / n_frames)
        same = same and repr(got["off"]) == repr(got["on"])
    for fs in streams.values():
        fs.close()
    res = {name: dict(ms_per_frame=float(np.median(v)), min=float(min(v)), max=float(max(v))) for name, v in per.items()}
    res["overhead_ms_per_frame"] = res["on"]["ms_per_frame"] - res["off"]["ms_per_frame"]
    res["people_equal"] = same
    print(f"FrameStream 480x640: {res['off']['ms_per_frame']:.3f} ms/frame without tracking, "
          f"{res['on']['ms_per_frame']:.3f} with (overhead {res['overhead_ms_per_frame'] * 1e3:.1f} us; "
          f"people equal: {same})", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "track.json"))
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_track needs a CUDA device")
    name, power = card()
    print(f"{name}, power limit {power}", flush=True)
    res = dict(card=name, power_limit=power, kernel=kernel_grid(a.calls, a.rounds),
               frame_stream=frame_stream(a.frames, a.rounds))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
