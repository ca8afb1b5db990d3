#!/usr/bin/env python
"""What smoothing costs: ``spg_smooth_frames`` alone, and ``FrameStream``'s time per frame with tracking against tracking
plus smoothing.

1. Kernel: CUDA-event time of one ``spg_smooth_frames`` call over a grid of streams x persons (1 / 8 / 64 streams, one
   frame each; 10 / 30 / 128 persons per frame, every person tracked and all 17 joints present).  Warm-up calls give
   every person a slot and every joint state, and each later call moves the persons by a pixel or two: the steady state
   of a video.  --calls calls per timed window, median of --rounds windows; back-to-back calls from Python set that
   pace, so the kernel's own time is also read from torch.profiler (CUDA activities) over 50 more calls.
2. FrameStream: ``submit`` per frame (slots=2, each result read one submit later) of --frames seeded 480 x 640 uint8
   frames at the reference's settings (boxsize 640, max_downsample 64, scale_search [1], rotation_search [0]) with
   imhn.IMHN at the reference's random initialisation, track=TrackParams() against track=TrackParams() +
   smooth=SmoothParams() alternated round by round in one process; wall time per frame, median and min-max over
   --rounds rounds.

The card's name and power limit are read in the same run.

usage: python tools/bench_smooth.py [--calls 200] [--rounds 5] [--frames 64] [--out profiles/smooth.json]"""
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
            centre = rng.uniform(0, 4000, (S, P, 1, 2))
            recs = np.zeros(S, dt)
            recs["n_persons"] = P
            recs["rows"]["present"][:, :P] = (1 << 17) - 1

            def fill():
                recs["rows"]["xy"][:, :P] = BASE[None, None] + centre + rng.normal(0, 1.0, (S, P, 17, 2))
                return torch.from_numpy(recs.view(np.uint8).reshape(S, -1).copy()).cuda()
            variants = [fill() for _ in range(4)]  # records moved by a pixel or two from call to call
            streams = torch.arange(S, dtype=torch.int32, device="cuda")
            ids = torch.full((S, g.capR), -1, dtype=torch.int64, device="cuda")
            ids[:, :P] = torch.arange(P, device="cuda")
            times = torch.zeros((4, S), dtype=torch.float64, device="cuda")
            xy = torch.empty((S, g.capR, 17, 2), dtype=torch.float64, device="cuda")
            tables = torch.zeros((S, grouping.SMOOTH_TABLE.itemsize), dtype=torch.uint8, device="cuda")
            frames = []
            for k, v in enumerate(variants):
                f = np.zeros(S, grouping.SMOOTH_FRAME)
                for s in range(S):
                    f[s]["record"], f[s]["stream"] = v[s].data_ptr(), streams.data_ptr() + 4 * s
                    f[s]["ids"], f[s]["time"] = ids[s].data_ptr(), times[k].data_ptr() + 8 * s
                    f[s]["xy"] = xy[s].data_ptr()
                frames.append(f)

            def run(n, start):
                for k in range(start, start + n):
                    times[k % 4].fill_(k / 30.0)  # each call 1/30 s after the last: a positive dt
                    g.smooth_frames(frames[k % 4], tables.data_ptr(), S, 1.0, 1.0, 1.0)
            run(8, 0)  # every person takes a slot, every joint gets state
            torch.cuda.synchronize()
            tb = tables.cpu().numpy().view(grouping.SMOOTH_TABLE).reshape(-1)
            assert (tb["slots"]["live"].sum(axis=1) == P).all() and (tb["slots"]["mask"][:, :P] == (1 << 17) - 1).all()
            # the fill_ kernels sit between the calls, as the upload does in a tick; they are timed with them and
            # measured alone below
            k0, times_us = 8, []
            for _ in range(rounds):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                run(calls, k0)
                b.record()
                b.synchronize()
                k0 += calls
                times_us.append(a.elapsed_time(b) * 1e3 / calls)
            fills = []
            for _ in range(rounds):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for k in range(calls):
                    times[k % 4].fill_(k / 30.0)
                b.record()
                b.synchronize()
                fills.append(a.elapsed_time(b) * 1e3 / calls)
            # the kernel's own device time, from the profiler in a window of its own
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                run(50, k0)
                torch.cuda.synchronize()
            k0 += 50
            ev = [e for e in prof.key_averages() if "smooth_kernel" in e.key]
            dev_us = sum(getattr(e, "device_time_total", 0) or e.cuda_time_total for e in ev) / sum(e.count for e in ev)
            assert int(tables.cpu().numpy().view(grouping.SMOOTH_TABLE).reshape(-1)["clock"].min()) == k0
            out.append(dict(streams=S, persons=P, us_per_call=float(np.median(times_us)), us_min=float(min(times_us)),
                            us_max=float(max(times_us)), fill_us=float(np.median(fills)), kernel_us=float(dev_us)))
            print(f"streams {S:3d} persons {P:3d}: {out[-1]['us_per_call']:8.2f} us per call "
                  f"({out[-1]['us_min']:.2f}-{out[-1]['us_max']:.2f}; the time fill alone {out[-1]['fill_us']:.2f}); "
                  f"smooth_kernel {dev_us:.2f} us", flush=True)
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

    streams = {"track": dropin.FrameStream(model, params, MODEL_PARAMS_REF, slots=2, track=dropin.TrackParams()),
               "smooth": dropin.FrameStream(model, params, MODEL_PARAMS_REF, slots=2, track=dropin.TrackParams(),
                                            smooth=dropin.SmoothParams())}

    def run(fs, smoothed):
        prev, out = None, []
        for f in frames:
            t = fs.submit(f)
            if prev is not None:
                out.append(fs.result(prev, ids=True, smoothed=smoothed))
            prev = t
        out.append(fs.result(prev, ids=True, smoothed=smoothed))
        return out

    for name, fs in streams.items():  # warm-up: both slots captured
        run(fs, name == "smooth")
    per = {"track": [], "smooth": []}
    same_ids = True
    for _ in range(rounds):
        got = {}
        for name, fs in streams.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            got[name] = run(fs, name == "smooth")
            per[name].append((time.perf_counter() - t) * 1e3 / n_frames)
        same_ids = same_ids and [i for _, i in got["track"]] == [i for _, i in got["smooth"]]
    for fs in streams.values():
        fs.close()
    res = {name: dict(ms_per_frame=float(np.median(v)), min=float(min(v)), max=float(max(v))) for name, v in per.items()}
    res["overhead_ms_per_frame"] = res["smooth"]["ms_per_frame"] - res["track"]["ms_per_frame"]
    res["ids_equal"] = same_ids
    print(f"FrameStream 480x640: {res['track']['ms_per_frame']:.3f} ms/frame with tracking, "
          f"{res['smooth']['ms_per_frame']:.3f} with tracking and smoothing (overhead "
          f"{res['overhead_ms_per_frame'] * 1e3:.1f} us; ids equal: {same_ids})", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "smooth.json"))
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_smooth needs a CUDA device")
    name, power = card()
    print(f"{name}, power limit {power}", flush=True)
    res = dict(card=name, power_limit=power, kernel=kernel_grid(a.calls, a.rounds),
               frame_stream=frame_stream(a.frames, a.rounds))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
