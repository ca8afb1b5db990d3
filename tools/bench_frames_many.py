#!/usr/bin/env python
"""Ticks of frames through ``dropin.FrameStream.submit_many`` (one CUDA graph per tick) against ``submit`` per frame,
alternated round by round in the same run.

Workload: --frames seeded ``synth.photo`` frames at the COCO val2017 shapes of tools/bench_frames.py, once as uint8 images
and once as quality-95 4:2:0 JPEG bytes, at the reference's settings (boxsize 640, max_downsample 64, scale_search [1],
rotation_search [0], stride 4); the network is imhn.IMHN at the reference's random initialisation, bf16 autocast,
channels-last, device input stage.  Modes, each with a stream of its own: ``submit`` per frame (each result read before
the next submit but one, slots=2), and ``submit_many`` at K = 1, 4, 8 and 16 with the frames in order (mixed shapes) and
sorted by shape (one shape per tick, but the last of a shape).  Each K and input kind runs in a process of its own (the
tool starts one per pair), and in it each mode is warmed up by passes over every frame until a pass captures no graph
(every tick key captured in every slot, the scratch at its final size).  Reports per mode and input kind frames/s (median and min-max over the rounds), per-frame
latency p50 / p90 (from its tick's submit to its result), and in a separate pass under torch.profiler the kernel time
per frame split into network, decode, pre-network, post-network and grouping.  The people of every mode are compared
with ``submit``'s (how many frames differ), and the largest difference of the maps at K = 8.  The card's name and
power limit are read in the same run.

usage: python tools/bench_frames_many.py [--frames 48] [--rounds 3] [--out profiles/frames_many.json]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_frames import MODEL_PARAMS_REF, SHAPES, card  # noqa: E402

STAGES = (("decode", ("jpeg_",)), ("prenet", ("prenet_",)), ("postnet", ("postnet",)),
          ("grouping", ("nms_peaks", "limb_", "match_assemble", "assemble_kernel")))


def stage_of(name: str) -> str:
    for stage, keys in STAGES:
        if any(k in name for k in keys):
            return stage
    return "network"  # every other kernel: the forward pass, its casts and copies


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=48)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ks", default="1,4,8,16")
    ap.add_argument("--kinds", default="uint8,jpeg")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "frames_many.json"))
    a = ap.parse_args()
    ks, kinds = [int(k) for k in a.ks.split(",")], a.kinds.split(",")
    if len(ks) * len(kinds) > 1:
        # one process per K and kind: only three streams' graph pools are alive at once, and every capture of a process
        # happens before its profiler pass (a process that captured graphs after a torch.profiler session died with a
        # segmentation fault; the cause was not established)
        import subprocess
        import tempfile
        res = {"runs": {}}
        with tempfile.TemporaryDirectory() as tmp:
            for kind in kinds:
                for k in ks:
                    out = os.path.join(tmp, f"{kind}_{k}.json")
                    subprocess.run([sys.executable, os.path.abspath(__file__), "--frames", str(a.frames), "--rounds",
                                    str(a.rounds), "--ks", str(k), "--kinds", kind, "--out", out], check=True)
                    with open(out) as f:
                        res["runs"][f"K={k} {kind}"] = json.load(f)
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
        return
    import cv2
    import torch
    from torch.profiler import ProfilerActivity, profile

    from improved_body_parts_b200 import dropin, imhn, skeleton, synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_frames_many needs a CUDA device")
    dropin.configure(device=0, limbs=dropin.LIMBS, input_stage="device")
    rng = np.random.default_rng(2033)
    images = [synth.photo(int(rng.integers(1 << 30)), *SHAPES[int(rng.integers(len(SHAPES)))]) for _ in range(a.frames)]
    jpegs = [cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 95, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, 0x221111])[1].tobytes()
             for img in images]
    inputs = {kind: {"uint8": images, "jpeg": jpegs}[kind] for kind in a.kinds.split(",")}
    order = {"mixed": list(range(a.frames)), "one shape": sorted(range(a.frames), key=lambda i: images[i].shape[:2])}
    params = dict(skeleton.default_params(), scale_search=[1.0], rotation_search=[0.0])
    runner = imhn.Runner(imhn.IMHN().init_like_reference_(0), device="cuda:0", use_graph=False)

    def model(x):
        return [[runner(x)]]

    streams = {}

    def ticks_of(k, o):
        idx = order[o]
        if o == "mixed":
            return [idx[i:i + k] for i in range(0, len(idx), k)]
        out, cur = [], []
        for i in idx:  # one shape per tick
            if cur and (len(cur) == k or images[cur[0]].shape != images[i].shape):
                out.append(cur)
                cur = []
            cur.append(i)
        return out + [cur]

    def run(mode, k, o, kind, lat, detail=False):
        fs, frames, people = streams[(mode, kind)], inputs[kind], {}
        if mode == "submit":
            pending = []
            for i in range(a.frames):
                pending.append((i, fs.submit(frames[i]), time.perf_counter()))
                if len(pending) == 2 or i == a.frames - 1:
                    for j, tk, t0 in pending:
                        people[j] = fs.result(tk, detail=detail)
                        lat.append(time.perf_counter() - t0)
                    pending = []
            return people
        for tick in ticks_of(k, o):
            t0 = time.perf_counter()
            tickets = fs.submit_many([frames[i] for i in tick])
            for i, tk in zip(tick, tickets):
                people[i] = fs.result(tk, detail=detail)
                lat.append(time.perf_counter() - t0)
        return people

    times, lats, split, differ, captures, host_decodes, maps_diff = {}, {}, {}, {}, {}, {}, None
    for kind in inputs:
        streams[("submit", kind)] = dropin.FrameStream(model, params, MODEL_PARAMS_REF, slots=2)
        ref = run("submit", 1, "mixed", kind, [])
        for k in ks:
            modes = [("submit", 1, "mixed")] + [(f"many K={k} {o}", k, o) for o in order]
            for m, _, _ in modes[1:]:
                streams[(m, kind)] = dropin.FrameStream(model, params, MODEL_PARAMS_REF, slots=2)
            for m, mk, o in modes:  # warm-up until a pass captures nothing; people compared with submit's
                for _ in range(6):
                    before = streams[(m, kind)].captures
                    got = run(m, mk, o, kind, [])
                    if streams[(m, kind)].captures == before:
                        break
                differ[(m, kind)] = differ.get((m, kind), 0) + sum(repr(got[i]) != repr(ref[i]) for i in range(a.frames))
            for _ in range(a.rounds):
                for m, mk, o in modes:
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    run(m, mk, o, kind, lats.setdefault((m, kind), []))
                    torch.cuda.synchronize()
                    times.setdefault((m, kind), []).append(time.perf_counter() - t)
            for m, mk, o in modes:
                if (m, kind) in split:
                    continue
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    run(m, mk, o, kind, [])
                    torch.cuda.synchronize()
                s = {stage: 0.0 for stage in ["network"] + [st for st, _ in STAGES]}
                for ev in prof.key_averages():
                    if ev.device_type is not None and "CUDA" in str(ev.device_type) and ev.device_time_total > 0:
                        s[stage_of(ev.key)] += ev.device_time_total / 1e3
                split[(m, kind)] = {st: v / a.frames for st, v in s.items()}
            if k == 8 and kind == "uint8":  # the largest map difference against submit
                got = run("many K=8 mixed", 8, "mixed", kind, [], detail=True)
                want = run("submit", 1, "mixed", kind, [], detail=True)
                maps_diff = 0.0
                for i in range(a.frames):
                    for x, y in ((got[i].heat, want[i].heat), (got[i].paf, want[i].paf)):
                        maps_diff = max(maps_diff, (x.tensor.double() - y.tensor.double()).abs().max().item())
            for m, _, _ in modes[1:]:
                fs = streams.pop((m, kind))
                captures[(m, kind)], host_decodes[(m, kind)] = fs.captures, fs.host_decodes
                fs.close()
            torch.cuda.empty_cache()
        fs = streams.pop(("submit", kind))
        captures[("submit", kind)], host_decodes[("submit", kind)] = fs.captures, fs.host_decodes
        fs.close()
        torch.cuda.empty_cache()
    name, pl = card()
    res = {"card": name, "power_limit": pl, "frames": a.frames, "rounds": a.rounds, "max_map_diff_k8": maps_diff,
           "modes": {}}
    print(f"{name}, power limit {pl}; {a.frames} frames, IMHN bf16, boxsize 640, scale_search [1], rotation_search [0]; "
          f"largest map difference at K=8 against submit: {maps_diff}")
    for (m, kind), ts in times.items():
        ts = sorted(ts)
        med = ts[len(ts) // 2]
        lat = np.asarray(lats[(m, kind)]) * 1e3
        row = dict(frames_per_s=a.frames / med, spread=[a.frames / ts[-1], a.frames / ts[0]],
                   latency_ms_p50=float(np.percentile(lat, 50)), latency_ms_p90=float(np.percentile(lat, 90)),
                   kernel_ms_per_frame=split[(m, kind)], frames_differing_from_submit=differ[(m, kind)],
                   captures=captures[(m, kind)], host_decodes=host_decodes[(m, kind)])
        res["modes"][f"{m} {kind}"] = row
        ks_txt = ", ".join(f"{st} {v:.2f}" for st, v in split[(m, kind)].items())
        print(f"  {m:>20} {kind:>5}: {row['frames_per_s']:6.1f} frames/s (min {row['spread'][0]:.1f}, max "
              f"{row['spread'][1]:.1f}); latency p50 {row['latency_ms_p50']:.1f} ms, p90 {row['latency_ms_p90']:.1f} ms; "
              f"kernel ms/frame: {ks_txt}; {row['frames_differing_from_submit']} frames differ from submit")
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
