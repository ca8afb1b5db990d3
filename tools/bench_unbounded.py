#!/usr/bin/env python
"""Time of the capacity-free grouping tier (``Grouper.group_unbounded``) on a crowded image, beside the bounded path on a
normal image and the CPU checker on the crowded one.  Prints one JSON line (and writes it to ``--out`` when given).

    python tools/bench_unbounded.py [--size 512] [--persons 160] [--normal-persons 30] [--reps 20] [--out FILE]

The tier sizes each stage from the previous one's counts, so a call synchronises the stream: its time is a host clock
around whole calls (each ends in a synchronise).  The bounded path is timed the same way (``group_device`` + the stream
synchronised), one image per call, so the two numbers are comparable.  The GPU's name and power limit are read in the
same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _gpu():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def _time(fn, reps):
    fn()  # warm-up: module load, workspace growth
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return float(np.median(t)) * 1e3, float(np.min(t)) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--persons", type=int, default=160)
    ap.add_argument("--normal-persons", type=int, default=30)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()

    import torch
    import __graft_entry__ as ge
    ge.build()
    from improved_body_parts_b200 import dropin, skeleton, synth
    from improved_body_parts_b200.grouping import Grouper
    from oracle import spg_oracle as so

    if not torch.cuda.is_available():
        raise SystemExit("bench_unbounded.py measures on a CUDA device; none is present")
    dev = torch.device("cuda:0")
    S = a.size
    params = skeleton.default_params()
    heat, paf = synth.make_batch(7, 1, S, S, a.persons)
    nheat, npaf = synth.make_batch(8, 1, S, S, a.normal_persons)
    g = Grouper(max_batch=1, max_h=S, max_w=S, max_peaks_per_part=dropin.CAP_PEAKS, max_cands_per_limb=dropin.CAP_CANDS,
                max_person_rows=dropin.CAP_ROWS)
    h, p = torch.from_numpy(heat).to(dev), torch.from_numpy(paf).to(dev)
    nh, np_ = torch.from_numpy(nheat).to(dev), torch.from_numpy(npaf).to(dev)
    st = torch.cuda.current_stream(dev)

    g.group_device(h, p, S, params)
    bounded_status = int(g.fetch(1).status[0])
    g.group_device(nh, np_, S, params)
    normal_status = int(g.fetch(1).status[0])

    def bounded():
        g.group_device(nh, np_, S, params)
        st.synchronize()

    tier_ms, tier_min = _time(lambda: g.group_unbounded(h, p, S, params), a.reps)
    bounded_ms, bounded_min = _time(bounded, a.reps)
    r = g.group_unbounded(h, p, S, params)
    o = so.group_batch(heat, paf, skeleton.LIMBS, S, params, cap_peaks=1 << 16, cap_conn=8192, cap_rows=8192)
    oracle_ms, oracle_min = _time(lambda: so.group_batch(heat, paf, skeleton.LIMBS, S, params, cap_peaks=1 << 16,
                                                          cap_conn=8192, cap_rows=8192), max(3, a.reps // 4))
    res = dict(
        gpu=_gpu(), map=f"{S}x{S}", crowd_persons=a.persons, normal_persons=a.normal_persons,
        crowd_bounded_status=hex(bounded_status), normal_status=hex(normal_status),
        crowd_max_peaks_per_part=int(r.peak_count[0].max()), crowd_candidates_max_limb=int(r.cand_count[0].max()),
        crowd_person_table_rows=int(r.subset.shape[1]), crowd_persons_found=int(r.n_persons[0]),
        tier_equals_checker=bool(int(o.n_persons[0]) == int(r.n_persons[0]) and
                                 np.array_equal(o.subset[0, :int(o.n_persons[0])], r.subset[0, :int(r.n_persons[0])])),
        tier_ms_median=round(tier_ms, 3), tier_ms_min=round(tier_min, 3),
        bounded_normal_ms_median=round(bounded_ms, 3), bounded_normal_ms_min=round(bounded_min, 3),
        checker_cpu_1thread_ms_median=round(oracle_ms, 3), checker_cpu_1thread_ms_min=round(oracle_min, 3))
    g.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
