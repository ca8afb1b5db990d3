#!/usr/bin/env python
"""Record the survivor counts of limb_score's screen for tests/test_gpu_screen_survivors.py (needs a CUDA device).

``python tests/golden/make_survivor_record.py [out.npz]`` writes ``tests/golden/screen/survivors.npz``: the published
survivor count per (image, limb) on the benchmark's p30 batch and on each random parameter case, with a CRC of each
case's maps.  The record in the repository was made while both screens looked at their samples in ascending order, so
the test checks that later forms of the screen keep exactly the same pairs."""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "tests"), HERE):
    sys.path.insert(0, p)

from test_gpu_screen_survivors import N_FUZZ, p30_case, survivor_counts  # noqa: E402
from test_oracle_vs_reference import fuzz_cases, maps_crc  # noqa: E402


def main(out: str) -> None:
    import torch

    dev = torch.device("cuda:0")
    heat, paf, extent, params = p30_case()
    surv, kernel = survivor_counts(torch, dev, heat, paf, extent, params, max_person_rows=64)
    rec = {"p30": surv.astype(np.int32), "p30_crc": np.int64(maps_crc(heat, paf))}
    print(f"p30: {kernel}, {int(surv.sum())} survivors")
    for trial, heat, paf, extent, params, cap in fuzz_cases(N_FUZZ):
        surv, kernel = survivor_counts(torch, dev, heat, paf, extent, params, max_peaks_per_part=cap, max_person_rows=128)
        rec[f"fuzz{trial}"] = surv.astype(np.int32)
        rec[f"fuzz{trial}_crc"] = np.int64(maps_crc(heat, paf))
        print(f"trial {trial}: {kernel}, {int(surv.sum())} survivors")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    np.savez_compressed(out, **rec)
    print("wrote", out)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "screen", "survivors.npz"))
