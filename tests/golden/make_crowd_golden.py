#!/usr/bin/env python
"""Generate the crowded golden fixtures of ``tests/golden/crowd/`` by EXECUTING THE REFERENCE's own functions, unmodified.

Same procedure as ``make_golden.py`` (seeded synthetic maps, ``find_peaks -> find_connections -> find_people`` lifted
verbatim from the reference's evaluate.py by oracle/ref_loader.py), for images past the bounded path's capacities: the
cases of the capacity-free tier (tests/test_gpu_unbounded.py).  They live in a subdirectory so that the fixture set every
bounded test runs (``tests/golden/*.npz``) stays as it is.  Smooth maps (``noise=0``) keep the files small; the spikes
are isolated noise peaks, more than 128 of them in a part on a 64 x 64 map.

Runs only where a reference checkout is available: ``python tests/golden/make_crowd_golden.py``.
Recorded environment and per-case counts: ``tests/golden/crowd/MANIFEST.json``.
"""
from __future__ import annotations

import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "crowd")
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from golden_io import save_case  # noqa: E402
from improved_body_parts_b200 import skeleton, synth  # noqa: E402
from oracle.ref_loader import Reference  # noqa: E402

# name -> make_image arguments
CASES = {
    "peaks_over_128": dict(seed=61, H=64, W=64, persons=4, spikes=3200, noise=0.0),
}


def main() -> None:
    import torch

    ref = Reference()
    assert tuple(ref.limbs) == skeleton.LIMBS, "limb table drifted from the reference"
    os.makedirs(OUT, exist_ok=True)
    manifest = {"generated_by": "tests/golden/make_crowd_golden.py", "reference": "hellojialee/Improved-Body-Parts",
                "numpy": np.__version__, "torch": torch.__version__, "python": sys.version.split()[0], "cases": {}}
    for name, gen in CASES.items():
        gen = dict(gen)
        seed, H, W, P = gen.pop("seed"), gen.pop("H"), gen.pop("W"), gen.pop("persons")
        heat, paf = synth.make_image(seed, H, W, P, **gen)
        params = skeleton.default_params()
        t0 = time.time()
        structs = ref.group(np.ascontiguousarray(heat.transpose(1, 2, 0)), np.ascontiguousarray(paf.transpose(1, 2, 0)),
                            H, params)
        dt_s = time.time() - t0
        path = os.path.join(OUT, name + ".npz")
        save_case(path, heat, paf, skeleton.LIMBS, H, params, structs,
                  meta=dict(seed=seed, H=H, W=W, persons=P, gen=gen, paf_dtype="f32", variant="evaluate"))
        peaks, conn, special, subset, _ = structs
        manifest["cases"][name] = dict(
            peaks=int(sum(len(p) for p in peaks)), max_peaks_per_part=int(max(len(p) for p in peaks)),
            connections=int(sum(0 if isinstance(c, list) else c.shape[0] for c in conn)), special_k=len(special),
            persons=int(subset.shape[0]), reference_seconds=round(dt_s, 3), bytes=os.path.getsize(path))
        print(f"{name:20s} {manifest['cases'][name]}")
    with open(os.path.join(OUT, "MANIFEST.json"), "w") as fh:
        json.dump(manifest, fh, indent=1)


if __name__ == "__main__":
    main()
