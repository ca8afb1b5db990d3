"""GPU: limb_score's screen keeps exactly the pairs it kept before its sample order changed.

Changes to the screen's tables or loops (the order in which it looks at a pair's samples, how a warp walks them) may
only change its speed: the survivor count of every (image, limb), which the library publishes next to the
candidates, must equal the count recorded with the ascending sample order (tests/golden/screen/survivors.npz, written
by tests/golden/make_survivor_record.py) on the benchmark's p30 batch and on the random parameter cases of the parity
tests."""
import os

import numpy as np
import pytest

from test_oracle_vs_reference import fuzz_cases, maps_crc

pytestmark = pytest.mark.gpu

RECORD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "screen", "survivors.npz")
P30 = dict(seed=20260921, batch=256, hw=128, persons=30)  # bench.py's p30 workload (BASE_SEED, rank 0)
N_FUZZ = 40


def survivor_counts(torch, dev, heat, paf, extent, params, **cfg):
    """Survivors of the screen per (image, limb), and the kernel that scored them."""
    from improved_body_parts_b200.grouping import Grouper

    N, _, H, W = heat.shape
    g = Grouper(max_batch=N, max_h=H, max_w=W, **cfg)
    try:
        g.group_device(torch.from_numpy(heat).to(dev), torch.from_numpy(paf).to(dev), extent, params)
        torch.cuda.synchronize()
        return g.device_tensors()["surv_count"][:N].cpu().numpy().copy(), g.stage_kernels()[1]
    finally:
        g.close()


def p30_case():
    from improved_body_parts_b200 import skeleton, synth

    heat, paf = synth.make_batch(P30["seed"], P30["batch"], P30["hw"], P30["hw"], P30["persons"])
    return heat, paf, P30["hw"], skeleton.default_params()


def test_survivors_equal_the_one_stage_screen(cuda_device):
    import torch

    with np.load(RECORD, allow_pickle=False) as z:
        rec = {k: z[k] for k in z.files}
    heat, paf, extent, params = p30_case()
    assert int(rec["p30_crc"]) == maps_crc(heat, paf), "the p30 maps are not the ones the record was made from"
    surv, kernel = survivor_counts(torch, cuda_device, heat, paf, extent, params, max_person_rows=64)
    assert "persist" in kernel
    assert np.array_equal(surv, rec["p30"]), f"{int((surv != rec['p30']).sum())} (image, limb) counts differ"
    persistent = 0
    for trial, heat, paf, extent, params, cap in fuzz_cases(N_FUZZ):
        assert int(rec[f"fuzz{trial}_crc"]) == maps_crc(heat, paf), f"trial {trial}: maps differ from the record"
        surv, kernel = survivor_counts(torch, cuda_device, heat, paf, extent, params, max_peaks_per_part=cap, max_person_rows=128)
        persistent += "persist" in kernel
        assert np.array_equal(surv, rec[f"fuzz{trial}"]), f"trial {trial} ({kernel}, {params}): survivor counts differ"
    assert persistent > 0  # draws with f32 maps and at most 64 peaks per part run the persistent kernel
