"""GPU: the persistent limb scorer's item queue scores every (image, limb) exactly once, and is back at 0 after a launch.

limb_score_persist_kernel deals its items from a handle-owned device counter that the last CTA resets.  One handle runs
the p30 batch, a 37-image call, a 2-image call (60 items: fewer than the SMs, so some CTAs draw nothing) and the p30
batch again; every call must give what a fresh handle gives for it alone, and p30 the recorded survivor counts.  A
counter left off 0 would skip items (their candidate and survivor counts stay stale) or score some twice."""
import numpy as np
import pytest

from test_gpu_screen_survivors import RECORD, p30_case

pytestmark = pytest.mark.gpu

CFG = dict(max_person_rows=64)


def run(torch, dev, g, heat, paf, extent, params):
    g.group_device(torch.from_numpy(heat).to(dev), torch.from_numpy(paf).to(dev), extent, params)
    r = g.fetch()
    N = heat.shape[0]
    surv = g.device_tensors()["surv_count"][:N].cpu().numpy().copy()
    return r, surv, g.stage_kernels()[1]


def assert_same(case, a, b):
    (ra, sa, _), (rb, sb, _) = a, b
    assert np.array_equal(sa, sb), f"{case}: survivor counts differ in {int((sa != sb).sum())} (image, limb)"
    assert np.array_equal(ra.cand_count, rb.cand_count), f"{case}: candidate counts differ"
    assert np.array_equal(ra.status, rb.status), f"{case}: status differs"
    assert np.array_equal(ra.n_persons, rb.n_persons), f"{case}: person counts differ"
    for i, P in enumerate(ra.n_persons.tolist()):
        for f in ("subset", "people_xy", "people_score"):
            assert np.array_equal(getattr(ra, f)[i, :P], getattr(rb, f)[i, :P]), f"{case}: image {i}: {f} differs"


def test_queue_resets_and_scores_every_item_once(cuda_device):
    import torch

    from improved_body_parts_b200 import skeleton, synth
    from improved_body_parts_b200.grouping import Grouper

    with np.load(RECORD, allow_pickle=False) as z:
        rec_p30 = z["p30"]
    heat30, paf30, extent, params = p30_case()
    calls = [("p30", heat30, paf30)]
    calls.append(("37 images", *synth.make_batch(7301, 37, 128, 128, 20)))
    calls.append(("2 images", *synth.make_batch(7302, 2, 128, 128, 30)))
    calls.append(("p30 again", heat30, paf30))

    fresh = {}
    for case, heat, paf in calls[:3]:
        with Grouper(max_batch=heat.shape[0], **CFG) as g:
            fresh[case] = run(torch, cuda_device, g, heat, paf, extent, params)
    fresh["p30 again"] = fresh["p30"]

    with Grouper(max_batch=256, **CFG) as g:
        for case, heat, paf in calls:
            got = run(torch, cuda_device, g, heat, paf, extent, params)
            assert "persist" in got[2], f"{case}: scored by {got[2]}"
            assert_same(case, got, fresh[case])
            if case.startswith("p30"):
                assert np.array_equal(got[1], rec_p30), f"{case}: survivor counts differ from the record"
        # spg_group_host runs its chunks on the handle's two streams, each with a queue of its own
        heat, paf = calls[1][1], calls[1][2]
        out = g.group_host(heat, paf, extent, params)
        rf = fresh["37 images"][0]
        assert np.array_equal(out["n_persons"], rf.n_persons) and np.array_equal(out["status"], rf.status)
        for i, P in enumerate(rf.n_persons.tolist()):
            assert np.array_equal(out["people_xy"][i, :P], rf.people_xy[i, :P]), f"group_host: image {i}: people_xy differs"
            assert np.array_equal(out["people_score"][i, :P], rf.people_score[i, :P]), f"group_host: image {i}: people_score differs"
