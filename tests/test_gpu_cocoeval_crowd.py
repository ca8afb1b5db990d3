"""GPU: the device COCOeval against the port (oracle/cocoeval_port.py) past one warp of ground truths and at user-set
parameters, with test_gpu_cocoeval.py's bar: evalImgs field by field, eval arrays, stats and summarize()'s text bit for
bit, and every seeded set kept off the thresholds.

coco_match_kernel walks a unit's ground truths in annotation order, 32 per step, coco_oks_kernel sums one term per
visible keypoint in numpy's pairwise order (blocks of 8, up to 128 terms) and coco_accumulate_kernel strides 256
threads over the recall thresholds.  Here units hold up to 97 ground truths and 100 kept detections, annotations 1 to
128 keypoints, and the parameters take counts and orders past one pass of each loop.  Each test first asserts that its
input reaches the path it is there for, so that a change to the generator cannot quietly stop exercising it; the
matcher's steps are counted in annotation order, its own, not in evaluateImg's."""
import numpy as np
import pytest

import cocoeval_cases as cc
from test_gpu_cocoeval import _run, assert_margin, assert_same

pytestmark = pytest.mark.gpu


def _units(ref):
    """Per (image, category, area range) with ground truths: their ignore flags in the unit's annotation order (the
    order coco_match_kernel steps through, 32 at a time) and the annotation indices of the ones some detection matched,
    at any threshold."""
    out = []
    for x in ref.evalImgs:
        if x is not None and x["gtIds"]:
            index = {g["id"]: j for j, g in enumerate(ref._gts[x["image_id"], x["category_id"]])}
            flags = np.zeros(len(index), bool)
            for gid, ig in zip(x["gtIds"], x["gtIgnore"]):
                flags[index[gid]] = ig
            out.append((flags, {index[int(m)] for m in x["dtMatches"].ravel() if m}))
    return out


def _matched_past(ref, first, ignored=False):
    """Whether some detection matched a ground truth at annotation index >= first (an ignored one if ``ignored``)."""
    return any(i >= first and (flags[i] or not ignored) for flags, matched in _units(ref) for i in matched)


def test_crowded_images():
    """31-97 ground truths and up to 100 detections per image, ignored ones on both sides of the first step's end."""
    ref, dev = _run(*cc.crowded_images())
    pk = dev._dev["pk"]
    assert set(cc.CROWDED_SIZES) <= set(pk.gt_count.tolist()) and pk.gt_count.max() >= 97
    assert pk.kept_count.max() == 100
    # evaluateImg's order: ignored ground truths at positions 31 and 32 (each lands at n_keep + ign_seen + lane)
    assert any(len(g) > 32 and g[31] and g[32] for g in (x["gtIgnore"] for x in ref.evalImgs if x is not None))
    # the matcher's order: kept and ignored ones before and after index 32 (keep_seen and ign_seen carried a step)
    assert any(f[:32].any() and not f[:32].all() and f[32:].any() and not f[32:].all() for f, _ in _units(ref))
    assert _matched_past(ref, 32, ignored=True), "no ignored ground truth matched past the first step (phase 1)"
    assert _matched_past(ref, 64), "no match in the third step"
    assert_margin(ref)
    assert_same(ref, dev)


@pytest.mark.parametrize("name", sorted(cc.CROWD_CASES))
def test_step_edges(name):
    """Ties, an earlier maximum, NaN OKS, the crowd skip, the break and the capped thresholds across 32-ground-truth
    steps, every OKS that decides a match exact (tests/test_cocoeval_port.py has the answers by hand)."""
    ref, dev = _run(*cc.CROWD_CASES[name]())
    assert _matched_past(ref, 32)
    if name in ("crowd_past_32", "break_past_32"):
        assert _matched_past(ref, 32, ignored=True), "phase 1 does not reach the second step"
    if name == "nan_steps":  # NaN OKS columns, in annotation order
        assert {int(c) for m in ref.ious.values() if len(m) for c in np.flatnonzero(np.isnan(m).all(0))} == {31, 32, 63}
    assert_same(ref, dev)


@pytest.mark.parametrize("k", cc.SIGMA_COUNTS)
def test_keypoint_counts(k):
    """k sigmas and 3k values per annotation: OKS of 1 to k terms, below 8, in whole blocks of 8 and with a tail."""
    ref, dev = _run(*cc.keypoint_count(k))
    pk = dev._dev["pk"]
    assert pk.gt_kpts.shape[1] == pk.dt_kpts.shape[1] == 3 * k and len(ref.params.kpt_oks_sigmas) == k
    k1 = set((pk.gt_kpts[:, 2::3] > 0).sum(1).tolist())
    assert 0 in k1 and k1 & set(range(1, 8)), k1
    if k >= 8:
        assert any(n % 8 == 0 for n in k1 - {0}), k1
    if k >= 18:
        assert any(n > 16 and n % 8 for n in k1), k1
    assert pk.gt_count.max() > 32
    assert_margin(ref)
    assert_same(ref, dev)


def _reaches(name, ref, pk):
    """The precondition of PARAM_SETS[name] on the port's params and results and the packed inputs."""
    p, ev = ref.params, ref.eval
    if name.startswith("iou"):
        t = np.asarray(p.iouThrs)
        return {"iou_one": len(t) == 1, "iou_unsorted": (np.diff(t) < 0).any(), "iou_20": len(t) == 20}[name]
    if name.startswith("rec"):
        r = np.asarray(p.recThrs)
        if name == "rec_one":
            return len(r) == 1
        # the slots past the first 256 hold precision, not only the zeros past the last reached threshold
        return len(r) > 256 and (ev["precision"][:, 256:] > 0).any() and \
            ((np.diff(r) < 0).any() == (name == "rec_unsorted"))
    if name == "area_one":
        return len(p.areaRng) == 1
    if name == "area_six":
        return len(p.areaRng) == 6 and (ev["recall"][:, :, 4:] == -1).all() and (ev["recall"][:, :, :4] > -1).any()
    if name == "max_dets_0":
        return pk.kept_count.max() == 0 and pk.dt_count.max() > 0
    return p.maxDets[-1] == 100 and pk.kept_count.max() == min(pk.dt_count.max(), 100)


@pytest.mark.parametrize("where", ["seeded", "crowded"])
@pytest.mark.parametrize("name", sorted(cc.PARAM_SETS))
def test_user_params(name, where):
    ref, dev = _run(*cc.param_set(name, where))
    assert _reaches(name, ref, dev._dev["pk"])
    assert_margin(ref)
    assert_same(ref, dev)


def test_two_categories_of_crowded_images():
    ref, dev = _run(*cc.two_categories())
    pk = dev._dev["pk"]
    assert dev.eval["counts"][2] == 2 and (pk.gt_count.reshape(2, -1) >= 33).all()
    assert pk.kept_count.max() == 100
    assert_margin(ref)
    assert_same(ref, dev)
