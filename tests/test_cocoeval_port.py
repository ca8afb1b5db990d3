"""CPU: the numpy restatement of pycocotools' keypoint evaluation (oracle/cocoeval_port.py) on hand-computed cases, one
per rule, and against pycocotools itself where it is installed."""
import contextlib
import copy
import functools
import io
import math

import numpy as np
import pytest

import cocoeval_cases as cases
from improved_body_parts_b200 import cocoeval, synth
from oracle import cocoeval_port as port

T = 10  # thresholds


def _run(name):
    ds, res, setup = (cases.CASES | cases.CROWD_CASES)[name]()
    c = cocoeval.COCO()
    c.dataset = copy.deepcopy(ds)
    c.createIndex()
    e = port.COCOevalPort(c, c.loadRes(res))
    if setup:
        setup(e.params)
    with contextlib.redirect_stdout(io.StringIO()):
        e.evaluate()
        e.accumulate()
        e.summarize()
    return e


def _img(e, img, a=0, cat=1):
    return next(x for x in e.evalImgs if x and x['image_id'] == img and x['category_id'] == cat and
                x['aRng'] == e.params.areaRng[a])


def test_crowd_region_matches_several_detections():
    e = _run("crowd")
    x = _img(e, 1)
    assert x['gtIds'] == [1, 2] and x['gtIgnore'].tolist() == [0, 1]
    assert (x['dtMatches'] == np.array([1, 2, 2, 2])).all()
    assert (x['dtIgnore'] == np.array([False, True, True, True])).all()
    assert (x['gtMatches'][:, 1] == 4).all(), "the crowd keeps the last detection's id"
    assert (e.eval['precision'][:, :, 0, 0, 0] == 1 / (1 + np.spacing(1))).all() and e.eval['recall'][:, 0, 0, 0].tolist() == [1.0] * T


def test_keypoint_less_ground_truth_scores_by_box_distance():
    e = _run("no_keypoints")
    var = (port.SIGMAS * 2) ** 2
    want = np.sum(np.exp(-(100.0 / var / (100.0 + np.spacing(1)) / 2))) / 17
    assert e.ious[1, 1][0, 0] == want
    x = _img(e, 1)
    assert x['gtIgnore'].tolist() == [1] and not x['dtMatches'].any()
    assert (e.eval['precision'][:, :, 0, 0, 0] == -1).all()


def test_scan_breaks_at_the_first_ignored_ground_truth_after_a_match():
    e = _run("ignore_break")
    assert e.ious[1, 1].tolist() == [[1.0, 1.0]]
    x = _img(e, 1)
    assert x['gtIds'] == [2, 1] and (x['dtMatches'] == 2).all() and not x['dtIgnore'].any()


def test_ties_go_to_the_last_ground_truth():
    e = _run("tie_last")
    x = _img(e, 1)
    assert x['gtIds'] == [1, 2, 3]
    assert (x['dtMatches'][:, 0] == 2).all() and (x['dtMatches'][:, 1] == 1).all() and (x['dtMatches'][:, 2] == 0).all()


def test_nan_oks_is_taken_then_replaced():
    e = _run("nan_oks")
    m = e.ious[1, 1]
    assert math.isnan(m[0, 0]) and m[0, 1] < 1e-200 and np.isnan(m[1]).all()
    x = _img(e, 1)
    assert (x['dtMatches'][:, 0] == 2).all(), "the NaN OKS gives way to the later ground truth at OKS ~0"
    assert (x['dtMatches'][:, 1] == 1).all(), "ground truth 2 is taken: the NaN one is matched"
    for a in (0, 1):
        assert not _img(e, 1, a)['dtIgnore'][:, 1].any(), "a NaN area is never outside a range"
    assert (_img(e, 1, 2)['dtMatches'][:, 1] == 2).all() and _img(e, 1, 2)['dtIgnore'][:, 1].all(), \
        "'large': ground truth 2 is ignored, and the NaN detection falls to it"


def test_ground_truth_id_zero_counts_as_unmatched():
    e = _run("gt_id_zero")
    x = _img(e, 1)
    assert (x['dtMatches'][:, 0] == 0).all() and (x['dtMatches'][:, 1] == 5).all()
    assert (x['gtMatches'][:, 0] == 1).all()
    assert e.eval['recall'][:, 0, 0, 0].tolist() == [0.5] * T


def test_score_ties_nan_and_signed_zero():
    e = _run("score_ties")
    assert _img(e, 1)['dtIds'] == [1, 2, 3, 8]
    assert _img(e, 2)['dtIds'] == [4, 9, 5]  # 0.5, 0.0, NaN
    assert _img(e, 3)['dtIds'] == [6, 7]      # -0.0 == 0.0: input order
    s = e.eval['scores'][0, :, 0, 0, 0]
    assert s[0] == 0.5 and s[-1] == 0.0


def test_more_detections_than_max_dets():
    e = _run("many_dets")
    assert e.params.maxDets == [5, 20]
    x = _img(e, 1)
    assert len(x['dtIds']) == 20 and x['dtIds'][:5] == [26, 24, 23, 22, 25] and x['dtScores'][-1] == 0.01 * 6
    assert e.eval['recall'][:, 0, 0, :].tolist() == [[0.5, 0.5]] * T


def test_images_without_ground_truth_or_detections():
    e = _run("empty_images")
    byimg = {(x['image_id'], x['aRng'][0], x['aRng'][1]) for x in e.evalImgs if x}
    assert [x is None for x in e.evalImgs[:4]] == [False, False, False, True]
    assert _img(e, 3)['dtIds'] == [] and _img(e, 2)['gtIds'] == []
    assert len(byimg) == 9
    assert e.eval['recall'][:, 0, 0, 0].tolist() == [0.5] * T


def test_area_range_edges_are_inside():
    e = _run("area_edges")
    assert _img(e, 1, 1)['gtIgnore'].tolist() == [0, 0, 1]  # 1024 and 9216 medium, 1023 not
    assert _img(e, 1, 2)['gtIgnore'].tolist() == [0, 1, 1]  # 9216 large


def test_area_range_without_positives_stays_minus_one():
    e = _run("no_positives")
    assert (e.eval['precision'][:, :, 0, 3, 0] == -1).all() and (e.eval['recall'][:, 0, 3, 0] == -1).all()
    assert (e.eval['scores'][:, :, 0, 3, 0] == -1).all()


def test_recall_short_of_the_thresholds_leaves_zeros():
    e = _run("short_recall")
    assert e.eval['recall'][:, 0, 0, 0].tolist() == [0.25] * T
    q = e.eval['precision'][0, :, 0, 0, 0]
    assert q[:26].tolist() == [0.5] * 26 and (q[26:] == 0).all()
    assert (e.eval['scores'][0, 26:, 0, 0, 0] == 0).all() and e.eval['scores'][0, 0, 0, 0, 0] == 0.95


def test_unsorted_duplicated_image_ids():
    e = _run("img_ids")
    assert e.params.imgIds == [1, 2, 3]
    assert [x['image_id'] for x in e.evalImgs[:3]] == [1, 2, 3]
    assert e.eval['recall'][:, 0, 0, 0].tolist() == [2 / 3] * T


def test_every_case_runs():
    for name in cases.CASES:
        assert _run(name).stats.shape == (10,)


def _against_pycocotools(ds, res, setup=None):
    pc = pytest.importorskip("pycocotools.cocoeval")
    from pycocotools.coco import COCO
    gt = COCO()
    gt.dataset = copy.deepcopy(ds)
    gt.createIndex()
    dt = gt.loadRes(copy.deepcopy(res))
    ref = pc.COCOeval(gt, dt, 'keypoints')
    mine = port.COCOevalPort(gt, dt)
    with contextlib.redirect_stdout(io.StringIO()):
        for e in (ref, mine):
            if setup:
                setup(e.params)
            e.evaluate()
            e.accumulate()
            e.summarize()
    assert len(ref.evalImgs) == len(mine.evalImgs)
    for a, b in zip(ref.evalImgs, mine.evalImgs):
        assert (a is None) == (b is None)
        if a is not None:
            for f in ('dtIds', 'gtIds', 'dtScores'):
                assert a[f] == b[f]
            for f in ('dtMatches', 'gtMatches', 'gtIgnore', 'dtIgnore'):
                assert np.array_equal(a[f], b[f])
    for f in ('precision', 'recall', 'scores'):
        assert np.array_equal(ref.eval[f], mine.eval[f])
    assert np.array_equal(ref.stats, mine.stats)


@pytest.mark.parametrize("seed, n", [(1, 37), (2, 200)])
def test_port_matches_pycocotools(seed, n):
    _against_pycocotools(*synth.coco_keypoint_set(seed, n))


_CROWD_SETS = {"crowded_images": cases.crowded_images, "two_categories": cases.two_categories,
               **cases.CROWD_CASES,
               **{f"keypoints_{k}": functools.partial(cases.keypoint_count, k) for k in cases.SIGMA_COUNTS},
               **{f"{name}_{where}": functools.partial(cases.param_set, name, where)
                  for name in cases.PARAM_SETS for where in ("seeded", "crowded")}}


@pytest.mark.parametrize("name", sorted(_CROWD_SETS))
def test_port_matches_pycocotools_past_one_warp(name):
    """The crowded sets, the step-edge cases and the user-set parameters of tests/test_gpu_cocoeval_crowd.py."""
    _against_pycocotools(*_CROWD_SETS[name]())


def test_categories_are_accumulated_on_their_own():
    e = _run("categories")
    assert e.params.catIds == [1, 2, 3] and e.eval['counts'][2] == 3
    assert e.eval['recall'][:, :, 0, 0].tolist() == [[1.0, 0.5, 0.0]] * T
    assert (e.eval['precision'][:, :, 0, 0, 0] == 2 / (2 + np.spacing(1))).all()  # the envelope: the second tp's
    q = e.eval['precision'][0, :, 1, 0, 0]
    assert (q[:51] == 1 / (2 + np.spacing(1))).all() and (q[51:] == 0).all()
    assert (e.eval['precision'][:, :, 2, 0, 0] == 0).all()
    s = _run("categories_subset")
    assert s.params.catIds == [1, 3] and s.eval['counts'][2] == 2
    assert np.array_equal(s.eval['precision'][:, :, 1], e.eval['precision'][:, :, 2])
    assert [x['category_id'] for x in s.evalImgs if x] == [1] * 6 + [3] * 6


# -- past one warp of ground truths: the device matcher's 32-ground-truth steps ----------------------------------------

def test_ties_across_steps_go_to_the_later_ground_truth():
    e = _run("dup_across_steps")
    assert set(np.unique(e.ious[1, 1]).tolist()) == {0.0, 1.0}
    x = _img(e, 1)
    assert x['gtIds'] == list(range(1, 71))
    # positions (5, 37), (31, 32), (0, 64): the later one first, then the earlier one; ids are positions + 1
    assert (x['dtMatches'] == np.array([38, 6, 33, 32, 65, 1])).all()
    m = x['gtMatches']
    assert (m[:, [37, 5, 32, 31, 64, 0]] == np.arange(1, 7)).all() and np.count_nonzero(m) == 6 * T


def test_an_earlier_step_maximum_holds_against_a_smaller_later_one():
    e = _run("earlier_max")
    m = e.ious[1, 1]
    assert m[0, 3] == 1.0 and m[0, 36] == 16 / 17 and np.count_nonzero(m[0]) == 2
    x = _img(e, 1)
    assert (x['dtMatches'][:, 0] == 4).all(), "OKS 1.0 at position 3 is kept against 16/17 at position 36"
    assert x['dtMatches'][:, 1].tolist() == [37] * 9 + [0], "16/17 at position 36 matches up to threshold 0.9"


def test_nan_oks_at_the_edges_of_a_step():
    e = _run("nan_steps")
    for img, q in ((1, 31), (2, 32), (3, 63)):
        m = e.ious[img, 1]
        assert np.isnan(m[:, q]).all() and np.isnan(m).sum() == 2
        assert m[0, 10] == 1.0 and m[0, q + 8] == 16 / 17
        x = _img(e, img)
        ids = x['gtIds']
        assert ids == list(range(72 * (img - 1) + 1, 72 * img + 1))
        # the NaN at q replaces OKS 1.0 at position 10; from there every ground truth is taken up to the 16/17
        assert (x['dtMatches'][:, 0] == ids[q + 8]).all(), q
        # the next detection: 16/17 taken, so OKS 0.0 carries the match on to the last free ground truth
        assert (x['dtMatches'][:, 1] == ids[71 if q + 8 < 71 else 70]).all(), q
        assert not x['dtIgnore'].any()


def test_a_matched_ground_truth_past_32_is_skipped():
    e = _run("taken_past_32")
    x = _img(e, 1)
    assert (x['dtMatches'][:, 0] == 36).all()
    assert x['dtMatches'][:, 1].tolist() == [39] * 9 + [0], "position 35 is taken: on to 16/17 at position 38"
    assert (x['dtMatches'][:, 2] == 0).all()
    assert (x['gtMatches'][:, 35] == 1).all()


def test_a_crowd_region_past_32_takes_several_detections():
    e = _run("crowd_past_32")
    assert [g['id'] for g in e._gts[1, 1]].index(100) == 34, "the crowd is in the second step of annotation order"
    x = _img(e, 1)
    assert x['gtIds'] == list(range(1, 37)) + [100] and x['gtIgnore'].tolist() == [0] * 36 + [1]
    assert (x['dtMatches'] == np.array([8, 100, 100, 100, 0])).all()
    assert (x['dtIgnore'] == np.array([False, True, True, True, False])).all()
    assert (x['gtMatches'][:, 36] == 4).all(), "the crowd keeps the last detection's id"
    assert (e.eval['recall'][:, 0, 0, 0] == 1 / 36).all()


def test_the_scan_breaks_at_an_ignored_ground_truth_past_32():
    e = _run("break_past_32")
    ids = [g['id'] for g in e._gts[1, 1]]
    assert [ids.index(i) for i in (101, 102, 103)] == [33, 38, 42], "annotation indices past the first step"
    x = _img(e, 1)
    assert x['gtIds'] == list(range(1, 41)) + [101, 102, 103]
    assert x['gtIgnore'].tolist() == [0] * 40 + [1] * 3
    assert e.ious[1, 1][0].tolist().count(1.0) == 2, "ground truths 21 and 101 tie at OKS 1.0"
    assert (x['dtMatches'] == np.array([21, 102, 0, 101])).all()
    assert (x['dtIgnore'] == np.array([False, True, False, True])).all()


def test_iou_thresholds_zero_and_one():
    e = _run("iou_thr_edges")
    x = _img(e, 1)
    assert e.params.iouThrs.tolist() == [0.0, 0.5, 1.0]
    assert x['dtMatches'].tolist() == [[13, 26, 40, 39], [13, 26, 0, 0], [13, 0, 0, 0]]
    assert e.eval['recall'][:, 0, 0, 0].tolist() == [4 / 40, 2 / 40, 1 / 40]
