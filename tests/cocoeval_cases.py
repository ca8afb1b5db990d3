"""Hand-built keypoint-evaluation cases, one per rule of pycocotools' keypoint path, shared by the port's CPU tests and
the device tests.  Every OKS that decides a match is exact: a detection equal to its ground truth has OKS 1.0, one far
from every point has OKS 0.0, one inside a keypoint-less ground truth's grown box has OKS 1.0, and a NaN area gives NaN.

``CASES[name]()`` returns ``(dataset, results, setup)``: a ground-truth dict, the ``format_results``-style list, and a
function applied to a ``COCOeval``'s ``params`` before ``evaluate()`` (or None).  ``CROWD_CASES`` has the same form,
each case's rule at the edges of the device matcher's 32-ground-truth steps.  ``crowded_set`` is a seeded set of given
ground-truth counts per image, up to 100 detections and k keypoints; ``PARAM_SETS`` holds user-set parameters."""
from __future__ import annotations

import copy
import math

import numpy as np

from improved_body_parts_b200 import synth

_T = np.array([(0, -17), (-2, -18), (2, -18), (-3, -17), (3, -17), (-5, -12), (5, -12), (-7, -6), (7, -6), (-8, 0),
               (8, 0), (-3, 0), (3, 0), (-3, 8), (3, 8), (-4, 16), (4, 16)], dtype=np.float64)


def pts(cx, cy, s=2.0):
    """17 integer points of a standing person centred at (cx, cy), s pixels per template unit."""
    return np.rint(np.stack([cx + _T[:, 0] * s, cy + _T[:, 1] * s], 1)).astype(np.int64)


def gt(aid, img, p=None, *, crowd=0, bbox=None, area=None, vis=2, cat=1):
    """A ground truth: points p (None: keypoint-less) with visibility vis, a bbox and area from them unless given."""
    if p is None:
        kp, nk = [0] * 51, 0
    else:
        kp = np.concatenate([p, np.full((17, 1), vis)], 1).reshape(-1).tolist()
        nk = 17 if vis else 0
    if bbox is None:
        x0, y0 = p.min(0)
        bbox = [float(x0), float(y0), float(p[:, 0].max() - x0), float(p[:, 1].max() - y0)]
    return {"id": aid, "image_id": img, "category_id": cat, "iscrowd": crowd, "num_keypoints": nk, "keypoints": kp,
            "bbox": bbox, "area": float(bbox[2] * bbox[3]) if area is None else area}


def det(img, p, score, cat=1):
    """A detection as format_results writes it: floats, visibility 1."""
    p = np.asarray(p, dtype=np.float64)
    return {"image_id": img, "category_id": cat, "score": score,
            "keypoints": np.concatenate([p, np.ones((17, 1))], 1).reshape(-1).tolist()}


def far(img, score):
    return det(img, pts(5000, 5000), score)


def dataset(anns, images, cats=(1,)):
    return {"images": [{"id": i, "file_name": f"{i}.jpg", "width": 640, "height": 480} for i in images],
            "annotations": anns,
            "categories": [{"id": c, "name": f"person{c}", "supercategory": "person"} for c in cats]}


def crowd():
    """Three detections inside a crowd region all match it (a crowd ground truth can be matched again), ignored."""
    a = pts(100, 100)
    anns = [gt(1, 1, a), gt(2, 1, None, crowd=1, bbox=[300.0, 300.0, 40.0, 40.0], area=1600.0)]
    inside = np.full((17, 2), 320.0)
    return dataset(anns, [1]), [det(1, a, 0.9), det(1, inside, 0.8), det(1, inside, 0.7), det(1, inside, 0.6)], None


def no_keypoints():
    """A keypoint-less ground truth scores by the distance to its box grown by its size on every side."""
    anns = [gt(1, 1, None, bbox=[10.0, 10.0, 10.0, 10.0], area=100.0)]
    p = np.tile([[40.0, 20.0]], (17, 1))  # x1 = 10 + 2 * 10 = 30: dx = 10, dy = 0
    return dataset(anns, [1]), [det(1, p, 0.5)], None


def ignore_break():
    """The scan stops at the first ignored ground truth once a match that is not ignored exists, though the ignored
    one has an equal OKS later in the order."""
    a = pts(100, 100)
    anns = [gt(1, 1, None, bbox=[80.0, 60.0, 40.0, 80.0], area=3200.0), gt(2, 1, a)]
    return dataset(anns, [1]), [det(1, a, 0.9)], None


def tie_last():
    """Equal OKS: the last ground truth wins; the next detection takes the other one."""
    a = pts(100, 100)
    anns = [gt(1, 1, a), gt(2, 1, a), gt(3, 1, pts(300, 100))]
    return dataset(anns, [1]), [det(1, a, 0.9), det(1, a, 0.8), det(1, a, 0.7)], None


def nan_oks():
    """A NaN OKS (NaN ground-truth area) is taken, then any later eligible ground truth replaces it, even at OKS 0; a
    detection with a NaN point has a NaN area, never outside an area range."""
    a = pts(100, 100)
    anns = [gt(1, 1, a, area=math.nan), gt(2, 1, pts(400, 300))]
    bad = a.astype(np.float64)
    bad[3, 0] = math.nan
    return dataset(anns, [1]), [det(1, a, 0.9), det(1, bad, 0.8)], None


def gt_id_zero():
    """A match to the ground truth with id 0 counts as unmatched in dtMatches and in accumulate."""
    a, b = pts(100, 100), pts(300, 100)
    anns = [gt(0, 1, a), gt(5, 1, b)]
    return dataset(anns, [1]), [det(1, a, 0.9), det(1, b, 0.8)], None


def score_ties():
    """Equal scores inside an image and across images keep their input order; -0.0 and 0.0 are equal; NaN sorts last."""
    a, b = pts(100, 100), pts(300, 100)
    anns = [gt(1, 1, a), gt(2, 1, b), gt(3, 2, a), gt(4, 3, b)]
    res = [det(1, b, 0.5), far(1, 0.5), det(1, a, 0.5), det(2, a, 0.5), far(2, math.nan), det(3, b, -0.0),
           far(3, 0.0), far(1, -0.0), det(2, a, 0.0)]
    return dataset(anns, [1, 2, 3]), res, None


def many_dets():
    """More than maxDets[-1] = 20 detections: only the 20 best count; maxDets [5, 20] truncates again per maxDet."""
    a = pts(100, 100)
    anns = [gt(1, 1, a), gt(2, 1, pts(300, 100))]
    res = [far(1, 0.01 * i) for i in range(24)] + [det(1, a, 0.205), det(1, a, 0.5)]

    def setup(p):
        p.maxDets = [20, 5]
    return dataset(anns, [1]), res, setup


def empty_images():
    """Images with no ground truth (false positives only), with no detection, and with neither (evalImgs None)."""
    a = pts(100, 100)
    anns = [gt(1, 1, a), gt(2, 3, a)]
    return dataset(anns, [1, 2, 3, 4]), [det(1, a, 0.9), far(2, 0.8), far(2, 0.3)], None


def area_edges():
    """Ground-truth areas exactly 32^2 and 96^2 are inside 'medium' (and 96^2 inside 'large'); detection areas too."""
    a, b, c = pts(100, 100), pts(300, 100), pts(500, 100)
    anns = [gt(1, 1, a, area=1024.0), gt(2, 1, b, area=9216.0), gt(3, 1, c, area=1023.0)]
    return dataset(anns, [1]), [det(1, a, 0.9), det(1, b, 0.8), det(1, c, 0.7)], None


def no_positives():
    """An extra area range no ground truth falls in: precision, recall and scores stay -1 there."""
    a = pts(100, 100)

    def setup(p):
        p.areaRng = list(p.areaRng) + [[1e11, 1e12]]
        p.areaRngLbl = list(p.areaRngLbl) + ['huge']
    return dataset([gt(1, 1, a)], [1]), [det(1, a, 0.9)], setup


def short_recall():
    """Recall 0.25 at best: the recall thresholds above it keep precision and score 0."""
    a = pts(100, 100)
    anns = [gt(1, 1, a), gt(2, 1, pts(300, 100)), gt(3, 1, pts(500, 100)), gt(4, 2, a)]
    return dataset(anns, [1, 2]), [far(1, 0.95), det(1, a, 0.9), far(2, 0.7)], None


def img_ids():
    """Unsorted, duplicated params.imgIds: evaluate() sorts them and drops the duplicates."""
    a = pts(100, 100)
    anns = [gt(1, 1, a), gt(2, 2, a), gt(3, 3, a)]

    def setup(p):
        p.imgIds = [3, 1, 3, 2, 1]
    return dataset(anns, [1, 2, 3, 4]), [det(3, a, 0.9), det(1, a, 0.4), far(2, 0.6), det(4, a, 0.3)], setup


def categories():
    """Three categories over the same images, each with its own outcome: category 1 finds both of its ground truths,
    category 2 one of two behind a false positive, category 3 nothing; each category is accumulated on its own."""
    a, b = pts(100, 100), pts(300, 100)
    anns = [gt(1, 1, a), gt(2, 2, b), gt(3, 1, a, cat=2), gt(4, 2, b, cat=2), gt(5, 1, a, cat=3)]
    res = [det(1, a, 0.9), det(2, b, 0.8), far(1, 0.95) | {"category_id": 2}, det(2, b, 0.5, cat=2),
           far(1, 0.7) | {"category_id": 3}, far(2, 0.6) | {"category_id": 3}]
    return dataset(anns, [1, 2], cats=(1, 2, 3)), res, None


def categories_subset():
    """User-set params.catIds: only categories 3 and 1 (evaluate() sorts them), category 2's annotations left out."""
    ds, res, _ = categories()

    def setup(p):
        p.catIds = [3, 1]
    return ds, res, setup


CASES = {f.__name__: f for f in (crowd, no_keypoints, ignore_break, tie_last, nan_oks, gt_id_zero, score_ties, many_dets,
                                 empty_images, area_edges, no_positives, short_recall, img_ids, categories,
                                 categories_subset)}


# -- past one warp of ground truths ------------------------------------------------------------------------------------
# The device matcher steps through a unit's ground truths 32 at a time in annotation order (indices 0-31, 32-63, ...),
# and computes each one's position in evaluateImg's order (not ignored first) on the way.  The two orders agree in a
# unit without ignored ground truths; where a case has ignored ones, it puts them at annotation index 32 or later, so
# that they sit past the first step in both.  The cases below put each of the matcher's rules at and across those step
# edges; CROWD_CASES holds them apart from CASES.

def spot(j):
    """The person at slot j: slots lie 1000 px apart, so a detection at one slot has OKS exactly 0.0 with a ground truth
    at any other (every term's exponent is below -746: exp underflows to 0)."""
    return pts(100 + 1000 * j, 100)


def moved(p):
    """p with its first point 5000 px lower: OKS exactly 16/17 against p (sixteen terms of 1.0 and one of 0.0)."""
    q = p.copy()
    q[0, 1] += 5000
    return q


def dup_across_steps():
    """70 ground truths with equal OKS 1.0 at sorted positions (5, 37), (31, 32) and (0, 64): the later one wins the
    tie, the next detection takes the earlier one."""
    slot = list(range(70))
    slot[37], slot[32], slot[64] = 5, 31, 0
    anns = [gt(j + 1, 1, spot(s)) for j, s in enumerate(slot)]
    res = [det(1, spot(s), sc) for s, sc in zip((5, 5, 31, 31, 0, 0), (0.9, 0.8, 0.7, 0.6, 0.5, 0.4))]
    return dataset(anns, [1]), res, None


def earlier_max():
    """OKS 1.0 at position 3 in the first step and 16/17 at position 36 in the second: the later, smaller one does not
    take the match; the next detection gets it where 16/17 reaches the threshold."""
    p = [spot(j) for j in range(40)]
    p[36] = moved(spot(3))
    anns = [gt(j + 1, 1, q) for j, q in enumerate(p)]
    return dataset(anns, [1]), [det(1, spot(3), 0.9), det(1, spot(3), 0.8)], None


def nan_steps():
    """Three images of 72 ground truths, a NaN ground-truth coordinate (NaN OKS with every detection) at sorted position
    31, 32 and 63: the last lane of a step, the first of the next, the last of the second.  Each detection has OKS 1.0
    at position 10 before the NaN and 16/17 eight positions after it: the NaN replaces the earlier maximum, and the next
    steps' ground truths are taken from OKS 0.0 up."""
    anns, res = [], []
    for img, q in ((1, 31), (2, 32), (3, 63)):
        p = [spot(j) for j in range(72)]
        p[q + 8] = moved(spot(10))
        row = [gt(len(anns) + j + 1, img, s) for j, s in enumerate(p)]
        row[q]["keypoints"][0] = math.nan
        anns += row
        res += [det(img, spot(10), 0.9), det(img, spot(10), 0.8)]
    return dataset(anns, [1, 2, 3]), res, None


def taken_past_32():
    """A ground truth at position 35, matched by the first detection, is skipped by the next ones, which scan on to the
    16/17 at position 38."""
    p = [spot(j) for j in range(40)]
    p[38] = moved(spot(35))
    anns = [gt(j + 1, 1, q) for j, q in enumerate(p)]
    return dataset(anns, [1]), [det(1, spot(35), sc) for sc in (0.9, 0.8, 0.7)], None


def crowd_past_32():
    """A crowd region at annotation index 34 among 36 persons (sorted position 36, behind them all) takes three
    detections."""
    anns = [gt(j + 1, 1, spot(j)) for j in range(36)]
    anns.insert(34, gt(100, 1, None, crowd=1, bbox=[100.0, 5000.0, 40.0, 40.0], area=1600.0))
    inside = np.tile([[120.0, 5020.0]], (17, 1))
    res = [det(1, spot(7), 0.9)] + [det(1, inside, sc) for sc in (0.8, 0.7, 0.6)] + [far(1, 0.5)]
    return dataset(anns, [1]), res, None


def break_past_32():
    """40 persons and three ignored ones (num_keypoints 0, visible points) at annotation indices 33, 38 and 42, sorted
    positions 40-42: the scan stops at the first ignored one after a match, though it ties; without a match among the
    persons the ignored ones are matched."""
    anns = [gt(j + 1, 1, spot(j)) for j in range(40)]
    for at, (aid, s) in zip((33, 38, 42), ((101, 20), (102, 50), (103, 51))):
        anns.insert(at, gt(aid, 1, spot(s)) | {"num_keypoints": 0})
    res = [det(1, spot(s), sc) for s, sc in zip((20, 50, 50, 20), (0.9, 0.8, 0.7, 0.6))]
    return dataset(anns, [1]), res, None


def iou_thr_edges():
    """iouThrs 0.0, 0.5 and 1.0 over 40 persons: 1.0 is capped at 1 - 1e-10, so OKS 1.0 still matches; at 0.0 a
    detection far from everyone matches at OKS 0.0, the last free ground truth (position 39, then 38)."""
    anns = [gt(j + 1, 1, spot(j)) for j in range(40)]
    res = [det(1, spot(12), 0.9), det(1, moved(spot(25)), 0.8), far(1, 0.7), far(1, 0.6)]

    def setup(p):
        p.iouThrs = np.array([0.0, 0.5, 1.0])
    return dataset(anns, [1]), res, setup


CROWD_CASES = {f.__name__: f for f in (dup_across_steps, earlier_max, nan_steps, taken_past_32, crowd_past_32,
                                       break_past_32, iou_thr_edges)}


CROWDED_SIZES = (31, 32, 33, 63, 64, 65, 97)
SIGMA_COUNTS = (1, 7, 8, 9, 16, 24, 127, 128)
_SIGMAS = np.array([.26, .25, .25, .35, .35, .79, .79, .72, .72, .62, .62, 1.07, 1.07, .87, .87, .89, .89]) / 10.0


def sigmas(k):
    """k per-keypoint OKS sigmas: COCO's 17, repeated."""
    return np.resize(_SIGMAS, k)


def crowded_set(seed, sizes, k=17, *, first_id=1, categories=1):
    """A seeded ground truth and result list, ``(dataset, results)`` as ``synth.coco_keypoint_set`` makes them, with
    ``sizes[i]`` ground truths in image i and k keypoints (3k values) per annotation.

    Persons stand in cells 500 px apart, so no detection comes near the grown boxes of two keypoint-less ground truths
    (a near-tie that cannot be pinned).  Between an eighth and a half of an image's ground truths are ignored --
    keypoint-less (num_keypoints 0, box distance) or crowd regions -- at random places in annotation order, the order
    the device matcher steps through 32 at a time: in the larger images on both sides of index 32 among kept ones, and
    matched past it.  evaluateImg's order puts them last: across positions 31/32 in an image of 33, past 64 in larger
    ones.  Areas run from below 32^2 to above 96^2, so 'medium' and 'large' ignore more.  The others have 1-7
    visible points, a multiple of 8, 17 or more (a tail after two blocks of 8) or all k, as k allows.

    Images of 60 ground truths or more get 100 detections, the others up to twice their count: three in four are noisy
    copies of a ground truth, the rest false positives, with scores that sometimes tie.  Copies of a keypoint-less
    ground truth miss no point: their points inside its grown box score exactly 1.0, and with others missed at (0, 0)
    the OKS would be a fraction j/k plus terms below the sum's rounding, on a threshold for k = 8, 16, 24 or 128.
    ``categories`` > 1: category c (1-based) is the set of seed ``seed + 100 (c - 1)``, its annotation ids offset by
    ``c x 10^6``."""
    if categories > 1:
        ds, res = crowded_set(seed, sizes, k, first_id=first_id)
        for c in range(2, categories + 1):
            d2, r2 = crowded_set(seed + 100 * (c - 1), sizes, k, first_id=first_id)
            for a in d2["annotations"]:
                a.update(category_id=c, id=a["id"] + c * 10 ** 6)
            for r in r2:
                r.update(category_id=c)
            ds["annotations"] += d2["annotations"]
            res += r2
        ds["categories"] = [{"id": c, "name": f"person{c}", "supercategory": "person"}
                            for c in range(1, categories + 1)]
        return ds, res
    rng = np.random.default_rng(seed)
    tmpl = np.random.default_rng(k).uniform(-8, 8, (k, 2))
    anns, results = [], []
    for n, G in enumerate(sizes):
        img = first_id + n
        side = max(1, int(np.ceil(np.sqrt(G))))
        cells = rng.permutation(side * side)[:G]
        ign = set(rng.choice(G, int(rng.integers(G // 8, G // 2 + 1)), replace=False).tolist()) if G else set()
        persons = []
        for j in range(G):
            scale = float(np.exp(rng.uniform(np.log(0.6), np.log(8.0))))
            c = np.array([250 + 500 * (cells[j] % side), 250 + 500 * (cells[j] // side)], np.float64)
            p = c + tmpl * scale + rng.normal(0, 0.5, (k, 2))
            x0, y0 = p.min(0) - scale
            bw, bh = p.max(0) - p.min(0) + 2 * scale
            area = float(bw * bh * rng.uniform(0.4, 0.7))
            vis = np.zeros(k, np.int64)
            if j not in ign:
                options = [int(rng.integers(1, min(k, 7) + 1)), k]
                if k >= 8:
                    options.append(8 * int(rng.integers(1, k // 8 + 1)))
                if k >= 17:
                    options.append(int(rng.integers(17, k + 1)))
                k1 = options[int(rng.integers(len(options)))]
                vis[rng.choice(k, k1, replace=False)] = rng.choice([1, 2], k1)
            crowd = int(j in ign and rng.random() < 1 / 3)
            kp = np.zeros((k, 3), np.int64)
            kp[vis > 0, :2] = np.rint(p[vis > 0]).astype(np.int64)
            kp[:, 2] = vis
            anns.append({"id": len(anns) + first_id, "image_id": img, "category_id": 1, "iscrowd": crowd,
                         "num_keypoints": int((vis > 0).sum()), "keypoints": kp.reshape(-1).tolist(),
                         "bbox": [float(x0), float(y0), float(bw), float(bh)], "area": area})
            persons.append((p, scale, bool(vis.any())))
        for _ in range(100 if G >= 60 else int(rng.integers(0, 2 * G + 1))):
            labelled = True
            if persons and rng.random() < 0.75:
                p, scale, labelled = persons[int(rng.integers(len(persons)))]
                xy = p + rng.normal(0, rng.uniform(0.1, 1.5) * scale, (k, 2))
            else:
                scale = float(np.exp(rng.uniform(np.log(0.6), np.log(8.0))))
                xy = rng.uniform(0, 500 * side, 2) + tmpl * scale
            miss = (rng.random(k) < 0.15) & labelled
            xy[miss] = 0.0
            kp = np.concatenate([xy, (~miss)[:, None].astype(np.float64)], 1)
            results.append({"image_id": img, "category_id": 1,
                            "keypoints": [v if j % 3 != 2 else int(v) for j, v in enumerate(kp.reshape(-1).tolist())],
                            "score": float(np.round(rng.uniform(0.05, 1.0), 2 if rng.random() < 0.3 else 12))})
    images = [{"id": first_id + n, "file_name": f"{first_id + n}.jpg", "width": 640, "height": 480}
              for n in range(len(sizes))]
    return {"images": images, "annotations": anns,
            "categories": [{"id": 1, "name": "person", "supercategory": "person"}]}, results


def set_params(*before, **values):
    """A setup that runs the setups ``before``, then sets each of ``values`` (a copy) on the params."""
    def setup(p):
        for s in before:
            s(p)
        for f, v in values.items():
            setattr(p, f, copy.deepcopy(v))
    return setup


# user-set parameters, each applied to a COCOeval's params before evaluate()
PARAM_SETS = {
    "iou_one": set_params(iouThrs=np.array([0.7])),
    "iou_unsorted": set_params(iouThrs=np.array([0.75, 0.5, 0.95, 0.6, 0.85])),
    "iou_20": set_params(iouThrs=np.linspace(0.5, 0.975, 20)),
    "rec_one": set_params(recThrs=np.array([0.3])),
    # up to recall 0.5, so that the thresholds past the first 256 are reached
    "rec_257": set_params(recThrs=np.linspace(0.0, 0.5, 257)),
    "rec_1000": set_params(recThrs=np.linspace(0.0, 1.0, 1000)),
    "rec_unsorted": set_params(recThrs=np.random.default_rng(5).permutation(np.linspace(0.0, 0.5, 301))),
    "area_one": set_params(areaRng=[[0.0, 1e10]], areaRngLbl=["all"]),
    "area_six": set_params(areaRng=[[0.0, 1e10], [32.0 ** 2, 96.0 ** 2], [96.0 ** 2, 1e10], [0.0, 32.0 ** 2],
                                    [5000.5, 5000.5], [96.0 ** 2, 32.0 ** 2]],
                           areaRngLbl=["all", "medium", "large", "small", "empty", "inverted"]),
    "max_dets_0": set_params(maxDets=[0]),
    "max_dets_100_1": set_params(maxDets=[100, 1]),
    "max_dets_1_20_100": set_params(maxDets=[1, 20, 100]),
}
UP_TO_100 = set_params(maxDets=[1, 20, 100])  # 100 kept per image; 20 stays, so summarize() reports numbers, not -1


def crowded_images():
    """``(dataset, results, setup)``: one image of each of CROWDED_SIZES ground truths, maxDets [1, 20, 100]."""
    return crowded_set(3, CROWDED_SIZES) + (UP_TO_100,)


def keypoint_count(k):
    """``(dataset, results, setup)``: crowded images of k keypoints, with k sigmas and maxDets [1, 20, 100]."""
    return crowded_set(11, (9, 33, 70), k) + (set_params(UP_TO_100, kpt_oks_sigmas=sigmas(k)),)


def two_categories():
    """``(dataset, results, setup)``: two categories of crowded images, maxDets [1, 20, 100]."""
    return crowded_set(9, (33, 65, 97), categories=2) + (UP_TO_100,)


def param_set(name, where):
    """``(dataset, results, setup)``: PARAM_SETS[name] on a seeded set of 60 images (``where`` 'seeded', from
    synth.coco_keypoint_set) or on crowded images ('crowded', with maxDets [1, 20, 100] unless maxDets is the parameter
    set)."""
    if where == "seeded":
        return synth.coco_keypoint_set(41, 60) + (PARAM_SETS[name],)
    base = () if name.startswith("max_dets") else (UP_TO_100,)
    return crowded_set(7, (33, 64, 97)) + (set_params(*base, PARAM_SETS[name]),)
