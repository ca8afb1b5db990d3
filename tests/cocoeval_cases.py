"""Hand-built keypoint-evaluation cases, one per rule of pycocotools' keypoint path, shared by the port's CPU tests and
the device tests.  Every OKS that decides a match is exact: a detection equal to its ground truth has OKS 1.0, one far
from every point has OKS 0.0, one inside a keypoint-less ground truth's grown box has OKS 1.0, and a NaN area gives NaN.

``CASES[name]()`` returns ``(dataset, results, setup)``: a ground-truth dict, the ``format_results``-style list, and a
function applied to a ``COCOeval``'s ``params`` before ``evaluate()`` (or None)."""
from __future__ import annotations

import math

import numpy as np

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
