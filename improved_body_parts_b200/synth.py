"""Seeded synthetic keypoint / body-part maps shaped like the network's output.

The recipe imitates the reference's ground-truth generator (SURVEY.md §8d):
keypoint map = per-channel MAX over persons of ``exp(-d^2 / 2 sigma^2)`` with
sigma = 9 px / stride 4 (``config/config.py:40``, ``py_data_heatmapper.py:133-149``);
body-part map of limb (a, b) = ``exp(-d_perp^2 / 2 sigma_p^2)``, sigma_p = 7/4 px, inside the
end-point bounding box grown by 1 px, small values floored to 0.01, AVERAGED where persons overlap
(``py_data_heatmapper.py:190-227,309-340``); plus U(0, 0.02) background noise; clipped to [0, 1].
Nothing here is on the product path: it feeds tests, golden fixtures and ``bench.py``.

Maps are returned channel-first (``[K, H, W]`` / ``[L, H, W]`` float32), the layout the CUDA path reads.
"Dirty" options steer inputs into the branches clean skeletons never reach (SURVEY.md §8a).
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np

from .skeleton import LIMBS, NUM_PARTS

# 18-joint standing template in map pixels at scale 1 (x right, y down), hips at the origin.
_TEMPLATE = np.array([
    (0.0, -17.0), (0.0, -12.0), (-5.0, -12.0), (-7.0, -6.0), (-8.0, 0.0), (5.0, -12.0), (7.0, -6.0), (8.0, 0.0),
    (-3.0, 0.0), (-3.5, 8.0), (-4.0, 16.0), (3.0, 0.0), (3.5, 8.0), (4.0, 16.0),
    (-1.5, -18.5), (1.5, -18.5), (-3.0, -17.5), (3.0, -17.5)], dtype=np.float64)

KEYPOINT_SIGMA = 9.0 / 4.0
LIMB_SIGMA = 7.0 / 4.0
LIMB_FLOOR_BELOW, LIMB_FLOOR_VALUE = 0.015, 0.01
NOISE_MAX = 0.02


def sample_skeletons(rng: np.random.Generator, persons: int, H: int, W: int, *, edge: bool = False,
                     scale_range: Tuple[float, float] = (0.8, 1.3), jitter: float = 0.6) -> np.ndarray:
    """Joint coordinates ``[persons, 18, 2]`` (x, y) in map pixels."""
    scale = rng.uniform(scale_range[0], scale_range[1], size=(persons, 1, 1))
    body = _TEMPLATE[None] * scale + rng.normal(0.0, jitter, size=(persons, NUM_PARTS, 2))
    if edge:  # let bodies straddle the border so the 5x5 refine box leaves the image
        cx = rng.uniform(0.0, W - 1.0, size=(persons, 1))
        cy = rng.uniform(0.0, H - 1.0, size=(persons, 1))
    else:
        cx = rng.uniform(min(12.0, W / 4), max(W - 13.0, W / 2), size=(persons, 1))
        cy = rng.uniform(min(26.0, H / 3), max(H - 23.0, H / 2), size=(persons, 1))
    body[..., 0] += cx
    body[..., 1] += cy
    return body


def _put_keypoint(plane: np.ndarray, x: float, y: float, sigma: float) -> None:
    H, W = plane.shape
    r = int(np.ceil(4.0 * sigma))
    x0, x1 = max(int(np.floor(x)) - r, 0), min(int(np.floor(x)) + r + 2, W)
    y0, y1 = max(int(np.floor(y)) - r, 0), min(int(np.floor(y)) + r + 2, H)
    if x0 >= x1 or y0 >= y1:
        return
    ex = np.exp(-(np.arange(x0, x1, dtype=np.float32) - np.float32(x)) ** 2 / np.float32(2.0 * sigma * sigma))
    ey = np.exp(-(np.arange(y0, y1, dtype=np.float32) - np.float32(y)) ** 2 / np.float32(2.0 * sigma * sigma))
    np.maximum(plane[y0:y1, x0:x1], np.outer(ey, ex), out=plane[y0:y1, x0:x1])


def _put_limb(acc: np.ndarray, cnt: np.ndarray, xa, ya, xb, yb, sigma: float) -> None:
    H, W = acc.shape
    dx, dy = xb - xa, yb - ya
    norm = float(np.hypot(dx, dy))
    if norm == 0.0:
        return
    x0, x1 = int(round(min(xa, xb) - 1.0)), int(round(max(xa, xb) + 1.0))
    y0, y1 = int(round(min(ya, yb) - 1.0)), int(round(max(ya, yb) + 1.0))
    if x1 < 0 or y1 < 0 or x0 >= W or y0 >= H:
        return
    x0, y0, x1, y1 = max(x0, 0), max(y0, 0), min(x1, W - 1), min(y1, H - 1)
    X = np.arange(x0, x1 + 1, dtype=np.float32)[None, :]
    Y = np.arange(y0, y1 + 1, dtype=np.float32)[:, None]
    d = np.abs(np.float32(dx) * (np.float32(ya) - Y) - (np.float32(xa) - X) * np.float32(dy)) / np.float32(norm + 1e-6)
    g = np.exp(-(d * d) / np.float32(2.0 * sigma * sigma))
    g[g <= LIMB_FLOOR_BELOW] = LIMB_FLOOR_VALUE
    acc[y0:y1 + 1, x0:x1 + 1] += g
    cnt[y0:y1 + 1, x0:x1 + 1] += 1


def render(joints: np.ndarray, visible: np.ndarray, H: int, W: int, rng: np.random.Generator,
           limbs: Sequence[Tuple[int, int]] = LIMBS, noise: float = NOISE_MAX,
           noise_levels: Optional[int] = None, sigma_scale: float = 1.0) -> Tuple[np.ndarray, np.ndarray]:
    """Rasterise ``joints [P,18,2]`` (``visible [P,18]`` bool) into ``heat [18,H,W]`` and ``paf [L,H,W]``."""
    P = joints.shape[0]
    heat = np.zeros((NUM_PARTS, H, W), np.float32)
    paf = np.zeros((len(limbs), H, W), np.float32)
    for p in range(P):
        for c in range(NUM_PARTS):
            if visible[p, c]:
                _put_keypoint(heat[c], joints[p, c, 0], joints[p, c, 1], KEYPOINT_SIGMA * sigma_scale)
    cnt = np.zeros((H, W), np.int32)
    for k, (a, b) in enumerate(limbs):
        cnt[:] = 0
        for p in range(P):
            if visible[p, a] and visible[p, b]:
                _put_limb(paf[k], cnt, joints[p, a, 0], joints[p, a, 1], joints[p, b, 0], joints[p, b, 1], LIMB_SIGMA * sigma_scale)
        np.divide(paf[k], cnt, out=paf[k], where=cnt > 0)
    if noise > 0:
        for arr in (heat, paf):
            if noise_levels:  # quantised noise: compressible fixtures, plateaus below every threshold
                n = rng.integers(0, noise_levels + 1, size=arr.shape).astype(np.float32) * np.float32(noise / noise_levels)
            else:
                n = rng.random(arr.shape, dtype=np.float32) * np.float32(noise)
            arr += n
    np.clip(heat, 0.0, 1.0, out=heat)
    np.clip(paf, 0.0, 1.0, out=paf)
    return heat, paf


def make_image(seed: int, H: int = 128, W: int = 128, persons: int = 10, *,
               limbs: Sequence[Tuple[int, int]] = LIMBS, drop_prob: float = 0.0, plateau: int = 0, spikes: int = 0,
               colocate: int = 0, missing_parts: Sequence[int] = (), edge: bool = False, negative_bias: float = 0.0,
               stretch: int = 0, noise_levels: Optional[int] = None, heat_gain: float = 1.0, paf_gain: float = 1.0,
               scale_range: Tuple[float, float] = (0.8, 1.3), sigma_scale: float = 1.0,
               noise: float = NOISE_MAX) -> Tuple[np.ndarray, np.ndarray]:
    """One synthetic image.  ``seed`` fully determines the result for a given numpy build.

    Dirty knobs: ``drop_prob`` removes joints at random; ``plateau`` copies that many peak values onto a
    neighbour pixel (equality NMS then yields two peaks, util.py:182); ``spikes`` adds isolated noise peaks
    above thre1; ``colocate`` snaps that many (person, part) joints onto another part of the same person
    (norm == 0, evaluate.py:228-230); ``missing_parts`` blanks whole part classes (special_k, :272-274);
    ``edge`` lets bodies leave the image (integer-coordinate border peaks, util.py:201-202);
    ``negative_bias`` shifts the body-part maps down so some samples are negative;
    ``stretch`` moves that many wrists far away (long-limb rejects, evaluate.py:324,353,409);
    ``heat_gain`` / ``paf_gain`` scale the maps (weak persons that the final prune removes, :491-496);
    ``scale_range`` / ``sigma_scale`` size the bodies and the blobs (4x for maps at image resolution, stride 4);
    ``noise`` is the amplitude of the uniform background noise (0 for smooth, up-sampled-looking maps).
    """
    rng = np.random.default_rng(seed)
    joints = sample_skeletons(rng, persons, H, W, edge=edge, scale_range=scale_range)
    visible = rng.random((persons, NUM_PARTS)) >= drop_prob
    for c in missing_parts:
        visible[:, c] = False
    for _ in range(colocate):
        if persons == 0:
            break
        p = int(rng.integers(persons))
        a, b = (int(v) for v in rng.choice(NUM_PARTS, size=2, replace=False))
        joints[p, a] = np.round(joints[p, b])  # both exactly on a pixel centre
        joints[p, b] = joints[p, a]
    for _ in range(stretch):
        if persons == 0:
            break
        p = int(rng.integers(persons))
        c = int(rng.choice([4, 7, 10, 13]))
        joints[p, c, 0] = rng.uniform(4, W - 5)
        joints[p, c, 1] = rng.uniform(4, H - 5)
    heat, paf = render(joints, visible, H, W, rng, limbs=limbs, noise=noise, noise_levels=noise_levels, sigma_scale=sigma_scale)
    for _ in range(spikes):
        c, y, x = int(rng.integers(NUM_PARTS)), int(rng.integers(H)), int(rng.integers(W))
        heat[c, y, x] = max(heat[c, y, x], np.float32(rng.uniform(0.12, 0.6)))
    if plateau:
        done = 0
        for c in rng.permutation(NUM_PARTS):
            if done >= plateau:
                break
            y, x = np.unravel_index(int(np.argmax(heat[c])), heat[c].shape)
            if heat[c, y, x] > 0.2:
                dy, dx = [(0, 1), (1, 0), (1, 1), (0, -1)][done % 4]
                yy, xx = min(max(y + dy, 0), H - 1), min(max(x + dx, 0), W - 1)
                heat[c, yy, xx] = heat[c, y, x]
                done += 1
    if heat_gain != 1.0:
        heat *= np.float32(heat_gain)
    if paf_gain != 1.0:
        paf *= np.float32(paf_gain)
    if negative_bias:
        paf -= np.float32(negative_bias)
    return heat, paf


def make_batch(base_seed: int, n: int, H: int = 128, W: int = 128, persons: int = 10, **kw):
    """``heat [n,18,H,W]``, ``paf [n,L,H,W]`` float32; image ``i`` uses seed ``base_seed + i``."""
    limbs = kw.get("limbs", LIMBS)
    heat = np.empty((n, NUM_PARTS, H, W), np.float32)
    paf = np.empty((n, len(limbs), H, W), np.float32)
    for i in range(n):
        heat[i], paf[i] = make_image(base_seed + i, H, W, persons, **kw)
    return heat, paf


def make_network_output(seed: int, h: int, w: int, persons: int, *, body_scale: float = 1.0, noise: float = 0.004,
                        base_hw: Tuple[int, int] = None, scale_range: Tuple[float, float] = (0.8, 1.3)) -> np.ndarray:
    """What the IMHN would answer for (image, mirrored image): ``[2, 50, h, w]`` float32 in the network's channel
    layout (body parts 0..29, keypoints 30..47, background 48..49; config/config.py:101-103).

    The first map holds the synthetic maps, the second a mirrored, channel-permuted copy plus a little noise, so that the
    flip ensemble (evaluate.py:139-140) has something to average.  ``body_scale`` renders the SAME skeletons (drawn for a
    ``base_hw`` map, default ``h / body_scale``) at another resolution -- the multi-scale search of predict()."""
    from .skeleton import FLIP_HEAT_ORD, FLIP_PAF_ORD
    rng = np.random.default_rng(seed)
    bh, bw = base_hw if base_hw is not None else (int(round(h / body_scale)), int(round(w / body_scale)))
    joints = sample_skeletons(rng, persons, bh, bw, scale_range=scale_range) * body_scale
    visible = np.ones((persons, NUM_PARTS), bool)
    heat, paf = render(joints, visible, h, w, np.random.default_rng(seed + 1), sigma_scale=body_scale)
    out = np.zeros((2, 50, h, w), np.float32)
    out[0, :30], out[0, 30:48] = paf, heat
    out[0, 48:] = rng.random((2, h, w), dtype=np.float32)
    out[1, :30] = paf[np.argsort(FLIP_PAF_ORD)][..., ::-1]
    out[1, 30:48] = heat[np.argsort(FLIP_HEAT_ORD[:NUM_PARTS])][..., ::-1]
    out[1] += (rng.random((50, h, w), dtype=np.float32) - 0.5) * np.float32(noise)
    return out


def coco_keypoint_set(seed: int, n_images: int, *, first_id: int = 1, categories: int = 1):
    """A seeded ground truth and result list shaped like ``person_keypoints_val2017`` and ``format_results``' output,
    for keypoint evaluation: ``(dataset, results)``.

    Per image 0-12 persons of every COCO area range, some of them with no labelled keypoint and about one image in
    eight with a crowd region (``iscrowd`` 1, no keypoints); 0-25 detections per image, most of them noisy copies of a
    person (points ``format_results`` writes as ``(0, 0, 0)`` where a joint is missing), the rest false positives, with
    scores that sometimes tie.  Ground-truth points are integers with visibility 0-2, as in the COCO files.
    ``categories`` > 1: category c (1-based) of the same images is the set of seed ``seed + 100 (c - 1)``, its
    annotation ids offset by ``c x 10^6``."""
    if categories > 1:
        dataset, results = coco_keypoint_set(seed, n_images, first_id=first_id)
        ids = [i["id"] for i in dataset["images"]]
        for c in range(2, categories + 1):
            d2, r2 = coco_keypoint_set(seed + 100 * (c - 1), n_images, first_id=first_id)
            remap = dict(zip([i["id"] for i in d2["images"]], ids))
            for a in d2["annotations"]:
                a.update(image_id=remap[a["image_id"]], category_id=c, id=a["id"] + c * 10 ** 6)
            for r in r2:
                r.update(image_id=remap[r["image_id"]], category_id=c)
            dataset["annotations"] += d2["annotations"]
            results += r2
        dataset["categories"] = [{"id": c, "name": f"person{c}", "supercategory": "person"}
                                 for c in range(1, categories + 1)]
        return dataset, results
    rng = np.random.default_rng(seed)
    images, anns, results = [], [], []
    tmpl = np.concatenate([_TEMPLATE[:1], _TEMPLATE[2:]])[:17]  # 17 points, the neck dropped
    ann_id = first_id
    for n in range(n_images):
        img_id = first_id + 7 * n + int(rng.integers(0, 7))
        W, H = int(rng.integers(320, 641)), int(rng.integers(240, 481))
        images.append({"id": img_id, "file_name": f"{img_id:012d}.jpg", "width": W, "height": H})
        persons, has_boxless = [], False
        for _ in range(int(rng.integers(0, 13)) if rng.random() < 0.9 else 0):
            scale = float(np.exp(rng.uniform(np.log(0.3), np.log(8.0))))
            cx, cy = rng.uniform(0, W), rng.uniform(0, H)
            pts = np.stack([cx + tmpl[:, 0] * scale, cy + tmpl[:, 1] * scale], 1) + rng.normal(0, 0.5, (17, 2))
            # at most one keypoint-less ground truth (a person or the crowd region) per image: two of them around one
            # detection give it OKS that differ only by the rounding of far points' terms, a near-tie no test can pin
            boxless = rng.random() < 0.1 and not has_boxless
            has_boxless |= boxless
            vis = np.zeros(17, int) if boxless else rng.choice([0, 1, 2], size=17, p=[0.25, 0.15, 0.6])
            kp = np.zeros((17, 3), np.int64)
            kp[vis > 0, 0:2] = np.rint(pts[vis > 0]).astype(np.int64)
            kp[:, 2] = vis
            x0, y0 = pts.min(0) - scale
            bw, bh = pts.max(0) - pts.min(0) + 2 * scale
            area = float(bw * bh * rng.uniform(0.4, 0.7))
            anns.append({"id": ann_id, "image_id": img_id, "category_id": 1, "iscrowd": 0,
                         "num_keypoints": int((vis > 0).sum()), "keypoints": kp.reshape(-1).tolist(),
                         "bbox": [float(x0), float(y0), float(bw), float(bh)], "area": area})
            ann_id += 1
            persons.append((pts, scale))
        if rng.random() < 0.125 and not has_boxless:
            bw, bh = rng.uniform(30, 200), rng.uniform(30, 200)
            anns.append({"id": ann_id, "image_id": img_id, "category_id": 1, "iscrowd": 1, "num_keypoints": 0,
                         "keypoints": [0] * 51, "bbox": [float(rng.uniform(0, W - bw)), float(rng.uniform(0, H - bh)),
                                                         float(bw), float(bh)], "area": float(bw * bh * 0.6)})
            ann_id += 1
        n_det = int(rng.integers(0, 26)) if persons or rng.random() < 0.3 else 0
        for _ in range(n_det):
            if persons and rng.random() < 0.75:
                pts, scale = persons[int(rng.integers(0, len(persons)))]
                xy = pts + rng.normal(0, rng.uniform(0.1, 1.5) * scale, (17, 2))
            else:
                scale = float(np.exp(rng.uniform(np.log(0.3), np.log(8.0))))
                xy = np.stack([rng.uniform(0, W) + tmpl[:, 0] * scale, rng.uniform(0, H) + tmpl[:, 1] * scale], 1)
            miss = rng.random(17) < 0.15
            xy[miss] = 0.0
            kp = np.concatenate([xy, (~miss)[:, None].astype(np.float64)], 1)
            score = float(np.round(rng.uniform(0.05, 1.0), 2 if rng.random() < 0.3 else 12))
            results.append({"image_id": img_id, "category_id": 1,
                            "keypoints": [v if j % 3 != 2 else int(v) for j, v in enumerate(kp.reshape(-1).tolist())],
                            "score": score})
    dataset = {"images": images, "annotations": anns,
               "categories": [{"id": 1, "name": "person", "supercategory": "person"}]}
    return dataset, results


def photo(seed: int, h: int, w: int, grey: bool = False) -> np.ndarray:
    """A seeded photo-like uint8 BGR (or grey) image: smooth noise at several scales plus fine grain, so that a JPEG of it
    has the size and coefficient statistics of a camera picture rather than of white noise."""
    import cv2
    rng = np.random.default_rng(seed)
    out = np.zeros((h, w, 3), np.float32)
    for s, amp in ((64, 45.0), (16, 30.0), (4, 18.0), (1, 8.0)):
        n = rng.standard_normal((h // s + 2, w // s + 2, 3)).astype(np.float32)
        out += cv2.resize(n, (w, h), interpolation=cv2.INTER_CUBIC) * amp
    img = np.clip(out + 128, 0, 255).astype(np.uint8)
    return cv2.cvtColor(img, cv2.COLOR_BGR2GRAY) if grey else img
