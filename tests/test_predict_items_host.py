"""CPU: the item planner of the batched multi-scale / rotation-search predict() (``dropin.plan_items``)."""
import itertools

import numpy as np

from oracle import prenet_port as pn

SEARCHES = [([1.0], [0.0]), ([0.5, 1.0, 1.5, 2.0], [0.0]), ([1.0], [0.0, 30.0, -30.0]), ([1.0, 0.5], [0.0, 30.0]),
            ([0.5, 1.0, 1.5, 2.0, 2.5], [0.0]), ([2.0], [45.0])]


def _shapes():
    rng = np.random.default_rng(8)
    return [(480, 640), (640, 480), (427, 640), (612, 612), (375, 500), (1, 1), (3, 7000), (5000, 20), (2000, 3000),
            (641, 639)] + [tuple(int(v) for v in rng.integers(1, 2000, 2)) for _ in range(60)]


def test_plan_items_is_the_prenet_geometry():
    """Every (image, item) of product(multiplier, rotation_search): the multiplier of evaluate.py:87, the clamped scale,
    the angle, cv2.resize's size and its padding -- clamped items included."""
    from improved_body_parts_b200 import dropin

    shapes = _shapes()
    clamped = 0
    for (scales, angles), (boxsize, md) in itertools.product(SEARCHES, ((640, 64), (368, 8), (160, 16))):
        params = dict(scale_search=scales, rotation_search=angles)
        plan, _ = dropin.plan_items(shapes, params, dict(boxsize=boxsize, max_downsample=md, stride=4))
        assert len(plan) == len(shapes)
        for i, (h, w) in enumerate(shapes):
            want = []
            for s, angle in itertools.product(scales, angles):
                multiplier = s * boxsize / h
                scale = pn.clamp_scale(multiplier, (h, w))
                clamped += scale != multiplier
                H1, W1 = pn.resized_size(h, w, scale)
                want.append((multiplier, scale, angle, H1, W1, -(-H1 // md) * md, -(-W1 // md) * md))
            assert plan[i] == want, (h, w, scales, angles, boxsize, md)
    assert clamped > 0


def test_buckets_hold_every_item_once_in_first_appearance_order():
    from improved_body_parts_b200 import dropin

    shapes = _shapes()
    for scales, angles in SEARCHES:
        plan, buckets = dropin.plan_items(shapes, dict(scale_search=scales, rotation_search=angles),
                                          dict(boxsize=640, max_downsample=64, stride=4))
        members = [m for ms in buckets.values() for m in ms]
        assert sorted(members) == [(i, t) for i in range(len(shapes)) for t in range(len(scales) * len(angles))]
        seen = []
        for i, items in enumerate(plan):
            for t, item in enumerate(items):
                assert (i, t) in buckets[item[5:]]
                if item[5:] not in seen:
                    seen.append(item[5:])
        assert list(buckets) == seen
        for ms in buckets.values():
            assert ms == sorted(ms)  # (image, item) order inside a bucket
    # a rotated item shares its scale's bucket
    _, b = dropin.plan_items([(480, 640)], dict(scale_search=[1.0, 0.5], rotation_search=[0.0, 30.0]),
                             dict(boxsize=640, max_downsample=64))
    assert b == {(640, 896): [(0, 0), (0, 1)], (320, 448): [(0, 2), (0, 3)]}


def test_bucket_planner_is_the_prenet_geometry():
    """One item per image: (multiplier, scale, angle, H1, W1, Hp, Wp) equals cv2.resize's size (cvRound) and its
    padding, the 2600 / 3800 clamp included, and images are bucketed by (Hp, Wp) in order of first appearance."""
    from improved_body_parts_b200 import dropin

    rng = np.random.default_rng(3)
    shapes = [(480, 640), (640, 480), (427, 640), (640, 427), (612, 612), (375, 500), (640, 640), (1, 1), (3, 7000),
              (5000, 20), (333, 333), (641, 639)] + [tuple(int(v) for v in rng.integers(1, 2000, 2)) for _ in range(200)]
    for boxsize, scale_search, md in ((640, 1.0, 64), (368, 1.0, 8), (640, 0.5, 32), (640, 2.0, 64), (160, 1.3, 16)):
        params = dict(scale_search=[scale_search], rotation_search=[0.0])
        model_params = dict(boxsize=boxsize, max_downsample=md, stride=4)
        plan, buckets = dropin.plan_items(shapes, params, model_params)
        assert len(plan) == len(shapes)
        seen = []
        for i, (h, w) in enumerate(shapes):
            multiplier = scale_search * boxsize / h
            scale = pn.clamp_scale(multiplier, (h, w))
            H1, W1 = pn.resized_size(h, w, scale)
            Hp, Wp = -(-H1 // md) * md, -(-W1 // md) * md
            assert plan[i] == [(multiplier, scale, 0.0, H1, W1, Hp, Wp)], (h, w, boxsize, scale_search, md)
            assert (i, 0) in buckets[(Hp, Wp)]
            if (Hp, Wp) not in seen:
                seen.append((Hp, Wp))
        assert list(buckets) == seen
        assert sorted(m for ms in buckets.values() for m in ms) == [(i, 0) for i in range(len(shapes))]
    # the reference's settings: images with one aspect ratio share an input size
    _, b = dropin.plan_items([(480, 640), (240, 320), (640, 480), (960, 1280)],
                             dict(scale_search=[1.0], rotation_search=[0.0]), dict(boxsize=640, max_downsample=64))
    assert b == {(640, 896): [(0, 0), (1, 0), (3, 0)], (640, 512): [(2, 0)]}
