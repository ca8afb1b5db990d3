"""CPU: the fixture of the validation-geometry tests (``coco_geometry``, used by test_gpu_coco_geometry.py) -- its item
sizes against ``dropin.plan_items`` and the CPU chain's coverage of the paths the GPU tests are meant to reach."""
import numpy as np
import pytest

import coco_geometry as cg


@pytest.mark.parametrize("name", list(cg.CONFIGS))
def test_geometry_restated_from_evaluate_is_dropins(name):
    from improved_body_parts_b200 import dropin
    cfg = cg.CONFIGS[name]
    shapes = [(s.H, s.W) for s in cg.FIXTURE]
    plan, buckets = dropin.plan_items(shapes, cfg.params(), cg.MODEL_PARAMS)
    for (H, W), items in zip(shapes, plan):
        want = [cg.geometry(H, W, s) for s in cfg.scale_search for _ in cfg.rotation_search]
        got = [(m, scale) + tuple(geo) for m, scale, _, *geo in items]
        assert got == want, (H, W)
    assert sum(len(v) for v in buckets.values()) == len(shapes) * len(cfg.scale_search) * len(cfg.rotation_search)


def test_geometry_of_the_validation_images():
    """The two shapes the stage is named after: 480 x 640 -> a 640 x 853 crop in a 640 x 896 input (second resize 0.75),
    640 x 427 -> multiplier 1, the crop is the image."""
    assert cg.geometry(480, 640, 1.0)[2:] == (640, 853, 640, 896)
    assert cg.geometry(427, 640, 1.0)[2:] == (640, 959, 640, 960)
    m, scale, H1, W1, Hp, Wp = cg.geometry(640, 427, 1.0)
    assert m == scale == 1.0 and (H1, W1, Hp, Wp) == (640, 427, 640, 448)
    assert cg.geometry(480, 640, 2.0)[2:] == (1280, 1707, 1280, 1728)
    assert {(s.H, s.W) for s in cg.FIXTURE} == set(cg.SHAPES) and len(cg.FIXTURE) == 24
    assert len(cg.CROWDED) == 2 and len(cg.TWINS) == 1
    for cfg in cg.CONFIGS.values():  # every configuration has a non-identity and an identity second resize
        assert {cg.FIXTURE[i].H == 640 for i in cfg.images} == {True, False} or len(cfg.images) == 1, cfg.name


def test_markers_are_distinct_and_above_the_padding():
    codes = [int(cg.image(i, s)[0, 0, 0]) for i, s in enumerate(cg.FIXTURE[:3])]
    assert codes == [cg.MARKER0, cg.MARKER0 + cg.MARKER_STEP, cg.MARKER0 + 2 * cg.MARKER_STEP]
    assert cg.MARKER0 > cg.MODEL_PARAMS["padValue"] and cg.MARKER0 + cg.MARKER_STEP * (len(cg.FIXTURE) - 1) <= 255


def test_persons_span_15_to_80_percent_of_the_image_and_straddle_the_border():
    heights, straddle = [], 0
    for s in cg.FIXTURE:
        _, _, H1, W1, _, _ = cg.geometry(s.H, s.W, 1.0)
        j = cg._skeletons(s, (H1 / 4, W1 / 4))
        heights += list((j[:, :, 1].max(1) - j[:, :, 1].min(1)) / (H1 / 4))
        out = (j[..., 0] < 0) | (j[..., 1] < 0) | (j[..., 0] > W1 / 4 - 1) | (j[..., 1] > H1 / 4 - 1)
        straddle += int((out.any(1) & ~out.all(1)).sum())
    assert 0.13 <= min(heights) and max(heights) <= 0.85 and np.median(heights) > 0.3, (min(heights), max(heights))
    assert straddle >= 5


@pytest.fixture(scope="module")
def chains():
    cfg = cg.CONFIGS["default"]
    picks = sorted(set(cg.CROWDED + cg.TWINS + [0, 1, 2, 4, 6, 7, 8]))
    return {i: cg.cpu_chain(cfg, i) for i in picks}


def test_the_chain_reaches_the_paths(chains):
    """A limb with more than 256 candidates, most scored pairs with all 20 samples, border peaks."""
    cov = cg.coverage(chains)
    assert cov["max_cands"] > 256, cov
    assert cov["full_samples"] > 0.5, cov
    assert cov["border_images"], cov
    assert all(int(chains[i].oracle.cand_count[0].max()) > 256 for i in cg.CROWDED)


def test_the_twins_tie(chains):
    """The twins' limbs are scored on exact translates of one map: the two rows of a limb tie on their priority, and
    only the matcher's tie-break (generation order) orders them."""
    c = chains[cg.TWINS[0]]
    ties = [k for k, rows in enumerate(c.structs[1]) if len(rows) >= 2 and rows[0, 2] == rows[1, 2]]
    assert len(ties) >= 10, ties
    for k in ties:  # i-major generation order: the left twin's row first
        rows = c.structs[1][k]
        assert rows[0, 3] < rows[1, 3] or (rows[0, 3] == rows[1, 3] and rows[0, 4] < rows[1, 4])
