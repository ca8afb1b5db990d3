"""CPU: the numpy port of the colour distortion (tests/tint_port.py) against cv2 over every 8-bit input, against exact
arithmetic for its fused multiply-add, and against the reference's goldens (tests/golden/tint/)."""
import json
import os
import random
from fractions import Fraction

import numpy as np
import pytest

import tint_port as tt
from improved_body_parts_b200 import targets

COLOR = tt.golden_paths("color")
GEN = tt.golden_paths("gen")


def _cv2():
    return pytest.importorskip("cv2")


def test_goldens_cover_every_tail_class_and_a_strided_source():
    with open(os.path.join(tt.golden_dir(), "MANIFEST.json")) as f:
        man = json.load(f)
    cases = man["cases"]
    widths = {c["source"][1] for n, c in cases.items() if n.startswith("color_")}
    assert {w % 32 for w in widths} >= {0, 11, 20, 1, 31} and {640, 427, 500, 1, 33} <= widths
    assert any(c["pad_cols"] > 0 for n, c in cases.items() if n.startswith("color_"))
    assert sum(sum(c["tint"]) for n, c in cases.items() if n.startswith("gen_")) >= 2
    assert man["row_block"] >= 1 and man["cv2"]
    for p in COLOR + GEN:
        z = np.load(p)
        assert int(z["row_block"]) == man["row_block"] and str(z["cv2_version"]) == man["cv2"]


def _exact_f32(q: Fraction) -> np.float32:
    """``q`` rounded once to float32, ties to even, by exact comparison of the candidates around it."""
    r = np.float32(float(q))
    cands = [np.nextafter(r, np.float32(-np.inf)), r, np.nextafter(r, np.float32(np.inf))]
    best = min(cands, key=lambda c: (abs(Fraction(float(c)) - q), int(c.view(np.uint32)) & 1))
    return best


def test_fma_emulation_rounds_once():
    """fma_f32 against exact rational arithmetic on the HSV->BGR operands and on random float32 triples, including
    operands built to put the float64 sum exactly halfway between two float32 values."""
    rng = np.random.default_rng(0)
    S = (np.arange(256, dtype=np.float32) * np.float32(1 / 255.)).astype(np.float32)
    hh = rng.random(2000).astype(np.float32)
    a = np.concatenate([-S[rng.integers(0, 256, 2000)], rng.standard_normal(2000).astype(np.float32),
                        np.full(4, np.float32(2.0 ** -24))])
    b = np.concatenate([hh, rng.standard_normal(2000).astype(np.float32), np.float32([1 + 2.0 ** -23, 1, -1, 1 - 2.0 ** -24])])
    c = 1.0
    got = tt.fma_f32(a, b, c)
    for x, y, g in zip(a, b, got):
        want = _exact_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(c))
        assert g.view(np.uint32) == want.view(np.uint32), (x, y, g, want)


def test_bgr2hsv_equals_cv2_on_every_triple():
    cv2 = _cv2()
    t = tt.all_triples()
    want = cv2.cvtColor(t.reshape(4096, 4096, 3), cv2.COLOR_BGR2HSV).reshape(-1, 3)
    assert np.array_equal(tt.bgr2hsv(t), want)


@pytest.mark.parametrize("position", ["body", "tail"])
def test_hsv2bgr_equals_cv2_on_every_triple(position):
    """Body: rows 4096 wide (no tail at any block up to 4096).  Tail: rows one pixel wide (all tail)."""
    cv2 = _cv2()
    t = tt.all_triples()
    img = t.reshape(4096, 4096, 3) if position == "body" else t.reshape(-1, 1, 3)
    assert np.array_equal(tt.hsv2bgr(img, 32), cv2.cvtColor(img, cv2.COLOR_HSV2BGR))


def test_cv2_row_block_is_what_the_goldens_were_made_with():
    _cv2()
    with open(os.path.join(tt.golden_dir(), "MANIFEST.json")) as f:
        made = json.load(f)["row_block"]
    block = targets.cv2_row_block()
    if block != made:
        pytest.skip(f"this host's cv2 has HSV->BGR row block {block}; the goldens were made with {made}")
    assert block == targets.TargetConfig().tint_row_block


@pytest.mark.parametrize("w", list(range(1, 65)) + [427])
def test_rows_of_every_width_match_cv2(w):
    cv2 = _cv2()
    block = targets.cv2_row_block()
    rng = np.random.default_rng(w)
    hsv = rng.integers(0, 256, (3, w, 3), dtype=np.uint8)  # hue >= 180 included: cv2 and the port still agree
    assert np.array_equal(tt.hsv2bgr(hsv, block), cv2.cvtColor(hsv, cv2.COLOR_HSV2BGR))
    bgr = hsv[::-1].copy()
    draws = (int(rng.integers(0, 21)), int(rng.integers(0, 81)), int(rng.integers(0, 61)))
    want = cv2.cvtColor(tt.shift_hsv(cv2.cvtColor(bgr, cv2.COLOR_BGR2HSV), draws), cv2.COLOR_HSV2BGR)
    assert np.array_equal(tt.distort_color(bgr, draws, block), want)


@pytest.mark.parametrize("path", COLOR, ids=lambda p: os.path.basename(p)[:-4])
def test_port_equals_the_reference_distort_color(path):
    z = np.load(path)
    img = tt.color_source(z)
    assert (int(z["pad_cols"]) > 0) == (not img.flags["C_CONTIGUOUS"])
    np.random.seed(int(z["seed"]))
    assert tt.draw() == tuple(int(v) for v in z["draws"])
    assert np.array_equal(tt.distort_color(img, z["draws"], int(z["row_block"])), z["out"])


def test_draws_are_the_reference_order_and_ranges():
    np.random.seed(3)
    d = [targets.draw_tint() for _ in range(2000)]
    np.random.seed(3)
    assert d == [tt.draw() for _ in range(2000)]
    a = np.array(d)
    assert a.min(0).tolist() == [0, 0, 0] and a.max(0).tolist() == [20, 80, 60]


@pytest.mark.parametrize("path", GEN, ids=lambda p: os.path.basename(p)[:-4])
def test_seeded_generators_reproduce_the_gen_loop_draws(path):
    """make_batch's order -- every selection from ``random`` first, then per tinted sample three ``np.random`` draws
    in sample order -- gives the draws of the reference's sequential loop."""
    z = np.load(path)
    cfg = targets.TargetConfig(int(z["size"]), int(z["size"]))
    random.seed(int(z["seed"]))
    np.random.seed(int(z["seed"]))
    augs = [targets.AugmentSelection.random(cfg.transform_params) for _ in range(len(z["draws"]))]
    got = [list(targets.draw_tint()) if a.tint else [0, 0, 0] for a in augs]
    assert np.array_equal(np.array(got), z["draws"])
    assert [a.tint for a in augs] == [bool(v) for v in z["aug"][:, 1]]
    for a, r in zip(augs, z["aug"]):
        assert [a.flip, a.tint, a.degree, a.crop[0], a.crop[1], a.scale] == r.tolist()
