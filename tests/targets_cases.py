"""The training-sample stage's case table: seeded (stride, output shape, Gaussian parameters, borders, row pitches, limb
table, joints) cases that together cover what ``spg_targets_warp`` / ``spg_targets_maps`` admit through the C ABI,
beyond the one configuration ``targets.make_batch`` uses.  ``tests/test_gpu_targets_space.py`` runs them against the
port (tests/targets_port.py); ``tests/test_targets_host.py`` checks the coverage.  ``area_probe`` builds masks whose
``f x f`` boxes hold the sums where cv2's ``INTER_AREA`` rounding is delicate."""
from __future__ import annotations

from typing import List, NamedTuple, Tuple

import numpy as np

from improved_body_parts_b200 import skeleton

FLT_MAX = float(np.finfo(np.float32).max)
DEFAULT_BORDERS = ((124, 127, 127), 255, 0)


def _limbs64(K: int, seed: int) -> Tuple[Tuple[int, int], ...]:
    """64 seeded limbs over K parts with a self-limb and a repeated limb: ``spg_create`` admits both."""
    rng = np.random.default_rng(seed)
    l = [tuple(int(v) for v in rng.integers(0, K, 2)) for _ in range(62)]
    return tuple(l + [(3, 3), l[0]])


class TargetCase(NamedTuple):
    name: str
    stride: int
    out_hw: Tuple[int, int]           # warped image rows, columns (the map is out_hw / stride)
    gaussian_size: int
    sigma: float
    paf_sigma: float
    limb_thre: float
    paf_thre: float
    borders: tuple                    # ((B, G, R), mask_miss, mask_all)
    limbs: Tuple[Tuple[int, int], ...]
    K: int
    sources: List[Tuple[int, int]]    # one (h, w) per sample
    persons: List[int]                # one count per sample
    pad: Tuple[int, int]              # bytes past each image row, each mask row
    edges: bool                       # joints on x / stride ties, at +-FLT_MAX, +-inf and NaN, v exactly 2 and NaN
    seed: int

    @property
    def map_hw(self) -> Tuple[int, int]:
        return self.out_hw[0] // self.stride, self.out_hw[1] // self.stride


_D = dict(sigma=9.0, paf_sigma=7.0, limb_thre=0.015)
CASES = [
    # stride 1: the map is the image; gaussian_size 0 (a one-pixel window); padded rows
    TargetCase("s1_48x48_g0", 1, (48, 48), 0, 2.0, 1.5, 0.015, 0.5, DEFAULT_BORDERS, skeleton.LIMBS, 18,
               [(60, 45), (1, 1)], [3, 1], (5, 3), True, 1),
    # stride 2, non-square, odd gaussian_size, non-default borders
    TargetCase("s2_64x96_g7_borders", 2, (64, 96), 7, 3.5, 2.25, 0.05, 1.75, ((0, 255, 17), 3, 250), skeleton.LIMBS, 18,
               [(120, 80), (33, 200)], [5, 0], (0, 0), True, 2),
    # stride 3 at 255 x 255 with the 24-limb table
    TargetCase("s3_255_limbs24", 3, (255, 255), 12, **_D, paf_thre=3.0, borders=DEFAULT_BORDERS,
               limbs=skeleton.LIMBS_24, K=18, sources=[(300, 420)], persons=[12], pad=(13, 1), edges=True, seed=3),
    # stride 4: a 1 x 1 map, gaussian_size larger than the map, one limb
    TargetCase("s4_1x1_one_limb", 4, (4, 4), 40, **_D, paf_thre=4.0, borders=DEFAULT_BORDERS, limbs=((1, 0),), K=18,
               sources=[(9, 7), (1, 1), (50, 3)], persons=[4, 2, 0], pad=(0, 0), edges=True, seed=4),
    # stride 5, non-square, 64 limbs over 32 parts
    TargetCase("s5_60x100_k32_l64", 5, (60, 100), 9, 4.0, 3.0, 0.02, 2.2, ((255, 0, 128), 0, 255), _limbs64(32, 5), 32,
               [(90, 110), (17, 23)], [6, 3], (7, 9), True, 5),
    # stride 6: 64 limbs over 18 parts, more than 256 persons x parts in a tile, a zero-person sample
    TargetCase("s6_96_l64_p300", 6, (96, 96), 6, 5.0, 4.0, 0.015, 6.0, DEFAULT_BORDERS, _limbs64(18, 6), 18,
               [(200, 150), (40, 40)], [300, 0], (1, 2), True, 6),
    # stride 8: the 46 x 46 map, the default parameters
    TargetCase("s8_368_default", 8, (368, 368), 8, **_D, paf_thre=8.0, borders=DEFAULT_BORDERS, limbs=skeleton.LIMBS,
               K=18, sources=[(480, 640), (640, 427)], persons=[10, 30], pad=(3, 0), edges=True, seed=8),
    # stride 8, non-square 1 x 2 map, 32 parts and one limb
    TargetCase("s8_8x16_k32", 8, (8, 16), 3, 1.5, 1.0, 0.1, 0.3, ((1, 2, 3), 128, 127), ((31, 0),), 32,
               [(16, 16)], [7], (0, 5), True, 9),
    # stride 22: the smallest stride whose mask area divides differently from cv2's product
    TargetCase("s22_132x88", 22, (132, 88), 2, 20.0, 15.0, 0.015, 22.0, DEFAULT_BORDERS, skeleton.LIMBS, 18,
               [(150, 100)], [5], (0, 0), True, 10),
]


def _matrix(rng, out_hw, src_hw) -> np.ndarray:
    """A seeded rotation, scale and (half the time) mirror taking the source's centre near the output's."""
    a, s = rng.uniform(-np.pi, np.pi), rng.uniform(0.5, 2.0) * max(out_hw) / max(src_hw)
    f = -1.0 if rng.random() < 0.5 else 1.0
    A, B = np.cos(a) * s, np.sin(a) * s
    cx, cy = src_hw[1] / 2, src_hw[0] / 2
    tx, ty = out_hw[1] / 2 + rng.uniform(-5, 5), out_hw[0] / 2 + rng.uniform(-5, 5)
    return np.array([[f * A, f * B, tx - f * (A * cx + B * cy)], [-B, A, ty - (-B * cx + A * cy)]])


def joints_of(case: TargetCase, P: int, rng) -> np.ndarray:
    """``[P, K, 3]`` float32 joints in output pixels around and beyond the map; with ``case.edges`` the first persons'
    joints sit on rounding ties (person 0) and at the non-finite and extreme values the ABI admits (person 1, or 0 when
    it is alone)."""
    H, W = case.out_hw
    j = np.zeros((P, case.K, 3), np.float32)
    j[:, :, 0] = rng.uniform(-0.2 * W, 1.2 * W, (P, case.K))
    j[:, :, 1] = rng.uniform(-0.2 * H, 1.2 * H, (P, case.K))
    j[:, :, 2] = rng.choice([0, 1, 2, 3], (P, case.K), p=[0.35, 0.45, 0.15, 0.05])
    if case.edges and P:
        s = case.stride
        k = np.arange(case.K)
        j[0, :, 0] = (k % max(W // s, 1) + 0.5) * s        # x / stride exactly k + 0.5: ties to even
        j[0, :, 1] = ((k // 2) % max(H // s, 1) + 0.5) * s
        j[0, :, 2] = 1
        specials = [(FLT_MAX, 3.0), (-FLT_MAX, 3.0), (3.0, FLT_MAX), (np.inf, 2.0), (-np.inf, 1.0), (1.0, -np.inf),
                    (np.nan, 2.0), (2.0, np.nan), (np.nan, np.nan)]
        p = min(1, P - 1)
        for i, (x, y) in enumerate(specials):
            j[p, i % case.K] = (x, y, i % 2)            # visible: the ABI's rule for non-finite joints applies
        j[p, (len(specials)) % case.K] = (1.0, 1.0, 2.0)   # v exactly 2: invisible
        j[p, (len(specials) + 1) % case.K] = (2.0, 2.0, np.nan)  # v NaN: invisible
        if P >= 3:  # the last person: a visible limb from a NaN joint to one in the middle of the map
            a, b = nan_limb(case)
            j[P - 1, a] = (np.nan, H / 2, 1.0)
            j[P - 1, b] = (W / 2, H / 2, 0.0)
    return j


def nan_limb(case: TargetCase) -> Tuple[int, int]:
    """The first limb of the case's table whose ends differ."""
    return next((a, b) for a, b in case.limbs if a != b)


def inputs(case: TargetCase):
    """Per sample ``(img [h, w, 3], mask_miss [h, w], mask_all [h, w], M, joints)``: uint8 sources (masks of 0, 255 and
    mid values), the warp matrix and float32 joints."""
    rng = np.random.default_rng(case.seed)
    out = []
    for (h, w), P in zip(case.sources, case.persons):
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        masks = []
        for _ in range(2):
            m = np.where(rng.random((h, w)) < 0.4, 0, 255).astype(np.uint8)
            m[rng.random((h, w)) < 0.1] = rng.integers(1, 255)
            masks.append(m)
        out.append((img, masks[0], masks[1], _matrix(rng, case.out_hw, (h, w)), joints_of(case, P, rng)))
    return out


# ---- INTER_AREA probes ----------------------------------------------------------------------------------------------
def area_sums(f: int, budget: int = 1 << 20, seed: int = 0) -> np.ndarray:
    """Box sums for an ``f x f`` area resize, at most ``budget // f^2`` of them (and at least 16): every sum whose cv2
    value ``rint(float32(s) * float32(1 / f^2))`` differs from the correctly rounded ``rint(s / f^2)``, the exact ties
    ``(q + 1/2) f^2`` and their neighbours, and seeded others -- in that priority."""
    area = f * f
    inv = np.float32(1) / np.float32(area)
    near = []
    for q in range(255):
        c = (2 * q + 1) * area // 2
        d = area // 32768 + 2
        near.append(np.arange(max(c - d, 0), min(c + d, 255 * area) + 1))
    s = np.unique(np.concatenate(near))
    mul = np.rint(s.astype(np.float32) * inv)
    div = np.rint(s.astype(np.float32) / np.float32(area))
    critical = s[mul != div]
    ties = s[2 * s % area == 0] if area % 2 == 0 else s[:0]
    cap = max(16, budget // area)
    rng = np.random.default_rng(seed + f)
    others = rng.integers(0, 255 * area + 1, 64)
    pick = [critical[np.linspace(0, len(critical) - 1, min(len(critical), cap // 2)).astype(int)] if len(critical) else critical]
    pick.append(ties[np.linspace(0, len(ties) - 1, min(len(ties), cap // 4)).astype(int)] if len(ties) else ties)
    pick += [np.array([0, 255 * area]), others]
    out = np.concatenate(pick)
    return out[:cap]


def box_with_sum(s: int, f: int, rng) -> np.ndarray:
    """A uint8 ``f x f`` box whose bytes sum to ``s`` (``0 <= s <= 255 f^2``), in a seeded order."""
    area = f * f
    v = np.full(area, s // area, np.int64)
    v[:s % area] += 1
    return rng.permutation(v).astype(np.uint8).reshape(f, f)


def area_probe(f: int, budget: int = 1 << 20, seed: int = 0, cols: int = 8):
    """``(mask, sums)``: a uint8 mask of ``rows x cols`` boxes of ``f x f`` whose box sums are ``area_sums(f)`` (the
    last row padded with zero boxes)."""
    sums = area_sums(f, budget, seed)
    rows = -(-len(sums) // cols)
    rng = np.random.default_rng(seed + 7 * f)
    m = np.zeros((rows * f, cols * f), np.uint8)
    for i, s in enumerate(sums):
        r, c = divmod(i, cols)
        m[r * f:(r + 1) * f, c * f:(c + 1) * f] = box_with_sum(int(s), f, rng)
    return m, sums
