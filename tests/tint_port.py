"""TEST INFRASTRUCTURE -- numpy restatement of the training augmentation's colour distortion, no cv2.

``distort_color`` is the reference's ``Transformer.distort_color`` (py_cocodata_server/py_data_transformer.py:97-110):
``cv2.cvtColor(img, COLOR_BGR2HSV)`` on uint8, three offsets clamped into range, ``cv2.cvtColor(.., COLOR_HSV2BGR)``.

- ``bgr2hsv`` is OpenCV's uint8 BGR->HSV: integer arithmetic on the 2^12 fixed-point tables ``sdiv`` / ``hdiv``.
- ``hsv2bgr`` is OpenCV's uint8 HSV->BGR: float32 arithmetic with two fused multiply-adds.  The result ``x * 255`` is
  truncated for the pixels OpenCV's SIMD loop handles and rounded to nearest even for the last ``width % row_block``
  pixels of every row, which its scalar tail handles (DESIGN.md §4).  ``row_block`` is 32 where OpenCV dispatches to
  AVX-512; ``improved_body_parts_b200.targets.cv2_row_block()`` measures it on a host with cv2.

The port is what the kernel (csrc/targets.cuh, targets_tint_kernel) must equal bit for bit.
"""
from __future__ import annotations

import numpy as np

_F, _D = np.float32, np.float64
#: cv2's HSV->RGB sector table: per sector, the entries of [V, V(1-S), V(1-S hh), V(1-S(1-hh))] giving B, G, R
SECTOR = np.array([[1, 3, 0], [1, 0, 2], [3, 0, 1], [0, 2, 1], [0, 1, 3], [2, 1, 0]])
#: the reference's draws: np.random.randint(n + 1) per channel, applied as draw - offset
DRAW_RANGE = (20, 80, 60)
DRAW_OFFSET = (10, 20, 20)


def sdiv() -> np.ndarray:
    """``round((255 << 12) / i)``, 0 at 0.  No quotient is a tie, so the integer form is exact."""
    i = np.arange(256, dtype=np.int64)
    return np.where(i == 0, 0, (2 * (255 << 12) + i) // np.maximum(2 * i, 1))


def hdiv() -> np.ndarray:
    """``round((180 << 12) / (6 i))``, 0 at 0."""
    i = np.arange(256, dtype=np.int64)
    return np.where(i == 0, 0, (2 * (180 << 12) + 6 * i) // np.maximum(12 * i, 1))


def bgr2hsv(img: np.ndarray) -> np.ndarray:
    """``cv2.cvtColor(img, COLOR_BGR2HSV)`` of uint8 ``[..., 3]``: hue in [0, 180)."""
    t = np.asarray(img)
    b, g, r = (t[..., i].astype(np.int64) for i in range(3))
    v = np.maximum(np.maximum(b, g), r)
    diff = v - np.minimum(np.minimum(b, g), r)
    vr, vg = -(v == r).astype(np.int64), -(v == g).astype(np.int64)
    s = (diff * sdiv()[v] + (1 << 11)) >> 12
    h = (vr & (g - b)) + (~vr & ((vg & (b - r + 2 * diff)) + (~vg & (r - g + 4 * diff))))
    h = (h * hdiv()[diff] + (1 << 11)) >> 12
    h = h + np.where(h < 0, 180, 0)
    return np.stack([h, s, v], -1).astype(np.uint8)


def fma_f32(a: np.ndarray, b: np.ndarray, c: float) -> np.ndarray:
    """``fmaf(a, b, c)`` of float32 arrays: ``a * b + c`` rounded once to float32.

    The product of two float32 values is exact in float64 (48 significant bits).  The float64 sum ``s = p + c`` is
    rounded, and its error ``e`` is exact by Knuth's TwoSum.  Rounding ``s`` to float32 then equals rounding the exact
    ``s + e`` unless ``s`` lies exactly halfway between two float32 values and ``e != 0``: there the exact value is on
    ``e``'s side of the midpoint, and that neighbour is taken."""
    p = np.asarray(a, _F).astype(_D) * np.asarray(b, _F).astype(_D)
    c = _D(c)
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.astype(_F)
    d = s - r.astype(_D)                                     # exact: s and r differ by at most half a float32 ulp
    other = np.nextafter(r, np.where(d > 0, np.inf, -np.inf).astype(_F))
    mid = (d != 0) & (r.astype(_D) + other.astype(_D) == 2 * s)
    return np.where(mid & (np.sign(e) == np.sign(d)) & (e != 0), other, r)


def hsv2bgr(hsv: np.ndarray, row_block: int = 32) -> np.ndarray:
    """``cv2.cvtColor(hsv, COLOR_HSV2BGR)`` of uint8 ``[H, W, 3]`` (or ``[W, 3]``, one row), ``row_block`` as above."""
    t = np.asarray(hsv)
    w = t.shape[-2]
    H = t[..., 0].astype(_F)
    S = t[..., 1].astype(_F) * _F(1 / 255.)
    V = t[..., 2].astype(_F) * _F(1 / 255.)
    hh = H * _F(6.0 / 180)
    hh = np.where(hh >= 6, hh - _F(6), hh)
    sector = np.floor(hh)
    hh = hh - sector
    one = _F(1)
    tab = np.stack([V, V * (one - S), V * fma_f32(-S, hh, 1.0), V * fma_f32(-S, one - hh, 1.0)], -1)
    out = np.take_along_axis(tab, SECTOR[sector.astype(np.int64)], -1)
    out = np.where((S == 0)[..., None], V[..., None], out)
    x = out * _F(255)
    tail = np.arange(w) >= w - w % int(row_block)            # per column of every row
    q = np.where(tail[:, None], np.rint(x), np.trunc(x))
    return q.clip(0, 255).astype(np.uint8)


def shift_hsv(hsv: np.ndarray, draws) -> np.ndarray:
    """``distort_color``'s offsets: ``draw - (10, 20, 20)`` added per channel, clamped to [0, 179], [0, 255], [0, 255]."""
    h = np.asarray(hsv).astype(np.int16)
    out = np.empty_like(h)
    for ch, (d, o, hi) in enumerate(zip(draws, DRAW_OFFSET, (179, 255, 255))):
        out[..., ch] = np.maximum(np.minimum(h[..., ch] - o + int(d), hi), 0)
    return out.astype(np.uint8)


def distort_color(img: np.ndarray, draws, row_block: int = 32) -> np.ndarray:
    """``Transformer.distort_color(img)`` with the given draws ``(hue, saturation, value)`` (0..20, 0..80, 0..60)."""
    return hsv2bgr(shift_hsv(bgr2hsv(img), draws), row_block)


def draw(rs=np.random) -> tuple:
    """The reference's three draws, in its order, from ``rs`` (``np.random`` or a ``RandomState``)."""
    return tuple(int(rs.randint(n + 1)) for n in DRAW_RANGE)


def all_triples() -> np.ndarray:
    """Every 8-bit triple once, ``[2^24, 3]`` uint8, first channel slowest."""
    v = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], -1).astype(np.uint8)


# ---- golden cases (tests/golden/tint/, made by tests/golden/make_tint_golden.py) -----------------------------------------
def golden_dir() -> str:
    import os
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tint")


def golden_paths(kind: str = "color"):
    """``kind="color"``: the distort_color cases; ``"gen"``: the gen()-style sample loops."""
    import glob
    import os
    return sorted(glob.glob(os.path.join(golden_dir(), f"{kind}_*.npz")))


def color_source(z) -> np.ndarray:
    """The uint8 source of a distort_color case, as the generator handed it to the reference (a strided view when
    ``pad_cols`` > 0)."""
    from make_targets_golden import source
    h, w = (int(v) for v in z["source_hw"])
    pad = int(z["pad_cols"])
    img, _, _ = source(h, w + pad)
    return img[:, pad // 2:pad // 2 + w]
