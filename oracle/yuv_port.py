"""numpy restatement of ``cv2.cvtColor(frame, COLOR_YUV2BGR_NV12 / _I420 / _YUYV)`` for uint8 frames.

OpenCV's integer BT.601 limited-range conversion (``ITUR_BT_601_*`` in modules/imgproc/src/color_yuv.simd.hpp): per
pixel, with ``y = max(0, Y - 16) * CY`` and the rounding ``1 << 19``,

    B = sat((y + round + CUB (U - 128)) >> 20)
    G = sat((y + round + CUG (U - 128) + CVG (V - 128)) >> 20)
    R = sat((y + round + CVR (V - 128)) >> 20)

in integers only.  A 2x2 block (4:2:0) or a 2x1 pair (4:2:2) shares one U and one V.  The planes are those
``spg_yuv_to_bgr`` takes (include/spgroup.h):

    nv12(y, uv)    y [H, W], uv [H/2, W] (U, V interleaved)
    i420(y, u, v)  y [H, W], u and v [H/2, W/2]
    yuyv(p)        p [H, 2W]: Y0 U Y1 V per pair of pixels

Each returns uint8 [H, W, 3] BGR.  ``cv2_layout`` gives the single array cv2 takes for the same planes.
"""
from __future__ import annotations

import numpy as np

CY, CUB, CUG, CVG, CVR = 1220542, 2116026, -409993, -852492, 1673527
SHIFT = 20
ROUND = 1 << (SHIFT - 1)

FORMATS = ("nv12", "i420", "yuyv")


def _sat(v: np.ndarray) -> np.ndarray:
    return np.clip(v >> SHIFT, 0, 255).astype(np.uint8)


def _bgr(Y: np.ndarray, U: np.ndarray, V: np.ndarray) -> np.ndarray:
    """The formula on luma Y and the chroma U, V already repeated to Y's shape."""
    y = np.maximum(Y.astype(np.int64) - 16, 0) * CY
    uu, vv = U.astype(np.int64) - 128, V.astype(np.int64) - 128
    return np.stack([_sat(y + ROUND + CUB * uu), _sat(y + ROUND + CUG * uu + CVG * vv), _sat(y + ROUND + CVR * vv)], -1)


def _up420(c: np.ndarray) -> np.ndarray:
    return np.repeat(np.repeat(c, 2, 0), 2, 1)


def nv12(y: np.ndarray, uv: np.ndarray) -> np.ndarray:
    return _bgr(y, _up420(uv[:, 0::2]), _up420(uv[:, 1::2]))


def i420(y: np.ndarray, u: np.ndarray, v: np.ndarray) -> np.ndarray:
    return _bgr(y, _up420(u), _up420(v))


def yuyv(p: np.ndarray) -> np.ndarray:
    return _bgr(p[:, 0::2], np.repeat(p[:, 1::4], 2, 1), np.repeat(p[:, 3::4], 2, 1))


def convert(fmt: str, planes) -> np.ndarray:
    """``nv12`` / ``i420`` / ``yuyv`` by name."""
    return {"nv12": nv12, "i420": i420, "yuyv": yuyv}[fmt](*planes)


def cv2_layout(fmt: str, planes) -> np.ndarray:
    """The single array ``cv2.cvtColor`` takes for these planes: ``[H*3/2, W]`` for NV12 and I420 (the planes back to
    back), ``[H, W, 2]`` for YUYV."""
    if fmt == "yuyv":
        (p,) = planes
        return np.ascontiguousarray(p).reshape(p.shape[0], p.shape[1] // 2, 2)
    H, W = planes[0].shape
    return np.concatenate([np.ascontiguousarray(p).reshape(-1) for p in planes]).reshape(H * 3 // 2, W)


def cv2_code(fmt: str) -> int:
    import cv2
    return {"nv12": cv2.COLOR_YUV2BGR_NV12, "i420": cv2.COLOR_YUV2BGR_I420, "yuyv": cv2.COLOR_YUV2BGR_YUYV}[fmt]


def plane_shapes(fmt: str, H: int, W: int):
    """The planes' shapes of an H x W frame."""
    return {"nv12": [(H, W), (H // 2, W)], "i420": [(H, W), (H // 2, W // 2), (H // 2, W // 2)],
            "yuyv": [(H, 2 * W)]}[fmt]


def random_planes(rng: np.random.Generator, fmt: str, H: int, W: int):
    return tuple(rng.integers(0, 256, s, dtype=np.uint8) for s in plane_shapes(fmt, H, W))


def every_triple(fmt: str):
    """Planes of a frame that holds every (Y, U, V) triple once: 4096 x 4096 pixels.  Each chroma sample (a 2x2 block,
    or a pair for YUYV) has its own (U, V); the 256 lumas of one (U, V) fill 64 blocks, or 128 pairs."""
    t = np.arange(1 << 24, dtype=np.int64)
    Y, U, V = (t & 255).astype(np.uint8), ((t >> 8) & 255).astype(np.uint8), (t >> 16).astype(np.uint8)
    if fmt == "yuyv":  # pair k: lumas 2k, 2k+1 and the (U, V) of triple 2k
        p = np.empty(1 << 25, np.uint8)
        p[0::4], p[1::4], p[2::4], p[3::4] = Y[0::2], U[0::2], Y[1::2], V[0::2]
        return (p.reshape(4096, 8192),)
    # block b (row-major over 2048 x 2048 blocks) holds triples 4b .. 4b+3 in its top-left, top-right, bottom-left,
    # bottom-right pixels
    y = Y.reshape(2048, 2048, 2, 2).transpose(0, 2, 1, 3).reshape(4096, 4096)
    u, v = U[0::4].reshape(2048, 2048), V[0::4].reshape(2048, 2048)
    if fmt == "nv12":
        uv = np.empty((2048, 4096), np.uint8)
        uv[:, 0::2], uv[:, 1::2] = u, v
        return y, uv
    return y, u, v
