"""TEST INFRASTRUCTURE -- CPU restatement of the rotation search of ``predict()`` (``rotation_search != [0]``), numpy only.

Extends ``oracle/postnet_port.py`` (the scale loop after the forward pass) by the one step an item with ``angle != 0``
adds, ``/root/reference/evaluate.py:143-158``: the x stride maps go through
``cv2.warpAffine(map, rotate_matrix_reverse, (0, 0))`` before the crop and the resize to the image.

Unlike ``cv2.resize`` (Intel IPP in the reference's wheels, pinned only within a float tolerance), ``cv2.warpAffine`` on
float32 maps runs OpenCV's generic fixed-point warp, and ``warp_affine_linear`` restates it BIT-IDENTICALLY
(``tests/test_postnet_rotation_port.py``): INTER_LINEAR, BORDER_CONSTANT 0, any channel count.  Nothing under
``improved_body_parts_b200/`` imports this file.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np

from oracle import postnet_port as pp

_F = np.float32


def invert_affine(M: np.ndarray) -> np.ndarray:
    """``invertAffineTransform`` in the operation order of ``warpAffine`` (imgproc/src/imgwarp.cpp): float64 ``[6]``."""
    m = [float(v) for v in np.asarray(M, np.float64).reshape(6)]
    D = m[0] * m[4] - m[1] * m[3]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22 = m[4] * D, m[0] * D
    m[0], m[1], m[3], m[4] = A11, m[1] * -D, m[3] * -D, A22
    b1 = -m[0] * m[2] - m[1] * m[5]
    b2 = -m[3] * m[2] - m[4] * m[5]
    m[2], m[5] = b1, b2
    return np.array(m, np.float64)


def _rhe(v: np.ndarray) -> np.ndarray:
    """``cvRound``: nearest integer, ties to even."""
    return np.rint(v).astype(np.int64)


def warp_affine_linear(src: np.ndarray, M: np.ndarray) -> np.ndarray:
    """``cv2.warpAffine(src, M, (0, 0))`` for float32 ``src [h, w]`` or ``[h, w, C]``: INTER_LINEAR, BORDER_CONSTANT 0.

    Destination pixel ``(x, y)`` reads the source at the inverted matrix's image of it in OpenCV's fixed point: 1/1024 px
    coordinates rounded ties-to-even per column and per row, then 1/32 px bilinear weights.  Taps outside the source
    read 0.  Every float32 product and sum is rounded on its own, the taps summed left to right (no FMA)."""
    a = np.asarray(src, np.float32)
    squeeze = a.ndim == 2
    if squeeze:
        a = a[:, :, None]
    h, w = a.shape[:2]
    m = invert_affine(M)
    x = np.arange(w, dtype=np.float64)
    y = np.arange(h, dtype=np.float64)
    adelta, bdelta = _rhe(m[0] * x * 1024), _rhe(m[3] * x * 1024)
    X0, Y0 = _rhe((m[1] * y + m[2]) * 1024) + 16, _rhe((m[4] * y + m[5]) * 1024) + 16
    X = (X0[:, None] + adelta[None, :]) >> 5
    Y = (Y0[:, None] + bdelta[None, :]) >> 5
    sx, sy = np.clip(X >> 5, -32768, 32767), np.clip(Y >> 5, -32768, 32767)  # saturate_cast<short>
    fx, fy = (X & 31).astype(np.float32) / _F(32), (Y & 31).astype(np.float32) / _F(32)
    one = _F(1)
    wts = ((one - fy) * (one - fx), (one - fy) * fx, fy * (one - fx), fy * fx)

    def tap(i, j):
        yy, xx = sy + i, sx + j
        inside = (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
        v = a[np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)]
        return np.where(inside[:, :, None], v, _F(0))

    with np.errstate(invalid="ignore"):  # 0 * inf = NaN, as in OpenCV
        out = tap(0, 0) * wts[0][:, :, None] + tap(0, 1) * wts[1][:, :, None]
        out = out + tap(1, 0) * wts[2][:, :, None]
        out = (out + tap(1, 1) * wts[3][:, :, None]).astype(np.float32)
    return out[:, :, 0] if squeeze else out


def rotation_matrices(padded_shape: Tuple[int, int], angle: float) -> Tuple[np.ndarray, np.ndarray]:
    """``evaluate.py:114-115``: ``(rotate_matrix, rotate_matrix_reverse)`` of a padded input of ``padded_shape``.  The
    centre is passed as ``(rows / 2, cols / 2)``, x and y swapped: on a non-square input the rotation is not about the
    image centre, and this keeps that quirk."""
    import cv2
    c = (padded_shape[0] / 2, padded_shape[1] / 2)
    return cv2.getRotationMatrix2D(c, angle, 1), cv2.getRotationMatrix2D(c, -angle, 1)


def post_network_item(out_pair: np.ndarray, stride: int, padded_shape: Tuple[int, int], pad: Sequence[int],
                      image_shape: Tuple[int, int], n_paf: int, n_layers: int, flip_paf_ord: Sequence[int],
                      flip_heat_ord: Sequence[int], resize=pp.resize_cubic,
                      rotate_matrix: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray]:
    """One ``(scale, angle)`` item after the forward pass (``evaluate.py:126-158``): ``postnet_port.post_network_scale``
    with the warp between the x stride resize and the crop.  ``rotate_matrix`` is ``rotate_matrix_reverse``; ``None``
    for ``angle == 0``, where the reference does not call ``warpAffine`` (an identity warp is not the identity on
    non-finite maps: 0 * inf = NaN).  Returns ``(heatmap, paf)`` at image size."""
    paf_avg, heat_avg = pp.flip_ensemble(out_pair, n_paf, n_layers, flip_paf_ord, flip_heat_ord)
    outs = []
    for m in (heat_avg, paf_avg):
        up = resize(np.ascontiguousarray(m, np.float32), None, fx=stride, fy=stride)
        if rotate_matrix is not None:
            up = warp_affine_linear(up, rotate_matrix)
        up = up[pad[0]:padded_shape[0] - pad[2], pad[1]:padded_shape[1] - pad[3], :]
        outs.append(resize(np.ascontiguousarray(up), (image_shape[1], image_shape[0])))
    return outs[0], outs[1]
