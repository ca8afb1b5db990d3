"""TEST INFRASTRUCTURE -- CPU restatement of the input side of ``predict()``, numpy only.

What it restates: the body of the ``(scale, angle)`` loop of ``predict()`` BEFORE the forward pass,
the reference's ``evaluate.py:94-121`` --

* the 2600 / 3800 clamp of the scale (:94-96),
* ``cv2.resize(image, (0, 0), fx=scale, fy=scale, INTER_CUBIC)`` of the uint8 BGR image (:98),
* ``util.padRightDownCorner`` with ``padValue`` (:99-100),
* ``np.float32(padded / 255)`` (:105),
* ``cv2.warpAffine(input_img, rotate_matrix, (0, 0))`` for ``angle != 0`` (:108-111),
* the mirrored copy and the concatenation into the ``[2, Hp, Wp, 3]`` pair the network receives (:116-119).

``cv2.resize`` of uint8 images runs Intel IPP's closed routine in the reference's opencv-python wheels; it differs from
OpenCV's own generic path by at most 1 LSB in some pixels.  ``resize_cubic_u8`` follows the GENERIC path
(``cv2.ipp.setUseIPP(False)``; ``modules/imgproc/src/resize.cpp``: ``resizeGeneric_`` with ``HResizeCubic<uchar, int,
short>`` and ``VResizeCubic<uchar, int, short, FixedPtCast<int, uchar, 22>, VResizeCubicVec_32s8u>``) BIT FOR BIT
(``tests/test_prenet_port.py``):

* coefficients as ``postnet_port.cubic_coeffs`` in float32 at source coordinate ``(d + 0.5) / fx - 0.5``, converted to
  ``short`` as ``rint(c * 2048)``; taps clamped to the image;
* horizontal pass: exact int32 sums of ``src * alpha``;
* vertical pass, vector body (``VResizeCubicVec_32s8u`` at the SSE baseline, no FMA): ``b_k = float(beta_k) * 2^-22``,
  ``v = S0*b0 + (S1*b1 + (S2*b2 + S3*b3))``, every product and sum rounded on its own, rounded ties-to-even and
  saturated to [0, 255];
* vertical pass, scalar tail: the last ``(dst_w * 3) % VEC_LANES`` values of each interleaved row take the integer
  path ``(sum S_k * beta_k + 2^21) >> 22``, saturated;
* ``dsize == ssize`` is a plain copy.

The warp is ``postnet_rotation_port.warp_affine_linear`` (bit-identical to cv2 on float32 images).  Nothing under
``improved_body_parts_b200/`` imports this file.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import numpy as np

from oracle import postnet_port as pp
from oracle import postnet_rotation_port as pr

#: values per vector iteration of ``VResizeCubicVec_32s8u`` (``v_int16::nlanes`` at the SSE baseline); the elements of
#: an interleaved row past the last whole group take the scalar integer path
VEC_LANES = 8

#: ``np.float32(u8 / 255)``: the float32 rounding of the float64 quotient, per byte value
U8_TO_F32 = np.float32(np.arange(256, dtype=np.float64) / 255)


def resized_size(h: int, w: int, fx: float) -> Tuple[int, int]:
    """``(rows, cols)`` of ``cv2.resize(src, (0, 0), fx=fx, fy=fx)``: ``saturate_cast<int>`` rounds ties to even."""
    return int(np.rint(h * fx)), int(np.rint(w * fx))


def _table(n_dst: int, n_src: int, scale: float) -> Tuple[np.ndarray, np.ndarray]:
    """Clamped source indices ``[n_dst, 4]`` and the fixed-point weights ``[n_dst, 4]`` (int64) of one axis."""
    idx, c = pp._axis_table(n_dst, n_src, scale)
    return idx, np.rint(c.astype(np.float32) * np.float32(2048)).astype(np.int64)


def resize_cubic_u8(src: np.ndarray, fx: float) -> np.ndarray:
    """``cv2.resize(src, (0, 0), fx=fx, fy=fx, interpolation=cv2.INTER_CUBIC)`` of uint8 ``src [h, w]`` or ``[h, w, C]``
    on OpenCV's generic path (IPP off).  The scale of either axis is ``1 / fx``."""
    a = np.asarray(src, np.uint8)
    squeeze = a.ndim == 2
    if squeeze:
        a = a[:, :, None]
    h, w, cn = a.shape
    H, W = resized_size(h, w, fx)
    if H <= 0 or W <= 0:
        raise ValueError(f"resized size {H}x{W} is empty")
    if (H, W) == (h, w):
        out = a.copy()
        return out[:, :, 0] if squeeze else out
    ix, ax = _table(W, w, 1.0 / fx)
    iy, ay = _table(H, h, 1.0 / fx)
    s = a.astype(np.int64)
    # horizontal pass on every source row: exact integer sums, [h, W, cn]
    hor = sum(s[:, ix[:, k], :] * ax[None, :, k, None] for k in range(4))
    rows = hor.reshape(h, W * cn)
    S = [rows[iy[:, k]] for k in range(4)]  # [H, W * cn] each
    # vector body: float32, products and sums rounded one at a time, nested from the right
    f32 = np.float32
    b = [ay[:, k].astype(np.float32)[:, None] * f32(2.0 ** -22) for k in range(4)]
    Sf = [v.astype(np.float32) for v in S]
    v = Sf[3] * b[3]
    v = (Sf[2] * b[2]).astype(f32) + v
    v = (Sf[1] * b[1]).astype(f32) + v
    v = (Sf[0] * b[0]).astype(f32) + v
    body = np.clip(np.rint(v.astype(f32)), 0, 255)
    # scalar tail: integer path
    acc = sum(S[k] * ay[:, k, None] for k in range(4))
    tail = np.clip((acc + (1 << 21)) >> 22, 0, 255)
    n_body = (W * cn) // VEC_LANES * VEC_LANES
    out = np.where(np.arange(W * cn)[None, :] < n_body, body, tail).astype(np.uint8).reshape(H, W, cn)
    return out[:, :, 0] if squeeze else out


def clamp_scale(scale: float, image_shape: Tuple[int, int]) -> float:
    """``evaluate.py:94-96``: shrink an item whose resized image would exceed 2600 rows or 3800 columns."""
    if scale * image_shape[0] > 2600 or scale * image_shape[1] > 3800:
        scale = min(2600 / image_shape[0], 3800 / image_shape[1])
    return scale


def pad_right_down(img: np.ndarray, stride: int, pad_value: int) -> Tuple[np.ndarray, List[int]]:
    """``util.padRightDownCorner``: pad below and to the right up to a multiple of ``stride`` with ``pad_value``."""
    h, w = img.shape[:2]
    pad = [0, 0, 0 if h % stride == 0 else stride - h % stride, 0 if w % stride == 0 else stride - w % stride]
    return np.pad(img, ((0, pad[2]), (0, pad[3]), (0, 0)), constant_values=pad_value), pad


def prenet_item(image: np.ndarray, scale: float, angle: float, max_downsample: int,
                pad_value: int) -> Tuple[np.ndarray, Tuple[int, int], List[int], Optional[np.ndarray]]:
    """One ``(scale, angle)`` item of ``evaluate.py:94-121``: returns ``(pair, imageToTest.shape[:2], pad,
    rotate_matrix_reverse)``; ``pair`` is the ``[2, Hp, Wp, 3]`` float32 tensor handed to the network (image, mirror),
    ``rotate_matrix_reverse`` is ``None`` for ``angle == 0``."""
    scale = clamp_scale(scale, image.shape[:2])
    image_to_test = resize_cubic_u8(image, scale)
    padded, pad = pad_right_down(image_to_test, max_downsample, pad_value)
    input_img = U8_TO_F32[padded]
    reverse = None
    if angle != 0:
        forward, reverse = pr.rotation_matrices(input_img.shape[:2], angle)
        input_img = pr.warp_affine_linear(input_img, forward)
    pair = np.stack([input_img, input_img[:, ::-1, :]]).astype(np.float32)
    return pair, image_to_test.shape[:2], pad, reverse
