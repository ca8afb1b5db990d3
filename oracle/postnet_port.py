"""TEST INFRASTRUCTURE -- CPU restatement of the reference's post-network stage (SURVEY.md §8 f-1), numpy only.

Groundwork for the next row of the scope table, not part of the product path: nothing under
``improved_body_parts_b200/`` imports this file.

What it restates: the body of the scale loop of ``predict()`` after the network has run,
``/root/reference/evaluate.py:126-161`` --

* split the two network outputs (image, mirrored image) into body-part and keypoint channels (:128-136),
* flip ensemble: mirror the second output back, permute its channels, average (:139-140),
* ``cv2.resize(..., fx=stride, fy=stride, INTER_CUBIC)`` (:143, :152),
* crop the padding (:148, :157), ``cv2.resize`` to the image size (:149, :158),
* accumulate ``map / n_scales`` in f64 (:160-161).

``cv2.resize`` in the reference's environment is Intel IPP's closed-source routine (opencv-python x86 wheels;
``cv2.ipp.setUseIPP(False)`` changes 47 % of the outputs by 1-2 ulp), so this stage is not bit-defined across hosts.
``resize_cubic`` follows OpenCV's own generic path (``modules/imgproc/src/resize.cpp``: ``resizeGeneric_`` with
``HResizeCubic`` / ``VResizeCubic``; coefficient formula ``interpolateCubic``, A = -0.75; source coordinate
``(dx + 0.5) * scale - 0.5``; taps clamped to the image) in float32 and is pinned to ``cv2`` within a float tolerance by
``tests/test_postnet_port.py`` -- the parity bar this stage can have (north_star: floats within 1e-4).
Rotation (``cv2.warpAffine``, :144-146, :153-155) is only used with ``rotation_search != [0]``; the reference's
config has ``rotation_search = 0`` (utils/config:27) and it is not restated.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np

_A = np.float32(-0.75)
_F = np.float32


def cubic_coeffs(fx: np.ndarray) -> np.ndarray:
    """``interpolateCubic`` (imgproc/src/resize.cpp): the four tap weights for fractional offsets ``fx`` (float32)."""
    x = fx.astype(np.float32)
    one = _F(1)
    c0 = ((_A * (x + one) - _F(5) * _A) * (x + one) + _F(8) * _A) * (x + one) - _F(4) * _A
    c1 = ((_A + _F(2)) * x - (_A + _F(3))) * x * x + one
    c2 = ((_A + _F(2)) * (one - x) - (_A + _F(3))) * (one - x) * (one - x) + one
    c3 = one - c0 - c1 - c2
    return np.stack([c0, c1, c2, c3], axis=-1).astype(np.float32)


def _axis_table(n_dst: int, n_src: int, scale: float) -> Tuple[np.ndarray, np.ndarray]:
    """Per destination index: the four clamped source indices and their weights (resize.cpp, the INTER_CUBIC branch)."""
    d = np.arange(n_dst, dtype=np.float64)
    f = ((d + 0.5) * scale - 0.5).astype(np.float32)  # `fx = (float)((dx+0.5)*scale_x - 0.5)`
    s = np.floor(f).astype(np.int64)
    frac = (f - s.astype(np.float32)).astype(np.float32)
    idx = np.clip(s[:, None] + np.arange(-1, 3)[None, :], 0, n_src - 1)
    return idx, cubic_coeffs(frac)


def resize_cubic(src: np.ndarray, dsize: Optional[Tuple[int, int]] = None, fx: float = 0.0, fy: float = 0.0) -> np.ndarray:
    """``cv2.resize(src, dsize, fx=fx, fy=fy, interpolation=cv2.INTER_CUBIC)`` for float32 ``src [h, w]`` or ``[h, w, C]``.

    ``dsize`` is ``(width, height)`` like OpenCV's; with ``dsize`` empty the size is ``round(w*fx), round(h*fy)``
    (``saturate_cast<int>``, round-half-even) and the scale is ``1/fx``; otherwise the scale is ``src/dst``.
    """
    a = np.asarray(src, np.float32)
    squeeze = a.ndim == 2
    if squeeze:
        a = a[:, :, None]
    h, w = a.shape[:2]
    if dsize is None or dsize == (0, 0):
        W, H = int(np.rint(w * fx)), int(np.rint(h * fy))
        sx, sy = 1.0 / fx, 1.0 / fy
    else:
        W, H = int(dsize[0]), int(dsize[1])
        sx, sy = 1.0 / (W / w), 1.0 / (H / h)  # inv_scale = dst/src; scale = 1/inv_scale (two roundings, as OpenCV)
    if (W, H) == (w, h):
        # resize.cpp: `if (dsize == ssize) { src.copyTo(dst); return; }` -- not the [0, 1, 0, 0] taps, which would turn
        # an infinite neighbour into NaN (inf * 0)
        out = a.copy()
        return out[:, :, 0] if squeeze else out
    ix, ax = _axis_table(W, w, sx)
    iy, ay = _axis_table(H, h, sy)
    # horizontal pass on every source row, float32, taps summed left to right
    hor = a[:, ix[:, 0], :] * ax[None, :, 0, None]
    for k in (1, 2, 3):
        hor = hor + a[:, ix[:, k], :] * ax[None, :, k, None]
    out = hor[iy[:, 0]] * ay[:, 0, None, None]
    for k in (1, 2, 3):
        out = out + hor[iy[:, k]] * ay[:, k, None, None]
    out = out.astype(np.float32)
    return out[:, :, 0] if squeeze else out


def flip_ensemble(out_pair: np.ndarray, n_paf: int, n_layers: int, flip_paf_ord: Sequence[int],
                  flip_heat_ord: Sequence[int]) -> Tuple[np.ndarray, np.ndarray]:
    """``evaluate.py:128-140``: ``out_pair [2, C, h, w]`` (image, mirrored image) -> averaged ``(paf, heat)`` in HWC."""
    blob = np.asarray(out_pair[0]).transpose(1, 2, 0)
    blob_flip = np.asarray(out_pair[1]).transpose(1, 2, 0)
    paf, heat = blob[:, :, :n_paf], blob[:, :, n_paf:n_layers]
    paf_f, heat_f = blob_flip[:, :, :n_paf], blob_flip[:, :, n_paf:n_layers]
    paf_avg = (paf + paf_f[:, ::-1, :][:, :, list(flip_paf_ord)]) / 2
    heat_avg = (heat + heat_f[:, ::-1, :][:, :, list(flip_heat_ord)]) / 2
    return paf_avg, heat_avg


def post_network_scale(out_pair: np.ndarray, stride: int, padded_shape: Tuple[int, int], pad: Sequence[int],
                       image_shape: Tuple[int, int], n_paf: int, n_layers: int, flip_paf_ord: Sequence[int],
                       flip_heat_ord: Sequence[int], resize=resize_cubic) -> Tuple[np.ndarray, np.ndarray]:
    """One iteration of the scale loop after the forward pass (``evaluate.py:126-158``, angle == 0).

    ``padded_shape`` is ``imageToTest_padded.shape[:2]``, ``pad`` the ``[up, left, down, right]`` list of
    ``util.padRightDownCorner``, ``image_shape`` the original ``image.shape[:2]``.  Returns ``(heatmap, paf)`` at image size.
    """
    paf_avg, heat_avg = flip_ensemble(out_pair, n_paf, n_layers, flip_paf_ord, flip_heat_ord)
    outs = []
    for m in (heat_avg, paf_avg):
        up = resize(np.ascontiguousarray(m, np.float32), None, fx=stride, fy=stride)
        up = up[pad[0]:padded_shape[0] - pad[2], pad[1]:padded_shape[1] - pad[3], :]
        outs.append(resize(np.ascontiguousarray(up), (image_shape[1], image_shape[0])))
    return outs[0], outs[1]


def accumulate(avg: np.ndarray, m: np.ndarray, n_items: int) -> np.ndarray:
    """``heatmap_avg = heatmap_avg + heatmap / n`` (:160-161): f64 accumulator, f32 map divided in f32 first."""
    return avg + m / n_items
