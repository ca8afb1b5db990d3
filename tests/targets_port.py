"""TEST INFRASTRUCTURE -- numpy restatement of the training-sample stage (improved_body_parts_b200/targets.py), no cv2.

``warp_sample`` is ``Transformer.transform``'s pixel work (py_data_transformer.py:132-149, 184) and ``label_maps`` is
``Heatmapper.create_heatmaps`` (py_data_heatmapper.py:50-97), vectorised.  The uint8 warp shares the coordinate code of
``oracle/postnet_rotation_port.warp_affine_linear`` (the inverted matrix, the 1/1024 -> 1/32 rounding) and adds OpenCV's
integer tap combine and the border value.  ``exp="numpy"`` evaluates the keypoint Gaussian with numpy's float32 ``exp``
and the limb length's float32 ``** 2`` as the reference does; ``exp="rounded"`` with float64 ``exp`` rounded to float32
and the correctly rounded square, as the kernel does (DESIGN.md §4).
"""
from __future__ import annotations

import numpy as np

from oracle.postnet_rotation_port import _rhe, invert_affine

_F = np.float32


def warp_affine_u8(src: np.ndarray, M: np.ndarray, dsize, border) -> np.ndarray:
    """``cv2.warpAffine(src, M, dsize, INTER_LINEAR, BORDER_CONSTANT, border)`` for uint8 ``src [h, w]`` or
    ``[h, w, C]``: weights ``32 (32 - ay)(32 - ax)`` ... summing to 2^15, taps outside the source read ``border``,
    ``(sum + 2^14) >> 15``."""
    a = np.asarray(src)
    squeeze = a.ndim == 2
    if squeeze:
        a = a[:, :, None]
    h, w, cn = a.shape
    W, H = dsize
    m = invert_affine(M)
    x, y = np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64)
    adelta, bdelta = _rhe(m[0] * x * 1024), _rhe(m[3] * x * 1024)
    X0, Y0 = _rhe((m[1] * y + m[2]) * 1024) + 16, _rhe((m[4] * y + m[5]) * 1024) + 16
    X = (X0[:, None] + adelta[None, :]) >> 5
    Y = (Y0[:, None] + bdelta[None, :]) >> 5
    sx, sy = np.clip(X >> 5, -32768, 32767), np.clip(Y >> 5, -32768, 32767)
    ax, ay = X & 31, Y & 31
    bv = np.broadcast_to(np.asarray(border, np.int64).reshape(-1)[:cn], (cn,))
    acc = np.zeros((H, W, cn), np.int64)
    for (i, j), wt in zip(((0, 0), (0, 1), (1, 0), (1, 1)),
                          ((32 - ay) * (32 - ax), (32 - ay) * ax, ay * (32 - ax), ay * ax)):
        yy, xx = sy + i, sx + j
        inside = (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
        v = a[np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)].astype(np.int64)
        acc += np.where(inside[:, :, None], v, bv[None, None, :]) * (32 * wt)[:, :, None]
    out = ((acc + (1 << 14)) >> 15).astype(np.uint8)
    return out[:, :, 0] if squeeze else out


def resize_area_int(a: np.ndarray, f: int) -> np.ndarray:
    """``cv2.resize(a, (w // f, h // f), INTER_AREA)`` of uint8 ``a [h, w]`` by the integer factor ``f`` dividing both
    sides, as OpenCV's fast-area code computes it from the box sum ``s``: ``(s + 2) >> 2`` at ``f = 2`` (ties up), else
    ``saturate_cast<uchar>(s * (1.f / f^2))`` -- the sum converted to float32, times the float32 reciprocal, rounded ties
    to even.  The product is not always the correctly rounded ``s / f^2`` (``f = 22, 34, 44, ...``); at ``f = 1`` cv2
    copies, which the product also gives."""
    h, w = a.shape
    s = a.reshape(h // f, f, w // f, f).astype(np.int64).sum(axis=(1, 3))
    if f == 2:
        return ((s + 2) >> 2).astype(np.uint8)
    inv = np.float32(1) / np.float32(f * f)
    return np.clip(np.rint(s.astype(np.float32) * inv), 0, 255).astype(np.uint8)


def erode3(m: np.ndarray) -> np.ndarray:
    """``cv2.erode(m, ones((3, 3)))``: the 3x3 min, neighbours outside the map ignored."""
    p = np.pad(m, 1, constant_values=np.inf)
    h, w = m.shape
    return np.min([p[i:i + h, j:j + w] for i in range(3) for j in range(3)], axis=0).astype(m.dtype)


def lut() -> np.ndarray:
    """``np.float32(u8) / 255.`` for every byte."""
    return np.arange(256, dtype=np.uint8).astype(np.float32) / 255.


BORDERS = ((124, 127, 127), 255, 0)  # the reference's borderValue for the image, mask_miss and mask_all


def warp_sample(img, mask_miss, mask_all, M, out_hw, stride, borders=BORDERS):
    """The float32 ``(img [H, W, 3], mask_miss [h, w], mask_all [h, w])`` of one sample; ``out_hw = (rows, cols)``,
    ``borders = (image (B, G, R), mask_miss, mask_all)``."""
    H, W = out_hw
    t = lut()
    im = warp_affine_u8(img, M, (W, H), borders[0])
    mm = resize_area_int(warp_affine_u8(mask_miss, M, (W, H), borders[1]), stride)
    ma = resize_area_int(warp_affine_u8(mask_all, M, (W, H), borders[2]), stride)
    return t[im], t[mm], t[ma]


def _kp_exp(arg: np.ndarray, exp: str) -> np.ndarray:
    if exp == "numpy":
        return np.exp(arg.astype(np.float32))
    if exp == "rounded":
        return np.exp(arg.astype(np.float64)).astype(np.float32)
    raise ValueError(exp)


def _window(lo: float, hi: float, n: int):
    """[lo, hi) clipped to the map: (a, b) or None when empty (Python slicing of the reference's window); None too when
    a bound is NaN."""
    a, b = max(lo, 0), min(hi, n)
    return (int(a), int(b)) if a < b else None


def label_maps(joints: np.ndarray, mask_all: np.ndarray, limbs, stride: int, sigma, paf_sigma, limb_thre, paf_thre,
               gsize: int, exp: str = "rounded") -> np.ndarray:
    """``Heatmapper.create_heatmaps(joints, mask_all)``: ``[L + K + 2, h, w]`` float32."""
    joints = np.asarray(joints, np.float32)
    h, w = mask_all.shape
    P, K = joints.shape[0], joints.shape[1] if joints.ndim == 3 else 18
    L = len(limbs)
    out = np.zeros((L + K + 2, h, w), np.float32)
    gx = (np.arange(w) * stride + stride / 2 - 0.5).astype(np.float32)
    gy = (np.arange(h) * stride + stride / 2 - 0.5).astype(np.float32)
    X = np.arange(w, dtype=np.float64) * stride + (stride / 2 - 0.5)
    Y = np.arange(h, dtype=np.float64) * stride + (stride / 2 - 0.5)
    ds2 = np.float32(2 * sigma * sigma)
    half = gsize // 2
    fs = np.float32(stride)
    for k in range(K):
        plane = out[L + k]
        for p in range(P):
            x, y, v = joints[p, k]
            if not v < 2:
                continue
            rx, ry = float(np.rint(x / fs)), float(np.rint(y / fs))
            wx, wy = _window(rx - half, rx + half + 1, w), _window(ry - half, ry + half + 1, h)
            if wx is None or wy is None:
                continue
            ex = _kp_exp(-(gx[wx[0]:wx[1]] - x) ** 2 / ds2, exp)
            ey = _kp_exp(-(gy[wy[0]:wy[1]] - y) ** 2 / ds2, exp)
            sl = (slice(*wy), slice(*wx))
            plane[sl] = np.maximum(plane[sl], np.outer(ey, ex))
    pt = np.float32(paf_thre)
    for l, (fr, to) in enumerate(limbs):
        acc = out[l]
        cnt = np.zeros((h, w), np.float32)
        for p in range(P):
            if not (joints[p, fr, 2] < 2 and joints[p, to, 2] < 2):
                continue
            x1, y1 = joints[p, fr, 0], joints[p, fr, 1]
            x2, y2 = joints[p, to, 0], joints[p, to, 1]
            dx, dy = x2 - x1, y2 - y1
            if dx * dx + dy * dy == 0:
                continue
            # the reference's (x1, x2) if x1 < x2 else (x2, x1), not min / max: with a NaN end both put the NaN in the box
            mnx, mxx = (x1, x2) if x1 < x2 else (x2, x1)
            mny, mxy = (y1, y2) if y1 < y2 else (y2, y1)
            lx, hx = float(np.rint((mnx - pt) / fs)), float(np.rint((mxx + pt) / fs))
            ly, hy = float(np.rint((mny - pt) / fs)), float(np.rint((mxy + pt) / fs))
            wx, wy = _window(lx, hx + 1, w), _window(ly, hy + 1, h)
            if wx is None or wy is None:
                continue
            detaX = np.float64(x1) - X[wx[0]:wx[1]][None, :]
            detaY = np.float64(y1) - Y[wy[0]:wy[1]][:, None]
            # numpy's float32 scalar ** 2 is not always the correctly rounded square dx * dx (DESIGN.md §4)
            sq = dx ** 2 + dy ** 2 if exp == "numpy" else dx * dx + dy * dy
            norm2 = np.sqrt(np.float64(sq))
            d = np.abs((np.float64(dx) * detaY - detaX * np.float64(dy)) / (norm2 + 1e-6))
            g = np.exp(-d ** 2 / (2 * paf_sigma ** 2))
            g[g <= limb_thre] = 0.01
            sl = (slice(*wy), slice(*wx))
            acc[sl] = (acc[sl].astype(np.float64) + g).astype(np.float32)
            cnt[sl] += 1
        nz = cnt > 0
        acc[nz] /= cnt[nz]
    out[L + K] = erode3(np.asarray(mask_all, np.float32))
    out[L + K + 1] = out[L:L + K].max(axis=0) if K else 0
    return np.clip(out, 0., 1.)


# ---- golden cases (tests/golden/targets/ and targets_space/, made by tests/golden/make_targets_golden.py) ---------------
def golden_paths(kind: str = "targets"):
    """The cases of ``tests/golden/<kind>/``: ``targets`` (the default configuration at 256 and 512) or
    ``targets_space`` (other strides, sizes, Gaussian parameters and limb tables)."""
    import glob
    import os
    d = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", kind)
    return sorted(p for p in glob.glob(os.path.join(d, "*.npz")) if not p.endswith("augment_draws.npz"))


def load_case(path: str) -> dict:
    """A golden case with its source rebuilt: ``img``, ``mask_miss_src``, ``mask_all_src`` and the recorded arrays."""
    from make_targets_golden import source
    z = dict(np.load(path))
    h, w = (int(v) for v in z["source_hw"])
    kinds = [k if k == "random" else int(k) for k in z["mask_kinds"].tolist()]
    z["img"], z["mask_miss_src"], z["mask_all_src"] = source(h, w, *kinds)
    z["image"] = z["image_codes"].astype(np.float32) / 255.
    z["size"] = int(z["size"])
    return z


def case_params(z: dict) -> dict:
    """The configuration a golden case was made with: the reference's defaults unless the case records its own."""
    from improved_body_parts_b200 import skeleton
    return dict(stride=int(z.get("stride", 4)), sigma=float(z.get("sigma", 9)), paf_sigma=float(z.get("paf_sigma", 7)),
                limb_thre=float(z.get("limb_gaussian_thre", 0.015)), paf_thre=float(z.get("paf_thre", 4)),
                gsize=int(z.get("gaussian_size", 14)), limbs=[tuple(int(v) for v in l) for l in z.get("limbs", skeleton.LIMBS)])


def target_config(z: dict):
    """A ``targets.TargetConfig`` with a golden case's size, stride, transform parameters and limb table."""
    from improved_body_parts_b200 import targets
    c = case_params(z)
    cfg = targets.TargetConfig(z["size"], z["size"], c["stride"])
    t = cfg.transform_params
    t.sigma, t.paf_sigma, t.limb_gaussian_thre, t.paf_thre = c["sigma"], c["paf_sigma"], c["limb_thre"], c["paf_thre"]
    t.keypoint_gaussian_thre = float(z.get("keypoint_gaussian_thre", 0.015))
    cfg.limbs_conn = c["limbs"]
    cfg.derive()
    return cfg


def port_case(z: dict, exp: str = "rounded"):
    """``(image, mask_miss, mask_all, labels)`` of a golden case by the port, from the case's M, joints and
    configuration."""
    c, n = case_params(z), z["size"]
    im, mm, ma = warp_sample(z["img"], z["mask_miss_src"], z["mask_all_src"], z["M"], (n, n), c["stride"])
    labels = label_maps(z["joints"].astype(np.float32), ma, c["limbs"], c["stride"], c["sigma"], c["paf_sigma"],
                        c["limb_thre"], c["paf_thre"], c["gsize"], exp=exp)
    return im, mm, ma, labels
