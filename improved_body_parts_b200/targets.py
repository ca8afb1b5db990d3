"""Training samples on the device: the reference data server's augmentation warp, masks and ground-truth maps.

The reference makes one sample on the CPU in ``RawDataIterator.gen`` (py_cocodata_server/py_data_iterator.py:35-72):
``Transformer.transform`` (py_data_transformer.py:112-184) warps the image and both masks with one affine matrix and
area-resizes the masks to the map size, and ``Heatmapper.create_heatmaps`` (py_data_heatmapper.py:50-97) rasterises the
joints into the ``[50, h, w]`` target whose channel layout is the network's output layout (body parts 0-29, keypoints
30-47, background 48-49).  Here the geometry -- the augmentation draw, the affine matrix and the joints it moves, a few
hundred numbers per sample -- stays on the host with the reference's own numpy expressions, and the per-pixel work runs in
two CUDA kernels (csrc/targets.cuh) through ``spg_targets_warp`` / ``spg_targets_maps``.

- ``AugmentSelection``, ``Transformer`` and ``Heatmapper`` keep the reference's signatures and returns, so that
  ``py_data_iterator.Transformer = targets.Transformer`` and ``py_data_iterator.Heatmapper = targets.Heatmapper`` drop
  them in.
- ``make_batch`` builds a whole batch of samples of any source sizes in one call and returns ``gen()``'s three outputs
  stacked, on the device, without a host synchronisation.

Colour distortion (``Transformer.distort_color``: an HSV round trip with three ``np.random`` draws) runs on the device
too, through ``spg_targets_tint``, when asked for: ``make_batch(..., tint=True)`` and ``Transformer(config, tint=True)``.
It equals cv2's result bit for bit given the row block of cv2's HSV->BGR vector loop (``TargetConfig.tint_row_block``,
``cv2_row_block()``; DESIGN.md §4).  Without ``tint=True`` a selection with ``tint`` set is refused, as before.
"""
from __future__ import annotations

import random
from math import ceil, cos, log, pi, sin, sqrt
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import grouping
from .skeleton import LIMBS, NUM_PARTS, PART_NAMES

_LEFT = ("Lsho", "Lelb", "Lwri", "Lhip", "Lkne", "Lank", "Leye", "Lear")
_RIGHT = ("Rsho", "Relb", "Rwri", "Rhip", "Rkne", "Rank", "Reye", "Rear")


class TransformParams:
    """The reference's ``TransformationParams(stride)`` (config/config.py): augmentation and target parameters."""

    def __init__(self, stride: int):
        self.target_dist = 0.6
        self.scale_prob = 0.8
        self.scale_min = 0.7
        self.scale_max = 1.3
        self.max_rotate_degree = 40.
        self.center_perterb_max = 50.
        self.flip_prob = 0.5
        self.tint_prob = 0.2
        self.sigma = 9
        self.keypoint_gaussian_thre = 0.015
        self.limb_gaussian_thre = 0.015
        self.paf_sigma = 7
        self.paf_thre = 1 * stride


class TargetConfig:
    """The parts of the reference's ``CanonicalConfig`` a training sample needs, with its defaults; the derived shapes
    follow ``width`` / ``height`` / ``stride``.  Any object with the same attributes (the reference's own config) works
    wherever a config is taken."""

    def __init__(self, width: int = 512, height: int = 512, stride: int = 4):
        self.width, self.height, self.stride = int(width), int(height), int(stride)
        #: cv2's HSV->BGR row block on the host whose results you want to match: the last ``width % tint_row_block``
        #: pixels of every row are rounded, the others truncated (32 where OpenCV dispatches to AVX-512;
        #: ``cv2_row_block()`` measures it)
        self.tint_row_block = 32
        self.num_parts = NUM_PARTS
        self.limbs_conn = list(LIMBS)
        self.leftParts = [PART_NAMES.index(p) for p in _LEFT]
        self.rightParts = [PART_NAMES.index(p) for p in _RIGHT]
        self.transform_params = TransformParams(self.stride)
        self.derive()

    def derive(self) -> None:
        self.paf_layers, self.heat_layers = len(self.limbs_conn), self.num_parts
        self.num_layers = self.paf_layers + self.heat_layers + 2
        self.paf_start, self.heat_start, self.bkg_start = 0, self.paf_layers, self.paf_layers + self.heat_layers
        self.mask_shape = (self.height // self.stride, self.width // self.stride)
        self.parts_shape = (self.height // self.stride, self.width // self.stride, self.num_layers)


def gaussian_size(config) -> int:
    """``Heatmapper.gaussian_size``: ``ceil(sqrt(-2 sigma^2 log(thre)) / stride) * 2`` (14 at the defaults)."""
    tp = config.transform_params
    double_sigma2 = 2 * tp.sigma * tp.sigma
    return ceil((sqrt(-double_sigma2 * log(tp.keypoint_gaussian_thre))) / config.stride) * 2


class AugmentSelection:
    """One augmentation: flip, tint, rotation in degrees, centre shift ``crop = (x, y)`` and scale."""

    def __init__(self, flip=False, tint=False, degree=0., crop=(0, 0), scale=1.):
        self.flip, self.tint, self.degree, self.crop, self.scale = flip, tint, degree, crop, scale

    @staticmethod
    def random(transform_params) -> "AugmentSelection":
        """The reference's draws from the ``random`` module in its order: flip, tint, degree, the scale's coin (then its
        value when it lands), x and y shift.  A seeded ``random`` gives the reference's selections."""
        tp = transform_params
        flip = random.uniform(0., 1.) < tp.flip_prob
        tint = random.uniform(0., 1.) < tp.tint_prob
        degree = random.uniform(-1., 1.) * tp.max_rotate_degree
        scale = 1.
        if random.uniform(0., 1.) < tp.scale_prob:
            scale = (tp.scale_max - tp.scale_min) * random.uniform(0., 1.) + tp.scale_min
        x_offset = int(random.uniform(-1., 1.) * tp.center_perterb_max)
        y_offset = int(random.uniform(-1., 1.) * tp.center_perterb_max)
        return AugmentSelection(flip, tint, degree, (x_offset, y_offset), scale)

    @staticmethod
    def unrandom() -> "AugmentSelection":
        return AugmentSelection(False, False, 0., (0, 0), 1.)

    def affine(self, center, scale_self, config) -> Tuple[np.ndarray, float]:
        """``(M, scale_size)``: the 2x3 float64 matrix taking source pixels to the output, composed as the reference
        does (centre to the origin, rotate, scale, flip, back to the output's centre plus the shift; the ``.dot`` chain
        left to right) so that it is the same to the last bit."""
        scale_self *= (config.height / (config.height - 1))
        A, B = cos(self.degree / 180. * pi), sin(self.degree / 180. * pi)
        scale_size = config.transform_params.target_dist / scale_self * self.scale
        center_x, center_y = center
        to_origin = np.array([[1., 0., -center_x], [0., 1., -center_y], [0., 0., 1.]])
        rotate = np.array([[A, B, 0], [-B, A, 0], [0, 0, 1.]])
        scale = np.array([[scale_size, 0, 0], [0, scale_size, 0], [0, 0, 1.]])
        flip = np.array([[-1 if self.flip else 1., 0., 0.], [0., 1., 0.], [0., 0., 1.]])
        to_centre = np.array([[1., 0., config.width / 2 - 0.5 + self.crop[0]],
                              [0., 1., config.height / 2 - 0.5 + self.crop[1]], [0., 0., 1.]])
        combined = to_centre.dot(flip).dot(scale).dot(rotate).dot(to_origin)
        return combined[0:2], scale_size


def transform_joints(joints: np.ndarray, M: np.ndarray, flip: bool, config) -> np.ndarray:
    """``meta['joints']`` after the warp (py_data_transformer.py:161-177): ``(x, y)`` through ``np.matmul(M, points)``,
    then left and right parts swapped when the image was flipped.  Returns a new array of ``joints``' dtype."""
    out = np.array(joints, copy=True)
    pts = out.copy()
    pts[:, :, 2] = 1
    out[:, :, 0:2] = np.matmul(M, pts.transpose([0, 2, 1])).transpose([0, 2, 1])
    if flip:
        left, right = out[:, config.leftParts, :], out[:, config.rightParts, :]
        out[:, config.leftParts, :] = right
        out[:, config.rightParts, :] = left
    return out


def target_params(config) -> np.ndarray:
    """The ``TARGET_PARAMS`` record of ``config``: the warp's output is ``dsize = (height, width)`` as the reference
    passes it, i.e. ``width`` rows of ``height`` columns."""
    if config.stride < 1 or config.height % config.stride or config.width % config.stride:
        raise ValueError(f"stride {config.stride} does not divide height {config.height} and width {config.width}")
    if config.height != config.width:
        raise ValueError("the reference's warp output (width x height) and label maps (height x width) only agree when "
                         f"height == width; got {config.height} x {config.width}")
    tp = config.transform_params
    p = np.zeros(1, grouping.TARGET_PARAMS)
    p["stride"], p["gaussian_size"] = config.stride, gaussian_size(config)
    p["out_h"], p["out_w"] = config.width, config.height
    p["sigma"], p["paf_sigma"], p["limb_gaussian_thre"], p["paf_thre"] = tp.sigma, tp.paf_sigma, tp.limb_gaussian_thre, \
        tp.paf_thre
    p["border_image"], p["border_mask_miss"], p["border_mask_all"] = (124, 127, 127), 255, 0
    return p


def _check_sample(i: int, img, mask_miss, mask_all, meta) -> None:
    img, mask_miss, mask_all = np.asarray(img), np.asarray(mask_miss), np.asarray(mask_all)
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3 or img.shape[0] < 1 or img.shape[1] < 1:
        raise ValueError(f"sample {i}: the source must be a uint8 HxWx3 array, got {img.dtype} {img.shape}")
    for name, m in (("mask_miss", mask_miss), ("mask_all", mask_all)):
        if m.dtype != np.uint8 or m.shape != img.shape[:2]:
            raise ValueError(f"sample {i}: {name} must be a uint8 array of the source's size {img.shape[:2]}, got "
                             f"{m.dtype} {m.shape}")
    if meta['scale_provided'][0] == 0:
        raise ValueError(f"sample {i}: scale_provided is zero (the affine matrix divides by it)")


def _check_joints(i: int, joints: np.ndarray) -> None:
    j = np.asarray(joints)
    if j.ndim != 3 or j.shape[2] != 3:
        raise ValueError(f"sample {i}: joints must be [persons, parts, 3], got {j.shape}")
    visible = j[:, :, 2] < 2
    if not np.isfinite(j[:, :, 0:2][visible]).all():
        raise ValueError(f"sample {i}: a visible joint (v < 2) has a non-finite coordinate")


def cv2_row_block(max_width: int = 4096) -> int:
    """The row block of the installed cv2's uint8 ``COLOR_HSV2BGR``, measured: for ``TargetConfig.tint_row_block``.

    cv2 truncates ``x * 255`` in its vector loop and rounds it in the scalar tail, the last ``width % block`` pixels of
    every row.  The probe is two rows of HSV ``(0, 1, 1)``, whose blue ``V (1 - S) * 255 ~ 0.996`` comes back 1 where
    rounded and 0 where truncated; the block is the narrowest width at which no pixel comes back rounded.  Needs cv2
    (the product path never imports it)."""
    import cv2
    for w in range(1, max_width + 1):
        out = cv2.cvtColor(np.full((2, w, 3), (0, 1, 1), np.uint8), cv2.COLOR_HSV2BGR)[:, :, 0]
        rounded = (out == 1).sum(axis=1)
        if rounded[0] != rounded[1]:
            raise RuntimeError(f"cv2's HSV->BGR rounded {rounded.tolist()} pixels in two equal rows of width {w}")
        if rounded[0] == 0:
            return w
    raise RuntimeError(f"cv2's HSV->BGR rounded every pixel of rows up to {max_width} wide: no vector loop to match")


def tint_records(images: Sequence[Tuple[int, int, int, int]], draws: Sequence[Tuple[int, int, int]],
                 row_block: int = 32) -> np.ndarray:
    """The ``TARGET_TINT`` records of ``images`` (per source ``(device pointer, row stride in bytes, height, width)``)
    with ``draws`` (per source ``(hue, saturation, value)`` as drawn: 0..20, 0..80, 0..60)."""
    recs = np.zeros(len(images), grouping.TARGET_TINT)
    for i, ((ptr, pitch, h, w), d) in enumerate(zip(images, draws)):
        recs[i] = (ptr, pitch, h, w, d[0], d[1], d[2], row_block)
    return recs


def draw_tint() -> Tuple[int, int, int]:
    """``distort_color``'s draws from ``np.random`` in its order: hue, saturation, value."""
    return int(np.random.randint(20 + 1)), int(np.random.randint(80 + 1)), int(np.random.randint(60 + 1))


def _row_block(config) -> int:
    """``config.tint_row_block`` (the reference's own config has none: 32)."""
    b = int(getattr(config, "tint_row_block", 32))
    if b < 1:
        raise ValueError(f"tint_row_block must be >= 1, got {b}")
    return b


class _Device:
    """One handle per (device, limb table): the training-sample calls use the handle's limb table only."""
    _handles = {}

    @classmethod
    def grouper(cls, config, device: int) -> grouping.Grouper:
        limbs = tuple(tuple(int(v) for v in l) for l in config.limbs_conn)
        key = (int(device), limbs, int(config.num_parts))
        if key not in cls._handles:
            cls._handles[key] = grouping.Grouper(limbs, config.num_parts, max_batch=1, max_h=16, max_w=16, device=device)
        return cls._handles[key]


def make_batch(samples: Sequence, augs: Sequence[Optional[AugmentSelection]], config=None, *, device: int = 0,
               stream=None, tint: bool = False):
    """``gen()``'s three outputs for a batch of samples, stacked, on ``cuda:device``.

    ``samples``: per sample ``(img, mask_miss, mask_all, meta)`` as ``gen`` reads them -- a uint8 HxWx3 source of any
    size, two uint8 HxW masks and the meta dict (``objpos``, ``scale_provided``, ``joints [P, 18, 3]``).  ``augs``: per
    sample an ``AugmentSelection`` (``None``: ``AugmentSelection.random``).  Returns ``(images [N, H, W, 3],
    mask_miss [N, 1, h, w], labels [N, 50, h, w])`` float32 CUDA tensors.  One host-to-device copy for all sources and
    one for all joints, one launch per chunk of each kernel, no host synchronisation; ``meta`` is not modified.
    Malformed input raises ``ValueError`` before anything is launched.

    ``tint=True`` applies ``distort_color`` to the samples whose selection has ``tint`` set: each draws its three offsets
    from ``np.random`` in sample order once the whole batch has passed validation, and one ``spg_targets_tint`` launch
    tints their sources in the device staging buffer before the warp, with ``config.tint_row_block``.  A seeded
    ``random`` and ``np.random`` thus give what a sequential ``gen()`` loop gives.  ``tint=False`` refuses such a
    selection."""
    import torch
    config = TargetConfig() if config is None else config
    samples, augs = list(samples), list(augs)
    if len(augs) != len(samples):
        raise ValueError("one augmentation per sample expected")
    params = target_params(config)
    row_block = _row_block(config) if tint else 0
    n = len(samples)
    out_h, out_w, s = int(params["out_h"][0]), int(params["out_w"][0]), config.stride
    mh, mw = out_h // s, out_w // s
    # host geometry and the two staging buffers: sources (image, mask_miss, mask_all back to back) and joints
    geo, src_off, jnt_off, tinted = [], [0], [0], []
    for i, ((img, mask_miss, mask_all, meta), aug) in enumerate(zip(samples, augs)):
        _check_sample(i, img, mask_miss, mask_all, meta)
        aug = AugmentSelection.random(config.transform_params) if aug is None else aug
        if aug.tint and not tint:
            raise ValueError(f"sample {i}: tint is not applied here; run the reference's Transformer.distort_color on "
                             "the uint8 image first and pass a selection with tint=False")
        if aug.tint:
            tinted.append(i)
        M, _ = aug.affine(meta['objpos'][0], meta['scale_provided'][0], config)
        joints = transform_joints(meta['joints'], M, aug.flip, config).astype(np.float32)
        _check_joints(i, joints)
        geo.append((M, joints))
        h, w = np.asarray(img).shape[:2]
        src_off.append(src_off[-1] + h * w * 5)
        jnt_off.append(jnt_off[-1] + joints.size)
    draws = [draw_tint() for _ in tinted]  # after validation: a refused batch consumes no draws
    dev = torch.device("cuda", device)
    g = _Device.grouper(config, device)
    src_host = torch.empty(src_off[-1], dtype=torch.uint8, pin_memory=True)
    jnt_host = torch.empty(max(jnt_off[-1], 1), dtype=torch.float32, pin_memory=True)
    sh, jh = src_host.numpy(), jnt_host.numpy()
    for i, (img, mask_miss, mask_all, _) in enumerate(samples):
        h, w = np.asarray(img).shape[:2]
        o = src_off[i]
        sh[o:o + h * w * 3] = np.asarray(img).reshape(-1)
        sh[o + h * w * 3:o + h * w * 4] = np.asarray(mask_miss).reshape(-1)
        sh[o + h * w * 4:o + h * w * 5] = np.asarray(mask_all).reshape(-1)
        jh[jnt_off[i]:jnt_off[i + 1]] = geo[i][1].reshape(-1)
    st = torch.cuda.current_stream(dev) if stream is None else stream
    with torch.cuda.stream(st):
        src = src_host.to(dev, non_blocking=True)
        jnt = jnt_host.to(dev, non_blocking=True)
        images = torch.empty((n, out_h, out_w, 3), dtype=torch.float32, device=dev)
        miss = torch.empty((n, 1, mh, mw), dtype=torch.float32, device=dev)
        all_ = torch.empty((n, mh, mw), dtype=torch.float32, device=dev)
        labels = torch.empty((n, config.num_layers, mh, mw), dtype=torch.float32, device=dev)
    ws = np.zeros(n, grouping.TARGET_SAMPLE)
    wj = np.zeros(n, grouping.TARGET_JOINTS)
    for i, (img, _, _, _) in enumerate(samples):
        h, w = np.asarray(img).shape[:2]
        base = src.data_ptr() + src_off[i]
        ws[i] = (base, base + h * w * 3, base + h * w * 4, w * 3, w, h, w, geo[i][0].reshape(6),
                 images[i].data_ptr(), miss[i].data_ptr(), all_[i].data_ptr())
        wj[i] = (jnt.data_ptr() + 4 * jnt_off[i], geo[i][1].shape[0], 0, all_[i].data_ptr(), labels[i].data_ptr())
    if tinted:  # in place in the staging buffer, ahead of the warp on the same stream
        shapes = [np.asarray(samples[i][0]).shape[:2] for i in tinted]
        g.targets_tint(tint_records([(src.data_ptr() + src_off[i], 3 * w, h, w) for i, (h, w) in zip(tinted, shapes)],
                                    draws, row_block), stream=st)
    g.targets_warp(params, ws, stream=st)
    g.targets_maps(params, wj, stream=st)  # src, jnt and all_ were allocated on st: their reuse is ordered after this
    return images, miss, labels


class Transformer:
    """The reference's ``Transformer``: ``transform`` warps one sample on the device and returns host arrays.  With
    ``tint=True`` it also applies ``distort_color`` when the selection asks for it, so that
    ``py_data_iterator.Transformer = targets.Transformer`` covers the whole of the reference's ``transform``."""

    def __init__(self, config, device: int = 0, tint: bool = False):
        self.config, self.device, self.tint = config, device, tint

    @staticmethod
    def distort_color(img, *, row_block: int = 32, device: Optional[int] = None) -> np.ndarray:
        """The reference's ``distort_color(img)``: uint8 ``[H, W, 3]`` BGR in, the tinted uint8 image out, on the host.
        Draws hue, saturation and value from ``np.random`` as the reference does; the HSV round trip runs on the
        device (``cuda:device``, the current device when ``None``) with cv2's HSV->BGR ``row_block``."""
        import torch
        a = np.asarray(img)
        if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3 or a.shape[0] < 1 or a.shape[1] < 1:
            raise ValueError(f"the source must be a uint8 HxWx3 array, got {a.dtype} {a.shape}")
        if row_block < 1:
            raise ValueError(f"row_block must be >= 1, got {row_block}")
        device = torch.cuda.current_device() if device is None else int(device)
        d = torch.from_numpy(np.ascontiguousarray(a)).to(torch.device("cuda", device))
        h, w = a.shape[:2]
        _Device.grouper(TargetConfig(), device).targets_tint(tint_records([(d.data_ptr(), 3 * w, h, w)], [draw_tint()],
                                                                          row_block))
        return d.cpu().numpy()

    def transform(self, img, mask_miss, mask_all, meta, aug=None):
        """``(img [H, W, 3], mask_miss [h, w], mask_all [h, w], meta)`` float32 in [0, 1], with ``meta['joints']``
        moved by the warp in place, as the reference returns them."""
        import torch
        aug = AugmentSelection.random(self.config.transform_params) if aug is None else aug
        _check_sample(0, img, mask_miss, mask_all, meta)
        if aug.tint and not self.tint:
            raise ValueError("tint is not applied here; run the reference's Transformer.distort_color on the uint8 "
                             "image first and pass a selection with tint=False")
        params = target_params(self.config)
        row_block = _row_block(self.config) if aug.tint else 0
        M, _ = aug.affine(meta['objpos'][0], meta['scale_provided'][0], self.config)
        dev = torch.device("cuda", self.device)
        out_h, out_w, s = int(params["out_h"][0]), int(params["out_w"][0]), self.config.stride
        src = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (img, mask_miss, mask_all)]
        out = [torch.empty(shape, dtype=torch.float32, device=dev) for shape in
               ((out_h, out_w, 3), (out_h // s, out_w // s), (out_h // s, out_w // s))]
        h, w = src[1].shape
        g = _Device.grouper(self.config, self.device)
        if aug.tint:  # the reference tints before it warps; np.random is drawn as its distort_color draws
            g.targets_tint(tint_records([(src[0].data_ptr(), 3 * w, h, w)], [draw_tint()], row_block))
        rec = np.zeros(1, grouping.TARGET_SAMPLE)
        rec[0] = (src[0].data_ptr(), src[1].data_ptr(), src[2].data_ptr(), w * 3, w, h, w, M.reshape(6),
                  out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr())
        g.targets_warp(params, rec)
        meta['joints'] = transform_joints(meta['joints'], M, aug.flip, self.config)
        return out[0].cpu().numpy(), out[1].cpu().numpy(), out[2].cpu().numpy(), meta


class Heatmapper:
    """The reference's ``Heatmapper``: ``create_heatmaps`` on the device, returning the host array."""

    def __init__(self, config, device: int = 0):
        self.config, self.device = config, device
        self.gaussian_size = gaussian_size(config)

    def create_heatmaps(self, joints, mask_all) -> np.ndarray:
        """``[num_layers, h, w]`` float32: body parts, keypoints, ``erode(mask_all)`` and the keypoints' max, clipped to
        [0, 1]."""
        import torch
        params = target_params(self.config)
        joints = np.ascontiguousarray(joints, np.float32)
        _check_joints(0, joints)
        dev = torch.device("cuda", self.device)
        mh, mw = int(params["out_h"][0]) // self.config.stride, int(params["out_w"][0]) // self.config.stride
        m = np.ascontiguousarray(mask_all, np.float32)
        if m.shape != (mh, mw):
            raise ValueError(f"mask_all must be {mh}x{mw}, got {m.shape}")
        jd, md = torch.from_numpy(joints).to(dev), torch.from_numpy(m).to(dev)
        labels = torch.empty((self.config.num_layers, mh, mw), dtype=torch.float32, device=dev)
        rec = np.zeros(1, grouping.TARGET_JOINTS)
        rec[0] = (jd.data_ptr(), joints.shape[0], 0, md.data_ptr(), labels.data_ptr())
        _Device.grouper(self.config, self.device).targets_maps(params, rec)
        return labels.cpu().numpy()
