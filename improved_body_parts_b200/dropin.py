"""Drop-in replacements for the reference's grouping call sites (evaluate.py:509-511).

The reference has no plugin interface: ``process()`` resolves three module-level functions by name,

    all_peaks                  = find_peaks(heatmap, params)                                  # evaluate.py:169
    connection_all, special_k  = find_connections(all_peaks, paf, oriImg.shape[0], params)    # evaluate.py:206
    subset, candidate          = find_people(connection_all, special_k, all_peaks, params)    # evaluate.py:279

so the boundary is "same names, same arguments, same Python return structures".  The functions below honour it
and run every stage on the GPU through ``libspgroup.so``; ``install(evaluate)`` rebinds the three names in an
already imported ``evaluate`` module (INTEGRATION.md shows the launcher).  Argument meaning and quirks follow
the reference: ``image_width`` is really the image height (evaluate.py:510), border peaks come back as integer
coordinates, ``special_k`` limbs get ``[]``, ``candidate`` is the flattened peak table.

Each stage is self-contained (it uploads what it is given), so the functions can be swapped in one at a time;
``group()`` is the fused call for code that owns the call site and wants one device round trip.
There is no CPU path: without the CUDA library / an sm_90 GPU these functions raise ``GroupingError``.
"""
from __future__ import annotations

import dataclasses
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import sharding, wire
from .grouping import ST_MEANING, Grouper, GroupingError, clamp_scale, input_geometry
from .skeleton import COCO_FROM_PART, LIMBS, NUM_PARTS, GroupParams

_limbs: Tuple[Tuple[int, int], ...] = LIMBS
_device = 0
_variant = "evaluate"
_input_stage = "host"
_groupers: Dict[int, Grouper] = {}  # the max_batch=1 handle of the per-image calls, per device
_ragged: Dict[int, Grouper] = {}  # the handle of the batched calls (group_many / predict_many), per device
CAP_PEAKS, CAP_CANDS, CAP_ROWS = 128, 4096, 128
MAX_DIM = 32767  # the C ABI's limit; the workspace does not depend on the map size, so ONE handle serves every image size


def _stage(input_stage: str) -> str:
    if input_stage not in ("host", "device"):
        raise ValueError("input_stage must be 'host' or 'device'")
    return input_stage


def _forward_batch(n) -> int:
    if int(n) < 1:
        raise ValueError("forward_batch must be >= 1")
    return int(n)


def configure(limbs: Optional[Sequence[Tuple[int, int]]] = None, device: Optional[int] = None,
              variant: Optional[str] = None, input_stage: Optional[str] = None) -> None:
    """Select the limb table (default: the Canonical ``limbs_conn``, config/config.py:94), the CUDA device, the
    behavioural variant: ``"evaluate"`` (evaluate.py, the default) or ``"demo"`` (demo_image.py's inlined copy, which
    differs at :288, :414-415 and :533 -- SURVEY.md 3.2), and where ``predict`` builds the network's input:
    ``"host"`` (cv2, the default) or ``"device"`` (``spg_prenet``)."""
    global _limbs, _device, _variant, _input_stage
    if input_stage is not None:
        _input_stage = _stage(input_stage)
    if limbs is not None:
        _limbs = tuple((int(a), int(b)) for a, b in limbs)
    if device is not None:
        _device = int(device)
    if variant is not None:
        if variant not in ("evaluate", "demo"):
            raise ValueError("variant must be 'evaluate' or 'demo'")
        _variant = variant
    for g in list(_groupers.values()) + list(_ragged.values()):
        g.close()
    _groupers.clear()
    _ragged.clear()


def _new_grouper(max_batch: int) -> Grouper:
    return Grouper(_limbs, NUM_PARTS, COCO_FROM_PART, max_batch=max_batch, max_h=MAX_DIM, max_w=MAX_DIM,
                   max_peaks_per_part=CAP_PEAKS, max_cands_per_limb=CAP_CANDS, max_person_rows=CAP_ROWS, device=_device)


def _grouper() -> Grouper:
    """The one native handle of the current device (evaluate.py runs over images of hundreds of different sizes: a
    handle per size, as in round 1, grew device memory and streams without bound)."""
    g = _groupers.get(_device)
    if g is None:
        g = _groupers[_device] = _new_grouper(1)
    return g


def _grouper_many(n: int) -> Grouper:
    """The handle of the batched calls on the current device; its max_batch grows on demand.  The max_batch=1 handle of
    the per-image calls stays separate: spg_postnet_rotated sizes its float64 accumulator by the handle's max_batch."""
    g = _ragged.get(_device)
    if g is None or g.max_batch < n:
        if g is not None:
            g.close()
        g = _ragged[_device] = _new_grouper(max(int(n), 1))
    return g


def _params(params):
    """The reference's params dict -> what the library runs with (the demo variant adds its three deviations)."""
    if isinstance(params, GroupParams):
        return params
    return GroupParams.demo(params) if _variant == "demo" else params


def _check_status(status: int) -> None:
    status = int(status)
    if status:
        why = [text for bit, text in ST_MEANING.items() if status & bit]
        raise GroupingError(f"grouping failed (status {status:#x}): " + ("; ".join(why) if why else
                            f"capacity exceeded; capacities: {CAP_PEAKS} peaks/part, {CAP_CANDS} candidates/limb, "
                            f"{CAP_ROWS} person rows"))


#: status bits of an image that went past the handle's capacities (SPG_ST_PEAK_OVERFLOW | SPG_ST_CAND_OVERFLOW |
#: SPG_ST_ROW_OVERFLOW): such an image is regrouped on the capacity-free tier (``Grouper.group_unbounded``)
CAPACITY_BITS = 0x7


def _over_capacity(status) -> bool:
    return bool(int(status) & CAPACITY_BITS)


def _unbounded(heat, paf, as_f64: bool, image_extent, params):
    """One image's device maps regrouped on the capacity-free tier: a one-image ``GroupResult``.  Its status can only
    carry the bits the reference raises for, which ``_check_status`` turns into ``GroupingError``."""
    return _grouper().group_unbounded(heat, paf, image_extent, _params(params), paf_as_f64=as_f64)


def _group_params(params) -> GroupParams:
    p = _params(params)
    return p if isinstance(p, GroupParams) else GroupParams.from_dict(dict(p or {}))


def _chain_params(params) -> GroupParams:
    """``params`` of a later stage with the peak-finding fields find_peaks ran with: what the tier regroups a chained
    image with, so that its peaks are the ones find_peaks returned."""
    return dataclasses.replace(_group_params(params), **_state["peak_params"])


def _tier_unavailable(stage: str, status) -> GroupingError:
    return GroupingError(f"{stage}: the image exceeds the grouping capacities (status {int(status):#x}; {CAP_PEAKS} "
                         f"peaks/part, {CAP_CANDS} candidates/limb, {CAP_ROWS} person rows) and the capacity-free tier "
                         f"needs the maps of the image: chain find_peaks -> find_connections -> find_people on each "
                         f"other's return values, or call group()")


def _people_of_result(r) -> list:
    """``process()``'s return value (evaluate.py:523-543) from a one-image ``GroupResult``, in the form
    ``wire.people_of`` gives it: ``np.float64`` coordinates and score, integer ``(0, 0)`` for a missing joint."""
    out = []
    for j in range(int(r.n_persons[0])):
        row = r.subset[0, j]
        pts = [(np.float64(x), np.float64(y)) if row[part, 0] >= 0 else (0, 0)
               for part, (x, y) in zip(COCO_FROM_PART, r.people_xy[0, j])]
        out.append((pts, np.float64(r.people_score[0, j])))
    return out


def _maps_to_device(hwc: np.ndarray, channels: int, dtype):
    """``[H, W, C]`` host maps (what predict() returns) -> ``[1, channels, H, W]`` device planes of torch ``dtype``.

    The array goes up as it is and is transposed / cast on the device: a numpy transpose of a 512x512x30 float64 array
    on the host costs more than the whole device path.  The float64 -> float32 cast rounds to nearest even on both sides."""
    import torch
    arr = np.asarray(hwc)
    if arr.dtype not in (np.float32, np.float64):
        arr = arr.astype(np.float64)
    t = torch.from_numpy(np.ascontiguousarray(arr)).to(f"cuda:{_device}")
    return t[:, :, :channels].permute(2, 0, 1).to(dtype).contiguous()[None]


def _heat_tensor(heat):
    """``DeviceMaps`` or host ``[H, W, >=18]`` keypoint maps -> ``[1, 18, H, W]`` float32 device planes (the cast of
    evaluate.py:173)."""
    import torch
    return heat.tensor if isinstance(heat, DeviceMaps) else _maps_to_device(heat, NUM_PARTS, torch.float32)


def _paf_tensor(paf):
    """``DeviceMaps`` or host ``[H, W, L]`` body-part maps -> ``(device planes, as_f64)``: host float64 maps stay
    float64, any other host maps become float32; ``as_f64`` says the planes are float32 storage of float64 values."""
    import torch
    if isinstance(paf, DeviceMaps):
        return paf.tensor, paf.as_f64
    dtype = torch.float64 if np.asarray(paf).dtype == np.float64 else torch.float32
    return _maps_to_device(paf, len(_limbs), dtype), False


class DeviceMaps:
    """Averaged maps that stay on the GPU between ``predict`` and the grouping functions (what ``dropin.predict``
    returns in place of the reference's ``[H, W, C]`` float64 host arrays).  ``numpy()`` gives the reference's array."""

    def __init__(self, tensor, as_f64: bool):
        self.tensor, self.as_f64 = tensor, as_f64  # [1, C, H, W]; as_f64: float32 storage of the float64 values
        self.shape = (int(tensor.shape[2]), int(tensor.shape[3]), int(tensor.shape[1]))

    def numpy(self) -> np.ndarray:
        return self.tensor[0].permute(1, 2, 0).double().cpu().numpy()


#: what the last stage left on the device, so that the next stage does not upload it again when it is handed the very
#: objects the previous stage returned (the call sequence of evaluate.py:509-511)
_state: Dict[str, object] = {}


def pad_right_down_corner(img: np.ndarray, stride: int, pad_value: int) -> Tuple[np.ndarray, list]:
    """utils/util.py:44-64: pad below / to the right up to a multiple of ``stride`` with ``pad_value``."""
    h, w = img.shape[:2]
    pad = [0, 0, 0 if h % stride == 0 else stride - h % stride, 0 if w % stride == 0 else stride - w % stride]
    return np.pad(img, ((0, pad[2]), (0, pad[3]), (0, 0)), constant_values=pad_value), pad


#: pinned host staging per slot ("image", "pairs") as ``(buffer, event of the last copy out of it)``
_staging: Dict[str, tuple] = {}


def _pinned(slot: str, n: int, dtype):
    """A pinned buffer of ``n`` elements of ``dtype`` for ``slot`` (grown on demand), once the slot's last copy has left
    it.  Record the next copy out of it with ``_copied(slot)``."""
    import torch
    buf, ev = _staging.get(slot, (None, None))
    if ev is not None:
        ev.synchronize()
    if buf is None or buf.numel() < n:
        buf = torch.empty(n, dtype=dtype, pin_memory=True)
    _staging[slot] = (buf, ev)
    return buf[:n]


def _copied(slot: str) -> None:
    """Mark the copy just enqueued on the current stream out of ``slot``'s buffer."""
    import torch
    ev = torch.cuda.Event()
    ev.record(torch.cuda.current_stream(_device))
    _staging[slot] = (_staging[slot][0], ev)


def _upload_images(images) -> list:
    """The ``[H, W, 3]`` uint8 CUDA image of every entry of ``images``: CUDA tensors as they are (on the current device),
    host images packed into one pinned buffer and sent up with one asynchronous copy into one device buffer, of which
    each gets a view."""
    import torch
    dev = f"cuda:{_device}"
    out = [img.to(dev) if isinstance(img, torch.Tensor) else None for img in images]
    host_imgs = {i: np.ascontiguousarray(img, np.uint8) for i, img in enumerate(images) if out[i] is None}
    if host_imgs:
        host = _pinned("image", sum(a.size for a in host_imgs.values()), torch.uint8)
        staged, at, off = host.numpy(), {}, 0
        for i, a in host_imgs.items():
            staged[off:off + a.size] = a.reshape(-1)
            at[i] = off
            off += a.size
        packed = host.to(dev, non_blocking=True)
        _copied("image")
        for i, a in host_imgs.items():
            out[i] = packed[at[i]:at[i] + a.size].view(a.shape)
    return out


def predict(image, params, model, model_params, heat_layers=None, paf_layers=None, input_image_path=None,
            input_stage: Optional[str] = None):
    """evaluate.py:83-166 with everything after the forward pass on the device.

    Same arguments as the reference's ``predict``.  For every item of ``product(multiplier, rotate_angle)`` (:87-90) the
    image is scaled, padded and -- for ``angle != 0`` -- rotated exactly as there, and the network runs on it and its
    mirror (:118-124).  With ``input_stage="host"`` (the default, see ``configure``) that input is built with cv2 on
    the host (:98-117); with ``"device"`` the uint8 image goes up once (``image`` may also be a uint8 CUDA tensor) and
    ``spg_prenet`` builds every item's pair on the GPU, with OpenCV's generic resize path (the IPP build of the
    reference's wheels differs from it by at most 1 LSB in some pixels).  The flip ensemble, both bicubic resizes, the
    inverse rotation of the maps, the crop and the float64 average over the items (:126-161) happen in
    ``spg_postnet_rotated`` -- the maps never visit the host.  Returns two ``DeviceMaps`` (heatmap, paf) that
    ``find_peaks`` / ``find_connections`` / ``group`` accept."""
    import torch
    stage = _stage(_input_stage if input_stage is None else input_stage)
    g = _grouper()
    multiplier = [x * model_params["boxsize"] / image.shape[0] for x in params["scale_search"]]
    if stage == "device":
        items = g.prenet(_upload_images([image])[0], multiplier, params["rotation_search"],
                         max_downsample=int(model_params["max_downsample"]), pad_value=int(model_params["padValue"]))
    else:
        items = _host_items(image, multiplier, params["rotation_search"], model_params)
    outs, crops, rotations = [], [], []
    for pair, crop, reverse in items:
        with torch.no_grad():
            outs.append(_network_output(model, pair)[None].contiguous())
        crops.append(crop)
        rotations.append(reverse)
    heat, paf = g.postnet(outs, crops, image.shape[:2], stride=int(model_params["stride"]), nan_scrub=_variant == "demo",
                          rotations=rotations)
    return DeviceMaps(heat, False), DeviceMaps(paf, paf.dtype == torch.float32)


def _host_items(image: np.ndarray, multiplier, angles, model_params):
    """The items of ``product(multiplier, angles)`` built with cv2 on the host, each pair moved to the device as it is
    yielded: a generator, so that the next item's cv2 work overlaps the network's kernels for this one."""
    import itertools

    import torch
    for scale, angle in itertools.product(multiplier, angles):
        pair, crop, reverse = _host_pair(image, clamp_scale(scale, image.shape[:2]), angle, model_params)
        yield torch.from_numpy(pair).to(f"cuda:{_device}"), crop, reverse


def _host_pair(image: np.ndarray, scale: float, angle: float, model_params, out: Optional[np.ndarray] = None):
    """evaluate.py:98-117 for one item with cv2 on the host: ``(pair, crop, rotate_matrix_reverse)`` -- ``pair`` the
    ``[2, Hp, Wp, 3]`` float32 network input (image, mirror), written into ``out`` when given; ``crop`` =
    ``imageToTest.shape[:2]``; the reverse matrix is ``None`` for angle 0.  ``scale`` is already clamped."""
    import cv2
    image_to_test = cv2.resize(image, (0, 0), fx=scale, fy=scale, interpolation=cv2.INTER_CUBIC)
    padded, _ = pad_right_down_corner(image_to_test, model_params["max_downsample"], model_params["padValue"])
    input_img = np.float32(padded / 255)
    reverse = None
    if angle != 0:  # evaluate.py:113-117, the centre's x and y swapped as there
        centre = (input_img.shape[0] / 2, input_img.shape[1] / 2)
        reverse = cv2.getRotationMatrix2D(centre, -angle, 1)
        input_img = cv2.warpAffine(input_img, cv2.getRotationMatrix2D(centre, angle, 1), (0, 0))
    if out is None:
        out = np.empty((2,) + input_img.shape, np.float32)
    out[0] = input_img
    out[1] = input_img[:, ::-1, :]
    return out, image_to_test.shape[:2], reverse


def _network_output(model, x):
    """The network's maps for the input batch ``x`` (evaluate.py:124-126): the last stack's finest scale, float32 unless
    the network answers in float16."""
    import torch
    out = model(x)[-1][0]
    if out.dtype not in (torch.float32, torch.float16):
        out = out.float()
    return out


def plan_items(image_shapes, params, model_params):
    """The batches of ``predict_batch`` for any ``scale_search x rotation_search``: per image, per item of
    ``product(multiplier, rotation_search)`` (evaluate.py:87-90) ``(multiplier, scale, angle, H1, W1, Hp, Wp)`` -- the
    scale after the clamp of :94-96, the crop size and the padded network input size of :98-100 -- and the items grouped
    by network input size ``{(Hp, Wp): [(image index, item index), ...]}`` in order of first appearance.  The rotated and
    unrotated items of one scale share a bucket: the rotation happens inside the padded input."""
    import itertools
    plan, buckets = [], {}
    md = int(model_params["max_downsample"])
    for i, shape in enumerate(image_shapes):
        h, w = int(shape[0]), int(shape[1])
        items = []
        multiplier = [x * model_params["boxsize"] / h for x in params["scale_search"]]
        for t, (m, angle) in enumerate(itertools.product(multiplier, params["rotation_search"])):
            scale = clamp_scale(m, (h, w))
            geo = input_geometry(h, w, scale, md)
            items.append((m, scale, angle) + geo)
            buckets.setdefault(geo[2:], []).append((i, t))
        plan.append(items)
    return plan, buckets


def predict_batch(images, params, model, model_params, *, forward_batch: int, input_stage: Optional[str] = None):
    """``predict`` for several images at once: one ``(heatmap, paf)`` pair of ``DeviceMaps`` per image, in input order.

    At stride 4 the items of every image -- one per element of ``scale_search x rotation_search`` -- are grouped by
    padded network input size (``plan_items``; an item's rotation does not change its size).  For each size in turn its
    items' inputs are built into one tensor as ``predict`` builds them (``input_stage`` as there: cv2 on the host, or one
    ``spg_prenet_ragged`` call per size that writes every item into its slot; the call's host images go up together,
    through one pinned buffer and one copy), forward passes take at most ``forward_batch``
    items (``2 * forward_batch`` samples: each item and its mirror), and the tensor is released.  One
    ``spg_postnet_ragged_items`` call then runs the post-network stage of the whole batch, reading each item's pair out
    of its forward pass in place.  Every network output lives until that call: at ``scale_search = [0.5, 1, 1.5, 2]``,
    boxsize 640, float32 that is about 100 MB per 480 x 640 image.

    Every kernel treats each image on its own, so the maps equal ``predict``'s bit for bit when the network's output for
    a sample does not depend on the batch it runs in (a network under cuDNN may pick another algorithm for another batch
    size).  Another stride runs ``predict`` per image."""
    import torch
    stage = _stage(_input_stage if input_stage is None else input_stage)
    fb = _forward_batch(forward_batch)
    images = list(images)
    if int(model_params["stride"]) != 4:
        return [predict(img, params, model, model_params, input_stage=stage) for img in images]
    plan, buckets = plan_items([img.shape[:2] for img in images], params, model_params)
    g = _grouper_many(len(images))
    dev = f"cuda:{_device}"
    md, pv = int(model_params["max_downsample"]), int(model_params["padValue"])
    uploaded = _upload_images(images) if stage == "device" else None
    entries = [[None] * len(items) for items in plan]
    for (Hp, Wp), members in buckets.items():
        k = len(members)
        x = torch.empty((2 * k, Hp, Wp, 3), dtype=torch.float32, device=dev)
        if stage == "host":
            built = []  # per member (crop, rotate_matrix_reverse)
            host = _pinned("pairs", x.numel(), torch.float32).view(x.shape)
            for j, (i, t) in enumerate(members):
                _, scale, angle = plan[i][t][:3]
                built.append(_host_pair(images[i], scale, angle, model_params, out=host[2 * j:2 * j + 2].numpy())[1:])
            x.copy_(host, non_blocking=True)
            _copied("pairs")
        else:
            pairs = g.prenet_ragged([(uploaded[i], plan[i][t][0], plan[i][t][2]) for i, t in members], max_downsample=md,
                                    pad_value=pv, out=[x[2 * j:2 * j + 2] for j in range(k)])
            built = [(crop, reverse) for _, crop, reverse in pairs]
        for c0 in range(0, k, fb):
            c1 = min(k, c0 + fb)
            with torch.no_grad():
                out = _network_output(model, x[2 * c0:2 * c1]).contiguous()
            for j in range(c0, c1):
                i, t = members[j]
                entries[i][t] = (out[2 * (j - c0):2 * (j - c0) + 2],) + built[j]
        del x
    maps = g.postnet_ragged_items([(e, tuple(int(v) for v in img.shape[:2])) for e, img in zip(entries, images)],
                                  nan_scrub=_variant == "demo")
    return [(DeviceMaps(heat, False), DeviceMaps(paf, paf.dtype == torch.float32)) for heat, paf in maps]


def _upload_peaks(g: Grouper, all_peaks) -> None:
    if _state.get("peaks") is all_peaks and _state.get("handle") is g:
        return  # still on the device from our own find_peaks
    _state.clear()
    counts = [len(p) for p in all_peaks]
    flat = [t for part in all_peaks for t in part]
    g.upload_peaks(0, counts, [float(t[0]) for t in flat], [float(t[1]) for t in flat], [np.float32(t[2]) for t in flat])


# ---- the three reference functions ---------------------------------------------------------------------
def find_peaks(heatmap_avg, params):
    """evaluate.py:169-203.  ``heatmap_avg [H,W,>=18]`` -> list[18] of [(x, y, score, id), ...]."""
    import torch
    g = _grouper()
    heat = _heat_tensor(heatmap_avg)
    g.nms_peaks(heat, _params(params))
    r = g.fetch(1)
    tier = _over_capacity(r.status[0])
    if tier:  # every peak of the image from the capacity-free tier; no body-part maps yet, so zero planes stand in
        zeros = torch.zeros((1, len(_limbs)) + tuple(heat.shape[2:]), dtype=torch.float32, device=heat.device)
        r = _unbounded(heat, zeros, False, heat.shape[2], params)
    else:
        _check_status(r.status[0])
    all_peaks = r.as_reference_structures(0)[0]
    gp = _group_params(params)
    _state.clear()
    _state.update(peaks=all_peaks, handle=g, heat=heat, tier_peaks=tier,
                  peak_params=dict(thre1=gp.thre1, offset_radius=gp.offset_radius))
    return all_peaks


def _chained_peaks(g: Grouper, all_peaks) -> bool:
    """``all_peaks`` is what our own find_peaks returned last, on handle ``g``, with its heat maps kept."""
    return _state.get("peaks") is all_peaks and _state.get("handle") is g and "heat" in _state


def find_connections(all_peaks, paf_avg, image_width, params):
    """evaluate.py:206-276.  ``paf_avg [H,W,L]`` float32 or float64 -> (connection_all, special_k)."""
    g = _grouper()
    chained = _chained_peaks(g, all_peaks)
    paf, as_f64 = _paf_tensor(paf_avg)
    tier = chained and bool(_state.get("tier_peaks"))
    if not tier:
        _upload_peaks(g, all_peaks)
        g.limb_score(paf, image_width, _params(params), paf_as_f64=as_f64)
        g.limb_match(1, _params(params))
        r = g.fetch(1)
        if _over_capacity(r.status[0]):
            if not chained:
                raise _tier_unavailable("find_connections", r.status[0])
            tier = True
    if tier:
        gp = _chain_params(params)
        r = _unbounded(_state["heat"], paf, as_f64, image_width, gp)
        _state.update(tier=r, tier_params=gp)  # find_people takes its persons from the same call
    _check_status(r.status[0])
    if chained:
        _state.update(paf=paf, as_f64=as_f64, extent=image_width)
    # ids in the rows are those of the caller's all_peaks (:267), not positions in our tables
    _, conns, special, _, _ = r.as_reference_structures(0)
    for k, rows in enumerate(conns):
        if isinstance(rows, list) or not len(rows):
            continue
        a, b = _limbs[k]
        rows[:, 0] = np.array([t[3] for t in all_peaks[a]], np.float64)[rows[:, 3].astype(np.int64)]
        rows[:, 1] = np.array([t[3] for t in all_peaks[b]], np.float64)[rows[:, 4].astype(np.int64)]
    _state.update(conns=conns, special=special)
    return conns, special


def find_people(connection_all, special_k, all_peaks, params):
    """evaluate.py:279-498 -> (subset [P,20,2] float64, candidate [N,4] float64)."""
    g = _grouper()  # assembly does not depend on the map size
    if _state.get("conns") is connection_all and _state.get("special") is special_k and _state.get("peaks") is all_peaks \
            and _state.get("handle") is g:  # evaluate.py:509-511 handing our own objects back: everything is still on the device
        r = _state.get("tier")
        if r is None:
            g.assemble(1, _params(params))
            r = g.fetch(1)
            if _over_capacity(r.status[0]):
                if "paf" not in _state:
                    raise _tier_unavailable("find_people", r.status[0])
                r = None
        if r is None or _state.get("tier_params") not in (None, _chain_params(params)):
            gp = _chain_params(params)  # the persons of the tier, with find_people's own assembly parameters
            r = _unbounded(_state["heat"], _state["paf"], _state["as_f64"], _state["extent"], gp)
            _state.update(tier=r, tier_params=gp)
        _check_status(r.status[0])
        return r.subset[0, :int(r.n_persons[0])].copy(), np.array([item for sublist in all_peaks for item in sublist])
    _upload_peaks(g, all_peaks)
    special = set(int(k) for k in special_k)
    counts, ij, sc, nm = [], [], [], []
    for k, rows in enumerate(connection_all):
        if k in special:
            counts.append(-1)
            continue
        rows = np.asarray(rows, np.float64).reshape(-1, 6)
        counts.append(len(rows))
        ij.append(rows[:, 3:5].astype(np.int32))
        sc.append(rows[:, 2])
        nm.append(rows[:, 5])
    g.upload_connections(0, counts, np.concatenate(ij) if ij else np.zeros((0, 2), np.int32),
                         np.concatenate(sc) if sc else np.zeros(0), np.concatenate(nm) if nm else np.zeros(0))
    g.assemble(1, _params(params))
    r = g.fetch(1)
    if _over_capacity(r.status[0]):
        raise _tier_unavailable("find_people", r.status[0])
    _check_status(r.status[0])
    subset = r.subset[0, :int(r.n_persons[0])].copy()
    candidate = np.array([item for sublist in all_peaks for item in sublist])  # evaluate.py:283, verbatim semantics
    # subset holds positions in the flattened table; the reference stores the peaks' own ids there (equal unless
    # the caller renumbered all_peaks)
    flat_ids = [t[3] for part in all_peaks for t in part]
    if flat_ids != list(range(len(flat_ids))):
        ids = np.asarray(flat_ids, np.float64)
        sel = subset[:, :-2, 0] >= 0
        subset[:, :-2, 0][sel] = ids[subset[:, :-2, 0][sel].astype(int)]
    return subset, candidate


def group(heatmap_avg, paf_avg, image_extent, params):
    """Fused peaks -> connections -> people: one upload, four kernels, one download.

    Returns ``(all_peaks, connection_all, special_k, subset, candidate)`` exactly as the three calls would."""
    g = _grouper()
    _state.clear()
    heat = _heat_tensor(heatmap_avg)
    paf, as_f64 = _paf_tensor(paf_avg)
    g.group_device(heat, paf, image_extent, _params(params), paf_as_f64=as_f64)
    r = g.fetch(1)
    if _over_capacity(r.status[0]):
        r = _unbounded(heat, paf, as_f64, image_extent, params)
    _check_status(r.status[0])
    return r.as_reference_structures(0)


def _ragged_maps(maps):
    """(heat, paf) pairs of ``DeviceMaps`` or host ``[H, W, C]`` arrays -> device tensors + whether paf is float32
    storage of float64 values (one answer for the whole call)."""
    pairs, as_f64 = [], set()
    for heat, paf in maps:
        h = _heat_tensor(heat)
        p, f64 = _paf_tensor(paf)
        pairs.append((h, p))
        as_f64.add(f64)
    if len(as_f64) > 1:
        raise GroupingError("the body-part maps of one call must all be float32, float32-held float64 or float64")
    return pairs, as_f64 == {True}


#: device buffers of the wire records ``predict_many`` downloads, per device
_records: Dict[int, object] = {}


def _group_ragged(maps, image_extents, params, records: bool = False):
    """The maps of a batch of images to the device and one ragged grouping call (``spg_group_ragged``) on the batched
    handle: ``(handle, n_images, wire, regroup)``.  With ``records`` the call also writes image i's wire record to row i
    of ``wire``, a per-device buffer; without, ``wire`` is None.  ``regroup(i)`` regroups image i on the capacity-free
    tier from the device maps of the call."""
    import torch
    pairs, as_f64 = _ragged_maps(maps)
    g = _grouper_many(len(pairs))
    _state.clear()
    buf = None
    if records:
        rec_bytes = g.wire_record_bytes()
        buf = _records.get(_device)
        if buf is None or buf.shape[0] < len(pairs) or buf.shape[1] != rec_bytes:
            buf = torch.empty((max(len(pairs), g.max_batch), rec_bytes), dtype=torch.uint8, device=f"cuda:{_device}")
            _records[_device] = buf
        g.set_wire_output(buf.data_ptr())
    try:
        g.group_ragged(pairs, image_extents, _params(params), paf_as_f64=as_f64)
    finally:
        if records:
            g.set_wire_output(None)

    def regroup(i: int):
        return _unbounded(pairs[i][0], pairs[i][1], as_f64, image_extents[i], params)
    return g, len(pairs), buf, regroup


def group_many(maps, image_extents, params):
    """``group()`` for several images of different sizes in ONE grouping call (``spg_group_ragged``) and one download.

    ``maps``: per image a ``(heatmap_avg, paf_avg)`` pair -- the ``DeviceMaps`` ``predict`` returns or host ``[H, W, C]``
    arrays; ``image_extents``: per image ``oriImg.shape[0]``.  Returns one ``(all_peaks, connection_all, special_k,
    subset, candidate)`` per image, equal to what ``group()`` returns for it."""
    image_extents = list(image_extents)
    g, n, _, regroup = _group_ragged(maps, image_extents, params)
    r = g.fetch(n)
    out = []
    for i in range(n):
        if _over_capacity(r.status[i]):
            ri = regroup(i)
            _check_status(ri.status[0])
            out.append(ri.as_reference_structures(0))
            continue
        _check_status(r.status[i])
        out.append(r.as_reference_structures(i))
    return out


def _people_of_batch(maps, extents, params) -> list:
    """One ragged grouping call for a batch of images, their wire records in one device-to-host copy, and per image
    ``process()``'s return value (evaluate.py:523-543)."""
    extents = list(extents)
    g, n, buf, regroup = _group_ragged(maps, extents, params, records=True)
    out = []
    for i, rec in enumerate(wire.as_records(buf[:n].cpu().numpy(), g.J, g.capR)):
        if _over_capacity(rec["status"]):  # the record holds at most capR persons: the tier's arrays hold them all
            ri = regroup(i)
            _check_status(ri.status[0])
            out.append(_people_of_result(ri))
            continue
        _check_status(rec["status"])
        out.append(wire.people_of(rec))
    return out


def predict_many(coco, images_directory, validation_ids, params, model, model_params, heat_layers, paf_layers,
                 batch: int = 16, image_name=None, forward_batch: int = 1):
    """evaluate.py:550-560 with the grouping of ``batch`` images at a time in one call.

    Same arguments, assert and result as the reference's ``predict_many``: ``{image_id: [([17 x (x, y)], score)]}`` in
    ``validation_ids`` order, with ``np.float64`` coordinates and scores and integer ``(0, 0)`` for a missing joint, so
    ``format_results`` writes the same file.  Per image: ``cv2.imread`` and ``predict`` (the maps stay on the device);
    every ``batch`` images and at the end: one ``group_many``-style ragged call, the batch's wire records in one copy.
    ``forward_batch > 1`` runs ``predict_batch`` on each group of ``batch`` images instead of ``predict`` per image, for
    any ``scale_search`` and ``rotation_search`` at stride 4 (see there for when its maps equal ``predict``'s).  A
    non-zero status raises ``GroupingError``.  ``image_name(coco, image_id)`` gives the file name (default: ``coco.imgs[image_id]['file_name']``, evaluate.py:546-547).  ``process()``
    is not called, so the reference's ``batch_time`` meter is not updated.

    In an initialised ``torch.distributed`` world of N > 1 processes (one per GPU) this is rank 0's call, and the other
    ranks run ``serve_predict_many``: the images are sharded over the ranks in contiguous blocks
    (``sharding.shard_range``), each rank runs its block exactly as above, and rank 0 returns the same dict a single
    process returns.  A block that raises on any rank raises ``GroupingError`` here, naming the rank and the image."""
    assert (not set(validation_ids).difference(set(coco.getImgIds())))
    if int(batch) < 1:
        raise ValueError("batch must be >= 1")
    fb = _forward_batch(forward_batch)
    names = [image_name(coco, iid) if image_name is not None else coco.imgs[iid]["file_name"] for iid in validation_ids]
    rank, world = sharding._world()
    if world == 1:
        return _predict_block(images_directory, list(zip(validation_ids, names)), params, model, model_params,
                              heat_layers, paf_layers, int(batch), fb)
    if rank != 0:
        raise RuntimeError(f"predict_many runs on rank 0; rank {rank} of {world} calls serve_predict_many")
    import os
    return _predict_sharded(dict(images_directory=os.path.abspath(images_directory), ids=list(validation_ids),
                                 names=names, params=params, model_params=model_params, heat_layers=heat_layers,
                                 paf_layers=paf_layers, batch=int(batch), forward_batch=fb), model)


def _predict_block(images_directory, named_ids, params, model, model_params, heat_layers, paf_layers, batch: int,
                   fb: int, at: Optional[list] = None) -> dict:
    """The body of ``predict_many`` over ``named_ids`` = ``[(image_id, file name)]``: ``{image_id: people}`` in that
    order.  ``at`` (a list) is kept holding the ids of the image or grouping batch being worked on, for error reports."""
    import os

    import cv2
    at = [] if at is None else at
    keypoints = {}
    pending = []  # (image_id, (heatmap, paf) -- or the image itself for predict_batch, oriImg.shape[0])

    def flush():
        if pending:
            at[:] = [iid for iid, _, _ in pending]  # the batch's ragged calls fail as one
            maps = [m for _, m, _ in pending]
            if fb > 1:
                maps = predict_batch(maps, dict(params), model, dict(model_params), forward_batch=fb)
            people = _people_of_batch(maps, [e for _, _, e in pending], params)
            for (iid, _, _), kp in zip(pending, people):
                keypoints[iid] = kp
            pending.clear()

    for image_id, name in named_ids:
        at[:] = [image_id]
        path = os.path.join(images_directory, name)
        ori = cv2.imread(path)  # B,G,R order (evaluate.py:502)
        if fb > 1:
            pending.append((image_id, ori, ori.shape[0]))
        else:
            pending.append((image_id, predict(ori, dict(params), model, dict(model_params), heat_layers + 2, paf_layers, path),
                            ori.shape[0]))
        if len(pending) >= batch:
            flush()
    flush()
    return keypoints


def _run_job(job: dict, model, rank: int, world: int):
    """This rank's block of ``job``: its ``{image_id: people}``, or, if the block raised, the text that says where and
    why (sent in place of the dict, so that the gather completes on every rank)."""
    lo, hi = sharding.shard_range(len(job["ids"]), rank, world)
    at: list = []
    try:
        return _predict_block(job["images_directory"], list(zip(job["ids"][lo:hi], job["names"][lo:hi])), job["params"],
                              model, job["model_params"], job["heat_layers"], job["paf_layers"], job["batch"],
                              job["forward_batch"], at)
    except Exception as e:  # noqa: BLE001 -- any failure of the block is reported to rank 0, which raises it
        where = f"image {at[0]}" if len(at) == 1 else f"images {at}"
        return f"{where}: {type(e).__name__}: {e}"


def _predict_sharded(job: dict, model) -> dict:
    """Rank 0 of ``predict_many`` in a world of N > 1: broadcast the job, run block 0, gather every rank's dict."""
    import torch.distributed as dist
    rank, world = sharding._world()
    dist.broadcast_object_list([job], src=0)
    mine = _run_job(job, model, rank, world)
    blocks: List[object] = [None] * world
    dist.gather_object(mine, blocks, dst=0)
    failed = [f"rank {r}, {b}" for r, b in enumerate(blocks) if isinstance(b, str)]
    if failed:
        raise GroupingError("predict_many failed on " + "; ".join(failed))
    keypoints = {}
    for b in blocks:  # rank order is image order: the blocks are contiguous
        keypoints.update(b)
    return keypoints


def serve_predict_many(model) -> None:
    """Ranks other than 0 of a ``torch.distributed`` world: run this rank's block of every ``predict_many`` call of
    rank 0 with the network ``model`` on this rank's device (``configure(device=local_rank)``), send rank 0 its
    ``{image_id: people}`` (or the text of the exception its block raised), and return at the empty job that
    ``end_serving`` on rank 0 broadcasts."""
    import torch.distributed as dist
    rank, world = sharding._world()
    if rank == 0:
        raise RuntimeError("serve_predict_many runs on the ranks other than 0")
    while True:
        job = [None]
        dist.broadcast_object_list(job, src=0)
        if not job[0]:
            return
        dist.gather_object(_run_job(job[0], model, rank, world), None, dst=0)


def end_serving() -> None:
    """Rank 0: broadcast the empty job that makes ``serve_predict_many`` return on the other ranks (call it once rank 0
    is done with ``predict_many``, also when it raised).  Nothing to do in a world of one process."""
    import torch.distributed as dist
    rank, world = sharding._world()
    if world > 1:
        if rank != 0:
            raise RuntimeError("end_serving runs on rank 0")
        dist.broadcast_object_list([None], src=0)


def keypoints(subset, candidate):
    """Tail of process() (evaluate.py:523-543): [(17 x (x, y) in COCO order, score)]."""
    out = []
    for row in subset:
        pts = []
        for part in COCO_FROM_PART:
            idx = row[part, 0]
            pts.append((0, 0) if idx == -1 else tuple(candidate[int(idx)][:2]))
        out.append((pts, 1 - 1.0 / row[-2, 0]))
    return out


def keypoint_heatmap_nms(heat, kernel: int = 3, thre: float = 0.1):
    """utils/util.py:177-183 -- the one seam demo_image.py offers (:213).  ``heat [1,C,H,W]`` tensor -> ``heat * keep``.

    Peaks come from the CUDA NMS kernel; the masked map is rebuilt from them (zeros elsewhere)."""
    import torch
    if kernel != 3:
        raise GroupingError("only the 3x3 NMS the reference uses is implemented")
    if heat.dim() != 4 or heat.shape[0] != 1:
        raise GroupingError("expected a [1,C,H,W] tensor")
    C = heat.shape[1]
    g = Grouper(((0, 0),), C, (0,), max_batch=1, max_h=MAX_DIM, max_w=MAX_DIM, max_peaks_per_part=CAP_PEAKS,
                device=_device) if C != NUM_PARTS else _grouper()
    src = heat.to(f"cuda:{_device}", torch.float32).contiguous()
    _state.clear()
    g.nms_peaks(src, dict(thre1=float(thre), offset_radius=0))
    r = g.fetch(1)
    _check_status(r.status[0])
    out = torch.zeros_like(src)
    for c in range(C):
        n = int(min(r.peak_count[0, c], r.peak_anchor.shape[2]))
        if n:
            a = r.peak_anchor[0, c, :n].astype(np.int64)
            ys = torch.as_tensor((a >> 16) & 0x7fff, device=src.device)
            xs = torch.as_tensor(a & 0xffff, device=src.device)
            out[0, c, ys, xs] = src[0, c, ys, xs]
    if C != NUM_PARTS:
        g.close()
    return out.to(heat.device)


def install(evaluate_module, device_predict: bool = False, device_input: bool = False, batch: int = 1,
            forward_batch: int = 1) -> None:
    """Rebind ``find_peaks / find_connections / find_people`` of an imported reference ``evaluate`` module.

    ``limbSeq`` is taken from the module (evaluate.py:54) so alternative skeletons keep working.  With
    ``device_predict`` the module's ``predict`` (:83-166) is replaced as well: the network of the module (the global
    ``posenet`` the reference's own predict uses, :124) feeds the device post-network stage and the maps stay on the GPU.
    ``device_input`` (with ``device_predict``) also builds the network's input on the GPU (``input_stage="device"``).
    ``batch > 1`` (with ``device_predict``) also replaces ``predict_many`` (:550-560) by ``predict_many`` above, which
    groups ``batch`` images per call; it uses the module's ``posenet`` and ``get_image_name`` and leaves the module's
    ``batch_time`` meter alone.  ``forward_batch > 1`` (with ``device_predict`` and ``batch > 1``) makes that
    ``predict_many`` run the network on up to ``forward_batch`` items (images, or with a multi-scale or rotation search
    their scaled and rotated copies) of the same input size at once (``predict_batch``).  In an initialised
    ``torch.distributed`` world of N > 1 processes, one per GPU, each with ``configure(device=local_rank)``, that
    ``predict_many`` shards the images over the ranks: rank 0 calls it (``evaluate.validation()``), the other ranks
    run ``serve_predict_many`` until rank 0 calls ``end_serving``."""
    if int(batch) > 1 and not device_predict:
        raise ValueError("batch > 1 needs device_predict=True: the batched grouping takes the maps predict() leaves on the device")
    fb = _forward_batch(forward_batch)
    if fb > 1 and (not device_predict or int(batch) < 2):
        raise ValueError("forward_batch > 1 needs device_predict=True and batch > 1: it batches predict_many's forward passes")
    configure(limbs=getattr(evaluate_module, "limbSeq", _limbs), input_stage="device" if device_input else "host")
    evaluate_module.find_peaks = find_peaks
    evaluate_module.find_connections = find_connections
    evaluate_module.find_people = find_people
    if device_predict:
        def _predict(image, params, model, model_params, heat_layers, paf_layers, input_image_path):
            return predict(image, params, getattr(evaluate_module, "posenet", model), model_params, heat_layers,
                           paf_layers, input_image_path)
        evaluate_module.predict = _predict
    if int(batch) > 1:
        def _predict_many(coco, images_directory, validation_ids, params, model, model_params, heat_layers, paf_layers):
            return predict_many(coco, images_directory, validation_ids, params, getattr(evaluate_module, "posenet", model),
                                model_params, heat_layers, paf_layers, batch=int(batch),
                                image_name=getattr(evaluate_module, "get_image_name", None), forward_batch=fb)
        evaluate_module.predict_many = _predict_many
