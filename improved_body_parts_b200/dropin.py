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
import functools
from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np

from . import sharding, wire
from .grouping import (JPEG_OK, JPEG_RECORD, SMOOTH_FRAME, SMOOTH_TABLE, ST_MEANING, TRACK_FRAME, TRACK_TABLE, YUV_I420,
                       YUV_MEMBER, YUV_NV12, YUV_YUYV, Grouper, GroupingError, clamp_scale, input_geometry, jpeg_parse,
                       prenet_item)
from .skeleton import COCO_FROM_PART, LIMBS, NUM_PARTS, GroupParams

_limbs: Tuple[Tuple[int, int], ...] = LIMBS
_device = 0
_variant = "evaluate"
_input_stage = "host"
_decode = "host"
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
              variant: Optional[str] = None, input_stage: Optional[str] = None, decode: Optional[str] = None) -> None:
    """Select the limb table (default: the Canonical ``limbs_conn``, config/config.py:94), the CUDA device, the
    behavioural variant: ``"evaluate"`` (evaluate.py, the default) or ``"demo"`` (demo_image.py's inlined copy, which
    differs at :288, :414-415 and :533 -- SURVEY.md 3.2), where ``predict`` builds the network's input:
    ``"host"`` (cv2, the default) or ``"device"`` (``spg_prenet``), and how ``predict_many`` reads the image files:
    ``"host"`` (``cv2.imread``, the default) or ``"device"`` (``imread_many``: each group of ``batch`` files decoded on
    the GPU in one call), which needs the device input stage.  The combination is checked after the call's changes:
    with ``decode="device"`` in effect, ``configure(input_stage="host")`` raises ``ValueError`` unless it also passes
    ``decode="host"``."""
    global _limbs, _device, _variant, _input_stage, _decode
    stage = _input_stage if input_stage is None else _stage(input_stage)
    dec = _decode if decode is None else decode
    if dec not in ("host", "device"):
        raise ValueError("decode must be 'host' or 'device'")
    if dec == "device" and stage != "device":
        raise ValueError("decode='device' needs input_stage='device': the network input is built from the decoded CUDA "
                         "image")
    _input_stage, _decode = stage, dec
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


def _new_grouper(max_batch: int, device: Optional[int] = None) -> Grouper:
    return Grouper(_limbs, NUM_PARTS, COCO_FROM_PART, max_batch=max_batch, max_h=MAX_DIM, max_w=MAX_DIM,
                   max_peaks_per_part=CAP_PEAKS, max_cands_per_limb=CAP_CANDS, max_person_rows=CAP_ROWS,
                   device=_device if device is None else device)


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


def _people_of_record(rec, regroup) -> list:
    """``process()``'s return value from one image's wire record, which holds at most capR persons: with a capacity bit
    the image's people come from ``regroup()``, its one-image ``GroupResult`` on the capacity-free tier."""
    if _over_capacity(rec["status"]):
        r = regroup()
        _check_status(r.status[0])
        return _people_of_result(r)
    _check_status(rec["status"])
    return wire.people_of(rec)


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


def _pack(slot: str, arrays) -> list:
    """The uint8 host ``arrays`` packed into ``slot``'s pinned buffer and sent up with one asynchronous copy into one
    device buffer: per array its flat view of that buffer."""
    import torch
    arrays = [a.reshape(-1) for a in arrays]
    host = _pinned(slot, sum(a.size for a in arrays), torch.uint8)
    staged, bounds = host.numpy(), np.cumsum([0] + [a.size for a in arrays]).tolist()
    for a, o in zip(arrays, bounds):
        staged[o:o + a.size] = a
    packed = host.to(f"cuda:{_device}", non_blocking=True)
    _copied(slot)
    return [packed[o0:o1] for o0, o1 in zip(bounds, bounds[1:])]


def _upload_images(images) -> list:
    """The ``[H, W, 3]`` uint8 CUDA image of every entry of ``images``: CUDA tensors as they are (on the current device),
    host images packed into one pinned buffer and sent up with one asynchronous copy into one device buffer, of which
    each gets a view."""
    import torch
    out = [img.to(f"cuda:{_device}") if isinstance(img, torch.Tensor) else None for img in images]
    host_imgs = {i: np.ascontiguousarray(img, np.uint8) for i, img in enumerate(images) if out[i] is None}
    if host_imgs:
        for (i, a), v in zip(host_imgs.items(), _pack("image", host_imgs.values())):
            out[i] = v.view(a.shape)
    return out


def imread_many(paths) -> Tuple[list, int]:
    """``cv2.imread(path)`` of every path as a ``[H, W, 3]`` uint8 CUDA tensor on the current device, in order, and the
    number of files that were read on the host.

    The files are read and parsed (``spg_jpeg_parse``); the ones the device decoder takes -- baseline and
    extended-sequential Huffman JPEGs, grey or YCbCr 4:4:4 / 4:2:2 / 4:4:0 / 4:2:0 -- go up together through one pinned
    buffer and one copy and are decoded in one ``spg_jpeg_decode_ragged`` call, bit-identical to ``cv2.imread``.  Every
    other file (progressive, another format, anything the parser or the decoder finds malformed) is read with
    ``cv2.imread`` and uploaded: those are the host fallbacks.  A file cv2 cannot read, a missing or unreadable path
    included, gives ``None``, as ``cv2.imread`` does."""
    import cv2
    import torch
    dev = torch.device("cuda", _device)
    datas = []
    for p in paths:
        try:
            with open(p, "rb") as f:
                datas.append(f.read())
        except OSError:  # missing or unreadable: cv2.imread below gives None for it
            datas.append(None)
    todo = [i for i, d in enumerate(datas) if d is not None]
    recs = {i: jpeg_parse(datas[i]) for i in todo}
    todo = [i for i in todo if recs[i]["status"] == JPEG_OK]
    out = [None] * len(datas)
    if todo:
        files = _pack("jpeg", [np.frombuffer(datas[i], np.uint8) for i in todo])
        sizes = [int(recs[i]["height"]) * int(recs[i]["width"]) * 3 for i in todo]
        images = torch.empty(sum(sizes), dtype=torch.uint8, device=dev)
        status = torch.empty(len(todo), dtype=torch.int32, device=dev)
        arr = np.zeros(len(todo), JPEG_RECORD)
        o = 0
        for k, i in enumerate(todo):
            arr[k] = recs[i]
            arr[k]["data"], arr[k]["out"] = files[k].data_ptr(), images.data_ptr() + o
            arr[k]["decode_status"] = status.data_ptr() + 4 * k
            out[i] = images[o:o + sizes[k]].view(int(recs[i]["height"]), int(recs[i]["width"]), 3)
            o += sizes[k]
        _grouper().jpeg_decode(arr)
        for k, st in enumerate(status.cpu().tolist()):  # synchronises the decode
            if st != JPEG_OK:
                out[todo[k]] = None
    host_reads = 0
    for i, p in enumerate(paths):
        if out[i] is None:
            host_reads += 1
            img = cv2.imread(p)
            out[i] = None if img is None else torch.from_numpy(img).to(dev)
    return out, host_reads


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


def _host_pairs(images, plan, members, model_params, out) -> list:
    """The cv2 pair of every member ``(image index, item index)`` of one network input size (``plan_items``), written
    into the pinned ``[2 * len(members), Hp, Wp, 3]`` float32 tensor ``out``; per member ``(crop, reverse)``."""
    return [_host_pair(images[i], plan[i][t][1], plan[i][t][2], model_params, out=out[2 * j:2 * j + 2].numpy())[1:]
            for j, (i, t) in enumerate(members)]


def _forward_bucket(model, x, members, built, step: int, entries) -> None:
    """Forward one input size's tensor ``x`` (the pairs of ``members``) ``step`` members at a time, and set each member's
    ``entries[i][t]`` to ``(output pair, crop, reverse)`` (``built``: per member its crop and reverse)."""
    import torch
    with torch.no_grad():
        for c in range(0, len(members), step):
            out = _network_output(model, x[2 * c:2 * (c + step)]).contiguous()
            for k, (i, t) in enumerate(members[c:c + step]):
                entries[i][t] = (out[2 * k:2 * k + 2],) + built[c + k]


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
            host = _pinned("pairs", x.numel(), torch.float32).view(x.shape)
            built = _host_pairs(images, plan, members, model_params, host)
            x.copy_(host, non_blocking=True)
            _copied("pairs")
        else:
            pairs = g.prenet_ragged([(uploaded[i], plan[i][t][0], plan[i][t][2]) for i, t in members], max_downsample=md,
                                    pad_value=pv, out=[x[2 * j:2 * j + 2] for j in range(k)])
            built = [(crop, reverse) for _, crop, reverse in pairs]
        _forward_bucket(model, x, members, built, fb, entries)
        del x
    maps = g.postnet_ragged_items([(e, tuple(int(v) for v in img.shape[:2])) for e, img in zip(entries, images)],
                                  nan_scrub=_variant == "demo")
    return [(DeviceMaps(heat, False), DeviceMaps(paf, paf.dtype == torch.float32)) for heat, paf in maps]


class FrameResult(NamedTuple):
    """``FrameStream.result(ticket, detail=True)``: the people, the frame's wire record (``include/spgroup.h``; only the
    header and the first ``n_persons`` rows are the frame's), copies of its averaged maps and, for a frame submitted as
    JPEG bytes or a ``YUVFrame``, the ``[H, W, 3]`` uint8 BGR image it was decoded or converted to (on the device, or by
    ``cv2.imdecode`` / ``cv2.cvtColor``), else None."""
    people: list
    record: np.ndarray
    heat: "DeviceMaps"
    paf: "DeviceMaps"
    image: Optional[np.ndarray] = None


#: the fields of a parsed JPEG that a frame graph's launches depend on: the format a graph serves
JPEG_FORMAT = ("frame_height", "frame_width", "n_components", "h_samp", "v_samp", "restart_interval", "orientation")


def _imdecode(data: np.ndarray) -> np.ndarray:
    """``cv2.imdecode(data, IMREAD_COLOR)``; ``ValueError`` for bytes cv2 cannot decode either."""
    import cv2
    img = cv2.imdecode(data, cv2.IMREAD_COLOR)
    if img is None:
        raise ValueError("the frame's bytes are not an image cv2.imdecode can decode")
    return img


#: cv2.cvtColor's code and spg_yuv_to_bgr's format of each YUV layout FrameStream takes
_YUV = {"nv12": ("COLOR_YUV2BGR_NV12", YUV_NV12), "i420": ("COLOR_YUV2BGR_I420", YUV_I420),
        "yuyv": ("COLOR_YUV2BGR_YUYV", YUV_YUYV)}


def _yuv_layout(fmt: str, H: int, W: int) -> List[Tuple[int, Tuple[int, int]]]:
    """Per plane of an H x W frame in ``fmt``: its offset in the packed planes and its shape."""
    shapes = {"nv12": [(H, W), (H // 2, W)], "i420": [(H, W), (H // 2, W // 2), (H // 2, W // 2)],
              "yuyv": [(H, 2 * W)]}[fmt]
    offsets = np.cumsum([0] + [h * w for h, w in shapes]).tolist()
    return list(zip(offsets, shapes))


def _yuv_bytes(fmt: str, H: int, W: int) -> int:
    """The packed planes' bytes: 1.5 per pixel for NV12 and I420, 2 for YUYV."""
    return H * W * 3 // 2 if fmt != "yuyv" else 2 * H * W


class YUVFrame:
    """A camera or video frame in YUV, for ``FrameStream.submit`` and ``submit_many``.

    ``format`` is ``"nv12"`` (NVDEC and GPU video readers), ``"i420"`` (FFmpeg / PyAV ``yuv420p``, software
    pipelines) or ``"yuyv"`` (V4L2 / UVC webcams), and ``planes`` a tuple of 2-D uint8 arrays, all numpy or all CUDA
    tensors on one device: NV12 Y ``[H, W]`` and interleaved UV ``[H/2, W]``; I420 Y ``[H, W]``, U and V
    ``[H/2, W/2]``; YUYV the packed ``[H, 2W]``.  A plane's rows may be pitched -- stride ``(pitch, 1)`` with ``pitch``
    at least its row's bytes -- so the views of a decoder's surface can be passed as they are.  H and W must be even
    (W for YUYV), as ``cv2.cvtColor`` requires.  The frame is posed as ``cv2.cvtColor(frame, COLOR_YUV2BGR_*)``, OpenCV's
    BT.601 limited-range conversion."""

    __slots__ = ("format", "planes", "height", "width", "device")

    def __init__(self, format: str, planes):
        import torch
        if format not in _YUV:
            raise ValueError(f"a YUV frame's format is one of {tuple(_YUV)}, not {format!r}")
        planes = tuple(p.numpy() if isinstance(p, torch.Tensor) and not p.is_cuda else p for p in planes)
        n = len(_yuv_layout(format, 2, 2))
        if len(planes) != n:
            raise ValueError(f"a {format} frame has {n} plane(s), not {len(planes)}")
        cuda = [isinstance(p, torch.Tensor) for p in planes]
        if any(cuda) and (not all(cuda) or len({p.device for p in planes}) != 1):
            raise ValueError("a YUV frame's planes are all numpy arrays or all CUDA tensors on one device")
        for k, p in enumerate(planes):
            if not (isinstance(p, np.ndarray) or cuda[k]) or p.dtype != (torch.uint8 if cuda[k] else np.uint8) or p.ndim != 2:
                raise ValueError(f"plane {k} of a YUV frame is a 2-D uint8 array")
            if p.shape[0] < 1 or p.shape[1] < 1:
                raise ValueError("a YUV frame is empty")
            row, col = p.stride() if cuda[k] else p.strides  # bytes and elements agree for uint8
            if col != 1 or (p.shape[0] > 1 and row < p.shape[1]):
                raise ValueError(f"plane {k} of a YUV frame needs rows of contiguous bytes, stride (pitch, 1) with pitch "
                                 f">= its {p.shape[1]} bytes per row (it has {(row, col)})")
        H, W = int(planes[0].shape[0]), int(planes[0].shape[1]) // (2 if format == "yuyv" else 1)
        if W % 2 or (format != "yuyv" and H % 2):
            raise ValueError(f"a {format} frame needs an even {'width' if format == 'yuyv' else 'height and width'} "
                             f"(cv2.cvtColor refuses {H}x{W})")
        want = [shape for _, shape in _yuv_layout(format, H, W)]
        got = [tuple(int(d) for d in p.shape) for p in planes]
        if got != want:
            raise ValueError(f"the planes of a {H}x{W} {format} frame are {want}, not {got}")
        self.format, self.planes, self.height, self.width = format, planes, H, W
        self.device = planes[0].device.index if cuda[0] else None

    def to_bgr(self) -> np.ndarray:
        """``cv2.cvtColor`` of a host frame, on cv2's single-array layout (``[H*3/2, W]`` or ``[H, W, 2]``)."""
        import cv2
        if self.device is not None:
            raise ValueError("to_bgr converts a host frame: its planes are CUDA tensors")
        if self.format == "yuyv":
            src = np.ascontiguousarray(self.planes[0]).reshape(self.height, self.width, 2)
        else:
            src = np.concatenate([np.ascontiguousarray(p).reshape(-1) for p in self.planes])
            src = src.reshape(self.height * 3 // 2, self.width)
        return cv2.cvtColor(src, getattr(cv2, _YUV[self.format][0]))


@dataclasses.dataclass(frozen=True)
class TrackParams:
    """``FrameStream``'s tracking: ``streams`` tables of tracks (one per camera or video, frames name theirs with
    ``submit(..., stream=s)``), the OKS at or above which a person may continue a track, and the frames of its stream a
    track outlives unmatched (``include/spgroup.h`` "tracking" has the rules)."""
    streams: int = 1
    oks_threshold: float = 0.5
    max_age: int = 30

    def __post_init__(self):
        for name in ("streams", "max_age"):
            v = getattr(self, name)
            if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
                raise ValueError(f"TrackParams.{name} is an int, not {v!r}")
        if not 1 <= self.streams < 1 << 31:
            raise ValueError(f"TrackParams.streams must be in [1, 2^31), not {self.streams}")
        if not 0 <= self.max_age < 1 << 31:
            raise ValueError(f"TrackParams.max_age must be in [0, 2^31), not {self.max_age}")
        t = self.oks_threshold
        if isinstance(t, bool) or not isinstance(t, (int, float, np.integer, np.floating)) or not 0.0 <= float(t) <= 1.0:
            raise ValueError(f"TrackParams.oks_threshold must be a number in [0, 1], not {t!r}")


def _number(v) -> bool:
    return not isinstance(v, bool) and isinstance(v, (int, float, np.integer, np.floating)) and bool(np.isfinite(v))


@dataclasses.dataclass(frozen=True)
class SmoothParams:
    """``FrameStream``'s smoothing of tracked people's keypoints: a One-Euro filter (Casiez, Roussel and Vogel, CHI 2012)
    per track and joint.  ``min_cutoff`` (Hz) is the cut-off at rest: lower removes more jitter; ``beta`` raises the
    cut-off with the joint's filtered speed in person sizes per second: higher lags less in motion; ``d_cutoff`` (Hz)
    filters that speed; ``rate`` (frames per second) spaces the frames submitted without a time
    (``include/spgroup.h`` "smoothing" has the rules).  The defaults are a starting point, not tuned on real video."""
    min_cutoff: float = 1.0
    beta: float = 1.0
    d_cutoff: float = 1.0
    rate: float = 30.0

    def __post_init__(self):
        for name in ("min_cutoff", "d_cutoff", "rate"):
            v = getattr(self, name)
            if not _number(v) or not float(v) > 0.0:
                raise ValueError(f"SmoothParams.{name} must be a finite number above 0, not {v!r}")
        if not _number(self.beta) or not float(self.beta) >= 0.0:
            raise ValueError(f"SmoothParams.beta must be a finite number at least 0, not {self.beta!r}")


class _Key(NamedTuple):
    """A frame's part of a tick key: its size, its source -- a host or CUDA BGR image (``"image"``, ``"cuda"``), JPEG
    bytes the device decodes (``"jpeg"``), a ``YUVFrame`` with host or CUDA planes (``"yuv"``, ``"yuv_cuda"``) -- and its
    ``JPEG_FORMAT`` values or YUV layout (None for an image)."""
    height: int
    width: int
    source: str
    format: object = None


class _Frame(NamedTuple):
    """A frame ``_admit`` took: its key, what is staged (a contiguous host or a CUDA image, JPEG bytes as uint8, the
    ``YUVFrame``), its parsed JPEG record, the image cv2 decoded or converted it to at submit, if it did, and with
    smoothing its time in seconds."""
    key: _Key
    data: object
    rec: Optional[np.ndarray] = None
    decoded: Optional[np.ndarray] = None
    t: Optional[float] = None


def _admit(frames, streams, *, input_stage: str, device: int, n_streams: Optional[int], times=None, previous=None,
           step: float = 0.0):
    """A tick's frames, stream indices and times checked before anything is staged: per frame its ``_Frame``, the
    stream indices as ints, and how many frames ``cv2.imdecode`` decoded.  ``n_streams``: ``TrackParams.streams``, or
    None without tracking (only stream 0 exists).  ``times``: None or per frame its time or None; ``previous``: with
    smoothing, per stream the time of its last frame (None before its first), and None without, when every time must
    be None.  With smoothing each frame's ``t`` is its time, or its stream's previous one plus ``step`` (0.0 for the
    stream's first frame), and must be finite and later than its stream's previous time.  A JPEG file the parser
    refuses, and with ``input_stage="host"`` every JPEG or YUV frame, is staged as cv2's image of it."""
    import torch
    checked = []
    for s in streams:
        if isinstance(s, bool) or not isinstance(s, (int, np.integer)):
            raise ValueError(f"a stream index is an int, not {s!r}")
        if n_streams is None:
            if s != 0:
                raise ValueError(f"stream {s}: streams other than 0 need tracking (FrameStream(track=TrackParams(...)))")
        elif not 0 <= s < n_streams:
            raise ValueError(f"stream {s} is outside [0, {n_streams})")
        checked.append(int(s))
    times = [None] * len(checked) if times is None else list(times)
    if previous is None and any(t is not None for t in times):
        raise ValueError("a frame's time needs smoothing (FrameStream(smooth=SmoothParams(...)))")
    resolved, last = [], {}
    if previous is not None:
        for s, t in zip(checked, times):
            prev = last.get(s, previous[s])
            if t is None:
                t = 0.0 if prev is None else prev + float(step)
            elif not _number(t):
                raise ValueError(f"a frame's time is a finite number of seconds, not {t!r}")
            t = float(t)
            if prev is not None and not t > prev:
                raise ValueError(f"stream {s}: time {t!r} is not later than its previous frame's {prev!r}")
            last[s] = t
            resolved.append(t)
    out, decodes = [], 0
    for frame in frames:
        decoded = None
        yuv = isinstance(frame, YUVFrame)
        cuda = frame.device is not None if yuv else isinstance(frame, torch.Tensor) and frame.is_cuda
        if cuda and input_stage == "host":
            raise ValueError("input_stage='host' builds the network input with cv2: pass host frames")
        if yuv:
            if cuda and frame.device != device:
                raise ValueError(f"a CUDA YUV frame's planes are on cuda:{device}, not cuda:{frame.device}")
            if input_stage == "device":
                out.append(_Frame(_Key(frame.height, frame.width, "yuv_cuda" if cuda else "yuv", frame.format), frame))
                continue
            frame = decoded = frame.to_bgr()
        elif isinstance(frame, (bytes, bytearray, memoryview)):
            data = np.frombuffer(frame, np.uint8)
            if data.size == 0:
                raise ValueError("a JPEG frame's bytes are empty")
            rec = jpeg_parse(data) if input_stage == "device" else None
            if rec is not None and rec["status"] == JPEG_OK:
                fmt = tuple(int(rec[k]) for k in JPEG_FORMAT)
                out.append(_Frame(_Key(int(rec["height"]), int(rec["width"]), "jpeg", fmt), data, rec))
                continue
            frame = decoded = _imdecode(data)
            decodes += 1
        if cuda:
            if frame.dtype != torch.uint8 or frame.dim() != 3 or frame.shape[2] != 3 or frame.device.index != device:
                raise ValueError(f"a CUDA frame is a [H, W, 3] uint8 tensor on cuda:{device}")
            source = "cuda"
        else:
            frame = np.ascontiguousarray(frame.numpy() if isinstance(frame, torch.Tensor) else frame)
            if frame.dtype != np.uint8 or frame.ndim != 3 or frame.shape[2] != 3:
                raise ValueError("a frame is a [H, W, 3] uint8 BGR image")
            source = "image"
        out.append(_Frame(_Key(int(frame.shape[0]), int(frame.shape[1]), source), frame, None, decoded))
    if resolved:
        out = [f._replace(t=t) for f, t in zip(out, resolved)]
    return out, checked, decodes


def _align(n: int) -> int:
    return -(-int(n) // 256) * 256


class _Tick:
    """One slot's buffers for one tick key, and the graph captured over them.  ``keys``: per frame its ``_Key``;
    ``caps``: per frame its capacity in bytes (0 for the others); ``recs``: per frame its parsed JPEG record or None."""

    def __init__(self, fs: "FrameStream", keys: tuple, caps: list, recs: list):
        import torch
        dev = torch.device("cuda", fs.device)
        host_stage = fs.input_stage == "host"
        self.keys, self.caps, self.graph = keys, list(caps), None
        self.stream, self.model_params = fs._stream, fs.model_params
        self.held: List[int] = []  # tickets of finished frames whose maps FrameStream._held still refers to
        self.plan, self.buckets = plan_items([k[:2] for k in keys], fs.params, fs.model_params)
        md = int(fs.model_params["max_downsample"])
        # per frame, per item: the crop and reverse rotation the post-network stage takes, as spg_prenet builds the item
        self.built = [[(geo[:2], reverse) for _, geo, _, reverse in
                       (prenet_item(k.height, k.width, item[0], item[2], md) for item in items)]
                      for k, items in zip(keys, self.plan)]
        self.jpeg = [j for j, k in enumerate(keys) if k.source == "jpeg"]
        self.yuv = [j for j, k in enumerate(keys) if k.source in ("yuv", "yuv_cuda")]
        # the one upload: the JPEG frames' records, with tracking the frames' stream indices (int32), with smoothing
        # then their times (float64), then per frame its bytes: a JPEG frame's capacity, a host image (with
        # input_stage="host" the pairs cv2 built go up instead) or a host YUV frame's packed planes.  A CUDA YUV frame's
        # planes are copied into packed planes of their own.
        self.at, off = {}, _align(len(self.jpeg) * JPEG_RECORD.itemsize)
        self.streams_at = self.times_at = None
        if fs._track is not None:
            self.streams_at, off = off, _align(off + 4 * len(keys))
        if fs._smooth is not None:
            self.times_at, off = off, _align(off + 8 * len(keys))
        for j, (H, W, source, fmt) in enumerate(keys):
            size = {"jpeg": self.caps[j], "yuv": _yuv_bytes(fmt, H, W), "image": None if host_stage else H * W * 3}
            if size.get(source) is not None:
                self.at[j], off = off, _align(off + size[source])
        self.yuv_dev = {j: torch.empty(_yuv_bytes(fmt, H, W), dtype=torch.uint8, device=dev)
                        for j, (H, W, source, fmt) in enumerate(keys) if source == "yuv_cuda"}
        self.up_host = torch.empty(off, dtype=torch.uint8, pin_memory=True)
        self.up = torch.empty(off, dtype=torch.uint8, device=dev)
        self.images = None if host_stage else [
            self.up[self.at[j]:self.at[j] + H * W * 3].view(H, W, 3) if source == "image" else
            torch.empty((H, W, 3), dtype=torch.uint8, device=dev) for j, (H, W, source, _) in enumerate(keys)]
        self.status = torch.zeros(max(len(self.jpeg), 1), dtype=torch.int32, device=dev)
        self.status_host = torch.zeros(self.status.shape, dtype=torch.int32, pin_memory=True)
        self.formats = np.zeros(len(self.jpeg), JPEG_RECORD)
        for jj, j in enumerate(self.jpeg):
            self.formats[jj] = recs[j]
            self.formats[jj]["data"] = self.up.data_ptr() + self.at[j]
            self.formats[jj]["out"] = self.images[j].data_ptr()
            self.formats[jj]["decode_status"] = self.status.data_ptr() + 4 * jj
        self.yuv_members = np.zeros(len(self.yuv), YUV_MEMBER)  # every address is the slot's own
        for jj, j in enumerate(self.yuv):
            H, W, source, fmt = keys[j]
            base = self.yuv_dev[j].data_ptr() if source == "yuv_cuda" else self.up.data_ptr() + self.at[j]
            m = self.yuv_members[jj]
            m["format"], m["height"], m["width"] = _YUV[fmt][1], H, W
            for k, (o, (_, w)) in enumerate(_yuv_layout(fmt, H, W)):
                m["planes"][k], m["pitches"][k] = base + o, w
            m["out"], m["out_pitch"] = self.images[j].data_ptr(), 3 * W
        self.inputs = {size: torch.empty((2 * len(members),) + size + (3,), dtype=torch.float32, device=dev)
                       for size, members in self.buckets.items()}
        self.pairs = {size: torch.empty(x.shape, dtype=torch.float32, pin_memory=True)
                      for size, x in self.inputs.items()} if host_stage else None
        self.n_items = len(self.plan[0])
        self.as_f64 = self.n_items == 1  # as predict() returns
        self.heat = [torch.empty((1, NUM_PARTS, H, W), dtype=torch.float32, device=dev) for H, W, _, _ in keys]
        self.paf = [torch.empty((1, len(fs.limbs), H, W), dtype=torch.float32 if self.as_f64 else torch.float64, device=dev)
                    for H, W, _, _ in keys]
        self.rec = torch.zeros((len(keys), fs._g.wire_record_bytes()), dtype=torch.uint8, device=dev)
        self.rec_host = torch.empty(self.rec.shape, dtype=torch.uint8, pin_memory=True)
        self.track = None
        if fs._track is not None:  # per frame its people's ids, and its spg_track_frames member
            self.ids = torch.empty((len(keys), fs._g.capR), dtype=torch.int64, device=dev)
            self.ids_host = torch.empty(self.ids.shape, dtype=torch.int64, pin_memory=True)
            self.track = np.zeros(len(keys), TRACK_FRAME)
            for j in range(len(keys)):
                self.track[j]["record"] = self.rec[j].data_ptr()
                self.track[j]["stream"] = self.up.data_ptr() + self.streams_at + 4 * j
                self.track[j]["jpeg_status"] = self.status.data_ptr() + 4 * self.jpeg.index(j) if j in self.jpeg else 0
                self.track[j]["ids"] = self.ids[j].data_ptr()
        self.smooth = None
        if fs._smooth is not None:  # per frame its people's smoothed joints, and its spg_smooth_frames member
            self.xy = torch.empty((len(keys), fs._g.capR, 17, 2), dtype=torch.float64, device=dev)
            self.xy_host = torch.empty(self.xy.shape, dtype=torch.float64, pin_memory=True)
            self.smooth = np.zeros(len(keys), SMOOTH_FRAME)
            for j in range(len(keys)):
                self.smooth[j]["record"] = self.rec[j].data_ptr()
                self.smooth[j]["stream"] = self.up.data_ptr() + self.streams_at + 4 * j
                self.smooth[j]["ids"] = self.ids[j].data_ptr()
                self.smooth[j]["time"] = self.up.data_ptr() + self.times_at + 8 * j
                self.smooth[j]["xy"] = self.xy[j].data_ptr()

    def stage(self, frames: List[_Frame], streams: List[int]) -> None:
        """Write a tick's frames into this slot's buffers: the upload's host side (with tracking the stream indices, -1
        skipping a frame, with smoothing the times), CUDA images and planes copied on the stream ahead of the graph, and
        with input_stage="host" each item's pair built by cv2 into the pinned copy of its input."""
        import torch
        host, copies = self.up_host.numpy(), []  # copies: (slot's device buffer, caller's CUDA tensor)
        if self.track is not None:
            host[self.streams_at:self.streams_at + 4 * len(frames)] = np.asarray(streams, np.int32).view(np.uint8)
        if self.smooth is not None:  # a re-posed frame (stream -1) has no time: it is skipped
            times = np.asarray([0.0 if f.t is None else f.t for f in frames], np.float64)
            host[self.times_at:self.times_at + 8 * len(frames)] = times.view(np.uint8)
        for j, (key, data, rec, _, _) in enumerate(frames):
            at = self.at.get(j)
            if key.source == "jpeg":
                jj = self.jpeg.index(j)
                host[at:at + data.size] = data
                for k in ("data", "out", "decode_status"):  # the tick's device addresses, as the format's
                    rec[k] = self.formats[jj][k]
                host[jj * JPEG_RECORD.itemsize:(jj + 1) * JPEG_RECORD.itemsize] = np.frombuffer(rec.tobytes(), np.uint8)
            elif key.source in ("yuv", "yuv_cuda"):
                for p, (o, (h, w)) in zip(data.planes, _yuv_layout(key.format, key.height, key.width)):
                    if key.source == "yuv":
                        host[at + o:at + o + h * w].reshape(h, w)[:] = p
                    else:
                        copies.append((self.yuv_dev[j][o:o + h * w].view(h, w), p))
            elif key.source == "cuda":
                copies.append((self.images[j], data))
            elif self.pairs is None:
                host[at:at + data.size] = data.reshape(-1)
        if copies:
            self.stream.wait_stream(torch.cuda.current_stream(self.stream.device))
            with torch.cuda.stream(self.stream):
                for dst, src in copies:
                    dst.copy_(src, non_blocking=True)
            for _, src in copies:
                src.record_stream(self.stream)
        if self.pairs is not None:
            for size, ms in self.buckets.items():
                _host_pairs([f.data for f in frames], self.plan, ms, self.model_params, self.pairs[size])


class FrameStream:
    """Frames posed at the GPU's rate: ``predict`` + ``group`` per frame, replayed from a CUDA graph per tick of frames.

    ``submit(frame)`` takes a ``[H, W, 3]`` uint8 BGR frame (numpy, or a CUDA tensor on the stream's device), a JPEG
    file's bytes or a ``YUVFrame`` and returns a ticket; ``submit_many(frames)`` takes a tick of several and returns
    one ticket each.  ``result(ticket)`` returns ``process()``'s value for that frame (evaluate.py:523-543), the
    ``[([17 x (x, y)], score)]`` of ``predict_many``: equal, value for value and type for type, to ``keypoints`` of
    ``group`` on the maps ``predict`` gives for the frame.  ``submit`` poses a tick of one frame and ``submit_many`` a
    tick of several, through the same calls.

    A tick holds one slot.  The slot keeps one CUDA graph per **tick key**: each frame's shape and source (host image,
    CUDA image, JPEG bytes of one format, or YUV planes of one layout on the host or on the device) in order.  The
    key's first tick in a slot runs call by call -- it is the key's warm-up (the network's lazy set-up, cuDNN's
    choices) -- and the slot then captures the graph over its buffers for that key; every later tick of that key in
    that slot is one graph launch.  The graph
    holds one upload from the slot's pinned buffer of the tick's host frames, host YUV planes, JPEG bytes and parsed
    records; ``spg_jpeg_decode_frames`` for every JPEG frame; one ``spg_yuv_to_bgr`` for every YUV frame;
    ``spg_prenet_ragged`` for every item of ``scale_search x rotation_search`` of every frame, into one input tensor per
    network input size (``input_stage="host"``: the upload of the pairs cv2 built on the host instead); the forward
    passes; ``spg_postnet_ragged_items``; ``spg_group_ragged`` writing each frame's wire record; and one copy of the
    records and JPEG statuses into pinned host memory.  A CUDA frame is copied into the slot's device image, and a CUDA
    YUV frame's planes into the slot's packed planes, ahead of the graph, so a graph never holds a caller's address.
    The graphs share one memory pool: they replay one at a time on the stream's own CUDA stream, and nothing allocated
    inside a capture outlives it.

    A tick of one frame forwards each item alone, as ``predict`` does, so ``submit`` equals ``predict`` + ``group``
    with any network.  A larger tick forwards each input size's items at once: every kernel treats each frame on its
    own, so with a network whose output for a sample does not depend on its batch each ticket equals ``submit``'s
    result for the frame; cuDNN may pick other algorithms for a larger batch, and the maps can then differ in the last
    bits.

    JPEG bytes (``bytes``, ``bytearray`` or ``memoryview``) are parsed on the host with ``spg_jpeg_parse``.  A file the
    device decoder takes (baseline or extended-sequential Huffman, grey or YCbCr 4:4:4 / 4:2:2 / 4:4:0 / 4:2:0) is
    decoded inside the graph, bit-identical to ``cv2.imdecode``; its key holds its format -- frame height and width,
    component count, luma sampling, restart interval and EXIF orientation -- and the scan's offset and length, the
    tables and the segments in front of the scan are read on the device from the frame's record, so they may change
    from frame to frame.  A slot reserves a capacity in bytes per JPEG frame of a key (the next power of two of the
    file's size, at least 64 KiB); a longer file grows it, which captures that key again.  A file the parser refuses
    (progressive, arithmetic-coded, other samplings and so on) is decoded with ``cv2.imdecode`` at submit and posed as
    a decoded frame; one the device decoder flags (corrupt data, or blocks outside the range where libjpeg-turbo's
    IDCTs agree) is decoded with cv2 from the slot's bytes when its result is read and posed again as a one-frame tick
    in the same slot, so a JPEG frame's result is always the one for ``cv2.imdecode(bytes, IMREAD_COLOR)``.
    ``host_decodes`` counts the JPEG frames ``cv2.imdecode`` decoded; with ``input_stage="host"`` that is every JPEG
    frame, decoded at submit.  Bytes cv2 cannot decode either raise ``ValueError``.

    A ``YUVFrame`` (NV12, I420 or YUYV planes, numpy or CUDA, rows possibly pitched) is converted inside the graph into
    the slot's device image, bit-identical to ``cv2.cvtColor(frame, COLOR_YUV2BGR_*)``: a host frame goes up packed at
    1.5 (NV12, I420) or 2 (YUYV) bytes per pixel.  With ``input_stage="host"`` a host YUV frame is converted with
    ``cv2.cvtColor`` at submit and posed as an image.  Either way its result is the one for cv2's image.

    ``slots`` ticks are in flight at most; each call to ``submit`` or ``submit_many`` takes the next slot in turn.  A
    slot owns its inputs, maps and records until its tick is finished, so the host stages tick k+1 while tick k's graph
    runs; a call to a slot whose tick is unread finishes that tick and keeps its results for ``result``.  A record with
    a capacity bit in its status (a crowded frame) is regrouped on the capacity-free tier from the frame's maps, as
    ``group`` does; any other status bit raises ``GroupingError`` from ``result``.  The variant
    (``configure(variant=...)``), the limb table and the default device are those in effect at construction.  The
    network's output is ``model(x)[-1][0]``, as for ``predict``; the model must be capture-safe after its first call at
    a shape (no host synchronisation, no host-to-device copy).  A stride other than 4 raises ``ValueError``, a capture
    that fails raises ``GroupingError``: there is no call-by-call fallback.

    ``track=TrackParams(...)`` follows people across frames: each frame belongs to a stream (``submit(frame,
    stream=s)``, ``submit_many(frames, streams=[...])``; stream 0 by default), and ``spg_track_frames``, recorded into
    the graph after the grouping, matches the frame's people to its stream's tracks by OKS and gives each an id
    (``result(ticket, ids=True)``).  Every graph replays on the stream's one CUDA stream in submit order, so a stream's
    frames are tracked in submit order, also across slots in flight; the stream indices travel in the tick's upload, so
    frames of any streams share a graph.  A frame whose record has a status bit (a crowded frame, whose people come from
    the capacity-free tier, or a grouping error) or whose JPEG decode was flagged is unobserved: its stream's tracks age
    and its people get id -1, also after the flagged frame is posed again.

    ``smooth=SmoothParams(...)`` (with ``track``) filters each tracked person's joints across its stream's frames: a
    One-Euro filter per track id and joint, ``spg_smooth_frames``, recorded into the graph after the tracking, with its
    state in one table per stream on the device.  Each frame has a time in seconds (``submit(frame, t=...)``,
    ``submit_many(frames, times=[...])``): a frame without one comes ``1 / rate`` after its stream's previous frame (its
    stream's first at 0.0), and a time that is not finite or not later than its stream's previous one is refused
    before anything is staged.  ``result(ticket, smoothed=True)`` gives each present joint of a tracked person its
    filtered position (float64).  People with id -1 (an unobserved frame, a crowded frame's, a flagged JPEG frame posed
    again) keep their raw joints; ``FrameResult.record`` and the maps stay raw."""

    _track: Optional[TrackParams] = None  # the tracking parameters, or None
    _smooth: Optional[SmoothParams] = None  # the smoothing parameters, or None

    def __init__(self, model, params, model_params, *, slots: int = 2, input_stage: str = "device",
                 device: Optional[int] = None, track: Optional[TrackParams] = None,
                 smooth: Optional[SmoothParams] = None):
        if int(model_params["stride"]) != 4:
            raise ValueError(f"FrameStream needs stride 4 (model_params['stride'] is {model_params['stride']}): the "
                             "ragged and rotated post-network kernels it records are stride-4 kernels")
        if int(slots) < 1:
            raise ValueError("slots must be >= 1")
        if track is not None and not isinstance(track, TrackParams):
            raise ValueError(f"track is a TrackParams or None, not {track!r}")
        if smooth is not None and not isinstance(smooth, SmoothParams):
            raise ValueError(f"smooth is a SmoothParams or None, not {smooth!r}")
        if smooth is not None and track is None:
            raise ValueError("smoothing follows tracked people: FrameStream(smooth=...) needs track=TrackParams(...)")
        import torch
        self.model, self.params, self.model_params = model, dict(params), dict(model_params)
        self.input_stage = _stage(input_stage)
        self.device = _device if device is None else int(device)
        self.limbs = _limbs
        self._gp = _group_params(params)
        self._nan_scrub = _variant == "demo"
        self._g = _new_grouper(1, self.device)     # the graphs' handle; its max_batch grows to the largest tick
        self._tier = _new_grouper(1, self.device)  # the capacity-free tier's, used while later graphs run
        self._stream = torch.cuda.Stream(device=self.device)
        self._tier_stream = torch.cuda.Stream(device=self.device)
        self._pool = None
        self._ticks: List[Dict[tuple, _Tick]] = [{} for _ in range(int(slots))]  # per slot, its _Tick per tick key
        self._busy: List[Optional[tuple]] = [None] * int(slots)  # per slot (tickets, _Tick, done event, _Frames)
        self._done: Dict[int, object] = {}  # finished tickets: (people, record) or the exception to raise
        self._held: Dict[int, tuple] = {}  # finished tickets' maps, while their tick's buffers hold them
        self._next = 0  # the next ticket
        self._calls = 0  # ticks launched: the next one takes slot _calls % slots
        self.captures = 0  # graphs captured so far (a tick key's first sight in a slot, or after a buffer moved)
        self.host_decodes = 0  # JPEG frames decoded with cv2.imdecode
        self._track = track
        if track is not None:  # every stream's table of tracks, empty
            self._tables = torch.zeros((track.streams, TRACK_TABLE.itemsize), dtype=torch.uint8, device=self.device)
        self._smooth = smooth
        if smooth is not None:  # every stream's filter slots, empty, and the time of its last frame
            self._smooth_tables = torch.zeros((track.streams, SMOOTH_TABLE.itemsize), dtype=torch.uint8,
                                              device=self.device)
            self._times: List[Optional[float]] = [None] * track.streams
            self._smoothed: Dict[int, list] = {}  # finished tickets' smoothed people

    def close(self) -> None:
        for ticks in self._ticks:
            ticks.clear()
        self._held.clear()
        self._g.close()
        self._tier.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def submit(self, frame, *, stream: int = 0, t: Optional[float] = None) -> int:
        """Pose ``frame`` as a tick of one frame in the next slot and return its ticket.  ``frame`` is a ``[H, W, 3]``
        uint8 BGR image (numpy, or a CUDA tensor on the stream's device), a JPEG file's bytes or a ``YUVFrame``.
        ``submit(f)`` and ``submit_many([f])`` form the same tick key, so in one slot they share one graph.  ``stream``:
        the frame's stream with tracking (``TrackParams.streams``); without, only 0.  ``t``: with smoothing, the frame's
        time in seconds, or None for its stream's previous time plus ``1 / SmoothParams.rate``; without, None."""
        return self._submit([frame], [stream], [t])[0]

    def submit_many(self, frames, *, streams=None, times=None) -> List[int]:
        """Pose a tick of ``K >= 1`` frames -- one frame per camera, or the next K frames of a video -- through one
        CUDA graph in the next slot, and return one ticket per frame, each read with ``result``.

        ``frames`` may mix every kind ``submit`` takes and every shape; it needs ``input_stage="device"``.  A frame
        ``submit`` would refuse refuses the whole tick before anything is staged; if the launch or its capture raises,
        no ticket is issued.  ``streams``: with tracking, None (every frame is stream 0's: the next K frames of one
        video) or one stream per frame (one per camera, say); without, None.  ``times``: with smoothing, None or one
        time (or None) per frame, as ``submit``'s ``t``; without, None."""
        if self.input_stage != "device":
            raise ValueError("submit_many needs input_stage='device': the tick's network inputs are built by "
                             "spg_prenet_ragged")
        frames = list(frames)
        streams = [0] * len(frames) if streams is None else list(streams)
        if len(streams) != len(frames):
            raise ValueError(f"{len(frames)} frames but {len(streams)} streams")
        times = [None] * len(frames) if times is None else list(times)
        if len(times) != len(frames):
            raise ValueError(f"{len(frames)} frames but {len(times)} times")
        if not frames:
            raise ValueError("submit_many needs at least one frame")
        return self._submit(frames, streams, times)

    def _submit(self, frames: list, streams: list, times: list) -> List[int]:
        """Admit a tick's frames, stream indices and times (``_admit``), launch it in the next slot and return its
        tickets."""
        sm = self._smooth
        frames, streams, decodes = _admit(frames, streams, input_stage=self.input_stage, device=self.device,
                                          n_streams=None if self._track is None else self._track.streams, times=times,
                                          previous=None if sm is None else self._times,
                                          step=0.0 if sm is None else 1.0 / float(sm.rate))
        self.host_decodes += decodes
        slot = self._calls % len(self._busy)
        if self._busy[slot] is not None:
            self._finish(slot)
        tk, done = self._launch(slot, frames, streams)
        tickets = list(range(self._next, self._next + len(frames)))  # issued once the tick runs
        self._next += len(frames)
        self._calls += 1
        self._busy[slot] = (tickets, tk, done, frames)
        if sm is not None:
            for f, s in zip(frames, streams):
                self._times[s] = f.t
        return tickets

    def _launch(self, slot: int, frames: List[_Frame], streams: List[int]):
        """Stage a tick's frames and stream indices (``_Tick.stage``) in the slot's ``_Tick`` for their keys (made on the
        key's first sight, made again when a JPEG frame outgrows its capacity) and run its graph, or reserve its
        scratch, run its calls and capture them; returns the ``_Tick`` and the event of the launch's end."""
        import torch
        keys = tuple(f.key for f in frames)
        if self._g.max_batch < len(keys):
            self._stream.synchronize()  # the old handle's scratch may be in use
            self._g.close()
            self._g = _new_grouper(len(keys), self.device)
            self._invalidate()
        tk = self._ticks[slot].get(keys)
        sizes = [f.data.size if f.key.source == "jpeg" else 0 for f in frames]
        if tk is None or any(s > c for s, c in zip(sizes, tk.caps)):
            caps = [max(1 << 16, 1 << (s - 1).bit_length()) if s else 0 for s in sizes]
            if tk is not None:
                caps = [max(a, b) for a, b in zip(caps, tk.caps)]
                self._drop_held(tk)
            tk = self._ticks[slot][keys] = _Tick(self, keys, caps, [f.rec for f in frames])
        if tk.graph is None:
            # Before every call-by-call run, not only on a key's first sight: a key whose graph was dropped (a buffer
            # moved, or the handle was replaced for a larger tick) would otherwise grow a buffer in its eager run and
            # free the address that graphs captured since then replay.
            members = [(k.height, k.width, item[0], item[2]) for k, items in zip(tk.keys, tk.plan) for item in items]
            moved = self._g.reserve_frames(members, tk.n_items, max_downsample=int(self.model_params["max_downsample"]))
            if tk.jpeg and self._g.jpeg_reserve_frames(tk.formats, [tk.caps[j] for j in tk.jpeg]):
                moved = True
            if moved:
                self._invalidate()
        self._drop_held(tk)  # the maps of the key's earlier tick are overwritten
        tk.stage(frames, streams)
        eager = tk.graph is None
        with torch.cuda.stream(self._stream):
            if eager:
                self._path(tk)
            else:
                tk.graph.replay()
            done = torch.cuda.Event()
            done.record(self._stream)
        if eager:
            self._capture(tk)
        return tk, done

    def _path(self, tk: _Tick) -> None:
        """One tick's work on the current stream: run as it is for the warm-up, recorded by ``_capture``."""
        g = self._g
        md, pv = int(self.model_params["max_downsample"]), int(self.model_params["padValue"])
        if tk.pairs is None or tk.track is not None:
            tk.up.copy_(tk.up_host, non_blocking=True)
        if tk.pairs is None:
            if tk.jpeg:
                g.jpeg_decode_frames(tk.up.data_ptr(), tk.formats, [tk.caps[j] for j in tk.jpeg])
                tk.status_host.copy_(tk.status, non_blocking=True)
            if tk.yuv:
                g.yuv_to_bgr(tk.yuv_members)
            members, outs = [], []
            for size, ms in tk.buckets.items():
                for k, (i, t) in enumerate(ms):
                    members.append((tk.images[i], tk.plan[i][t][0], tk.plan[i][t][2]))
                    outs.append(tk.inputs[size][2 * k:2 * k + 2])
            g.prenet_ragged(members, max_downsample=md, pad_value=pv, out=outs)
        else:
            for size, x in tk.inputs.items():
                x.copy_(tk.pairs[size], non_blocking=True)
        # A tick of one frame forwards each item alone, as predict does, so that submit equals predict + group with any
        # network; a larger tick forwards each input size's items at once.
        entries = [[None] * tk.n_items for _ in tk.keys]
        for size, ms in tk.buckets.items():
            _forward_bucket(self.model, tk.inputs[size], ms, [tk.built[i][t] for i, t in ms],
                            1 if len(tk.keys) == 1 else len(ms), entries)
        maps = list(zip(tk.heat, tk.paf))
        g.postnet_ragged_items([(e, k[:2]) for e, k in zip(entries, tk.keys)], outs=maps, nan_scrub=self._nan_scrub)
        g.set_wire_output(tk.rec.data_ptr())
        try:
            g.group_ragged(maps, [k.height for k in tk.keys], self._gp, paf_as_f64=tk.as_f64)
        finally:
            g.set_wire_output(None)
        if tk.track is not None:
            t = self._track
            g.track_frames(tk.track, self._tables.data_ptr(), t.streams, t.oks_threshold, t.max_age)
            tk.ids_host.copy_(tk.ids, non_blocking=True)
        if tk.smooth is not None:
            sm = self._smooth
            g.smooth_frames(tk.smooth, self._smooth_tables.data_ptr(), self._track.streams, sm.min_cutoff, sm.beta,
                            sm.d_cutoff)
            tk.xy_host.copy_(tk.xy, non_blocking=True)
        tk.rec_host.copy_(tk.rec, non_blocking=True)

    def _capture(self, tk: _Tick) -> None:
        """Capture ``_path(tk)`` into ``tk.graph``."""
        import torch
        graph = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(graph, pool=self._pool, stream=self._stream):
                self._path(tk)
        except Exception as e:
            raise GroupingError(f"capturing the path of a tick of {len(tk.keys)} frame(s) failed (a model that "
                                "synchronises with the host or copies from it in its forward cannot be captured): "
                                f"{type(e).__name__}: {e}") from e
        if self._pool is None:
            self._pool = graph.pool()
        tk.graph = graph
        self.captures += 1

    def _finish(self, slot: int) -> None:
        """Wait for the slot's tick and keep every frame's result (or the error it raises) under its ticket, with its
        maps for ``result(detail=True)``; frees the slot.  A JPEG frame the device decoder flagged is decoded with cv2
        from the slot's bytes and posed again as a one-frame tick in the same slot."""
        tickets, tk, done, frames = self._busy[slot]
        self._busy[slot] = None
        done.synchronize()
        records = tk.rec_host.numpy().copy()
        ids = tk.ids_host.numpy().copy() if tk.track is not None else None
        xy = tk.xy_host.numpy().copy() if self._smooth is not None else None
        for j, ticket in enumerate(tickets):
            record, heat, paf, image = records[j], tk.heat[j], tk.paf[j], frames[j].decoded
            frame_ids = None if ids is None else ids[j]
            frame_xy = None if xy is None else xy[j]
            if j in tk.jpeg and int(tk.status_host[tk.jpeg.index(j)]) != JPEG_OK:
                image = _imdecode(tk.up_host[tk.at[j]:tk.at[j] + frames[j].data.size].numpy())
                self.host_decodes += 1
                frame = _Frame(_Key(image.shape[0], image.shape[1], "image"), image, None, image)
                # the tick tracked the frame as unobserved: posing it again tracks and smooths nothing, and its people
                # get -1 and keep their raw joints
                again, d = self._launch(slot, [frame], [-1])
                d.synchronize()
                record, heat, paf = again.rec_host[0].numpy().copy(), again.heat[0].clone(), again.paf[0].clone()
                frame_ids = frame_xy = None
            elif j in tk.jpeg or j in tk.yuv:
                image = tk.images[j]  # decoded or converted on the device: copied to the host if detail asks for it
            self._keep(ticket, record, heat, paf, tk.keys[j].height, tk.as_f64, frame_ids, frame_xy)
            self._held[ticket] = (heat, paf, tk.as_f64, image)
            tk.held.append(ticket)

    def _drop_held(self, tk: _Tick) -> None:
        """Forget the maps of ``tk``'s finished frames whose result is unread: its buffers are about to be overwritten
        or dropped.  Their people stay readable; ``detail=True`` then raises."""
        for ticket in tk.held:
            self._held.pop(ticket, None)
        tk.held.clear()

    def _invalidate(self) -> None:
        """A scratch buffer of the graphs' handle moved, or the handle was replaced: every graph recorded it."""
        for ticks in self._ticks:
            for tk in ticks.values():
                tk.graph = None

    def result(self, ticket: int, *, detail: bool = False, ids: bool = False, smoothed: bool = False):
        """``process()``'s value for the frame of ``ticket`` (waits for it); each ticket is read once.  ``detail=True``
        returns a ``FrameResult`` with the frame's wire record and copies of its maps, which needs the frame's buffers
        to still hold them: read it before ``slots`` later calls to ``submit`` or ``submit_many``.  ``ids=True`` (with
        tracking) returns ``(value, ids)``: per person its track's id within the frame's stream, -1 for the people of an
        unobserved frame.  ``smoothed=True`` (with smoothing) gives each present joint of a tracked person its filtered
        position as float64; ``FrameResult.record`` and the maps stay raw."""
        if ids and self._track is None:
            raise ValueError("ids=True needs tracking (FrameStream(track=TrackParams(...)))")
        if smoothed and self._smooth is None:
            raise ValueError("smoothed=True needs smoothing (FrameStream(smooth=SmoothParams(...)))")
        for slot, busy in enumerate(self._busy):
            if busy is not None and ticket in busy[0]:
                self._finish(slot)
                break
        if ticket not in self._done:
            raise ValueError(f"ticket {ticket} is not a submitted frame whose result is unread")
        held = self._held.pop(ticket, None)
        if detail and held is None:
            raise ValueError(f"ticket {ticket}: its slot holds a later frame; read detail=True before {len(self._busy)} "
                             "later submits")
        out = self._done.pop(ticket)
        filtered = self._smoothed.pop(ticket, None) if self._smooth is not None else None
        if isinstance(out, Exception):
            raise out
        people, record, person_ids = out
        if smoothed:
            people = filtered
        value = people
        if detail:
            heat, paf, as_f64, image = held
            if image is not None and not isinstance(image, np.ndarray):
                image = image.cpu().numpy()
            value = FrameResult(people, record, DeviceMaps(heat.clone(), False), DeviceMaps(paf.clone(), as_f64), image)
        return (value, person_ids) if ids else value

    def _keep(self, ticket: int, record: np.ndarray, heat, paf, H: int, as_f64: bool, ids=None, xy=None) -> None:
        """Keep the people of one frame's wire record (or the error they raise) under its ticket, with their ids: with
        tracking, ``ids`` the frame's ids output, or None for -1 each; and with smoothing their smoothed joints from
        ``xy``, the frame's smoothed output, or None for the raw joints.  A record with a capacity bit is regrouped on
        the capacity-free tier from the frame's maps."""
        rec = wire.as_records(record, self._g.J, self._g.capR)[0]
        try:
            people = _people_of_record(rec, lambda: self._tier.group_unbounded(heat, paf, H, self._gp, paf_as_f64=as_f64,
                                                                              stream=self._tier_stream))
            person_ids = None
            if self._track is not None:
                person_ids = [-1] * len(people) if ids is None or rec["status"] else [int(v) for v in ids[:len(people)]]
            if self._smooth is not None:
                self._smoothed[ticket] = people if xy is None or rec["status"] else _smoothed_people(people, rec, xy)
            self._done[ticket] = (people, record, person_ids)
        except GroupingError as e:
            self._done[ticket] = e


def _smoothed_people(people: list, rec, xy: np.ndarray) -> list:
    """``process()``-style people of a wire record with each present joint's ``(x, y)`` taken from ``xy`` (the frame's
    ``spg_smooth_frames`` output, ``[rows][17][2]``) as float64; absent joints stay as they are."""
    out = []
    for p, (pts, score) in enumerate(people):
        present = int(rec["rows"][p]["present"])
        out.append(([(np.float64(xy[p, g, 0]), np.float64(xy[p, g, 1])) if (present >> g) & 1 else pt
                     for g, pt in enumerate(pts)], score))
    return out


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
    return [_people_of_record(rec, functools.partial(regroup, i))
            for i, rec in enumerate(wire.as_records(buf[:n].cpu().numpy(), g.J, g.capR))]


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
    order.  ``at`` (a list) is kept holding the ids of the image or grouping batch being worked on, for error reports.
    With ``configure(decode="device")`` each group of ``batch`` files is read with one ``imread_many`` call."""
    import os

    import cv2
    at = [] if at is None else at
    named_ids = list(named_ids)
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

    for g0 in range(0, len(named_ids), batch):
        group = named_ids[g0:g0 + batch]
        paths = [os.path.join(images_directory, name) for _, name in group]
        decoded = None
        if _decode == "device":
            at[:] = [iid for iid, _ in group]
            decoded = imread_many(paths)[0]
        for k, (image_id, _) in enumerate(group):
            at[:] = [image_id]
            ori = decoded[k] if decoded is not None else cv2.imread(paths[k])  # B,G,R order (evaluate.py:502)
            if fb > 1:
                pending.append((image_id, ori, int(ori.shape[0])))
            else:
                pending.append((image_id, predict(ori, dict(params), model, dict(model_params), heat_layers + 2, paf_layers,
                                                  paths[k]), int(ori.shape[0])))
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
            forward_batch: int = 1, device_decode: bool = False) -> None:
    """Rebind ``find_peaks / find_connections / find_people`` of an imported reference ``evaluate`` module.

    ``limbSeq`` is taken from the module (evaluate.py:54) so alternative skeletons keep working.  With
    ``device_predict`` the module's ``predict`` (:83-166) is replaced as well: the network of the module (the global
    ``posenet`` the reference's own predict uses, :124) feeds the device post-network stage and the maps stay on the GPU.
    ``device_input`` (with ``device_predict``) also builds the network's input on the GPU (``input_stage="device"``).
    ``batch > 1`` (with ``device_predict``) also replaces ``predict_many`` (:550-560) by ``predict_many`` above, which
    groups ``batch`` images per call; it uses the module's ``posenet`` and ``get_image_name`` and leaves the module's
    ``batch_time`` meter alone.  ``forward_batch > 1`` (with ``device_predict`` and ``batch > 1``) makes that
    ``predict_many`` run the network on up to ``forward_batch`` items (images, or with a multi-scale or rotation search
    their scaled and rotated copies) of the same input size at once (``predict_batch``).  ``device_decode`` (with
    ``device_input`` and ``batch > 1``) makes that ``predict_many`` decode each group of ``batch`` JPEG files on the GPU
    (``imread_many``) instead of ``cv2.imread`` per file.  In an initialised
    ``torch.distributed`` world of N > 1 processes, one per GPU, each with ``configure(device=local_rank)``, that
    ``predict_many`` shards the images over the ranks: rank 0 calls it (``evaluate.validation()``), the other ranks
    run ``serve_predict_many`` until rank 0 calls ``end_serving``."""
    if int(batch) > 1 and not device_predict:
        raise ValueError("batch > 1 needs device_predict=True: the batched grouping takes the maps predict() leaves on the device")
    fb = _forward_batch(forward_batch)
    if fb > 1 and (not device_predict or int(batch) < 2):
        raise ValueError("forward_batch > 1 needs device_predict=True and batch > 1: it batches predict_many's forward passes")
    if device_decode and (not (device_predict and device_input) or int(batch) < 2):
        raise ValueError("device_decode needs device_predict=True, device_input=True and batch > 1: it replaces the "
                         "cv2.imread of predict_many, whose images feed the device input stage")
    configure(limbs=getattr(evaluate_module, "limbSeq", _limbs), input_stage="device" if device_input else "host",
              decode="device" if device_decode else "host")
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
