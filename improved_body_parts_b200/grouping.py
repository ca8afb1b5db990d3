"""ctypes binding of ``libspgroup.so`` (include/spgroup.h) -- the H100 grouping path.

This module is the host-side mirror of the reference's grouping interface: ``Grouper`` owns one native
handle (one per GPU / stream) and exposes the whole path (``group_device`` / ``group_host``) and the four
stages.  There is no CPU implementation behind it: if the CUDA library is missing or no sm_90 device is
present, construction raises.  PyTorch is used only as plumbing (device memory, streams, NCCL).
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import os
from typing import Optional, Sequence, Tuple

import numpy as np

from . import wire
from .skeleton import COCO_FROM_PART, LIMBS, NUM_PARTS, GroupParams

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libspgroup.so")
ABI_VERSION = 2

ST_PEAK_OVERFLOW, ST_CAND_OVERFLOW, ST_ROW_OVERFLOW, ST_SAMPLE_INDEX, ST_ASSERT, ST_WIRE_OVERFLOW = 1, 2, 4, 8, 16, 32
ST_NONFINITE, ST_NAN_PRIORITY = 64, 128
#: what the reference does where a status bit is set (the bits of the conditions it would raise for, and the one whose
#: outputs it computes in an order that is not reproduced)
ST_MEANING = {ST_SAMPLE_INDEX: "SAMPLE_INDEX: a line sample index outside the map (the reference raises IndexError, "
                               "evaluate.py:235)",
              ST_ASSERT: "ASSERT: a keypoint shared by two persons (the reference raises at evaluate.py:437-439)",
              ST_NONFINITE: "NONFINITE: a limb pair with a non-finite length (the reference raises ValueError, "
                            "evaluate.py:226)",
              ST_NAN_PRIORITY: "NAN_PRIORITY: a NaN candidate priority among others (the reference's sort order at "
                               "evaluate.py:259 is undefined)"}
F32, F64, F32_AS_F64, F16, BF16 = 0, 1, 2, 3, 4


class GroupingError(RuntimeError):
    pass


class _Config(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("device", C.c_int32), ("n_parts", C.c_int32), ("n_limbs", C.c_int32),
                ("limbs", C.POINTER(C.c_int32)), ("n_out_joints", C.c_int32), ("out_from_part", C.POINTER(C.c_int32)),
                ("max_batch", C.c_int32), ("max_h", C.c_int32), ("max_w", C.c_int32),
                ("max_peaks_per_part", C.c_int32), ("max_cands_per_limb", C.c_int32), ("max_person_rows", C.c_int32)]


class _Params(C.Structure):
    _fields_ = [("thre1", C.c_double), ("thre2", C.c_double), ("connect_ration", C.c_double),
                ("len_rate", C.c_double), ("connection_tole", C.c_double), ("min_mean_score", C.c_double),
                ("mid_num", C.c_int32), ("offset_radius", C.c_int32), ("remove_recon", C.c_int32),
                ("min_parts", C.c_int32), ("crit1_strict", C.c_int32), ("refresh_len_check", C.c_int32)]


class _PostnetScale(C.Structure):
    _fields_ = [("net_out", C.c_void_p), ("dtype", C.c_int32), ("image_stride", C.c_int64), ("pair_stride", C.c_int64),
                ("chan_stride", C.c_int64), ("h", C.c_int32), ("w", C.c_int32), ("crop_h", C.c_int32), ("crop_w", C.c_int32)]


class _PostnetDesc(C.Structure):
    _fields_ = [("n_scales", C.c_int32), ("scales", C.POINTER(_PostnetScale)), ("stride", C.c_int32),
                ("paf_chan0", C.c_int32), ("heat_chan0", C.c_int32), ("flip_paf_ord", C.POINTER(C.c_int32)),
                ("flip_heat_ord", C.POINTER(C.c_int32)), ("nan_scrub", C.c_int32)]


class _PostnetRotation(C.Structure):
    _fields_ = [("apply", C.c_int32), ("reserved", C.c_int32), ("matrix", C.c_double * 6)]


class _PostnetCommon(C.Structure):
    _fields_ = [("stride", C.c_int32), ("paf_chan0", C.c_int32), ("heat_chan0", C.c_int32),
                ("flip_paf_ord", C.POINTER(C.c_int32)), ("flip_heat_ord", C.POINTER(C.c_int32)), ("nan_scrub", C.c_int32),
                ("net_dtype", C.c_int32)]


class _PostnetImage(C.Structure):
    _fields_ = [("net_out", C.c_void_p), ("pair_stride", C.c_int64), ("chan_stride", C.c_int64), ("h", C.c_int32),
                ("w", C.c_int32), ("crop_h", C.c_int32), ("crop_w", C.c_int32), ("height", C.c_int32), ("width", C.c_int32),
                ("heat_out", C.c_void_p), ("paf_out", C.c_void_p)]


class _PrenetItem(C.Structure):
    _fields_ = [("scale", C.c_double), ("rotate", C.c_int32), ("reserved", C.c_int32), ("matrix", C.c_double * 6),
                ("out", C.c_void_p), ("out_image_stride", C.c_int64)]


#: one ``spg_prenet_member`` (include/spgroup.h) per record: a ragged call fills hundreds of them, which a numpy record
#: array takes without a Python object per member
PRENET_MEMBER = np.dtype([("image", np.uint64), ("row_stride", np.int64), ("height", np.int32), ("width", np.int32),
                          ("scale", np.float64), ("rotate", np.int32), ("reserved", np.int32), ("matrix", np.float64, (6,)),
                          ("out", np.uint64)], align=True)


#: ``spg_target_params``, ``spg_target_sample`` and ``spg_target_joints`` (include/spgroup.h) as numpy records: a batch of
#: training samples fills one record per sample
TARGET_PARAMS = np.dtype([("stride", np.int32), ("gaussian_size", np.int32), ("out_h", np.int32), ("out_w", np.int32),
                          ("sigma", np.float64), ("paf_sigma", np.float64), ("limb_gaussian_thre", np.float64),
                          ("paf_thre", np.float64), ("border_image", np.int32, (3,)), ("border_mask_miss", np.int32),
                          ("border_mask_all", np.int32), ("reserved", np.int32)], align=True)
TARGET_SAMPLE = np.dtype([("image", np.uint64), ("mask_miss", np.uint64), ("mask_all", np.uint64),
                          ("image_row_stride", np.int64), ("mask_row_stride", np.int64), ("height", np.int32),
                          ("width", np.int32), ("matrix", np.float64, (6,)), ("image_out", np.uint64),
                          ("mask_miss_out", np.uint64), ("mask_all_out", np.uint64)], align=True)
TARGET_JOINTS = np.dtype([("joints", np.uint64), ("n_persons", np.int32), ("reserved", np.int32), ("mask_all", np.uint64),
                          ("labels", np.uint64)], align=True)
#: ``spg_target_tint``: one source to tint in place, the reference's three draws and cv2's HSV->BGR row block
TARGET_TINT = np.dtype([("image", np.uint64), ("row_stride", np.int64), ("height", np.int32), ("width", np.int32),
                        ("hue", np.int32), ("saturation", np.int32), ("value", np.int32), ("row_block", np.int32)],
                       align=True)

#: ``spg_loss_params`` and ``spg_loss_pred`` (include/spgroup.h): the training loss's shared record and one record per
#: prediction tensor (``pred_tuple[k][j]`` at ``k * 5 + j``)
LOSS_FOCAL, LOSS_L2 = 0, 1
LOSS_PARAMS = np.dtype([("mode", np.int32), ("nstack", np.int32), ("batch", np.int32), ("channels", np.int32),
                        ("height", np.int32), ("width", np.int32), ("heat_start", np.int32), ("bkg_start", np.int32),
                        ("multi_task_weight", np.float64), ("keypoint_task_weight", np.float64),
                        ("nstack_weight", np.float64, (8,)), ("scale_weight", np.float64, (5,)),
                        ("batch_divisor", np.float64), ("scale_weight_sum", np.float64),
                        ("nstack_weight_sum", np.float64)], align=True)
LOSS_PRED = np.dtype([("data", np.uint64), ("grad", np.uint64), ("batch_stride", np.int64), ("chan_stride", np.int64),
                      ("row_stride", np.int64), ("grad_batch_stride", np.int64), ("grad_chan_stride", np.int64),
                      ("grad_row_stride", np.int64)], align=True)


class _ImageMaps(C.Structure):
    _fields_ = [("heat", C.c_void_p), ("paf", C.c_void_p), ("heat_chan_stride", C.c_int64),
                ("paf_chan_stride", C.c_int64), ("height", C.c_int32), ("width", C.c_int32), ("image_extent", C.c_double)]


class _DeviceView(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("max_batch", "n_parts", "n_limbs", "n_out_joints", "cap_peaks", "cap_cands",
                                          "cap_rows")] + \
               [(n, C.c_void_p) for n in ("peak_x", "peak_y", "peak_score", "peak_anchor", "peak_count", "conn_ij",
                                          "conn_score", "conn_norm", "conn_count", "cand_count", "surv_count", "subset",
                                          "n_persons", "people_xy", "people_score", "status")]


_ptr, _i32, _i64, _u64, _f64, _int, _P = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64, C.c_double, C.c_int, C.POINTER

#: export name -> (restype, argtypes) of every function include/spgroup.h declares (tests/test_abi.py checks the table
#: against the header and the built library).  Handles, streams and data pointers are all ``c_void_p``.
_PROTOTYPES = {
    "spg_create": (_int, [_P(_Config), _P(C.c_void_p)]),
    "spg_destroy": (None, [_ptr]),
    "spg_last_error": (C.c_char_p, [_ptr]),
    "spg_abi_version": (_int, []),
    "spg_get_device_view": (_int, [_ptr, _P(_DeviceView)]),
    "spg_group_batch": (_int, [_ptr, _ptr, _i64, _i64, _ptr, _i32, _i64, _i64, _i32, _i32, _i32, _f64, _P(_Params), _ptr]),
    "spg_group_ragged": (_int, [_ptr, _P(_ImageMaps), _i32, _i32, _P(_Params), _ptr]),
    "spg_group_unbounded": (_int, [_ptr, _P(_ImageMaps), _i32, _P(_Params), _ptr]),
    # spg_unbounded_sizes is four 32-bit words: cap_peaks, cap_rows, n_persons, status (uint32)
    "spg_download_unbounded": (_int, [_ptr, _P(C.c_int32)] + [_ptr] * 14),
    "spg_group_host": (_int, [_ptr, _ptr, _ptr, _i32, _i32, _i32, _i32, _f64, _P(_Params), _ptr, _ptr, _ptr, _ptr]),
    "spg_host_alloc": (_int, [_P(C.c_void_p), _u64]),
    "spg_host_free": (_int, [_ptr]),
    "spg_postnet": (_int, [_ptr, _P(_PostnetDesc), _i32, _i32, _i32, _ptr, _ptr, _i32, _ptr]),
    "spg_postnet_rotated": (_int, [_ptr, _P(_PostnetDesc), _P(_PostnetRotation), _i32, _i32, _i32, _ptr, _ptr, _i32, _ptr]),
    "spg_postnet_ragged": (_int, [_ptr, _P(_PostnetCommon), _P(_PostnetImage), _i32, _i32, _ptr]),
    "spg_postnet_ragged_items": (_int, [_ptr, _P(_PostnetCommon), _P(_PostnetImage), _P(_PostnetRotation), _i32, _i32, _i32,
                                        _ptr]),
    "spg_prenet": (_int, [_ptr, _ptr, _i64, _i64, _i32, _i32, _i32, _i32, _i32, _P(_PrenetItem), _i32, _ptr]),
    "spg_prenet_ragged": (_int, [_ptr, _i32, _i32, _ptr, _i32, _ptr]),  # members: a PRENET_MEMBER array
    # params: a TARGET_PARAMS record; samples: a TARGET_SAMPLE / TARGET_JOINTS array
    "spg_targets_warp": (_int, [_ptr, _ptr, _ptr, _i32, _ptr]),
    "spg_targets_maps": (_int, [_ptr, _ptr, _ptr, _i32, _ptr]),
    "spg_targets_tint": (_int, [_ptr, _ptr, _i32, _ptr]),  # samples: a TARGET_TINT array
    # params: a LOSS_PARAMS record; preds: a LOSS_PRED array
    "spg_loss_forward": (_int, [_ptr, _ptr, _ptr, _ptr, _ptr, _i32, _ptr, _ptr, _ptr]),
    "spg_loss_backward": (_int, [_ptr, _ptr, _ptr, _ptr, _ptr, _i32, _ptr, _ptr]),
    "spg_nms_peaks": (_int, [_ptr, _ptr, _i64, _i64, _i32, _i32, _i32, _P(_Params), _ptr]),
    "spg_limb_score": (_int, [_ptr, _ptr, _i32, _i64, _i64, _i32, _i32, _i32, _f64, _P(_Params), _ptr]),
    "spg_limb_match": (_int, [_ptr, _i32, _P(_Params), _ptr]),
    "spg_assemble": (_int, [_ptr, _i32, _P(_Params), _ptr]),
    "spg_match_assemble": (_int, [_ptr, _i32, _P(_Params), _ptr]),
    "spg_upload_peaks": (_int, [_ptr, _i32, _ptr, _ptr, _ptr, _ptr, _ptr]),
    "spg_upload_connections": (_int, [_ptr, _i32, _ptr, _ptr, _ptr, _ptr, _ptr]),
    "spg_download_peaks": (_int, [_ptr, _i32, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr]),
    "spg_download_connections": (_int, [_ptr, _i32, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr]),
    "spg_download_people": (_int, [_ptr, _i32, _ptr, _ptr, _ptr, _ptr, _ptr]),
    "spg_download_status": (_int, [_ptr, _i32, _ptr, _ptr]),
    "spg_wire_record_bytes": (_i64, [_ptr]),
    "spg_set_wire_output": (_int, [_ptr, _ptr, _i64, _i32]),
    "spg_arm_wire_signal": (_int, [_ptr, _ptr, _u64]),
    "spg_wire_create": (_int, [_i32, _u64, _P(C.c_void_p), C.c_char_p]),
    "spg_wire_open": (_int, [_i32, C.c_char_p, _P(C.c_void_p)]),
    "spg_wire_close": (_int, [_ptr]),
    "spg_wire_destroy": (_int, [_i32, _ptr]),
    "spg_wire_signal": (_int, [_i32, _ptr, _u64, _ptr]),
    "spg_wire_signal_many": (_int, [_i32, _P(C.c_void_p), _i32, _u64, _ptr]),
    "spg_wire_wait": (_int, [_i32, _ptr, _u64, _ptr]),
    "spg_launch_count": (_i64, [_ptr]),
    "spg_stage_kernel": (C.c_char_p, [_ptr, _i32]),
}
EXPORTS = tuple(_PROTOTYPES)

_lib = None


def load_library() -> C.CDLL:
    """Load ``libspgroup.so`` from the package directory.  Fails loudly; there is no fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise GroupingError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; "
                                f"g.build()'` (or `make -C improved_body_parts_b200/csrc`).  There is no CPU fallback.")
        lib = C.CDLL(LIB_PATH)
        for name, (restype, argtypes) in _PROTOTYPES.items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = restype, argtypes
        if lib.spg_abi_version() != ABI_VERSION:
            raise GroupingError("libspgroup.so ABI version mismatch")
        _lib = lib
    return _lib


def params_struct(params) -> _Params:
    """``params``: the reference's dict (utils/config keys), a GroupParams, or None for the defaults."""
    if params is None:
        gp = GroupParams()
    elif isinstance(params, GroupParams):
        gp = params
    else:
        gp = GroupParams.from_dict(dict(params))
    return _Params(gp.thre1, gp.thre2, gp.connect_ration, gp.len_rate, gp.connection_tole, gp.min_mean_score,
                   gp.mid_num, gp.offset_radius, gp.remove_recon, gp.min_parts, gp.crit1_strict, gp.refresh_len_check)


def clamp_scale(scale: float, image_hw) -> float:
    """evaluate.py:94-96: an item whose resized image would exceed 2600 rows or 3800 columns is shrunk to fit."""
    h, w = image_hw
    if scale * h > 2600 or scale * w > 3800:
        scale = min(2600 / h, 3800 / w)
    return scale


def input_geometry(h: int, w: int, scale: float, max_downsample: int) -> Tuple[int, int, int, int]:
    """``(H1, W1, Hp, Wp)`` of one item (evaluate.py:98-100): the size of ``cv2.resize(image, (0, 0), fx=scale,
    fy=scale)`` (``cvRound``: ties to even) = the crop, and that size padded up to multiples of ``max_downsample`` = the
    network's input."""
    H1, W1 = int(np.rint(h * scale)), int(np.rint(w * scale))
    md = int(max_downsample)
    return H1, W1, -(-H1 // md) * md, -(-W1 // md) * md


def prenet_item(h: int, w: int, scale: float, angle: float, max_downsample: int):
    """One pre-network item of an ``h x w`` image (evaluate.py:94-110): ``(scale, (H1, W1, Hp, Wp), forward, reverse)``
    -- the scale after the clamp of :94-96, the crop and padded network input sizes of :98-100 (zeros for a scale that
    is not finite and positive, which the library rejects), and for ``angle != 0`` the forward 2x3 matrix warpAffine
    takes and the reverse one ``postnet`` takes (the centre's x and y swapped as at :108-110), else ``None`` twice."""
    scale = clamp_scale(float(scale), (h, w))
    geo = input_geometry(h, w, scale, max_downsample) if np.isfinite(scale) and scale > 0 else (0, 0, 0, 0)
    forward = reverse = None
    if angle != 0:
        import cv2
        centre = (geo[2] / 2, geo[3] / 2)
        forward, reverse = cv2.getRotationMatrix2D(centre, angle, 1), cv2.getRotationMatrix2D(centre, -angle, 1)
    return scale, geo, forward, reverse


def _vp(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _stream_handle(stream, device: int) -> int:
    """The ``cudaStream_t`` of ``stream`` (a torch stream or a raw handle); ``None``: ``device``'s current stream."""
    if stream is None:
        import torch
        stream = torch.cuda.current_stream(device)  # the handle's device, not torch's current one
    return int(getattr(stream, "cuda_stream", stream))


def _check(rc: int, what: str, handle=None) -> None:
    """Raise for a non-zero return code, with the library's message (``handle`` None: the handle-less calls' slot)."""
    if rc != 0:
        msg = load_library().spg_last_error(handle)
        raise GroupingError(f"{what} failed ({rc}): {msg.decode() if msg else ''}")


class _CudaView:
    """Zero-copy torch view of handle-owned device memory (``__cuda_array_interface__``)."""

    def __init__(self, ptr: int, shape: Tuple[int, ...], typestr: str):
        self.__cuda_array_interface__ = {"shape": tuple(int(s) for s in shape), "typestr": typestr,
                                         "data": (int(ptr), False), "version": 2, "strides": None}


@dataclasses.dataclass
class GroupResult:
    """Host copy of everything one call produced (dense arrays with the handle's capacities)."""
    K: int
    L: int
    limbs: np.ndarray
    peak_count: np.ndarray   # [N,K]
    peak_x: np.ndarray       # [N,K,capP] f64
    peak_y: np.ndarray
    peak_score: np.ndarray   # f32
    peak_anchor: np.ndarray  # u32: (y<<16)|x, bit 31 = border peak
    conn_count: np.ndarray   # [N,L], -1 = special_k
    cand_count: np.ndarray   # [N,L]
    conn_ij: np.ndarray      # [N,L,capP] u32 (i<<16)|j
    conn_score: np.ndarray
    conn_norm: np.ndarray
    n_persons: np.ndarray    # [N]
    subset: np.ndarray       # [N,capR,K+2,2]
    people_xy: np.ndarray    # [N,capR,J,2]
    people_score: np.ndarray  # [N,capR]
    status: np.ndarray       # [N] u32

    def as_reference_structures(self, n: int):
        """(all_peaks, connection_all, special_k, subset, candidate) exactly as evaluate.py:203,276,498 return them."""
        K, L = self.K, self.L
        capP = self.peak_x.shape[2]
        cnt = np.minimum(self.peak_count[n], capP)
        off = np.concatenate([[0], np.cumsum(cnt)])
        all_peaks, flat = [], []
        for c in range(K):
            lst = []
            for q in range(int(cnt[c])):
                anchor = int(self.peak_anchor[n, c, q])
                gid = int(off[c] + q)
                if anchor >> 31:
                    xy = (np.int64(anchor & 0xffff), np.int64((anchor >> 16) & 0x7fff))
                else:
                    xy = (np.float64(self.peak_x[n, c, q]), np.float64(self.peak_y[n, c, q]))
                lst.append(xy + (np.float32(self.peak_score[n, c, q]), gid))
                flat.append((float(self.peak_x[n, c, q]), float(self.peak_y[n, c, q]),
                             float(self.peak_score[n, c, q]), float(gid)))
            all_peaks.append(lst)
        connection_all, special_k = [], []
        for k in range(L):
            m = int(self.conn_count[n, k])
            if m < 0:
                special_k.append(k)
                connection_all.append([])
                continue
            a, b = (int(v) for v in self.limbs[k])
            ij = self.conn_ij[n, k, :m].astype(np.int64)
            rows = np.zeros((m, 6))
            rows[:, 3] = ij >> 16
            rows[:, 4] = ij & 0xffff
            rows[:, 0] = off[a] + rows[:, 3]
            rows[:, 1] = off[b] + rows[:, 4]
            rows[:, 2] = self.conn_score[n, k, :m]
            rows[:, 5] = self.conn_norm[n, k, :m]
            connection_all.append(rows)
        P = int(self.n_persons[n])
        subset = self.subset[n, :P].copy()
        candidate = np.array(flat, np.float64).reshape(-1, 4) if flat else np.zeros((0,))
        return all_peaks, connection_all, special_k, subset, candidate

    def keypoints(self, n: int):
        """process() tail (evaluate.py:523-543): list of ([17 x (x, y)], score)."""
        P = int(self.n_persons[n])
        return [([tuple(xy) for xy in self.people_xy[n, j]], float(self.people_score[n, j])) for j in range(P)]


# ---- peer memory + stream-ordered signalling (the NVLink gather; sharding.py drives it) ------------------------
def wire_create(device: int, nbytes: int) -> Tuple[int, bytes]:
    """Zero-filled device buffer other processes can map: ``(device address, 64-byte IPC handle)``."""
    ptr, hd = C.c_void_p(), C.create_string_buffer(64)
    _check(load_library().spg_wire_create(device, nbytes, C.byref(ptr), hd), "spg_wire_create")
    return int(ptr.value), hd.raw


def wire_open(device: int, ipc_handle: bytes) -> int:
    ptr = C.c_void_p()
    _check(load_library().spg_wire_open(device, ipc_handle, C.byref(ptr)), "spg_wire_open")
    return int(ptr.value)


def wire_close(peer_ptr: int) -> None:
    load_library().spg_wire_close(peer_ptr)


def wire_destroy(device: int, dev_ptr: int) -> None:
    load_library().spg_wire_destroy(device, dev_ptr)


def wire_signal(device: int, word_ptr: int, value: int, stream) -> None:
    """Release-store ``value`` into a 64-bit word (local or peer memory) after everything earlier on ``stream``."""
    _check(load_library().spg_wire_signal(device, word_ptr, value, _stream_handle(stream, device)), "spg_wire_signal")


def wire_signal_many(device: int, word_ptrs: Sequence[int], value: int, stream) -> None:
    """One launch that release-stores ``value`` into every word of ``word_ptrs`` (<= 32, local or peer memory)."""
    arr = (C.c_void_p * len(word_ptrs))(*word_ptrs)
    _check(load_library().spg_wire_signal_many(device, arr, len(word_ptrs), value, _stream_handle(stream, device)),
           "spg_wire_signal_many")


def wire_wait(device: int, word_ptr: int, value: int, stream) -> None:
    """Make ``stream`` wait until the LOCAL 64-bit word is >= ``value`` (a stream memory operation, no SM involved)."""
    _check(load_library().spg_wire_wait(device, word_ptr, value, _stream_handle(stream, device)), "spg_wire_wait")


def device_bytes_view(ptr: int, nbytes: int, device: int):
    """Zero-copy uint8 torch view of raw device memory."""
    import torch
    return torch.as_tensor(_CudaView(ptr, (int(nbytes),), "|u1"), device=torch.device("cuda", device))


class Grouper:
    """One native grouping handle.  Not thread-safe; use one per stream / GPU."""

    def __init__(self, limbs: Sequence[Tuple[int, int]] = LIMBS, n_parts: int = NUM_PARTS,
                 out_from_part: Sequence[int] = COCO_FROM_PART, *, max_batch: int = 256, max_h: int = 128,
                 max_w: int = 128, max_peaks_per_part: int = 64, max_cands_per_limb: int = 1024,
                 max_person_rows: int = 96, device: int = 0):
        self._lib = load_library()
        self._h = C.c_void_p()
        self.limbs = np.ascontiguousarray(np.asarray(limbs, np.int32).reshape(-1, 2))
        self.out_from_part = np.ascontiguousarray(np.asarray(out_from_part, np.int32))
        self.K, self.L, self.J = int(n_parts), int(self.limbs.shape[0]), int(self.out_from_part.shape[0])
        self.max_batch, self.max_h, self.max_w = int(max_batch), int(max_h), int(max_w)
        self.capP, self.capC, self.capR = int(max_peaks_per_part), int(max_cands_per_limb), int(max_person_rows)
        self.device = int(device)
        cfg = _Config(ABI_VERSION, self.device, self.K, self.L, self.limbs.ctypes.data_as(C.POINTER(C.c_int32)), self.J,
                      self.out_from_part.ctypes.data_as(C.POINTER(C.c_int32)), self.max_batch, self.max_h, self.max_w,
                      self.capP, self.capC, self.capR)
        rc = self._lib.spg_create(C.byref(cfg), C.byref(self._h))
        if rc != 0:
            self._h = C.c_void_p()
            _check(rc, "spg_create")

    # -- lifetime ------------------------------------------------------------------------------
    def close(self) -> None:
        if getattr(self, "_h", None) and self._h.value:
            self._lib.spg_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    @property
    def launch_count(self) -> int:
        return int(self._lib.spg_launch_count(self._h))

    def stage_kernels(self):
        """Names of the kernel variants the last launches used: (nms_peaks, limb_score, limb_match, assemble)."""
        return tuple((self._lib.spg_stage_kernel(self._h, i) or b"").decode() for i in range(4))

    def postnet_kernel(self) -> str:
        """Name of the kernel the last ``postnet`` call launched."""
        return (self._lib.spg_stage_kernel(self._h, 4) or b"").decode()

    # -- wire records (include/spgroup.h; wire.py is the host-side view) -------------------------------
    def wire_record_bytes(self, rows: Optional[int] = None) -> int:
        """Bytes of one image's record with ``rows`` person rows (default: ``max_person_rows``)."""
        return wire.record_bytes(self.J, self.capR if rows is None else rows)

    def set_wire_output(self, dev_ptr: Optional[int], first_record: int = 0, rows: Optional[int] = None) -> None:
        """Make the assemble stage also write one wire record per image to ``dev_ptr`` (a raw device address: local
        memory or a peer GPU's buffer opened with ``wire_open``); ``None`` switches it off."""
        rc = self._lib.spg_set_wire_output(self._h, dev_ptr, first_record, self.capR if rows is None else rows)
        _check(rc, "spg_set_wire_output", self._h)

    def arm_wire_signal(self, word_ptr: Optional[int], value: int = 0) -> None:
        """The next single-launch assemble stage release-stores ``value`` into the 64-bit word at ``word_ptr`` (local or
        peer memory) when its last CTA is done: the "records landed" signal without a separate kernel.  One shot."""
        _check(self._lib.spg_arm_wire_signal(self._h, word_ptr, value), "spg_arm_wire_signal", self._h)

    # -- helpers ---------------------------------------------------------------------------------
    def _stream_ptr(self, stream) -> int:
        return _stream_handle(stream, self.device)

    def _check_maps(self, t, name: str, channels: int, dtypes) -> None:
        """Shape / dtype / channel checks shared by the whole-path and the stage entry points."""
        import torch
        self._dev_tensor(t, name)
        if t.device.index != self.device:
            raise GroupingError(f"{name} lives on cuda:{t.device.index}, the handle on cuda:{self.device}")
        if t.dtype not in dtypes:
            raise GroupingError(f"{name} must be " + " or ".join(str(d).replace("torch.", "") for d in dtypes))
        if t.shape[1] < channels:
            raise GroupingError(f"{name} has {t.shape[1]} channels, the skeleton needs {channels}")
        if t.shape[0] > self.max_batch:
            raise GroupingError(f"{name} holds {t.shape[0]} images, the handle was created for {self.max_batch}")

    @staticmethod
    def _dev_tensor(t, name: str):
        if not t.is_cuda:
            raise GroupingError(f"{name} must be a CUDA tensor")
        if t.dim() != 4 or t.stride(3) != 1 or t.stride(2) != t.shape[3]:
            raise GroupingError(f"{name} must be [N,C,H,W] with contiguous rows (pixel stride 1, row stride W)")
        return t

    def _paf_dtype(self, paf, as_f64: bool = False) -> int:
        import torch
        if paf.dtype == torch.float32:
            return F32_AS_F64 if as_f64 else F32
        if paf.dtype == torch.float64:
            return F64
        raise GroupingError("body-part maps must be float32 or float64")

    def _check_net_out(self, o, channels: int, n: Optional[int] = None, prefix: str = "") -> None:
        """A network output the post-network stage reads: ``[N,2,C,h,w]`` (``n`` images) or, for ``n=None``, one pair
        ``[2,C,h,w]``; float32 / float16 on the handle's device, rows contiguous, at least ``channels`` channels."""
        import torch
        lead = (2,) if n is None else (n, 2)
        if not o.is_cuda or o.device.index != self.device or o.dim() != len(lead) + 3 or tuple(o.shape[:len(lead)]) != lead:
            layout = "[2,C,h,w]" if n is None else "[N,2,C,h,w]"
            raise GroupingError(f"{prefix}network output must be a {layout} CUDA tensor on the handle's device")
        if o.stride(-1) != 1 or o.stride(-2) != o.shape[-1]:
            raise GroupingError(f"{prefix}network output rows must be contiguous")
        if o.dtype not in (torch.float32, torch.float16):
            raise GroupingError(f"{prefix}network output must be float32 or float16")
        if o.shape[-3] < channels:
            raise GroupingError(f"{prefix}network output has too few channels")

    # -- whole path --------------------------------------------------------------------------------
    def group_device(self, heat, paf, image_extent: float, params=None, stream=None, paf_as_f64: bool = False) -> None:
        """peaks -> connections -> people on device-resident maps; asynchronous on ``stream``.

        ``heat [N,>=K,H,W] float32`` (first K channels are used) and ``paf [N,>=L,H,W] float32|float64`` CUDA
        tensors; channel slices of the network's [N,50,h,w] output work without copies.  ``image_extent`` is the
        reference's ``oriImg.shape[0]`` (evaluate.py:510).
        """
        import torch
        self._check_maps(heat, "heat", self.K, (torch.float32,))  # find_peaks casts to float32, evaluate.py:173
        self._check_maps(paf, "paf", self.L, (torch.float32, torch.float64))
        N, _, H, W = heat.shape
        if paf.shape[0] != N or tuple(paf.shape[2:]) != (H, W):
            raise GroupingError("heat/paf shapes do not agree")
        p = params_struct(params)
        rc = self._lib.spg_group_batch(self._h, heat.data_ptr(), heat.stride(0), heat.stride(1), paf.data_ptr(),
                                       self._paf_dtype(paf, paf_as_f64), paf.stride(0), paf.stride(1), N, H, W,
                                       float(image_extent), C.byref(p), self._stream_ptr(stream))
        _check(rc, "spg_group_batch", self._h)
        self._peaks_shape = (N, H, W)
        self._last_n = N

    def group_ragged(self, maps, image_extents, params=None, stream=None, paf_as_f64: bool = False) -> None:
        """``group_device`` for images of different sizes in one asynchronous call; image i's results in slot i.

        ``maps``: per image a ``(heat, paf)`` pair of CUDA tensors, ``[C, H, W]`` or ``[1, C, H, W]`` with contiguous
        rows (channel slices of the network's output work), heat float32 and paf float32 / float64 -- one paf dtype for
        the whole call.  ``image_extents``: per image the reference's ``oriImg.shape[0]``.  Each image's results equal
        those of ``group_device`` on that image alone.  ``fetch(n)`` / ``as_reference_structures(i)`` read them back."""
        import torch
        maps = list(maps)
        extents = [float(e) for e in image_extents]
        if len(extents) != len(maps):
            raise GroupingError(f"{len(maps)} images but {len(extents)} image extents")
        if len(maps) > self.max_batch:
            raise GroupingError(f"{len(maps)} images, the handle was created for {self.max_batch}")
        arr = (_ImageMaps * max(len(maps), 1))()
        dtype = None
        for i, (heat, paf) in enumerate(maps):
            heat = heat[None] if heat.dim() == 3 else heat
            paf = paf[None] if paf.dim() == 3 else paf
            try:
                self._check_maps(heat, "heat", self.K, (torch.float32,))
                self._check_maps(paf, "paf", self.L, (torch.float32, torch.float64))
            except GroupingError as e:
                raise GroupingError(f"image {i}: {e}") from None
            if heat.shape[0] != 1 or paf.shape[0] != 1 or tuple(paf.shape[2:]) != tuple(heat.shape[2:]):
                raise GroupingError(f"image {i}: heat and paf must be one image each, of the same size")
            d = self._paf_dtype(paf, paf_as_f64)
            if dtype is not None and d != dtype:
                raise GroupingError(f"image {i}: every image of a call needs the same paf dtype")
            dtype = d
            arr[i] = _ImageMaps(heat.data_ptr(), paf.data_ptr(), heat.stride(1), paf.stride(1), heat.shape[2],
                                heat.shape[3], extents[i])
        p = params_struct(params)
        rc = self._lib.spg_group_ragged(self._h, arr, len(maps), F32 if dtype is None else dtype, C.byref(p),
                                        self._stream_ptr(stream))
        _check(rc, "spg_group_ragged", self._h)
        self._peaks_shape = None
        self._last_n = len(maps)

    def group_unbounded(self, heat, paf, image_extent: float, params=None, paf_as_f64: bool = False,
                        stream=None) -> GroupResult:
        """One image on the capacity-free tier (``spg_group_unbounded``): the reference's answer whatever the image's
        number of peaks, candidates and persons, where the other calls set a capacity status bit.  Synchronous.

        ``heat`` / ``paf``: the image's maps as for ``group_ragged`` (``[C, H, W]`` or ``[1, C, H, W]``).  Returns a
        one-image ``GroupResult`` with the tier's sizes (``peak_x.shape[2]`` = the largest part's peak count,
        ``subset.shape[1]`` = the person table's rows), so ``as_reference_structures(0)`` and ``keypoints(0)`` read it
        as they read ``fetch``'s.  The handle's results of earlier calls are left as they were."""
        import torch
        heat = heat[None] if heat.dim() == 3 else heat
        paf = paf[None] if paf.dim() == 3 else paf
        self._check_maps(heat, "heat", self.K, (torch.float32,))
        self._check_maps(paf, "paf", self.L, (torch.float32, torch.float64))
        if heat.shape[0] != 1 or paf.shape[0] != 1 or tuple(paf.shape[2:]) != tuple(heat.shape[2:]):
            raise GroupingError("heat and paf must be one image each, of the same size")
        im = _ImageMaps(heat.data_ptr(), paf.data_ptr(), heat.stride(1), paf.stride(1), heat.shape[2], heat.shape[3],
                        float(image_extent))
        p = params_struct(params)
        st = self._stream_ptr(stream)
        _check(self._lib.spg_group_unbounded(self._h, C.byref(im), self._paf_dtype(paf, paf_as_f64), C.byref(p), st),
               "spg_group_unbounded", self._h)
        sz = (C.c_int32 * 4)()  # spg_unbounded_sizes: cap_peaks, cap_rows, n_persons, status
        _check(self._lib.spg_download_unbounded(self._h, sz, *([None] * 13), st), "spg_download_unbounded", self._h)
        K, L, J, cP, cR = self.K, self.L, self.J, int(sz[0]), int(sz[1])
        r = GroupResult(
            K=K, L=L, limbs=self.limbs, peak_count=np.zeros((1, K), np.int32), peak_x=np.zeros((1, K, cP)),
            peak_y=np.zeros((1, K, cP)), peak_score=np.zeros((1, K, cP), np.float32),
            peak_anchor=np.zeros((1, K, cP), np.uint32), conn_count=np.zeros((1, L), np.int32),
            cand_count=np.zeros((1, L), np.int32), conn_ij=np.zeros((1, L, cP), np.uint32),
            conn_score=np.zeros((1, L, cP)), conn_norm=np.zeros((1, L, cP)),
            n_persons=np.array([sz[2]], np.int32), subset=np.zeros((1, cR, K + 2, 2)),
            people_xy=np.zeros((1, cR, J, 2)), people_score=np.zeros((1, cR)),
            status=np.array([sz[3] & 0xffffffff], np.uint32))
        _check(self._lib.spg_download_unbounded(
            self._h, sz, _vp(r.peak_count), _vp(r.peak_x), _vp(r.peak_y), _vp(r.peak_score), _vp(r.peak_anchor),
            _vp(r.conn_count), _vp(r.cand_count), _vp(r.conn_ij), _vp(r.conn_score), _vp(r.conn_norm), _vp(r.subset),
            _vp(r.people_xy), _vp(r.people_score), st), "spg_download_unbounded", self._h)
        return r

    def group_host(self, heat: np.ndarray, paf: np.ndarray, image_extent: float, params=None, out=None) -> dict:
        """Host maps in, person lists out (H2D / kernels / D2H pipelined inside the library).  Synchronous.

        ``heat [N,K,H,W] float32`` and ``paf [N,L,H,W] float32|float64`` C-contiguous numpy arrays (pinned memory
        gives full copy/compute overlap).  ``out`` may carry preallocated result arrays to reuse.
        """
        if heat.dtype != np.float32 or not heat.flags.c_contiguous or heat.ndim != 4 or heat.shape[1] != self.K:
            raise GroupingError("heat must be a C-contiguous float32 [N,K,H,W] array")
        if paf.dtype not in (np.float32, np.float64) or not paf.flags.c_contiguous or paf.ndim != 4 or paf.shape[1] != self.L:
            raise GroupingError("paf must be a C-contiguous float32/float64 [N,L,H,W] array")
        N, _, H, W = heat.shape
        if paf.shape[0] != N or paf.shape[2:] != (H, W):
            raise GroupingError("heat/paf shapes differ")
        if out is None:
            out = {}
        o_n = out.setdefault("n_persons", np.zeros((N,), np.int32))
        o_xy = out.setdefault("people_xy", np.zeros((N, self.capR, self.J, 2), np.float64))
        o_sc = out.setdefault("people_score", np.zeros((N, self.capR), np.float64))
        o_st = out.setdefault("status", np.zeros((N,), np.uint32))
        p = params_struct(params)
        rc = self._lib.spg_group_host(self._h, _vp(heat), _vp(paf), F64 if paf.dtype == np.float64 else F32, N, H, W,
                                      float(image_extent), C.byref(p), _vp(o_n), _vp(o_xy), _vp(o_sc), _vp(o_st))
        _check(rc, "spg_group_host", self._h)
        self._last_n = N
        return out

    # -- post-network stage ---------------------------------------------------------------------------
    def postnet(self, net_outs, crops, out_hw, *, stride: int = 4, paf_dtype=None, heat_out=None, paf_out=None,
                paf_chan0: int = 0, heat_chan0: Optional[int] = None, flip_paf_ord=None, flip_heat_ord=None,
                nan_scrub: bool = False, stream=None, rotations=None):
        """The scale loop of ``predict()`` after the forward pass (evaluate.py:126-161) on the device.

        ``net_outs``: one CUDA tensor ``[N, 2, C, h, w]`` (float32 / float16; image, mirrored image) per item of
        ``product(multiplier, rotate_angle)``; ``crops``: per item ``(crop_h, crop_w)`` = ``imageToTest.shape[:2]``;
        ``out_hw``: the image size.  ``rotations``: ``None``, or per item ``None`` (angle 0) or the 2x3 matrix the
        reference warps that item's x stride maps with (``rotate_matrix_reverse``, evaluate.py:115, :144, :153).
        Returns ``(heat [N,K,H,W] float32, paf [N,L,H,W])`` -- ``paf`` float32 for a single item (pass
        ``paf_as_f64=True`` to the grouping calls: the reference's float64 values are exactly these), float64 otherwise.
        """
        import torch
        if len(net_outs) != len(crops) or not net_outs:
            raise GroupingError("one crop size per scale expected")
        H, W = (int(v) for v in out_hw)
        N = int(net_outs[0].shape[0])
        dev = torch.device("cuda", self.device)
        single = len(net_outs) == 1
        if paf_dtype is None:
            paf_dtype = torch.float32 if single else torch.float64
        if paf_dtype == torch.float32 and not single:
            raise GroupingError("float32 body-part planes hold the reference's float64 values only for a single scale")
        heat_chan0 = self.L if heat_chan0 is None else heat_chan0
        fp, fh = self._flip_orders(flip_paf_ord, flip_heat_ord)
        scales = (_PostnetScale * len(net_outs))()
        for t, (o, (ch, cw)) in enumerate(zip(net_outs, crops)):
            self._check_net_out(o, max(heat_chan0 + self.K, paf_chan0 + self.L), N)
            scales[t] = _PostnetScale(o.data_ptr(), F32 if o.dtype == torch.float32 else F16, o.stride(0), o.stride(1),
                                      o.stride(2), o.shape[3], o.shape[4], int(ch), int(cw))
        if heat_out is None:
            heat_out = torch.empty((N, self.K, H, W), dtype=torch.float32, device=dev)
        if paf_out is None:
            paf_out = torch.empty((N, self.L, H, W), dtype=paf_dtype, device=dev)
        if not (heat_out.is_contiguous() and paf_out.is_contiguous()) or paf_out.dtype != paf_dtype:
            raise GroupingError("heat_out / paf_out must be contiguous tensors of the requested dtype")
        desc = _PostnetDesc(len(net_outs), scales, int(stride), int(paf_chan0), int(heat_chan0),
                            fp.ctypes.data_as(C.POINTER(C.c_int32)), fh.ctypes.data_as(C.POINTER(C.c_int32)), int(bool(nan_scrub)))
        rot = None
        if rotations is not None:
            if len(rotations) != len(net_outs):
                raise GroupingError("one rotation entry (None or a 2x3 matrix) per item expected")
            rot = (_PostnetRotation * len(net_outs))()
            for t, m in enumerate(rotations):
                if m is not None:
                    m = np.asarray(m, np.float64)
                    if m.shape != (2, 3):
                        raise GroupingError("a rotation matrix is 2x3")
                    rot[t] = _PostnetRotation(1, 0, (C.c_double * 6)(*m.reshape(6).tolist()))
        rc = self._lib.spg_postnet_rotated(self._h, C.byref(desc), rot, N, H, W, heat_out.data_ptr(), paf_out.data_ptr(),
                                           F32 if paf_dtype == torch.float32 else F64, self._stream_ptr(stream))
        _check(rc, "spg_postnet_rotated", self._h)
        return heat_out, paf_out

    def _flip_orders(self, flip_paf_ord, flip_heat_ord):
        """The flip permutations of the body-part / keypoint channels (default: the canonical skeleton's)."""
        from .skeleton import FLIP_HEAT_ORD, FLIP_PAF_ORD, NUM_LIMBS
        if flip_paf_ord is None and self.L != NUM_LIMBS:
            raise GroupingError("flip_paf_ord is needed for a non-canonical skeleton")
        fp = np.ascontiguousarray(np.asarray(FLIP_PAF_ORD if flip_paf_ord is None else flip_paf_ord, np.int32)[:self.L])
        fh = np.ascontiguousarray(np.asarray(FLIP_HEAT_ORD if flip_heat_ord is None else flip_heat_ord, np.int32)[:self.K])
        return fp, fh

    def postnet_ragged(self, images, *, stride: int = 4, paf_dtype=None, outs=None, paf_chan0: int = 0,
                       heat_chan0: Optional[int] = None, flip_paf_ord=None, flip_heat_ord=None, nan_scrub: bool = False,
                       stream=None):
        """``postnet`` for a batch of images of different sizes with one item each (one scale, no rotation) in one
        asynchronous call.

        ``images``: per image ``(net_out, (crop_h, crop_w), (H, W))`` -- ``net_out`` the ``[2, C, h, w]`` CUDA tensor of
        its pair (float32 / float16, one dtype per call; slices of a shared ``[2k, C, h, w]`` batch output work without
        copies).  ``outs``: optional per-image ``(heat, paf)`` contiguous tensors to write into.  Returns per image
        ``(heat [1,K,H,W] float32, paf [1,L,H,W])``, equal to what ``postnet`` returns for that image alone; ``paf`` is
        float32 by default (float32 storage of the float64 values, ``paf_as_f64=True`` for the grouping calls)."""
        return self._postnet_ragged([([(o, crop, None)], hw) for o, crop, hw in images], stride, paf_dtype, outs, paf_chan0,
                                    heat_chan0, flip_paf_ord, flip_heat_ord, nan_scrub, stream)

    def postnet_ragged_items(self, images, *, paf_dtype=None, outs=None, paf_chan0: int = 0,
                             heat_chan0: Optional[int] = None, flip_paf_ord=None, flip_heat_ord=None,
                             nan_scrub: bool = False, stream=None):
        """``postnet`` for a batch of images of different sizes with several items each -- the multi-scale and rotation
        search of ``predict()`` -- in one asynchronous call (stride 4).

        ``images``: per image ``(items, (H, W))``; ``items``: per item of ``product(multiplier, rotate_angle)`` a
        ``(net_out, (crop_h, crop_w), rotate_matrix_reverse or None)`` triple -- what ``prenet`` returns with the
        ``[2, C, h, w]`` network output of the pair in place of the pair (float32 / float16, one dtype per call).  Every
        image has the same number of items, and item t is rotated in every image or in none.  ``outs``: optional
        per-image ``(heat, paf)`` contiguous tensors to write into.  Returns per image ``(heat [1,K,H,W] float32,
        paf [1,L,H,W])``, equal to what ``postnet(..., rotations=...)`` returns for that image alone; ``paf`` is
        float64 for more than one item and float32 for a single one, as there."""
        return self._postnet_ragged(images, 4, paf_dtype, outs, paf_chan0, heat_chan0, flip_paf_ord, flip_heat_ord,
                                    nan_scrub, stream)

    def _postnet_ragged(self, images, stride, paf_dtype, outs, paf_chan0, heat_chan0, flip_paf_ord, flip_heat_ord,
                        nan_scrub, stream):
        """``postnet_ragged_items`` at any ``stride`` (the C call rejects all but 4): one ``spg_postnet_ragged_items``
        call.  Errors name ``image i``, or ``image i item t`` when the images have several items."""
        import torch
        images = list(images)
        if outs is not None and len(outs) != len(images):
            raise GroupingError("one (heat, paf) output pair per image expected")
        if len(images) > self.max_batch:
            raise GroupingError(f"{len(images)} images, the handle was created for {self.max_batch}")
        n_items = len(images[0][0]) if images else 1
        if any(len(items) != n_items for items, _ in images):
            raise GroupingError("every image of a call needs the same number of items")
        if n_items < 1:
            raise GroupingError("every image needs at least one item")
        if paf_dtype is None:
            paf_dtype = torch.float32 if n_items == 1 else torch.float64
        if paf_dtype not in (torch.float32, torch.float64):
            raise GroupingError("paf_dtype must be float32 or float64")
        heat_chan0 = self.L if heat_chan0 is None else heat_chan0
        fp, fh = self._flip_orders(flip_paf_ord, flip_heat_ord)
        dev = torch.device("cuda", self.device)
        n_all = max(len(images) * n_items, 1)
        arr, rot = (_PostnetImage * n_all)(), (_PostnetRotation * n_all)()
        net_dtype, any_rot, results = None, False, []
        for i, (items, (H, W)) in enumerate(images):
            H, W = int(H), int(W)
            if outs is not None:
                heat, paf = outs[i]
            else:
                heat = torch.empty((1, self.K, H, W), dtype=torch.float32, device=dev)
                paf = torch.empty((1, self.L, H, W), dtype=paf_dtype, device=dev)
            if not (heat.is_contiguous() and paf.is_contiguous()) or heat.dtype != torch.float32 or paf.dtype != paf_dtype \
                    or heat.numel() != self.K * H * W or paf.numel() != self.L * H * W:
                raise GroupingError(f"image {i}: heat / paf outputs must be contiguous float32 [K,H,W] / {paf_dtype} [L,H,W]")
            for t, (o, (ch, cw), m) in enumerate(items):
                prefix = f"image {i}: " if n_items == 1 else f"image {i} item {t}: "
                self._check_net_out(o, max(heat_chan0 + self.K, paf_chan0 + self.L), prefix=prefix)
                if net_dtype is not None and o.dtype != net_dtype:
                    raise GroupingError(f"{prefix}every network output of a call needs the same dtype")
                net_dtype = o.dtype
                k = i * n_items + t
                arr[k] = _PostnetImage(o.data_ptr(), o.stride(0), o.stride(1), o.shape[2], o.shape[3], int(ch), int(cw), H, W,
                                       heat.data_ptr(), paf.data_ptr())
                if m is not None:
                    m = np.asarray(m, np.float64)
                    if m.shape != (2, 3):
                        raise GroupingError(f"{prefix}a rotation matrix is 2x3")
                    rot[k] = _PostnetRotation(1, 0, (C.c_double * 6)(*m.reshape(6).tolist()))
                    any_rot = True
            results.append((heat, paf))
        common = _PostnetCommon(int(stride), int(paf_chan0), int(heat_chan0), fp.ctypes.data_as(C.POINTER(C.c_int32)),
                                fh.ctypes.data_as(C.POINTER(C.c_int32)), int(bool(nan_scrub)),
                                F16 if net_dtype == torch.float16 else F32)
        rc = self._lib.spg_postnet_ragged_items(self._h, C.byref(common), arr, rot if any_rot else None, len(images), n_items,
                                                F32 if paf_dtype == torch.float32 else F64, self._stream_ptr(stream))
        _check(rc, "spg_postnet_ragged_items", self._h)
        return results

    # -- pre-network stage ----------------------------------------------------------------------------
    @property
    def prenet_kernel(self) -> str:
        """Name of the kernel the last pre-network launch used (``""`` before the first)."""
        return (self._lib.spg_stage_kernel(self._h, 5) or b"").decode()

    def prenet(self, image, scales, angles, *, max_downsample: int, pad_value: int, out=None, stream=None):
        """The item loop of ``predict()`` before the forward pass (evaluate.py:94-121) on the device.

        ``image``: ``[N, H, W, 3]`` or ``[H, W, 3]`` uint8 CUDA tensor (BGR as read) with contiguous rows; ``scales`` the
        reference's ``multiplier`` and ``angles`` its ``rotate_angle``: one item per entry of ``product(scales, angles)``
        (:90), each scale clamped as at :94-96.  ``out``: optional per-item output tensors to reuse.  Returns per item
        ``(pair, crop, rotate_matrix_reverse)``: ``pair`` the ``[N, 2, Hp, Wp, 3]`` float32 tensor the network receives
        (image, mirror; ``[2, Hp, Wp, 3]`` for a 3-D ``image``), ``crop`` = ``imageToTest.shape[:2]`` and the reverse
        matrix (``None`` for angle 0) -- the ``crops`` and ``rotations`` ``postnet`` takes.  Asynchronous on ``stream``.
        """
        import itertools

        import torch
        if not getattr(image, "is_cuda", False) or image.dtype != torch.uint8 or image.dim() not in (3, 4):
            raise GroupingError("image must be a [N,H,W,3] or [H,W,3] uint8 CUDA tensor")
        if image.device.index != self.device:
            raise GroupingError(f"image lives on cuda:{image.device.index}, the handle on cuda:{self.device}")
        batched = image.dim() == 4
        img = image if batched else image[None]
        N, h, w, cn = (int(v) for v in img.shape)
        if cn != 3 or img.stride(3) != 1 or img.stride(2) != 3:
            raise GroupingError("image must have 3 channels and contiguous rows (channel stride 1, pixel stride 3)")
        md, pv = int(max_downsample), int(pad_value)
        if md < 1:
            raise GroupingError("max_downsample must be >= 1")
        pairs = list(itertools.product(scales, angles))
        if out is not None and len(out) != len(pairs):
            raise GroupingError("one output tensor per item expected")
        items = (_PrenetItem * max(len(pairs), 1))()
        results = []
        for t, (scale, angle) in enumerate(pairs):
            scale, (H1, W1, Hp, Wp), forward, reverse = prenet_item(h, w, scale, angle, md)
            o = self._prenet_out(None if out is None else out[t] if batched else out[t][None], (N, 2, Hp, Wp, 3),
                                 f"out[{t}]", f"[N,2,{Hp},{Wp},3] CUDA tensor with contiguous images")
            m = (C.c_double * 6)(*(np.asarray(forward, np.float64).reshape(6).tolist() if forward is not None else [0.0] * 6))
            items[t] = _PrenetItem(scale, int(forward is not None), 0, m, o.data_ptr(), o.stride(0))
            results.append((o if batched else o[0], (H1, W1), reverse))
        rc = self._lib.spg_prenet(self._h, img.data_ptr(), img.stride(0), img.stride(1), N, h, w, md, pv, items, len(pairs),
                                  self._stream_ptr(stream))
        _check(rc, "spg_prenet", self._h)
        return results

    def prenet_ragged(self, members, *, max_downsample: int, pad_value: int, out=None, stream=None):
        """``prenet`` for images of different sizes, each with its own items, in one asynchronous call.

        ``members``: per member ``(image, scale, angle)`` -- ``image`` a ``[H, W, 3]`` uint8 CUDA tensor (BGR as read)
        with contiguous rows, ``scale`` a ``multiplier`` entry (clamped as at evaluate.py:94-96) and ``angle`` a
        ``rotate_angle`` entry; several members may read one image.  ``out``: optional per-member ``[2, Hp, Wp, 3]``
        float32 contiguous tensors to write into (slices of one batch tensor work).  Returns per member the
        ``(pair, crop, rotate_matrix_reverse)`` triple ``prenet`` returns for that image and item alone."""
        import torch
        members = list(members)
        if out is not None and len(out) != len(members):
            raise GroupingError("one output tensor per member expected")
        md, pv = int(max_downsample), int(pad_value)
        if md < 1:
            raise GroupingError("max_downsample must be >= 1")
        arr = np.zeros(max(len(members), 1), PRENET_MEMBER)
        results = []
        for i, (image, scale, angle) in enumerate(members):
            if not getattr(image, "is_cuda", False) or image.dtype != torch.uint8 or image.dim() != 3:
                raise GroupingError(f"member {i}: image must be a [H,W,3] uint8 CUDA tensor")
            if image.device.index != self.device:
                raise GroupingError(f"member {i}: image lives on cuda:{image.device.index}, the handle on cuda:{self.device}")
            h, w, cn = (int(v) for v in image.shape)
            if cn != 3 or image.stride(2) != 1 or image.stride(1) != 3:
                raise GroupingError(f"member {i}: image must have 3 channels and contiguous rows")
            scale, (H1, W1, Hp, Wp), forward, reverse = prenet_item(h, w, scale, angle, md)
            o = self._prenet_out(None if out is None else out[i], (2, Hp, Wp, 3), f"out[{i}]",
                                 f"contiguous [2,{Hp},{Wp},3] CUDA tensor")
            arr[i] = (image.data_ptr(), image.stride(0), h, w, scale, int(forward is not None), 0,
                      np.zeros(6) if forward is None else np.asarray(forward, np.float64).reshape(6), o.data_ptr())
            results.append((o, (H1, W1), reverse))
        rc = self._lib.spg_prenet_ragged(self._h, md, pv, arr.ctypes.data, len(members), self._stream_ptr(stream))
        _check(rc, "spg_prenet_ragged", self._h)
        return results

    def _prenet_out(self, o, shape, name, form):
        """A pre-network output of ``shape`` on the handle's device: ``o`` checked (the leading pair contiguous), or a new
        tensor for ``None``."""
        import torch
        if o is None:
            return torch.empty(shape, dtype=torch.float32, device=torch.device("cuda", self.device))
        if o.dtype != torch.float32 or not o.is_cuda or o.device.index != self.device or tuple(o.shape) != shape or \
                not o[(0,) * (len(shape) - 4)].is_contiguous():
            raise GroupingError(f"{name} must be a float32 {form}")
        return o

    # -- training samples (targets.py builds the records) ----------------------------------------------------------
    def targets_warp(self, params: np.ndarray, samples: np.ndarray, stream=None) -> None:
        """``spg_targets_warp``: ``params`` one ``TARGET_PARAMS`` record, ``samples`` a ``TARGET_SAMPLE`` array of device
        addresses on the handle's device.  Asynchronous on ``stream``."""
        p, s = self._records(params, TARGET_PARAMS), self._records(samples, TARGET_SAMPLE)
        _check(self._lib.spg_targets_warp(self._h, p.ctypes.data, s.ctypes.data, len(s), self._stream_ptr(stream)),
               "spg_targets_warp", self._h)

    def targets_maps(self, params: np.ndarray, samples: np.ndarray, stream=None) -> None:
        """``spg_targets_maps``: ``samples`` a ``TARGET_JOINTS`` array; the limb table is the handle's."""
        p, s = self._records(params, TARGET_PARAMS), self._records(samples, TARGET_JOINTS)
        _check(self._lib.spg_targets_maps(self._h, p.ctypes.data, s.ctypes.data, len(s), self._stream_ptr(stream)),
               "spg_targets_maps", self._h)

    def targets_tint(self, records: np.ndarray, stream=None) -> None:
        """``spg_targets_tint``: ``records`` a ``TARGET_TINT`` array; each source is tinted in place on the device."""
        s = self._records(records, TARGET_TINT)
        _check(self._lib.spg_targets_tint(self._h, s.ctypes.data, len(s), self._stream_ptr(stream)), "spg_targets_tint",
               self._h)

    # -- training loss (loss.py builds the records) ---------------------------------------------------------------
    def loss_forward(self, params: np.ndarray, mask_miss: int, labels: int, preds: np.ndarray, dtype: int,
                     stack_sums: int, loss: int, stream=None) -> None:
        """``spg_loss_forward``: ``params`` one ``LOSS_PARAMS`` record, ``preds`` a ``LOSS_PRED`` array; the tensors are
        device addresses on the handle's device.  Asynchronous on ``stream``."""
        p, r = self._records(params, LOSS_PARAMS), self._records(preds, LOSS_PRED)
        _check(self._lib.spg_loss_forward(self._h, p.ctypes.data, mask_miss, labels, r.ctypes.data, dtype, stack_sums, loss,
                                          self._stream_ptr(stream)), "spg_loss_forward", self._h)

    def loss_backward(self, params: np.ndarray, mask_miss: int, labels: int, preds: np.ndarray, dtype: int,
                      grad_output: int, stream=None) -> None:
        """``spg_loss_backward``: every ``preds[i]["grad"]`` written from the float32 device scalar at ``grad_output``."""
        p, r = self._records(params, LOSS_PARAMS), self._records(preds, LOSS_PRED)
        _check(self._lib.spg_loss_backward(self._h, p.ctypes.data, mask_miss, labels, r.ctypes.data, dtype, grad_output,
                                           self._stream_ptr(stream)), "spg_loss_backward", self._h)

    def loss_kernel(self) -> str:
        """Name of the kernel the last loss call launched."""
        return (self._lib.spg_stage_kernel(self._h, 7) or b"").decode()

    @staticmethod
    def _records(a: np.ndarray, dtype: np.dtype) -> np.ndarray:
        a = np.ascontiguousarray(a).reshape(-1)
        if a.dtype != dtype:
            raise GroupingError(f"records of dtype {dtype} expected")
        return a

    # -- stages -------------------------------------------------------------------------------------
    def nms_peaks(self, heat, params=None, stream=None) -> None:
        """find_peaks (evaluate.py:169-203) on ``heat [N,>=K,H,W]`` float32 CUDA."""
        import torch
        self._check_maps(heat, "heat", self.K, (torch.float32,))
        N, _, H, W = heat.shape
        self._peaks_shape = (N, H, W)
        p = params_struct(params)
        rc = self._lib.spg_nms_peaks(self._h, heat.data_ptr(), heat.stride(0), heat.stride(1), N, H, W, C.byref(p),
                                     self._stream_ptr(stream))
        _check(rc, "spg_nms_peaks", self._h)
        self._last_n = N

    def limb_score(self, paf, image_extent: float, params=None, stream=None, paf_as_f64: bool = False) -> None:
        """Scoring half of find_connections (evaluate.py:211-255) for peaks already on the device."""
        import torch
        self._check_maps(paf, "paf", self.L, (torch.float32, torch.float64))
        N, _, H, W = paf.shape
        ps = getattr(self, "_peaks_shape", None)  # peaks from spg_nms_peaks: the maps must agree (uploaded peaks carry no shape)
        if ps is not None and (ps[0] < N or ps[1:] != (H, W)):
            raise GroupingError(f"paf is {N}x{H}x{W} but the peaks on the device come from {ps[0]}x{ps[1]}x{ps[2]} heat maps")
        p = params_struct(params)
        rc = self._lib.spg_limb_score(self._h, paf.data_ptr(), self._paf_dtype(paf, paf_as_f64), paf.stride(0),
                                      paf.stride(1), N, H, W, float(image_extent), C.byref(p), self._stream_ptr(stream))
        _check(rc, "spg_limb_score", self._h)
        self._last_n = N

    def limb_match(self, n_images: int, params=None, stream=None) -> None:
        """Matching half of find_connections (evaluate.py:259-274)."""
        p = params_struct(params)
        _check(self._lib.spg_limb_match(self._h, n_images, C.byref(p), self._stream_ptr(stream)),
               "spg_limb_match", self._h)

    def assemble(self, n_images: int, params=None, stream=None) -> None:
        """find_people + process() tail (evaluate.py:279-498, 523-543)."""
        p = params_struct(params)
        _check(self._lib.spg_assemble(self._h, n_images, C.byref(p), self._stream_ptr(stream)), "spg_assemble", self._h)

    def match_assemble(self, n_images: int, params=None, stream=None) -> None:
        """limb_match + assemble fused in one kernel (what the whole-path calls run)."""
        p = params_struct(params)
        _check(self._lib.spg_match_assemble(self._h, n_images, C.byref(p), self._stream_ptr(stream)),
               "spg_match_assemble", self._h)

    # -- state transfer ---------------------------------------------------------------------------------
    def upload_peaks(self, image_index: int, part_count, x, y, score, stream=None) -> None:
        self._peaks_shape = None
        pc = np.ascontiguousarray(part_count, np.int32)
        x = np.ascontiguousarray(x, np.float64)
        y = np.ascontiguousarray(y, np.float64)
        s = np.ascontiguousarray(score, np.float32)
        _check(self._lib.spg_upload_peaks(self._h, image_index, _vp(pc), _vp(x), _vp(y), _vp(s),
                                          self._stream_ptr(stream)), "spg_upload_peaks", self._h)

    def upload_connections(self, image_index: int, conn_count, ij, score, norm, stream=None) -> None:
        cc = np.ascontiguousarray(conn_count, np.int32)
        ij = np.ascontiguousarray(ij, np.int32).reshape(-1, 2)
        sc = np.ascontiguousarray(score, np.float64)
        nm = np.ascontiguousarray(norm, np.float64)
        _check(self._lib.spg_upload_connections(self._h, image_index, _vp(cc), _vp(ij), _vp(sc), _vp(nm),
                                                self._stream_ptr(stream)), "spg_upload_connections", self._h)

    def fetch(self, n_images: Optional[int] = None, stream=None) -> GroupResult:
        """Synchronise and copy every result of the last call to the host."""
        N = int(self._last_n if n_images is None else n_images)
        K, L, J, cP, cR = self.K, self.L, self.J, self.capP, self.capR
        st = self._stream_ptr(stream)
        r = GroupResult(
            K=K, L=L, limbs=self.limbs, peak_count=np.zeros((N, K), np.int32), peak_x=np.zeros((N, K, cP)),
            peak_y=np.zeros((N, K, cP)), peak_score=np.zeros((N, K, cP), np.float32),
            peak_anchor=np.zeros((N, K, cP), np.uint32), conn_count=np.zeros((N, L), np.int32),
            cand_count=np.zeros((N, L), np.int32), conn_ij=np.zeros((N, L, cP), np.uint32),
            conn_score=np.zeros((N, L, cP)), conn_norm=np.zeros((N, L, cP)), n_persons=np.zeros((N,), np.int32),
            subset=np.zeros((N, cR, K + 2, 2)), people_xy=np.zeros((N, cR, J, 2)), people_score=np.zeros((N, cR)),
            status=np.zeros((N,), np.uint32))
        _check(self._lib.spg_download_peaks(self._h, N, _vp(r.peak_count), _vp(r.peak_x), _vp(r.peak_y), _vp(r.peak_score),
                                            _vp(r.peak_anchor), st), "spg_download_peaks", self._h)
        _check(self._lib.spg_download_connections(self._h, N, _vp(r.conn_count), _vp(r.cand_count), _vp(r.conn_ij),
                                                  _vp(r.conn_score), _vp(r.conn_norm), st),
               "spg_download_connections", self._h)
        _check(self._lib.spg_download_people(self._h, N, _vp(r.n_persons), _vp(r.subset), _vp(r.people_xy),
                                             _vp(r.people_score), st), "spg_download_people", self._h)
        _check(self._lib.spg_download_status(self._h, N, _vp(r.status), st), "spg_download_status", self._h)
        return r

    def device_tensors(self) -> dict:
        """Zero-copy torch views of the device-resident person lists (what the NCCL gather sends)."""
        import torch
        v = _DeviceView()
        _check(self._lib.spg_get_device_view(self._h, C.byref(v)), "spg_get_device_view", self._h)
        dev = torch.device("cuda", self.device)
        N, cR, J, K = self.max_batch, self.capR, self.J, self.K

        def view(ptr, shape, typestr):
            return torch.as_tensor(_CudaView(ptr, shape, typestr), device=dev)

        return {"n_persons": view(v.n_persons, (N,), "<i4"),
                "people_xy": view(v.people_xy, (N, cR, J, 2), "<f8"),
                "people_score": view(v.people_score, (N, cR), "<f8"),
                "subset": view(v.subset, (N, cR, K + 2, 2), "<f8"),
                "status": view(v.status, (N,), "<i4"),
                "cand_count": view(v.cand_count, (N, self.L), "<i4"),
                "surv_count": view(v.surv_count, (N, self.L), "<i4")}
