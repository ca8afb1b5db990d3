"""Keypoint evaluation on the device: a drop-in ``COCOeval`` for ``iouType='keypoints'`` and a minimal ``COCO`` loader.

``evaluate.py``'s ``validation()`` (``:585-622``) scores a checkpoint with pycocotools: ``COCO(annFile)``,
``cocoGt.loadRes(resFile)``, then ``COCOeval(cocoGt, cocoDt, 'keypoints')`` and ``evaluate()``, ``accumulate()``,
``summarize()``.  pycocotools runs computeOks, the greedy matcher and the precision/recall accumulation in nested Python
loops on one core.  Here they are CUDA kernels (csrc/cocoeval.cuh) behind ``spg_coco_evaluate`` /
``spg_coco_accumulate``:

- ``COCOeval(cocoGt, cocoDt, iouType='keypoints')`` has pycocotools' ``params``, ``evaluate()``, ``accumulate()``,
  ``summarize()``, ``stats`` and ``eval``; ``evalImgs`` and ``ious`` are built from the device arrays when first read.
  It takes pycocotools' ``COCO`` objects or the ones below.  It honours user-set ``imgIds``, ``catIds``, ``iouThrs``,
  ``recThrs``, ``areaRng``, ``maxDets`` and ``kpt_oks_sigmas``; ``iouType`` other than ``'keypoints'`` and
  ``useCats = 0`` raise ``NotImplementedError``, malformed annotations ``ValueError`` before any launch.
- ``evalImgs`` and ``eval`` equal pycocotools' as long as no OKS lies within CUDA's ``exp`` rounding (DESIGN §4) of a
  threshold or of a competing OKS; ``ious`` agree to within that rounding.
- ``COCO(annotation_file)`` loads a COCO json with ``dataset``, ``imgs``, ``anns``, ``cats``, ``getImgIds``,
  ``getCatIds``, ``getAnnIds``, ``loadAnns``, ``loadImgs``, ``loadCats`` and ``loadRes`` for keypoint results, so that
  ``validation()`` runs where pycocotools is not installed.

The handle is the per-device one ``targets`` caches; there is no CPU path.
"""
from __future__ import annotations

import copy
import datetime
import json
from collections import defaultdict

import numpy as np
import torch

from . import grouping, targets

INT32_MAX = 2 ** 31 - 1
MAX_KEYPOINTS = 128


class COCO:
    """A COCO annotation file in memory with the lookups ``validation()`` and ``COCOeval`` use."""

    def __init__(self, annotation_file=None):
        self.dataset, self.anns, self.cats, self.imgs = {}, {}, {}, {}
        self.imgToAnns, self.catToImgs = defaultdict(list), defaultdict(list)
        if annotation_file is not None:
            with open(annotation_file) as f:
                dataset = json.load(f)
            if not isinstance(dataset, dict):
                raise ValueError(f"{annotation_file}: a COCO annotation file holds a JSON object, not {type(dataset).__name__}")
            self.dataset = dataset
            self.createIndex()

    def createIndex(self):
        self.anns, self.cats, self.imgs = {}, {}, {}
        self.imgToAnns, self.catToImgs = defaultdict(list), defaultdict(list)
        for ann in self.dataset.get('annotations', []):
            self.imgToAnns[ann['image_id']].append(ann)
            self.anns[ann['id']] = ann
        for img in self.dataset.get('images', []):
            self.imgs[img['id']] = img
        for cat in self.dataset.get('categories', []):
            self.cats[cat['id']] = cat
        for ann in self.dataset.get('annotations', []):
            if 'category_id' in ann:
                self.catToImgs[ann['category_id']].append(ann['image_id'])

    def getAnnIds(self, imgIds=[], catIds=[], areaRng=[], iscrowd=None):
        imgIds, catIds = _as_list(imgIds), _as_list(catIds)
        if len(imgIds) == len(catIds) == len(areaRng) == 0:
            anns = self.dataset.get('annotations', [])
        else:
            anns = self.dataset.get('annotations', []) if len(imgIds) == 0 else \
                [a for i in imgIds if i in self.imgToAnns for a in self.imgToAnns[i]]
            if len(catIds):
                cats = set(catIds)
                anns = [a for a in anns if a['category_id'] in cats]
            if len(areaRng):
                anns = [a for a in anns if areaRng[0] < a['area'] < areaRng[1]]
        if iscrowd is not None:
            return [a['id'] for a in anns if a['iscrowd'] == iscrowd]
        return [a['id'] for a in anns]

    def getCatIds(self, catNms=[], supNms=[], catIds=[]):
        catNms, supNms, catIds = _as_list(catNms), _as_list(supNms), _as_list(catIds)
        cats = self.dataset.get('categories', [])
        if len(catNms):
            cats = [c for c in cats if c['name'] in catNms]
        if len(supNms):
            cats = [c for c in cats if c['supercategory'] in supNms]
        if len(catIds):
            cats = [c for c in cats if c['id'] in catIds]
        return [c['id'] for c in cats]

    def getImgIds(self, imgIds=[], catIds=[]):
        imgIds, catIds = _as_list(imgIds), _as_list(catIds)
        if len(imgIds) == len(catIds) == 0:
            return list(self.imgs.keys())
        ids = set(imgIds)
        for i, c in enumerate(catIds):
            ids = set(self.catToImgs[c]) if i == 0 and len(ids) == 0 else ids & set(self.catToImgs[c])
        return list(ids)

    def loadAnns(self, ids=[]):
        return [self.anns[i] for i in _as_list(ids)]

    def loadCats(self, ids=[]):
        return [self.cats[i] for i in _as_list(ids)]

    def loadImgs(self, ids=[]):
        return [self.imgs[i] for i in _as_list(ids)]

    def loadRes(self, resFile):
        """Keypoint results (a json file's name or a list of dicts) as a ``COCO``: each result's ``area`` and ``bbox``
        from the extent of all its points, the ones ``format_results`` writes as ``(0, 0, 0)`` included, and ``id`` its
        1-based position in the list.  A result for an image the ground truth lacks raises ``ValueError``."""
        if isinstance(resFile, str):
            with open(resFile) as f:
                anns = json.load(f)
        else:
            anns = resFile
        if not isinstance(anns, list):
            raise ValueError(f"results must be a list of dicts, got {type(anns).__name__}")
        anns = [dict(a) for a in anns]
        unknown = {a.get('image_id') for a in anns} - set(self.imgs)
        if unknown:
            raise ValueError(f"results for images the ground truth does not have: {sorted(unknown, key=str)[:5]}")
        for i, a in enumerate(anns):
            if 'keypoints' not in a:
                raise NotImplementedError("only keypoint results are supported (bbox and segm evaluation are not)")
            s = a['keypoints']
            x, y = s[0::3], s[1::3]
            if len(x) == 0:
                raise ValueError(f"result {i}: no keypoints")
            x0, x1, y0, y1 = np.min(x), np.max(x), np.min(y), np.max(y)
            a['area'] = (x1 - x0) * (y1 - y0)
            a['id'] = i + 1
            a['bbox'] = [x0, y0, x1 - x0, y1 - y0]
        res = COCO()
        res.dataset = {'images': list(self.dataset.get('images', [])),
                       'categories': copy.deepcopy(self.dataset.get('categories', [])), 'annotations': anns}
        res.createIndex()
        return res


def _as_list(v):
    return list(v) if isinstance(v, (list, tuple, np.ndarray, range)) else [v]


class Params:
    """pycocotools' ``Params(iouType='keypoints')``."""

    def __init__(self, iouType='keypoints'):
        if iouType != 'keypoints':
            raise NotImplementedError(f"iouType {iouType!r}: only 'keypoints' is evaluated on the device")
        self.imgIds = []
        self.catIds = []
        self.iouThrs = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
        self.recThrs = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
        self.maxDets = [20]
        self.areaRng = [[0 ** 2, 1e5 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
        self.areaRngLbl = ['all', 'medium', 'large']
        self.useCats = 1
        self.kpt_oks_sigmas = np.array([.26, .25, .25, .35, .35, .79, .79, .72, .72, .62, .62, 1.07, 1.07, .87, .87,
                                        .89, .89]) / 10.0
        self.iouType = iouType
        self.useSegm = None


def _column(anns, key, what, kind="f", width=None):
    """``ann[key]`` of every annotation as one float64 (``kind`` "f") or int64 (``kind`` "i") array, ``[n]`` or
    ``[n, width]``; ``ValueError`` for a missing key, a non-numeric value or a wrong length."""
    try:
        vals = [a[key] for a in anns]
    except KeyError:
        raise ValueError(f"{what}: an annotation has no {key!r}") from None
    except TypeError:
        raise ValueError(f"{what}: annotations must be dicts") from None
    try:
        arr = np.array(vals) if vals else np.zeros((0,) if width is None else (0, width))
    except ValueError:
        raise ValueError(f"{what}: {key!r} has entries of different lengths") from None
    shape = (len(anns),) if width is None else (len(anns), width)
    if arr.shape != shape:
        raise ValueError(f"{what}: {key!r} must be {'a number' if width is None else f'{width} numbers'} per annotation, "
                         f"got an array of shape {arr.shape}")
    if len(anns) and (arr.dtype.kind not in ("b", "i", "u", "f") or (kind == "i" and arr.dtype.kind == "f")):
        raise ValueError(f"{what}: {key!r} must be {'integers' if kind == 'i' else 'numbers'}, got {arr.dtype}")
    return arr.astype(np.int64 if kind == "i" else np.float64)


class _Packed:
    """One evaluate() call's inputs on the host: per unit (category-major, images in sorted order) the ground truths
    and detections in annotation order, and the sizes every device array is allocated from."""

    def __init__(self, gts, dts, img_ids, cat_ids, n_kpt, max_det):
        I, K = len(img_ids), len(cat_ids)
        img_ix, cat_ix = {v: i for i, v in enumerate(img_ids)}, {v: k for k, v in enumerate(cat_ids)}

        def units(anns, what):
            u = np.empty(len(anns), np.int64)
            for j, a in enumerate(anns):
                try:
                    i, k = img_ix.get(a['image_id']), cat_ix.get(a['category_id'])
                except (KeyError, TypeError):
                    raise ValueError(f"{what}: annotation {j} lacks image_id or category_id") from None
                u[j] = -1 if i is None or k is None else k * I + i
            keep = np.flatnonzero(u >= 0)
            order = keep[np.argsort(u[keep], kind="stable")]
            return [anns[j] for j in order], u[order]

        gts, gu = units(gts, "ground truth")
        dts, du = units(dts, "detections")
        U = I * K
        self.n_images, self.n_cats, self.n_units = I, K, U
        self.gt_kpts = _column(gts, 'keypoints', "ground truth", width=3 * n_kpt)
        self.gt_bbox = _column(gts, 'bbox', "ground truth", width=4)
        self.gt_area = _column(gts, 'area', "ground truth")
        self.gt_id = _column(gts, 'id', "ground truth", kind="i")
        crowd = _column(gts, 'iscrowd', "ground truth")
        nkp = _column(gts, 'num_keypoints', "ground truth")
        if np.isnan(crowd).any():
            raise ValueError("ground truth: 'iscrowd' is NaN")
        self.gt_flags = (((crowd != 0) | (nkp == 0)) * grouping.COCO_IGNORE +
                         (np.trunc(crowd) != 0) * grouping.COCO_CROWD).astype(np.uint8)
        self.dt_kpts = _column(dts, 'keypoints', "detections", width=3 * n_kpt)
        self.dt_area = _column(dts, 'area', "detections")
        self.dt_score = _column(dts, 'score', "detections")
        self.dt_id = _column(dts, 'id', "detections", kind="i")
        self.gt_count = np.bincount(gu, minlength=U).astype(np.int64)
        self.dt_count = np.bincount(du, minlength=U).astype(np.int64)
        self.kept_count = np.minimum(self.dt_count, max_det)
        self.dt_unit = du.astype(np.int32)
        start = lambda c: np.concatenate([[0], np.cumsum(c)])  # noqa: E731
        self.gt_start, self.dt_start = start(self.gt_count), start(self.dt_count)
        self.kept_start, self.iou_start = start(self.kept_count), start(self.kept_count * self.gt_count)
        self.n_gt, self.n_dt = len(gts), len(dts)
        self.n_kept, self.n_ious = int(self.kept_start[-1]), int(self.iou_start[-1])


class COCOeval:
    """pycocotools' ``COCOeval`` for ``iouType='keypoints'``, with the per-image matching and the accumulation on the
    device.  ``device`` defaults to torch's current CUDA device."""

    def __init__(self, cocoGt=None, cocoDt=None, iouType='keypoints', device=None):
        if iouType != 'keypoints':
            raise NotImplementedError(f"iouType {iouType!r}: only 'keypoints' is evaluated on the device")
        self.cocoGt, self.cocoDt = cocoGt, cocoDt
        self.params = Params(iouType)
        self._paramsEval = {}
        self.eval = {}
        self.stats = []
        self._device = device
        self._dev = None  # the last evaluate()'s device arrays
        self._evalImgs = self._ious = None
        if cocoGt is not None:
            self.params.imgIds = sorted(cocoGt.getImgIds())
            self.params.catIds = sorted(cocoGt.getCatIds())

    # -- evaluate ---------------------------------------------------------------------------------------------------
    def _tables(self, p):
        """The float64 / int32 tables the kernels read, checked."""
        if p.useCats != 1:
            raise NotImplementedError("useCats = 0 is not supported: keypoint evaluation is per category")
        iou = np.asarray(p.iouThrs, dtype=np.float64).reshape(-1)
        rec = np.asarray(p.recThrs, dtype=np.float64).reshape(-1)
        area = np.asarray(p.areaRng, dtype=np.float64)
        sig = np.asarray(p.kpt_oks_sigmas, dtype=np.float64)
        md = np.asarray(p.maxDets)
        if len(iou) == 0 or len(rec) == 0:
            raise ValueError("params.iouThrs and params.recThrs must not be empty")
        if area.ndim != 2 or area.shape[1] != 2 or area.shape[0] == 0:
            raise ValueError(f"params.areaRng must be a list of [lo, hi] pairs, got shape {area.shape}")
        if sig.ndim != 1 or not 1 <= len(sig) <= MAX_KEYPOINTS:
            raise ValueError(f"params.kpt_oks_sigmas must hold 1..{MAX_KEYPOINTS} sigmas, got shape {sig.shape}")
        if md.ndim != 1 or len(md) == 0 or md.dtype.kind not in "iu" or (md < 0).any() or (md > INT32_MAX).any():
            raise ValueError(f"params.maxDets must be non-negative integers, got {p.maxDets!r}")
        return iou, rec, area, md.astype(np.int32), (sig * 2) ** 2

    def evaluate(self):
        p = self.params
        p.imgIds = list(np.unique(p.imgIds))
        p.catIds = list(np.unique(p.catIds))
        p.maxDets = sorted(p.maxDets)
        iou, rec, area, md, kvars = self._tables(p)
        gts = self.cocoGt.loadAnns(self.cocoGt.getAnnIds(imgIds=p.imgIds, catIds=p.catIds))
        dts = self.cocoDt.loadAnns(self.cocoDt.getAnnIds(imgIds=p.imgIds, catIds=p.catIds))
        pk = _Packed(gts, dts, p.imgIds, p.catIds, len(kvars), int(md[-1]))
        T, A = len(iou), len(area)
        if self._device is None:
            self._device = torch.cuda.current_device()
        for what, n in (("units", pk.n_units + 1), ("OKS entries", pk.n_ious), ("ground truths x thresholds x areas",
                        pk.n_gt * T * A), ("detections x thresholds x areas", pk.n_dt * T * A * len(md))):
            if n > INT32_MAX:
                raise ValueError(f"{what}: {n} is above 2^31 - 1")
        dev = torch.device("cuda", self._device)
        put = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(dev)  # noqa: E731
        i32 = np.int32
        d = dict(iou_thrs=put(iou, np.float64), rec_thrs=put(rec, np.float64), area_rng=put(area, np.float64),
                 max_dets=put(md, i32), kpt_vars=put(kvars, np.float64),
                 gt_start=put(pk.gt_start, i32), dt_start=put(pk.dt_start, i32), kept_start=put(pk.kept_start, i32),
                 iou_start=put(pk.iou_start, i32), dt_unit=put(pk.dt_unit, i32), gt_kpts=put(pk.gt_kpts, np.float64),
                 gt_bbox=put(pk.gt_bbox, np.float64), gt_area=put(pk.gt_area, np.float64), gt_id=put(pk.gt_id, np.int64),
                 gt_flags=put(pk.gt_flags, np.uint8), dt_kpts=put(pk.dt_kpts, np.float64),
                 dt_area=put(pk.dt_area, np.float64), dt_score=put(pk.dt_score, np.float64),
                 dt_id=put(pk.dt_id, np.int64))
        e = dict(ious=torch.empty(pk.n_ious, dtype=torch.float64, device=dev),
                 dt_order=torch.empty(pk.n_dt, dtype=torch.int32, device=dev),
                 dt_rank=torch.empty(pk.n_dt, dtype=torch.int32, device=dev),
                 cat_order=torch.empty(pk.n_dt, dtype=torch.int32, device=dev),
                 gt_order=torch.empty((A, pk.n_gt), dtype=torch.int32, device=dev),
                 gt_ignore=torch.empty((A, pk.n_gt), dtype=torch.uint8, device=dev),
                 gt_matches=torch.empty((A, T, pk.n_gt), dtype=torch.int64, device=dev),
                 dt_matches=torch.empty((A, T, pk.n_kept), dtype=torch.int64, device=dev),
                 dt_ignore=torch.empty((A, T, pk.n_kept), dtype=torch.uint8, device=dev))
        params = np.zeros(1, grouping.COCO_PARAMS)
        for f in ("iou_thrs", "rec_thrs", "area_rng", "max_dets", "kpt_vars"):
            params[f] = d[f].data_ptr()
        params["n_iou"], params["n_rec"], params["n_area"], params["n_max_dets"], params["n_kpt"] = \
            T, len(rec), A, len(md), len(kvars)
        data = np.zeros(1, grouping.COCO_DATA)
        for f in grouping.COCO_DATA.names[6:]:
            data[f] = d[f].data_ptr()
        for f in ("n_images", "n_cats", "n_gt", "n_dt", "n_kept", "n_ious"):
            data[f] = getattr(pk, f)
        ev = np.zeros(1, grouping.COCO_EVAL)
        for f in grouping.COCO_EVAL.names:
            ev[f] = e[f].data_ptr()
        g = targets._Device.for_device(self._device)
        g.coco_evaluate(params, data, ev)
        self._dev = dict(pk=pk, tensors=d, eval=e, records=(params, data, ev), grouper=g, T=T, A=A, R=len(rec),
                         M=len(md))
        self._evalImgs = self._ious = None
        self._paramsEval = copy.deepcopy(p)

    def _host(self):
        """The device results of evaluate() on the host, once."""
        dv = self._dev
        if dv is None:
            raise RuntimeError("Please run evaluate() first")
        if "host" not in dv:
            dv["host"] = {k: v.cpu().numpy() for k, v in dv["eval"].items()}
        return dv["host"]

    @property
    def ious(self):
        """``{(imgId, catId): [D, G] OKS matrix, or [] when either list is empty}``, as pycocotools' ``ious``."""
        if self._ious is None and self._dev is not None:
            pk, h, p = self._dev["pk"], self._host(), self._paramsEval
            out = {}
            for i, img in enumerate(p.imgIds):
                for k, cat in enumerate(p.catIds):
                    u = k * pk.n_images + i
                    D, G = int(pk.kept_count[u]), int(pk.gt_count[u])
                    out[img, cat] = h["ious"][pk.iou_start[u]:pk.iou_start[u + 1]].reshape(D, G) if D and G else []
            self._ious = out
        return {} if self._ious is None else self._ious

    @property
    def evalImgs(self):
        """pycocotools' per (category, area range, image) list of evaluateImg results (``None`` for an image with
        neither ground truth nor detections)."""
        if self._evalImgs is None and self._dev is not None:
            pk, h, p = self._dev["pk"], self._host(), self._paramsEval
            max_det = p.maxDets[-1]
            out = []
            for k, cat in enumerate(p.catIds):
                for a, rng in enumerate(p.areaRng):
                    for i, img in enumerate(p.imgIds):
                        u = k * pk.n_images + i
                        g0, g1, d0 = pk.gt_start[u], pk.gt_start[u + 1], pk.dt_start[u]
                        k0, k1 = pk.kept_start[u], pk.kept_start[u + 1]
                        if g0 == g1 and pk.dt_count[u] == 0:
                            out.append(None)
                            continue
                        dets = h["dt_order"][d0:d0 + (k1 - k0)]
                        out.append({'image_id': img, 'category_id': cat, 'aRng': rng, 'maxDet': max_det,
                                    'dtIds': pk.dt_id[dets].tolist(), 'gtIds': pk.gt_id[h["gt_order"][a, g0:g1]].tolist(),
                                    'dtMatches': h["dt_matches"][a, :, k0:k1].astype(np.float64),
                                    'gtMatches': h["gt_matches"][a, :, g0:g1].astype(np.float64),
                                    'dtScores': pk.dt_score[dets].tolist(),
                                    # np.array of an empty list is float64, as pycocotools' gtIgnore of no GT
                                    'gtIgnore': h["gt_ignore"][a, g0:g1].astype(np.int64) if g1 > g0 else np.array([]),
                                    'dtIgnore': h["dt_ignore"][a, :, k0:k1].astype(bool)})
            self._evalImgs = out
        return [] if self._evalImgs is None else self._evalImgs

    # -- accumulate / summarize -------------------------------------------------------------------------------------
    def accumulate(self, p=None):
        """Precision, recall and scores of every (threshold, recall threshold, category, area range, maxDet) from the
        last evaluate().  ``p`` (default: ``params``, as in pycocotools) must hold the tables evaluate() ran with:
        accumulating a different selection raises ``ValueError`` (run evaluate() again with those params)."""
        dv = self._dev
        if dv is None:
            raise RuntimeError("Please run evaluate() first")
        pe = self._paramsEval
        p = self.params if p is None else p
        for f in ("imgIds", "catIds", "iouThrs", "recThrs", "maxDets", "areaRng", "useCats"):
            a, b = getattr(p, f, None), getattr(pe, f)
            try:
                same = np.shape(a) == np.shape(b) and np.array_equal(np.asarray(a, np.float64), np.asarray(b, np.float64),
                                                                     equal_nan=True)
            except (TypeError, ValueError):
                same = False
            if not same:
                raise ValueError(f"accumulate(): params.{f} differs from the one evaluate() ran with; run evaluate() again")
        T, R, K, A, M = dv["T"], dv["R"], len(pe.catIds), dv["A"], dv["M"]
        dev = torch.device("cuda", self._device)
        prec = torch.empty((T, R, K, A, M), dtype=torch.float64, device=dev)
        rec = torch.empty((T, K, A, M), dtype=torch.float64, device=dev)
        sc = torch.empty((T, R, K, A, M), dtype=torch.float64, device=dev)
        dv["grouper"].coco_accumulate(*dv["records"], prec.data_ptr(), rec.data_ptr(), sc.data_ptr())
        self.eval = {'params': pe, 'counts': [T, R, K, A, M],
                     'date': datetime.datetime.now().strftime('%Y-%m-%d %H:%M:%S'),
                     'precision': prec.cpu().numpy(), 'recall': rec.cpu().numpy(), 'scores': sc.cpu().numpy()}

    def summarize(self):
        """The ten lines of pycocotools' ``_summarizeKps``, printed; ``stats`` holds their values."""
        if not self.eval:
            raise RuntimeError("Please run accumulate() first")
        p = self.params

        def line(ap=1, iouThr=None, areaRng='all', maxDets=20):
            iStr = ' {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}'
            titleStr = 'Average Precision' if ap == 1 else 'Average Recall'
            typeStr = '(AP)' if ap == 1 else '(AR)'
            iouStr = '{:0.2f}:{:0.2f}'.format(p.iouThrs[0], p.iouThrs[-1]) if iouThr is None else '{:0.2f}'.format(iouThr)
            aind = [i for i, aRng in enumerate(p.areaRngLbl) if aRng == areaRng]
            mind = [i for i, mDet in enumerate(p.maxDets) if mDet == maxDets]
            s = self.eval['precision'] if ap == 1 else self.eval['recall']
            if iouThr is not None:
                s = s[np.where(iouThr == p.iouThrs)[0]]
            s = s[:, :, :, aind, mind] if ap == 1 else s[:, :, aind, mind]
            mean_s = -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
            print(iStr.format(titleStr, typeStr, iouStr, areaRng, maxDets, mean_s))
            return mean_s

        stats = np.zeros((10,))
        stats[0] = line(1, maxDets=20)
        stats[1] = line(1, maxDets=20, iouThr=.5)
        stats[2] = line(1, maxDets=20, iouThr=.75)
        stats[3] = line(1, maxDets=20, areaRng='medium')
        stats[4] = line(1, maxDets=20, areaRng='large')
        stats[5] = line(0, maxDets=20)
        stats[6] = line(0, maxDets=20, iouThr=.5)
        stats[7] = line(0, maxDets=20, iouThr=.75)
        stats[8] = line(0, maxDets=20, areaRng='medium')
        stats[9] = line(0, maxDets=20, areaRng='large')
        self.stats = stats
