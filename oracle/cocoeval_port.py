"""CPU restatement of pycocotools 2.0.x's keypoint evaluation, the checker of improved_body_parts_b200/cocoeval.py.

``COCOevalPort(cocoGt, cocoDt)`` follows ``pycocotools.cocoeval.COCOeval`` for ``iouType='keypoints'`` loop for loop:
``_prepare``, ``computeOks``, ``evaluateImg``, ``accumulate`` and ``_summarizeKps``, in numpy, on one core.  ``load_res``
restates ``COCO.loadRes`` for keypoint results.  Both take any object with pycocotools' ``COCO`` interface
(``getImgIds``, ``getCatIds``, ``getAnnIds``, ``loadAnns``, ``dataset``).  Written from the behaviour pycocotools
documents and exhibits, not from its source; tests/test_cocoeval_port.py checks it by hand-computed cases and, where
pycocotools is installed, against it.
"""
from __future__ import annotations

import copy
from collections import defaultdict

import numpy as np

SIGMAS = np.array([.26, .25, .25, .35, .35, .79, .79, .72, .72, .62, .62, 1.07, 1.07, .87, .87, .89, .89]) / 10.0


class Params:
    """``Params(iouType='keypoints')``: ``setKpParams``."""

    def __init__(self):
        self.imgIds = []
        self.catIds = []
        self.iouThrs = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
        self.recThrs = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
        self.maxDets = [20]
        self.areaRng = [[0 ** 2, 1e5 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
        self.areaRngLbl = ['all', 'medium', 'large']
        self.useCats = 1
        self.kpt_oks_sigmas = SIGMAS.copy()
        self.iouType = 'keypoints'


def load_res(coco_gt, anns):
    """``COCO.loadRes`` for keypoint results: a dict with the GT's images and categories and the results as
    annotations, each with ``area`` and ``bbox`` from all its points' extent and ``id`` = its 1-based position."""
    anns = [dict(a) for a in anns]
    img_ids = set(coco_gt.getImgIds())
    for a in anns:
        if a['image_id'] not in img_ids:
            raise ValueError('Results do not correspond to current coco set')
    for i, a in enumerate(anns):
        s = a['keypoints']
        x, y = s[0::3], s[1::3]
        x0, x1, y0, y1 = np.min(x), np.max(x), np.min(y), np.max(y)
        a['area'] = (x1 - x0) * (y1 - y0)
        a['id'] = i + 1
        a['bbox'] = [x0, y0, x1 - x0, y1 - y0]
    return {'images': list(coco_gt.dataset['images']), 'categories': copy.deepcopy(coco_gt.dataset['categories']),
            'annotations': anns}


class COCOevalPort:
    def __init__(self, cocoGt, cocoDt):
        self.cocoGt, self.cocoDt = cocoGt, cocoDt
        self.params = Params()
        self.params.imgIds = sorted(cocoGt.getImgIds())
        self.params.catIds = sorted(cocoGt.getCatIds())
        self.evalImgs = []
        self.eval = {}
        self.ious = {}
        self.stats = []

    def _prepare(self):
        p = self.params
        gts = self.cocoGt.loadAnns(self.cocoGt.getAnnIds(imgIds=p.imgIds, catIds=p.catIds))
        dts = self.cocoDt.loadAnns(self.cocoDt.getAnnIds(imgIds=p.imgIds, catIds=p.catIds))
        self._gts, self._dts = defaultdict(list), defaultdict(list)
        for gt in gts:
            ig = gt['ignore'] if 'ignore' in gt else 0
            ig = 'iscrowd' in gt and gt['iscrowd']
            ig = (gt['num_keypoints'] == 0) or ig
            self._gts[gt['image_id'], gt['category_id']].append(dict(gt, ignore=ig))
        for dt in dts:
            self._dts[dt['image_id'], dt['category_id']].append(dt)

    def evaluate(self):
        p = self.params
        p.imgIds = list(np.unique(p.imgIds))
        p.catIds = list(np.unique(p.catIds))
        p.maxDets = sorted(p.maxDets)
        self._prepare()
        self.ious = {(i, c): self.computeOks(i, c) for i in p.imgIds for c in p.catIds}
        maxDet = p.maxDets[-1]
        self.evalImgs = [self.evaluateImg(i, c, a, maxDet) for c in p.catIds for a in p.areaRng for i in p.imgIds]
        self._paramsEval = copy.deepcopy(p)

    def computeOks(self, imgId, catId):
        p = self.params
        gts, dts = self._gts[imgId, catId], self._dts[imgId, catId]
        inds = np.argsort([-d['score'] for d in dts], kind='mergesort')
        dts = [dts[i] for i in inds]
        if len(dts) > p.maxDets[-1]:
            dts = dts[0:p.maxDets[-1]]
        if len(gts) == 0 or len(dts) == 0:
            return []
        ious = np.zeros((len(dts), len(gts)))
        vars = (np.asarray(p.kpt_oks_sigmas) * 2) ** 2
        k = len(vars)
        for j, gt in enumerate(gts):
            g = np.array(gt['keypoints'])
            xg, yg, vg = g[0::3], g[1::3], g[2::3]
            k1 = np.count_nonzero(vg > 0)
            bb = gt['bbox']
            x0, x1 = bb[0] - bb[2], bb[0] + bb[2] * 2
            y0, y1 = bb[1] - bb[3], bb[1] + bb[3] * 2
            for i, dt in enumerate(dts):
                d = np.array(dt['keypoints'])
                xd, yd = d[0::3], d[1::3]
                if k1 > 0:
                    dx, dy = xd - xg, yd - yg
                else:
                    z = np.zeros(k)
                    dx = np.max((z, x0 - xd), axis=0) + np.max((z, xd - x1), axis=0)
                    dy = np.max((z, y0 - yd), axis=0) + np.max((z, yd - y1), axis=0)
                e = (dx ** 2 + dy ** 2) / vars / (gt['area'] + np.spacing(1)) / 2
                if k1 > 0:
                    e = e[vg > 0]
                ious[i, j] = np.sum(np.exp(-e)) / e.shape[0]
        return ious

    def evaluateImg(self, imgId, catId, aRng, maxDet):
        p = self.params
        gt, dt = self._gts[imgId, catId], self._dts[imgId, catId]
        if len(gt) == 0 and len(dt) == 0:
            return None
        _ig = [1 if (g['ignore'] or (g['area'] < aRng[0] or g['area'] > aRng[1])) else 0 for g in gt]
        gtind = np.argsort(_ig, kind='mergesort')
        gt = [gt[i] for i in gtind]
        gtIg = np.array([_ig[i] for i in gtind])
        dtind = np.argsort([-d['score'] for d in dt], kind='mergesort')
        dt = [dt[i] for i in dtind[0:maxDet]]
        iscrowd = [int(o['iscrowd']) for o in gt]
        ious = self.ious[imgId, catId][:, gtind] if len(self.ious[imgId, catId]) > 0 else self.ious[imgId, catId]
        T, G, D = len(p.iouThrs), len(gt), len(dt)
        gtm, dtm, dtIg = np.zeros((T, G)), np.zeros((T, D)), np.zeros((T, D))
        if not len(ious) == 0:
            for tind, t in enumerate(p.iouThrs):
                for dind, d in enumerate(dt):
                    iou = min([t, 1 - 1e-10])
                    m = -1
                    for gind, g in enumerate(gt):
                        if gtm[tind, gind] > 0 and not iscrowd[gind]:
                            continue
                        if m > -1 and gtIg[m] == 0 and gtIg[gind] == 1:
                            break
                        if ious[dind, gind] < iou:
                            continue
                        iou = ious[dind, gind]
                        m = gind
                    if m == -1:
                        continue
                    dtIg[tind, dind] = gtIg[m]
                    dtm[tind, dind] = gt[m]['id']
                    gtm[tind, m] = d['id']
        a = np.array([d['area'] < aRng[0] or d['area'] > aRng[1] for d in dt]).reshape((1, len(dt)))
        dtIg = np.logical_or(dtIg, np.logical_and(dtm == 0, np.repeat(a, T, 0)))
        return {'image_id': imgId, 'category_id': catId, 'aRng': aRng, 'maxDet': maxDet,
                'dtIds': [d['id'] for d in dt], 'gtIds': [g['id'] for g in gt], 'dtMatches': dtm, 'gtMatches': gtm,
                'dtScores': [d['score'] for d in dt], 'gtIgnore': gtIg, 'dtIgnore': dtIg}

    def accumulate(self):
        p = self._paramsEval
        T, R, K, A, M = len(p.iouThrs), len(p.recThrs), len(p.catIds), len(p.areaRng), len(p.maxDets)
        precision, recall, scores = -np.ones((T, R, K, A, M)), -np.ones((T, K, A, M)), -np.ones((T, R, K, A, M))
        I0, A0 = len(p.imgIds), len(p.areaRng)
        for k in range(K):
            for a in range(A):
                for m, maxDet in enumerate(p.maxDets):
                    E = [self.evalImgs[k * A0 * I0 + a * I0 + i] for i in range(I0)]
                    E = [e for e in E if e is not None]
                    if len(E) == 0:
                        continue
                    dtScores = np.concatenate([e['dtScores'][0:maxDet] for e in E])
                    inds = np.argsort(-dtScores, kind='mergesort')
                    dtScoresSorted = dtScores[inds]
                    dtm = np.concatenate([e['dtMatches'][:, 0:maxDet] for e in E], axis=1)[:, inds]
                    dtIg = np.concatenate([e['dtIgnore'][:, 0:maxDet] for e in E], axis=1)[:, inds]
                    gtIg = np.concatenate([e['gtIgnore'] for e in E])
                    npig = np.count_nonzero(gtIg == 0)
                    if npig == 0:
                        continue
                    tps = np.logical_and(dtm, np.logical_not(dtIg))
                    fps = np.logical_and(np.logical_not(dtm), np.logical_not(dtIg))
                    tp_sum = np.cumsum(tps, axis=1).astype(dtype=np.float64)
                    fp_sum = np.cumsum(fps, axis=1).astype(dtype=np.float64)
                    for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
                        tp, fp = np.array(tp), np.array(fp)
                        nd = len(tp)
                        rc = tp / npig
                        pr = tp / (fp + tp + np.spacing(1))
                        q, ss = np.zeros((R,)), np.zeros((R,))
                        recall[t, k, a, m] = rc[-1] if nd else 0
                        pr, q = pr.tolist(), q.tolist()
                        for i in range(nd - 1, 0, -1):
                            if pr[i] > pr[i - 1]:
                                pr[i - 1] = pr[i]
                        inds = np.searchsorted(rc, p.recThrs, side='left')
                        try:
                            for ri, pi in enumerate(inds):
                                q[ri] = pr[pi]
                                ss[ri] = dtScoresSorted[pi]
                        except IndexError:
                            pass
                        precision[t, :, k, a, m] = np.array(q)
                        scores[t, :, k, a, m] = np.array(ss)
        self.eval = {'params': p, 'counts': [T, R, K, A, M], 'precision': precision, 'recall': recall, 'scores': scores}

    def summarize(self):
        p = self.params

        def one(ap, iouThr=None, areaRng='all', maxDets=20):
            iStr = ' {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}'
            iouStr = '{:0.2f}:{:0.2f}'.format(p.iouThrs[0], p.iouThrs[-1]) if iouThr is None else '{:0.2f}'.format(iouThr)
            aind = [i for i, lbl in enumerate(p.areaRngLbl) if lbl == areaRng]
            mind = [i for i, m in enumerate(p.maxDets) if m == maxDets]
            s = self.eval['precision' if ap else 'recall']
            if iouThr is not None:
                s = s[np.where(iouThr == p.iouThrs)[0]]
            s = s[:, :, :, aind, mind] if ap else s[:, :, aind, mind]
            mean_s = -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
            print(iStr.format('Average Precision' if ap else 'Average Recall', '(AP)' if ap else '(AR)', iouStr, areaRng,
                              maxDets, mean_s))
            return mean_s

        stats = np.zeros((10,))
        for i, args in enumerate([(1,), (1, .5), (1, .75), (1, None, 'medium'), (1, None, 'large'),
                                  (0,), (0, .5), (0, .75), (0, None, 'medium'), (0, None, 'large')]):
            stats[i] = one(*args)
        self.stats = stats
