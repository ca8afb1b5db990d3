"""GPU: the device COCOeval (improved_body_parts_b200/cocoeval.py) against the numpy port (oracle/cocoeval_port.py).

evalImgs equal field by field, eval arrays and stats bit for bit, ious within OKS_ULPS units in the last place (CUDA's
exp against numpy's, DESIGN §4).  Every seeded set first asserts that no OKS lies within that bound of a threshold or
of a different OKS of the same detection, the condition under which the matches cannot differ."""
import contextlib
import copy
import io
import json
import os

import numpy as np
import pytest
import torch

from cocoeval_cases import CASES
from improved_body_parts_b200 import cocoeval, synth
from oracle import cocoeval_port as port

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OKS_ULPS = 32


def _coco(ds):
    c = cocoeval.COCO()
    c.dataset = copy.deepcopy(ds)
    c.createIndex()
    return c


def _run(ds, res, setup=None, stream=None):
    gt = _coco(ds)
    dt = gt.loadRes(res)
    ref = port.COCOevalPort(gt, dt)
    dev = cocoeval.COCOeval(gt, dt, 'keypoints')
    for e in (ref, dev):
        if setup:
            setup(e.params)
    with contextlib.redirect_stdout(io.StringIO()) as out_ref:
        ref.evaluate()
        ref.accumulate()
        ref.summarize()
    with contextlib.redirect_stdout(io.StringIO()) as out_dev, torch.cuda.stream(stream or torch.cuda.current_stream()):
        dev.evaluate()
        dev.accumulate()
        dev.summarize()
    assert out_dev.getvalue() == out_ref.getvalue()
    return ref, dev


def assert_margin(ref):
    """No OKS within the bound of a threshold, or of another OKS of its detection that it does not equal."""
    thr = np.minimum(np.asarray(ref.params.iouThrs), 1 - 1e-10)
    for key, m in ref.ious.items():
        if len(m) == 0:
            continue
        tol = OKS_ULPS * np.spacing(np.abs(np.nan_to_num(m)))
        near = np.abs(m[..., None] - thr) <= tol[..., None]
        assert not near.any(), f"seed violates the margin: OKS near a threshold at {key}"
        for row, t in zip(m, tol):  # only OKS that can be matched compete
            live = row >= thr.min() - t
            d = np.abs(row[live, None] - row[None, live])
            assert not ((d > 0) & (d <= t[live, None])).any(), f"seed violates the margin: close OKS at {key}"


def assert_same(ref, dev):
    assert list(dev.ious) == list(ref.ious)
    for key, m in ref.ious.items():
        got = dev.ious[key]
        if len(m) == 0:
            assert len(got) == 0, key
            continue
        assert got.shape == m.shape, key
        both_nan = np.isnan(m) & np.isnan(got)
        diff = np.where(both_nan, 0, np.abs(got - m))
        assert (diff <= OKS_ULPS * np.spacing(np.abs(np.nan_to_num(m)))).all(), (key, got, m)
    assert len(dev.evalImgs) == len(ref.evalImgs)
    for j, (a, b) in enumerate(zip(ref.evalImgs, dev.evalImgs)):
        if a is None:
            assert b is None, j
            continue
        assert b is not None, j
        assert a.keys() == b.keys(), j
        for f in a:
            x, y = a[f], b[f]
            if isinstance(x, np.ndarray):
                assert x.shape == y.shape and np.array_equal(x, y), (j, f, x, y)
                assert np.asarray(x).dtype.kind == np.asarray(y).dtype.kind, (j, f)
            elif f == 'dtScores':
                assert np.array_equal(np.asarray(x, dtype=np.float64), np.asarray(y), equal_nan=True), (j, f)
            else:
                assert x == y, (j, f, x, y)
    for f in ('precision', 'recall', 'scores'):
        x, y = ref.eval[f], dev.eval[f]
        assert x.shape == y.shape, f
        assert np.array_equal(x.view(np.int64), y.view(np.int64)), (f, np.argwhere(x.view(np.int64) != y.view(np.int64))[:5])
    assert dev.eval['counts'] == ref.eval['counts']
    assert np.array_equal(np.asarray(ref.stats).view(np.int64), np.asarray(dev.stats).view(np.int64))


@pytest.mark.parametrize("name", sorted(CASES))
def test_hand_cases(name):
    ref, dev = _run(*CASES[name]())
    assert_same(ref, dev)


@pytest.mark.parametrize("n_images", [1, 37, 5000])
def test_seeded_sets(n_images):
    ds, res = synth.coco_keypoint_set(1000 + n_images, n_images)
    ref, dev = _run(ds, res)
    assert_margin(ref)
    assert_same(ref, dev)
    assert sum(e is not None for e in ref.evalImgs) > 0


def test_reference_format_results():
    """The detections format_results wrote for the reference's grouping (tests/golden/reference) against a seeded
    ground truth of the same images."""
    res = json.load(open(os.path.join(ROOT, "tests", "golden", "reference", "format_results.json")))
    ds, _ = synth.coco_keypoint_set(77, 40)
    ids = sorted({r["image_id"] for r in res})
    extra, _ = synth.coco_keypoint_set(78, len(ids), first_id=max(i["id"] for i in ds["images"]) + 1)
    remap = dict(zip([i["id"] for i in extra["images"]], ids))
    for a in extra["annotations"]:
        a["image_id"] = remap[a["image_id"]]
        a["id"] += 10 ** 6
    for i in extra["images"]:
        i["id"] = remap[i["id"]]
    ds["images"] += extra["images"]
    ds["annotations"] += extra["annotations"]
    ref, dev = _run(ds, res)
    assert_margin(ref)
    assert_same(ref, dev)


def test_nonfinite_keypoints():
    """Detections built from grouping's non-finite goldens: the peaks of maps with NaN values, whose refined coordinates
    are NaN where the peak's score is NaN (grouping carries them into the results), and their NaN scores."""
    ds, res = synth.coco_keypoint_set(5, 60)
    rows = []
    for name in ("border_nan_score_one", "nan_border_row0", "nan_border_row1"):
        c = np.load(os.path.join(ROOT, "tests", "golden", "nonfinite", f"{name}.npz"))["candidate"]
        xy = np.where(np.isnan(c[:, 2:3]), np.nan, c[:, :2])
        rows.append((xy, c[:, 2]))
    for j, r in enumerate(res[::4]):
        xy, sc = rows[j % len(rows)]
        pick = (np.arange(17) * 7 + j) % len(xy)
        kp = np.asarray(r["keypoints"], dtype=np.float64).reshape(17, 3)
        kp[::2, :2] = xy[pick][::2] + kp[::2, :2] * 0.0
        r["keypoints"] = kp.reshape(-1).tolist()
        if j % 5 == 0:
            r["score"] = float(np.nan if np.isnan(sc).any() else sc[0])
    assert any(np.isnan(r["keypoints"]).any() for r in res)
    ref, dev = _run(ds, res)
    assert_same(ref, dev)


@pytest.mark.parametrize("cat_ids", [None, [3, 1]])
def test_seeded_categories(cat_ids):
    """Three categories over 400 images (user-set catIds: two of them), against the port; the same bits again on
    another stream."""
    ds, res = synth.coco_keypoint_set(21, 400, categories=3)
    setup = None if cat_ids is None else (lambda p: setattr(p, "catIds", list(cat_ids)))
    ref, dev = _run(ds, res, setup)
    assert_margin(ref)
    assert dev.eval["counts"][2] == (3 if cat_ids is None else 2)
    assert_same(ref, dev)
    _, again = _run(ds, res, setup, stream=torch.cuda.Stream())
    for f in ('precision', 'recall', 'scores'):
        assert np.array_equal(dev.eval[f].view(np.int64), again.eval[f].view(np.int64)), f


def test_repeatable_across_calls_and_streams():
    ds, res = synth.coco_keypoint_set(9, 300)
    _, a = _run(ds, res)
    _, b = _run(ds, res, stream=torch.cuda.Stream())
    assert_same(a, b)
    for key, m in a.ious.items():
        assert np.array_equal(np.asarray(m).view(np.int64), np.asarray(b.ious[key]).view(np.int64)), key


def test_validation_through_launcher(tmp_path):
    """validation() of a stand-in evaluate module, run through prepare(device_cocoeval=True) without pycocotools,
    returns the device COCOeval with the port's stats."""
    from test_cocoeval_host import launch_stand_in
    ds, res = synth.coco_keypoint_set(11, 50)
    out = launch_stand_in(tmp_path, ds, res, device_cocoeval=True, run_validation=True)
    gt = _coco(ds)
    ref = port.COCOevalPort(gt, gt.loadRes(res))
    ref.params.imgIds = gt.getImgIds()
    with contextlib.redirect_stdout(io.StringIO()):
        ref.evaluate()
        ref.accumulate()
        ref.summarize()
    assert out["cls"] == "improved_body_parts_b200.cocoeval.COCOeval"
    assert out["stats"] == [float(v) for v in ref.stats]
    assert len(out["lines"]) == 10
