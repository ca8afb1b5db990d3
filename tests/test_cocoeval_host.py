"""CPU: the host side of keypoint evaluation (improved_body_parts_b200/cocoeval.py) -- the minimal COCO loader, the
checks that run before any launch, the summarize text -- and the launcher's --device-cocoeval binding on a stand-in
``evaluate`` module."""
import contextlib
import copy
import io
import json
import math
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from cocoeval_cases import dataset, det, gt, pts
from improved_body_parts_b200 import cocoeval
from oracle import cocoeval_port as port

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _coco(ds):
    c = cocoeval.COCO()
    c.dataset = ds
    c.createIndex()
    return c


def test_loader_reads_a_file_and_indexes_it(tmp_path):
    a = pts(100, 100)
    ds = dataset([gt(5, 2, a), gt(3, 1, a, crowd=1), gt(4, 2, pts(300, 100))], [2, 1])
    f = tmp_path / "ann.json"
    f.write_text(json.dumps(ds))
    c = cocoeval.COCO(str(f))
    assert c.getImgIds() == [2, 1] and c.getCatIds() == [1]
    assert c.getAnnIds(imgIds=[1, 2], catIds=[1]) == [3, 5, 4]
    assert c.getAnnIds(imgIds=2) == [5, 4] and c.getAnnIds(iscrowd=1) == [3]
    assert [x["id"] for x in c.loadAnns([4, 3])] == [4, 3]
    assert c.loadImgs(1)[0]["file_name"] == "1.jpg" and c.imgs[2]["id"] == 2 and set(c.anns) == {3, 4, 5}


def test_load_res_area_from_all_points_and_ids(tmp_path):
    ds = dataset([gt(1, 1, pts(100, 100))], [1, 2])
    c = _coco(ds)
    p = pts(100, 100).astype(float)
    p[4] = 0.0  # a missing joint, written as (0, 0, 0)
    res = [det(1, p, 0.5) | {"id": 99}, det(2, pts(50, 60), 0.25)]
    res[0]["keypoints"][14] = 0
    f = tmp_path / "res.json"
    f.write_text(json.dumps(res))
    r = c.loadRes(str(f))
    a0 = r.anns[1]
    x, y = np.array(res[0]["keypoints"][0::3]), np.array(res[0]["keypoints"][1::3])
    assert a0["area"] == (x.max() - 0.0) * (y.max() - 0.0)  # the (0, 0) point sets the minimum
    assert a0["bbox"] == [0.0, 0.0, x.max(), y.max()]
    assert sorted(r.anns) == [1, 2] and r.anns[2]["image_id"] == 2
    assert r.getImgIds() == [1, 2] and r.getCatIds() == [1]
    assert res[0]["id"] == 99, "the caller's list is not modified"
    p_ = port.load_res(c, res)
    assert [(q["id"], q["area"], q["bbox"]) for q in p_["annotations"]] == \
           [(r.anns[i]["id"], r.anns[i]["area"], r.anns[i]["bbox"]) for i in (1, 2)]


def test_load_res_rejects_unknown_images_and_other_result_types():
    c = _coco(dataset([gt(1, 1, pts(100, 100))], [1]))
    with pytest.raises(ValueError, match="ground truth does not have"):
        c.loadRes([det(7, pts(1, 1), 0.5)])
    with pytest.raises(NotImplementedError):
        c.loadRes([{"image_id": 1, "category_id": 1, "bbox": [0, 0, 1, 1], "score": 1.0}])
    with pytest.raises(ValueError):
        c.loadRes({"not": "a list"})


def _eval(ds, res):
    c = _coco(ds)
    return cocoeval.COCOeval(c, c.loadRes(res), 'keypoints')


@pytest.mark.parametrize("bad, match", [
    (lambda g, d: g[0].update(keypoints=[1] * 50), "51 numbers"),
    (lambda g, d: d[0].update(keypoints=d[0]["keypoints"][:-3]), "51 numbers"),
    (lambda g, d: g[0].update(keypoints=["1"] * 51), "numbers"),
    (lambda g, d: g[0].update(bbox=[1, 2, 3]), "4 numbers"),
    (lambda g, d: g[0].pop("iscrowd"), "iscrowd"),
    (lambda g, d: g[0].update(num_keypoints=None), "num_keypoints"),
    (lambda g, d: g[0].update(id=1.5), "integers"),
    (lambda g, d: d[0].update(score="high"), "score"),
    (lambda g, d: g[0].update(iscrowd=math.nan), "NaN"),
])
def test_malformed_annotations_raise_before_any_launch(bad, match):
    a = pts(100, 100)
    ds = dataset([gt(1, 1, a)], [1])
    e = _eval(ds, [det(1, a, 0.5)])
    bad(e.cocoGt.dataset["annotations"], e.cocoDt.dataset["annotations"])
    e.cocoGt.createIndex()
    e.cocoDt.createIndex()
    with pytest.raises(ValueError, match=match):
        e.evaluate()


def test_unsupported_settings():
    c = _coco(dataset([gt(1, 1, pts(100, 100))], [1]))
    with pytest.raises(NotImplementedError):
        cocoeval.COCOeval(c, c, 'bbox')
    e = cocoeval.COCOeval(c, c.loadRes([det(1, pts(100, 100), 0.5)]))
    e.params.useCats = 0
    with pytest.raises(NotImplementedError):
        e.evaluate()
    for field, value in (("kpt_oks_sigmas", np.ones(129)), ("maxDets", [-1]), ("areaRng", [[0, 1, 2]])):
        e = cocoeval.COCOeval(c, c.loadRes([det(1, pts(100, 100), 0.5)]))
        setattr(e.params, field, value)
        with pytest.raises(ValueError):
            e.evaluate()
    with pytest.raises(RuntimeError, match="evaluate"):
        e.accumulate()
    with pytest.raises(RuntimeError, match="accumulate"):
        e.summarize()


def test_default_params_are_pycocotools_keypoint_params():
    p = cocoeval.Params()
    q = port.Params()
    for f in ("iouThrs", "recThrs", "kpt_oks_sigmas"):
        assert np.array_equal(getattr(p, f), getattr(q, f))
    assert p.maxDets == [20] and p.areaRng == [[0, 1e10], [1024, 9216], [9216, 1e10]]
    assert p.areaRngLbl == ['all', 'medium', 'large'] and p.useCats == 1


def test_summarize_text():
    """The ten _summarizeKps lines from a known eval: threshold rows chosen by equality, means over s > -1."""
    c = _coco(dataset([gt(1, 1, pts(100, 100))], [1]))
    e = cocoeval.COCOeval(c, c)
    p = e.params
    prec = np.full((10, 101, 1, 3, 1), 0.5)
    prec[0] = 1.0       # IoU 0.50
    prec[5] = 0.25      # IoU 0.75
    prec[:, :, :, 2] = -1  # large: nothing
    rec = np.full((10, 1, 3, 1), 0.75)
    rec[:, :, 1] = -1
    e.eval = {'precision': prec, 'recall': rec, 'scores': prec}
    with contextlib.redirect_stdout(io.StringIO()) as out:
        e.summarize()
    lines = out.getvalue().splitlines()
    assert lines[0] == ' Average Precision  (AP) @[ IoU=0.50:0.95 | area=   all | maxDets= 20 ] = 0.525'
    assert lines[1] == ' Average Precision  (AP) @[ IoU=0.50      | area=   all | maxDets= 20 ] = 1.000'
    assert lines[2] == ' Average Precision  (AP) @[ IoU=0.75      | area=   all | maxDets= 20 ] = 0.250'
    assert lines[4] == ' Average Precision  (AP) @[ IoU=0.50:0.95 | area= large | maxDets= 20 ] = -1.000'
    assert lines[8] == ' Average Recall     (AR) @[ IoU=0.50:0.95 | area=medium | maxDets= 20 ] = -1.000'
    assert lines[9] == ' Average Recall     (AR) @[ IoU=0.50:0.95 | area= large | maxDets= 20 ] = 0.750'
    assert len(lines) == 10 and e.stats[4] == -1 and e.stats[0] == np.mean(prec[:, :, :, 0, 0])
    ref = port.COCOevalPort(c, c)
    ref.eval = e.eval
    with contextlib.redirect_stdout(io.StringIO()) as out2:
        ref.summarize()
    assert out2.getvalue() == out.getvalue() and np.array_equal(ref.stats, e.stats)
    assert p.iouThrs[5] == 0.75


# ---- the launcher ------------------------------------------------------------------------------------------------

_STAND_IN = r'''
import json, os, sys
import pycocotools.coco, pycocotools.cocoeval, matplotlib.pyplot, configobj, apex
from pycocotools.coco import COCO
from pycocotools.cocoeval import COCOeval

os.environ["CUDA_VISIBLE_DEVICES"] = "0"
limbSeq = [(1, 0), (1, 2), (2, 3)]


def find_peaks(heatmap, params):
    raise AssertionError("stand-in find_peaks called")


def find_connections(all_peaks, paf, image_width, params):
    raise AssertionError("stand-in find_connections called")


def find_people(connection_all, special_k, all_peaks, params):
    raise AssertionError("stand-in find_people called")


def predict_many(coco, images_dir, validation_ids, *rest):
    return json.load(open(os.environ["STAND_IN_RESULTS"]))


def format_results(keypoints, resFile):
    json.dump(keypoints, open(resFile, "w"))


def validation(model, dump_name, validation_ids=None, dataset="val2017"):
    annType = "keypoints"
    cocoGt = COCO(os.environ["STAND_IN_ANNOTATIONS"])
    if validation_ids == None:
        validation_ids = cocoGt.getImgIds()[:500]
    resFile = os.path.join(os.environ["STAND_IN_OUT"], "%s_results.json" % dump_name)
    keypoints = predict_many(cocoGt, None, validation_ids)
    format_results(keypoints, resFile)
    cocoDt = cocoGt.loadRes(resFile)
    cocoEval = COCOeval(cocoGt, cocoDt, annType)
    cocoEval.params.imgIds = validation_ids
    cocoEval.evaluate()
    cocoEval.accumulate()
    cocoEval.summarize()
    return cocoEval
'''

_CHILD = r'''
import contextlib, io, json, os, sys
sys.path.insert(0, {root!r})
import importlib.util
spec = importlib.util.spec_from_file_location("run_evaluate_b200", os.path.join({root!r}, "tools", "run_evaluate_b200.py"))
L = importlib.util.module_from_spec(spec); spec.loader.exec_module(L)
ev = L.prepare({ref!r}, device_cocoeval={flag!r})
out = dict(stubbed=ev.__spg_stubbed__, COCOeval=f"{{ev.COCOeval.__module__}}.{{ev.COCOeval.__qualname__}}",
           COCO=f"{{ev.COCO.__module__}}.{{ev.COCO.__qualname__}}")
if {run!r}:
    with contextlib.redirect_stdout(io.StringIO()) as text:
        e = ev.validation(None, "stand_in")
    out.update(cls=f"{{type(e).__module__}}.{{type(e).__qualname__}}", stats=[float(v) for v in e.stats],
               lines=[l for l in text.getvalue().splitlines() if l.startswith(" Average")])
print("RESULT " + json.dumps(out))
'''


def launch_stand_in(tmp_path, ds, res, device_cocoeval, run_validation=False):
    """Run the launcher's prepare() on the stand-in in a child process; what it bound (and validation()'s result)."""
    ref = tmp_path / "checkout"
    (ref / "utils").mkdir(parents=True, exist_ok=True)
    (ref / "evaluate.py").write_text(_STAND_IN)
    shutil.copy(os.path.join(ROOT, "tests", "golden", "reference_utils_config.ini"), ref / "utils" / "config")
    (tmp_path / "ann.json").write_text(json.dumps(ds))
    (tmp_path / "res.json").write_text(json.dumps(res))
    env = dict(os.environ, STAND_IN_ANNOTATIONS=str(tmp_path / "ann.json"), STAND_IN_RESULTS=str(tmp_path / "res.json"),
               STAND_IN_OUT=str(tmp_path))
    code = _CHILD.format(root=ROOT, ref=str(ref), flag=device_cocoeval, run=run_validation)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, cwd=str(tmp_path),
                       env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(next(line for line in r.stdout.splitlines() if line.startswith("RESULT "))[7:])


def test_launcher_flag_binds_the_device_cocoeval(tmp_path):
    ds = dataset([gt(1, 1, pts(100, 100))], [1])
    default = launch_stand_in(tmp_path / "a", ds, [], device_cocoeval=False)
    bound = launch_stand_in(tmp_path / "b", ds, [], device_cocoeval=True)
    stubbed = "pycocotools.coco" in default["stubbed"]
    assert default["COCOeval"] != "improved_body_parts_b200.cocoeval.COCOeval"
    assert default["COCO"] != "improved_body_parts_b200.cocoeval.COCO"
    assert bound["COCOeval"] == "improved_body_parts_b200.cocoeval.COCOeval"
    assert (bound["COCO"] == "improved_body_parts_b200.cocoeval.COCO") == stubbed
    if stubbed:
        assert default["COCOeval"] == "builtins.object" and default["COCO"] == "builtins.object"


def test_accumulate_refuses_params_other_than_evaluated():
    """The check runs before any device work: a Params whose tables differ from evaluate()'s is refused."""
    c = _coco(dataset([gt(1, 1, pts(100, 100))], [1]))
    e = cocoeval.COCOeval(c, c)
    e._dev = {"T": 10}  # as after evaluate(); the refusal comes first
    e._paramsEval = copy.deepcopy(e.params)
    for f, v in (("recThrs", np.linspace(0, 1, 11)), ("catIds", [1, 2]), ("maxDets", [10]), ("areaRng", [[0, 1]])):
        q = copy.deepcopy(e.params)
        setattr(q, f, v)
        with pytest.raises(ValueError, match=f):
            e.accumulate(q)
    e.params.iouThrs = e.params.iouThrs[:5]
    with pytest.raises(ValueError, match="iouThrs"):
        e.accumulate()
