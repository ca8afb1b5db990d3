"""CPU: the host side of the batched predict(): the bucket planner of ``dropin.predict_batch`` and the launcher's
``--forward-batch``."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import prenet_port as pn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_bucket_planner_is_the_prenet_geometry():
    """(H1, W1, Hp, Wp) of every image equals cv2.resize's size (cvRound) and its padding, the 2600 / 3800 clamp
    included, and images are bucketed by (Hp, Wp) in order of first appearance."""
    from improved_body_parts_b200 import dropin

    rng = np.random.default_rng(3)
    shapes = [(480, 640), (640, 480), (427, 640), (640, 427), (612, 612), (375, 500), (640, 640), (1, 1), (3, 7000),
              (5000, 20), (333, 333), (641, 639)] + [tuple(int(v) for v in rng.integers(1, 2000, 2)) for _ in range(200)]
    for boxsize, scale_search, md in ((640, 1.0, 64), (368, 1.0, 8), (640, 0.5, 32), (640, 2.0, 64), (160, 1.3, 16)):
        params = dict(scale_search=[scale_search], rotation_search=[0.0])
        model_params = dict(boxsize=boxsize, max_downsample=md, stride=4)
        plan, buckets = dropin.plan_buckets(shapes, params, model_params)
        assert len(plan) == len(shapes)
        seen = []
        for i, (h, w) in enumerate(shapes):
            multiplier = scale_search * boxsize / h
            scale = pn.clamp_scale(multiplier, (h, w))
            H1, W1 = pn.resized_size(h, w, scale)
            Hp, Wp = -(-H1 // md) * md, -(-W1 // md) * md
            assert plan[i] == (multiplier, scale, H1, W1, Hp, Wp), (h, w, boxsize, scale_search, md)
            assert i in buckets[(Hp, Wp)]
            if (Hp, Wp) not in seen:
                seen.append((Hp, Wp))
        assert list(buckets) == seen
        assert sorted(i for idx in buckets.values() for i in idx) == list(range(len(shapes)))
    # the reference's settings: images with one aspect ratio share an input size
    _, b = dropin.plan_buckets([(480, 640), (240, 320), (640, 480), (960, 1280)],
                               dict(scale_search=[1.0], rotation_search=[0.0]), dict(boxsize=640, max_downsample=64))
    assert b == {(640, 896): [0, 1, 3], (640, 512): [2]}


def _launcher(args, tmp_path):
    ref = tmp_path / "checkout"
    (ref / "utils").mkdir(parents=True, exist_ok=True)
    (ref / "evaluate.py").write_text("limbSeq = [(1, 0), (1, 2)]\n")
    import shutil
    shutil.copy(os.path.join(ROOT, "tests", "golden", "reference_utils_config.ini"), ref / "utils" / "config")
    return subprocess.run([sys.executable, os.path.join(ROOT, "tools", "run_evaluate_b200.py"), "--reference", str(ref)] + args,
                          capture_output=True, text=True, timeout=300, cwd=str(tmp_path))


def test_launcher_takes_forward_batch(tmp_path):
    r = _launcher(["--batch", "8", "--forward-batch", "4"], tmp_path)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "evaluate imported from" in r.stdout
    for bad, msg in ((["--batch", "8", "--forward-batch", "0"], "--forward-batch must be >= 1"),
                     (["--batch", "8", "--forward-batch", "-3"], "--forward-batch must be >= 1"),
                     (["--forward-batch", "4"], "needs --batch > 1")):
        r = _launcher(bad, tmp_path)
        assert r.returncode == 2 and msg in r.stderr, (bad, r.stderr[-2000:])


def test_install_checks_forward_batch():
    import types

    from improved_body_parts_b200 import dropin
    mod = types.ModuleType("evaluate")
    try:
        with pytest.raises(ValueError, match="forward_batch"):
            dropin.install(mod, device_predict=True, batch=1, forward_batch=2)
        with pytest.raises(ValueError, match="forward_batch"):
            dropin.install(mod, device_predict=False, batch=1, forward_batch=2)
        with pytest.raises(ValueError, match="forward_batch"):
            dropin.install(mod, device_predict=True, batch=4, forward_batch=0)
        dropin.install(mod, device_predict=True, batch=4, forward_batch=4)
        assert mod.predict_many.__name__ == "_predict_many"
    finally:
        dropin.configure(limbs=dropin.LIMBS, input_stage="host")
