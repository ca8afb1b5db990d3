"""CPU: the host geometry of the training-sample stage (improved_body_parts_b200/targets.py) against the reference's
goldens, its input checks, and the numpy records mirroring include/spgroup.h."""
import os
import random
import subprocess

import numpy as np
import pytest

import targets_port as tp
from improved_body_parts_b200 import grouping, targets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = tp.golden_paths()


def _config(size):
    c = targets.TargetConfig(size, size)
    return c


@pytest.mark.parametrize("path", CASES, ids=lambda p: os.path.basename(p)[:-4])
def test_affine_and_joints_equal_the_goldens(path):
    z = tp.load_case(path)
    cfg = _config(z["size"])
    aug = targets.AugmentSelection(bool(z["aug_flip"]), False, float(z["aug_degree"]), tuple(int(v) for v in z["aug_crop"]),
                                   float(z["aug_scale"]))
    M, _ = aug.affine(list(z["objpos"]), float(z["scale_provided"]), cfg)
    assert np.array_equal(M, z["M"])
    assert np.array_equal(targets.transform_joints(z["joints_src"], M, aug.flip, cfg), z["joints"])


def test_seeded_random_draws_equal_the_reference():
    d = np.load(os.path.join(ROOT, "tests", "golden", "targets", "augment_draws.npz"))
    random.seed(int(d["seed"]))
    tp_ = targets.TargetConfig().transform_params
    got = []
    for _ in range(len(d["draws"])):
        a = targets.AugmentSelection.random(tp_)
        got.append([a.flip, a.tint, a.degree, a.crop[0], a.crop[1], a.scale])
    assert np.array_equal(np.array(got, np.float64), d["draws"])


def test_gaussian_size_default():
    assert targets.gaussian_size(targets.TargetConfig()) == 14


def _sample(h=40, w=50, P=2):
    rng = np.random.default_rng(0)
    j = np.zeros((P, 18, 3))
    j[:, :, 0:2] = rng.uniform(0, 40, (P, 18, 2))
    return (np.zeros((h, w, 3), np.uint8), np.full((h, w), 255, np.uint8), np.zeros((h, w), np.uint8),
            {"objpos": [[20.0, 20.0]], "scale_provided": [0.5], "joints": j})


def test_make_batch_rejects_malformed_input_before_any_device_work():
    un = targets.AugmentSelection.unrandom()
    img, mm, ma, meta = _sample()
    bad_joints = dict(meta, joints=meta["joints"].copy())
    bad_joints["joints"][1, 3, 0] = np.nan
    cases = [
        ([(img, mm, ma, bad_joints)], "non-finite"),
        ([(img, mm, ma, dict(meta, scale_provided=[0]))], "scale_provided"),
        ([(img.astype(np.float32), mm, ma, meta)], "uint8 HxWx3"),
        ([(img[:, :, :2].copy(), mm, ma, meta)], "uint8 HxWx3"),
        ([(img, mm[:-1], ma, meta)], "mask_miss"),
        ([(img, mm, ma[:, :-1], meta)], "mask_all"),
    ]
    for samples, match in cases:
        with pytest.raises(ValueError, match=match):
            targets.make_batch(samples, [un])
    with pytest.raises(ValueError, match="does not divide"):
        targets.make_batch([(img, mm, ma, meta)], [un], targets.TargetConfig(510, 510, 4))
    with pytest.raises(ValueError, match="distort_color"):
        targets.make_batch([(img, mm, ma, meta)], [targets.AugmentSelection(tint=True)])
    # an invisible joint may hold anything
    ok = dict(meta, joints=meta["joints"].copy())
    ok["joints"][1, 3] = (np.nan, np.inf, 2)
    targets._check_joints(0, ok["joints"].astype(np.float32))


def test_records_match_the_header(tmp_path):
    """TARGET_PARAMS / TARGET_SAMPLE / TARGET_JOINTS against spg_target_params / spg_target_sample / spg_target_joints."""
    recs = {"spg_target_params": grouping.TARGET_PARAMS, "spg_target_sample": grouping.TARGET_SAMPLE,
            "spg_target_joints": grouping.TARGET_JOINTS}
    lines = []
    for name, dt in recs.items():
        args = ", ".join([f"sizeof({name})"] + [f"offsetof({name}, {f})" for f in dt.names])
        lines.append(f'printf("{name}{" %zu" * (1 + len(dt.names))}\\n", {args});')
    probe, exe = tmp_path / "probe.c", tmp_path / "probe"
    probe.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "spgroup.h"\nint main(void){\n' + "\n".join(lines) +
                     "\nreturn 0;}\n")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(probe), "-o", str(exe)])
    got = {n: [int(v) for v in vals] for n, *vals in (l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())}
    want = {n: [dt.itemsize] + [dt.fields[f][1] for f in dt.names] for n, dt in recs.items()}
    assert got == want
