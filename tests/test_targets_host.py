"""CPU: the host geometry of the training-sample stage (improved_body_parts_b200/targets.py) against the reference's
goldens, its input checks, and the numpy records mirroring include/spgroup.h."""
import os
import random
import subprocess

import numpy as np
import pytest

import targets_cases as tc
import targets_port as tp
from improved_body_parts_b200 import grouping, skeleton, targets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = tp.golden_paths()
SPACE = tp.golden_paths("targets_space")


@pytest.mark.parametrize("path", CASES + SPACE, ids=lambda p: os.path.basename(p)[:-4])
def test_affine_and_joints_equal_the_goldens(path):
    z = tp.load_case(path)
    cfg = tp.target_config(z)
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


@pytest.mark.parametrize("path", SPACE, ids=lambda p: os.path.basename(p)[:-4])
def test_target_params_equal_the_goldens_configuration(path):
    """target_params of a TargetConfig carrying a golden's stride, transform parameters and limb table: the
    reference's gaussian_size, shapes and the values the kernels take."""
    z = tp.load_case(path)
    c = tp.case_params(z)
    cfg = tp.target_config(z)
    assert targets.gaussian_size(cfg) == c["gsize"]
    assert cfg.num_layers == z["labels"].shape[0] and cfg.mask_shape == z["mask_miss"].shape
    p = targets.target_params(cfg)[0]
    assert (int(p["stride"]), int(p["gaussian_size"]), int(p["out_h"]), int(p["out_w"])) == \
        (c["stride"], c["gsize"], z["size"], z["size"])
    assert (p["sigma"], p["paf_sigma"], p["limb_gaussian_thre"], p["paf_thre"]) == \
        (c["sigma"], c["paf_sigma"], c["limb_thre"], c["paf_thre"])


def test_case_table_covers_every_axis():
    """tests/targets_cases.py against the axes spg_targets_warp / spg_targets_maps admit."""
    cases = tc.CASES
    assert len({c.name for c in cases}) == len(cases)
    assert {c.stride for c in cases} >= {1, 2, 3, 4, 5, 6, 8}
    maps = [c.map_hw for c in cases]
    assert any(h == w > 1 for h, w in maps) and any(h != w for h, w in maps) and (1, 1) in maps
    for c in cases:
        assert c.out_hw[0] % c.stride == 0 and c.out_hw[1] % c.stride == 0
        assert len(c.sources) == len(c.persons) and all(0 <= a < c.K and 0 <= b < c.K for a, b in c.limbs)
        assert 1 <= len(c.limbs) <= 64 and c.K <= 32
    g = [(c.gaussian_size, c.map_hw) for c in cases]
    assert any(s == 0 for s, _ in g) and any(s % 2 for s, _ in g) and any(s // 2 >= max(hw) for s, hw in g)
    assert any(c.borders != tc.DEFAULT_BORDERS for c in cases)
    assert any(c.pad[0] > 0 for c in cases) and any(c.pad[1] > 0 for c in cases)
    assert any(c.pad[0] % 4 for c in cases)  # an image pitch that is no multiple of 4
    tables = {(len(c.limbs), c.K) for c in cases}
    assert {(1, 18), (24, 18), (64, 18), (64, 32), (1, 32)} <= tables
    assert any(tuple(c.limbs) == tuple(skeleton.LIMBS) for c in cases)
    assert any(a == b for c in cases for a, b in c.limbs)  # a self-limb
    assert any(len(set(c.limbs)) < len(c.limbs) for c in cases)  # a repeated limb
    assert len({(c.sigma, c.paf_sigma, c.limb_thre, c.paf_thre) for c in cases}) >= 6
    assert any(c.paf_thre != int(c.paf_thre) for c in cases)
    # joints: ties, +-FLT_MAX, +-inf, NaN (visible), v exactly 2 and v NaN; 0 persons and > 256 persons x parts
    allj = []
    for c in cases:
        for (_, _, _, M, j) in tc.inputs(c):
            assert M.shape == (2, 3) and np.isfinite(M).all() and j.dtype == np.float32 and j.shape[1:] == (c.K, 3)
            if len(j) > 1:  # person 0 on x / stride ties (person 1 holds the special values)
                vis = j[0, :, 2] < 2
                x = j[0, vis, 0] / np.float32(c.stride)
                assert vis.any() and np.array_equal(x - np.floor(x), np.full(x.shape, 0.5, np.float32)), c.name
            allj.append(j.reshape(-1, 3))
    a = np.concatenate(allj)
    vis = a[:, 2] < 2
    xy = a[vis, :2]
    fmax = np.float32(tc.FLT_MAX)
    assert (xy == fmax).any() and (xy == -fmax).any() and np.isposinf(xy).any() and np.isneginf(xy).any()
    assert np.isnan(xy[:, 0]).any() and np.isnan(xy[:, 1]).any()
    assert (a[:, 2] == 2).any() and np.isnan(a[:, 2]).any()
    for c in cases:  # every case has a visible limb with one NaN end and the other end on the map
        a, b = tc.nan_limb(c)
        j = [d[4] for d in tc.inputs(c) if len(d[4]) >= 3]
        assert j and np.isnan(j[0][-1, a, 0]) and np.isfinite(j[0][-1, b, :2]).all() and (j[0][-1, [a, b], 2] < 2).all()
    counts = [p for c in cases for p in c.persons]
    assert 0 in counts and any(p * c.K > 256 for c in cases for p in c.persons)


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
