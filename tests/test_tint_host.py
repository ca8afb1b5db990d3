"""CPU: the host side of the device colour distortion -- the TARGET_TINT record against include/spgroup.h, and make_batch's
checks and draws with tint=True before any device work."""
import os
import subprocess

import numpy as np
import pytest

from improved_body_parts_b200 import grouping, targets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_tint_record_matches_the_header(tmp_path):
    """TARGET_TINT against spg_target_tint, by the probe pattern of test_targets_host.py."""
    name, dt = "spg_target_tint", grouping.TARGET_TINT
    args = ", ".join([f"sizeof({name})"] + [f"offsetof({name}, {f})" for f in dt.names])
    probe, exe = tmp_path / "probe.c", tmp_path / "probe"
    probe.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "spgroup.h"\nint main(void){\n'
                     f'printf("{" %zu" * (1 + len(dt.names))}\\n", {args});\nreturn 0;}}\n')
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(probe), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert got == [dt.itemsize] + [dt.fields[f][1] for f in dt.names]


def test_tint_records():
    r = targets.tint_records([(1 << 40, 3000, 7, 1000), (16, 3, 1, 1)], [(0, 0, 0), (20, 80, 60)], 32)
    assert r.dtype == grouping.TARGET_TINT
    assert r["image"].tolist() == [1 << 40, 16] and r["row_stride"].tolist() == [3000, 3]
    assert r[["hue", "saturation", "value"]].tolist() == [(0, 0, 0), (20, 80, 60)] and (r["row_block"] == 32).all()


def _sample(h=40, w=50):
    j = np.zeros((1, 18, 3))
    j[:, :, 0:2] = 10.0
    return (np.zeros((h, w, 3), np.uint8), np.full((h, w), 255, np.uint8), np.zeros((h, w), np.uint8),
            {"objpos": [[20.0, 20.0]], "scale_provided": [0.5], "joints": j})


def test_make_batch_with_tint_rejects_before_any_draw_or_device_work():
    """A refused batch consumes no np.random draws: the tinted sample 0 is valid, sample 1 is not."""
    img, mm, ma, meta = _sample()
    tinted = targets.AugmentSelection(tint=True)
    bad = [(img, mm, ma, meta), (img, mm[:-1], ma, meta)]
    np.random.seed(5)
    before = np.random.get_state()
    with pytest.raises(ValueError, match="mask_miss"):
        targets.make_batch(bad, [tinted, tinted], tint=True)
    after = np.random.get_state()
    assert np.array_equal(after[1], before[1]) and after[2] == before[2]
    cfg = targets.TargetConfig(256, 256)
    cfg.tint_row_block = 0
    with pytest.raises(ValueError, match="tint_row_block"):
        targets.make_batch([(img, mm, ma, meta)], [tinted], cfg, tint=True)
    with pytest.raises(ValueError, match="distort_color"):  # tint=False: today's refusal
        targets.make_batch([(img, mm, ma, meta)], [tinted])
    with pytest.raises(ValueError, match="distort_color"):
        targets.Transformer(cfg).transform(img, mm, ma, meta, tinted)
    with pytest.raises(ValueError, match="uint8 HxWx3"):
        targets.Transformer.distort_color(img[:, :, :2].copy())
