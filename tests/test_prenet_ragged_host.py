"""CPU: the host side of the ragged pre-network call (``Grouper.prenet_ragged``): the one item helper that it and
``Grouper.prenet`` size their outputs with, and the member records it hands to ``spg_prenet_ragged``."""
import itertools
import os
import subprocess

import numpy as np

from oracle import postnet_rotation_port as pr
from oracle import prenet_port as pn
from test_predict_items_host import SEARCHES, _shapes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_item_helper_is_the_planner_and_the_port():
    """Every member of every search: the clamped scale and (H1, W1, Hp, Wp) of ``plan_items`` and of
    ``prenet_port.resized_size``, and the rotation matrices of the port -- clamped items included."""
    from improved_body_parts_b200 import dropin, grouping

    shapes = _shapes()
    clamped = rotated = 0
    for (scales, angles), (boxsize, md) in itertools.product(SEARCHES, ((640, 64), (368, 8), (160, 16))):
        params = dict(scale_search=scales, rotation_search=angles)
        plan, _ = dropin.plan_items(shapes, params, dict(boxsize=boxsize, max_downsample=md, stride=4))
        for i, (h, w) in enumerate(shapes):
            for (multiplier, scale, angle, *geo) in plan[i]:
                got_scale, got_geo, forward, reverse = grouping.prenet_item(h, w, multiplier, angle, md)
                assert got_scale == scale and got_geo == tuple(geo), (h, w, multiplier, angle, md)
                want_scale = pn.clamp_scale(multiplier, (h, w))
                H1, W1 = pn.resized_size(h, w, want_scale)
                assert got_scale == want_scale and got_geo == (H1, W1, -(-H1 // md) * md, -(-W1 // md) * md)
                clamped += scale != multiplier
                if angle == 0:
                    assert forward is None and reverse is None
                else:
                    rotated += 1
                    f, r = pr.rotation_matrices(got_geo[2:], angle)
                    assert np.array_equal(forward, f) and np.array_equal(reverse, r)
    assert clamped > 0 and rotated > 0


def test_item_helper_leaves_bad_scales_to_the_library():
    from improved_body_parts_b200 import grouping

    for scale in (float("nan"), 0.0, -1.0):  # an infinite scale is clamped to the 2600 x 3800 bound, as evaluate.py does
        assert grouping.prenet_item(20, 30, scale, 0, 8)[1] == (0, 0, 0, 0)


def test_member_record_is_the_header_struct(tmp_path):
    """``PRENET_MEMBER`` against ``spg_prenet_member`` of the real header: sizeof and the offset of every field."""
    from improved_body_parts_b200 import grouping

    dt = grouping.PRENET_MEMBER
    fields = {"image": "image", "row_stride": "row_stride", "height": "height", "width": "width", "scale": "scale",
              "rotate": "rotate", "reserved": "reserved", "matrix": "matrix", "out": "out"}
    assert set(dt.names) == set(fields)
    args = ", ".join(["sizeof(spg_prenet_member)"] + [f"offsetof(spg_prenet_member, {f})" for f in fields.values()])
    probe, exe = tmp_path / "probe.c", tmp_path / "probe"
    probe.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "spgroup.h"\nint main(void){\nprintf("' +
                     " %zu" * (1 + len(fields)) + '\\n", ' + args + ");\nreturn 0;}\n")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(probe), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert got == [dt.itemsize] + [dt.fields[f][1] for f in fields]
    assert got == [96, 0, 8, 16, 20, 24, 32, 36, 40, 88]
