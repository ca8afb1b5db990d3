"""CPU: the host side of the ragged grouping call -- the ``spg_image_maps`` mirror against the header, ``install``'s
batch argument, and the launcher's ``--batch`` reaching ``install``."""
import ctypes
import json
import os
import subprocess
import sys
import types

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_image_maps_layout_matches_the_header(tmp_path):
    from improved_body_parts_b200 import grouping

    probe = tmp_path / "probe.c"
    probe.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "spgroup.h"\n'
        'int main(void){printf("%zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(spg_image_maps), '
        'offsetof(spg_image_maps, heat), offsetof(spg_image_maps, paf), offsetof(spg_image_maps, heat_chan_stride), '
        'offsetof(spg_image_maps, paf_chan_stride), offsetof(spg_image_maps, height), offsetof(spg_image_maps, width), '
        'offsetof(spg_image_maps, image_extent));return 0;}\n')
    exe = tmp_path / "probe"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(probe), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    M = grouping._ImageMaps
    assert got == [ctypes.sizeof(M), M.heat.offset, M.paf.offset, M.heat_chan_stride.offset, M.paf_chan_stride.offset,
                   M.height.offset, M.width.offset, M.image_extent.offset]
    assert "spg_group_ragged" in grouping.EXPORTS


def test_batched_predict_many_needs_the_device_predict():
    from improved_body_parts_b200 import dropin

    mod = types.ModuleType("evaluate")
    sentinel = object()
    mod.find_peaks = mod.predict_many = sentinel
    with pytest.raises(ValueError, match="device_predict"):
        dropin.install(mod, batch=2)
    assert mod.find_peaks is sentinel and mod.predict_many is sentinel  # nothing rebound


_CHILD = r'''
import json, os, sys
sys.path.insert(0, {root!r})
sys.argv = ["launcher"]
from improved_body_parts_b200 import dropin
seen = []
dropin.install = lambda mod, **kw: seen.append(kw)
import importlib.util
spec = importlib.util.spec_from_file_location("run_evaluate_b200", os.path.join({root!r}, "tools", "run_evaluate_b200.py"))
L = importlib.util.module_from_spec(spec); spec.loader.exec_module(L)
sys.argv = ["launcher", "--reference", {ref!r}, "--batch", "8"]
L.main()
print("RESULT " + json.dumps(seen))
'''


def test_launcher_batch_reaches_install(tmp_path):
    from test_launcher import _STAND_IN

    ref = tmp_path / "checkout"
    (ref / "utils").mkdir(parents=True)
    (ref / "evaluate.py").write_text(_STAND_IN)
    with open(os.path.join(ROOT, "tests", "golden", "reference_utils_config.ini")) as f:
        (ref / "utils" / "config").write_text(f.read())
    r = subprocess.run([sys.executable, "-c", _CHILD.format(root=ROOT, ref=str(ref))], capture_output=True, text=True,
                       timeout=300, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr[-3000:]
    seen = json.loads(next(l for l in r.stdout.splitlines() if l.startswith("RESULT "))[7:])
    assert seen == [{"device_predict": True, "batch": 8}]
