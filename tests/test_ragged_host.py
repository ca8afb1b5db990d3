"""CPU: the host side of the ragged grouping call -- ``install``'s batch argument, and the launcher's ``--batch`` reaching
``install``."""
import json
import os
import subprocess
import sys
import types

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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
