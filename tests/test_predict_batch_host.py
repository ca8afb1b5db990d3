"""CPU: the host side of the batched predict(): the launcher's ``--forward-batch`` and ``install``'s check of it (the
item planner of ``dropin.predict_batch`` is in test_predict_items_host.py)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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
