"""CPU: the C-ABI library loads and exports every symbol include/spgroup.h declares; host-side logic."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "spgroup.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(spg_[a-z_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    import __graft_entry__ as ge
    from improved_body_parts_b200 import grouping

    ge.build()
    lib = ctypes.CDLL(grouping.LIB_PATH)
    declared = _declared()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/spgroup.h but not exported"
    assert sorted(grouping.EXPORTS) == declared
    assert lib.spg_abi_version() == grouping.ABI_VERSION


def test_struct_layouts_match_the_header(tmp_path):
    """ctypes mirrors vs the real header: compile a C probe that prints sizeof/offsetof."""
    import subprocess

    from improved_body_parts_b200 import grouping

    probe = tmp_path / "probe.c"
    probe.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "spgroup.h"\n'
        'int main(void){printf("%zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(spg_config), sizeof(spg_params), '
        'sizeof(spg_device_view), offsetof(spg_config, limbs), offsetof(spg_config, out_from_part), '
        'offsetof(spg_config, max_batch), offsetof(spg_params, mid_num), offsetof(spg_device_view, peak_x));return 0;}\n')
    exe = tmp_path / "probe"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(probe), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    C, V, P = grouping._Config, grouping._DeviceView, grouping._Params
    assert got == [ctypes.sizeof(C), ctypes.sizeof(P), ctypes.sizeof(V), C.limbs.offset, C.out_from_part.offset,
                   C.max_batch.offset, P.mid_num.offset, V.peak_x.offset]


def test_no_gpu_means_a_loud_failure_not_a_fallback():
    import torch
    from improved_body_parts_b200.grouping import Grouper, GroupingError

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(GroupingError, match="no CUDA device|CUDA"):
        Grouper()


def test_product_package_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "improved_body_parts_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f), encoding="utf-8").read()
                assert "spg_oracle" not in txt and "import oracle" not in txt and "from oracle" not in txt, f


def test_params_struct_from_reference_dict():
    from improved_body_parts_b200 import grouping, skeleton

    p = grouping.params_struct(dict(skeleton.default_params(), thre1=0.25, mid_num=12, unrelated="x"))
    assert (p.thre1, p.mid_num, p.min_parts, p.min_mean_score) == (0.25, 12, 2, 0.45)
    p = grouping.params_struct(None)
    assert (p.thre2, p.connect_ration, p.len_rate, p.connection_tole, p.offset_radius, p.remove_recon) == \
           (0.1, 0.8, 16.0, 0.7, 2, 0)


def test_ini_reader_reproduces_config_reader_quirks():
    from improved_body_parts_b200 import skeleton

    path = os.path.join(ROOT, "tests", "golden", "reference_utils_config.ini")
    param, model = skeleton.read_reference_ini(path)
    assert param["scale_search"] == [1.0] and param["rotation_search"] == [0.0]  # chars of '1' / '0'
    assert (param["thre1"], param["thre2"], param["mid_num"], param["len_rate"]) == (0.1, 0.1, 20, 16.0)
    assert model["stride"] == 4 and model["boxsize"] == 640


def test_skeleton_tables():
    from improved_body_parts_b200 import skeleton

    assert skeleton.NUM_LIMBS == 30 and skeleton.NUM_PARTS == 18 and skeleton.NUM_LAYERS == 50
    assert len(skeleton.COCO_FROM_PART) == 17 and 1 not in skeleton.COCO_FROM_PART  # neck dropped
    for g, part in enumerate(skeleton.COCO_FROM_PART):
        assert skeleton.DT_GT_MAPPING[part] == g


def test_synth_is_seed_deterministic_and_shaped():
    from improved_body_parts_b200 import synth

    a = synth.make_image(5, 64, 80, 3)
    b = synth.make_image(5, 64, 80, 3)
    assert a[0].shape == (18, 64, 80) and a[1].shape == (30, 64, 80)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert a[0].max() <= 1.0 and a[0].min() >= 0.0


def test_environment_is_read_only_in_spg_create():
    """No debug mode and no result-changing knob: the library has no SPG_DEBUG build, and the tuning switches that
    remain are read once in spg_create -- no other getenv exists in the host code or in any kernel header."""
    from improved_body_parts_b200 import grouping
    blob = open(grouping.LIB_PATH, "rb").read()
    assert b"SPG_DEBUG" not in blob
    for name in (b"SPG_PERSIST", b"SPG_NO_SCREEN", b"SPG_EXACT_WARPS"):
        assert name in blob
    src = open(os.path.join(ROOT, "improved_body_parts_b200", "csrc", "spgroup.cu")).read()
    body = src.split("int spg_create(")[1].split("\nvoid spg_destroy")[0]
    outside = src.replace(body, "")
    assert body.count("getenv(") >= 3
    assert "getenv(" not in outside
    for name in os.listdir(os.path.join(ROOT, "improved_body_parts_b200", "csrc")):
        if name.endswith(".cuh"):
            assert "getenv(" not in open(os.path.join(ROOT, "improved_body_parts_b200", "csrc", name)).read(), name
