"""CPU: the C-ABI library loads and exports every symbol include/spgroup.h declares; host-side logic."""
import ctypes
import os
import re

import numpy as np
import pytest

from improved_body_parts_b200 import grouping

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


#: ctypes mirror in grouping.py -> the struct of include/spgroup.h it mirrors
MIRRORS = {grouping._Config: "spg_config", grouping._Params: "spg_params", grouping._DeviceView: "spg_device_view",
           grouping._ImageMaps: "spg_image_maps", grouping._PostnetScale: "spg_postnet_scale",
           grouping._PostnetDesc: "spg_postnet_desc", grouping._PostnetRotation: "spg_postnet_rotation",
           grouping._PostnetCommon: "spg_postnet_common", grouping._PostnetImage: "spg_postnet_image",
           grouping._PrenetItem: "spg_prenet_item"}
#: layouts pinned by value too: sizeof, then the offset of every field
PINNED = {"spg_postnet_rotation": [56, 0, 4, 8], "spg_prenet_item": [80, 0, 8, 12, 16, 64, 72]}


def test_struct_layouts_match_the_header(tmp_path):
    """Every ctypes mirror against the real header: one generated C probe prints sizeof and the offset of every field of
    each mirrored struct."""
    import subprocess

    mirrors = {c for c in vars(grouping).values() if isinstance(c, type) and issubclass(c, ctypes.Structure)}
    assert mirrors == set(MIRRORS)
    lines = []
    for cls, name in MIRRORS.items():
        args = ", ".join([f"sizeof({name})"] + [f"offsetof({name}, {f})" for f, _ in cls._fields_])
        lines.append(f'printf("{name}{" %zu" * (1 + len(cls._fields_))}\\n", {args});')
    probe, exe = tmp_path / "probe.c", tmp_path / "probe"
    probe.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "spgroup.h"\nint main(void){\n' + "\n".join(lines) +
                     "\nreturn 0;}\n")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(probe), "-o", str(exe)])
    got = {name: [int(v) for v in vals] for name, *vals in
           (line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())}
    want = {name: [ctypes.sizeof(cls)] + [getattr(cls, f).offset for f, _ in cls._fields_] for cls, name in MIRRORS.items()}
    assert got == want
    for name, layout in PINNED.items():
        assert got[name] == layout, name


_C_SCALARS = {"int32_t": ctypes.c_int32, "int64_t": ctypes.c_int64, "uint64_t": ctypes.c_uint64, "double": ctypes.c_double}
_C_RESULTS = {"int": ctypes.c_int, "void": None, "int64_t": ctypes.c_int64, "const char *": ctypes.c_char_p}


def _prototypes():
    """name -> (return type, [parameter declarations]) of every function include/spgroup.h declares."""
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "spgroup.h")).read(), flags=re.S)
    out = {}
    for ret, name, params in re.findall(r"^([\w ]*?\**)\s*\b(spg_\w+)\s*\(([^)]*)\)\s*;", src, flags=re.M):
        params = " ".join(params.split())
        out[name] = (ret.strip(), [] if params == "void" else [p.strip() for p in params.split(",")])
    return out


def test_prototype_table_matches_the_header():
    """The binding's argtypes / restype of every export against its C prototype: the parameter count, and per parameter
    its kind -- a pointer (arrays such as ``ipc_handle[64]`` included) or the exact integer / floating-point type."""
    protos = _prototypes()
    assert sorted(protos) == sorted(grouping.EXPORTS)
    for name, (ret, params) in protos.items():
        restype, argtypes = grouping._PROTOTYPES[name]
        assert restype is _C_RESULTS[ret], name
        assert len(argtypes) == len(params), name
        for decl, t in zip(params, argtypes):
            if "*" in decl or "[" in decl:
                assert t in (ctypes.c_void_p, ctypes.c_char_p) or issubclass(t, ctypes._Pointer), (name, decl, t)
            else:
                assert t is _C_SCALARS[decl.rsplit(" ", 1)[0]], (name, decl, t)


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
    csrc = os.path.join(ROOT, "improved_body_parts_b200", "csrc")
    src = open(os.path.join(csrc, "spgroup.cu")).read()
    body = src.split("int spg_create(")[1].split("\nvoid spg_destroy")[0]
    assert body.count("getenv(") >= 3
    for name in os.listdir(csrc):
        if name.endswith((".cu", ".cuh")):
            txt = open(os.path.join(csrc, name)).read()
            assert "getenv(" not in (txt.replace(body, "") if name == "spgroup.cu" else txt), name


def test_every_handle_launch_goes_through_launch():
    """launch() (runtime.cuh) is the one place a kernel is launched on a handle: it records the stage's kernel, counts the
    launch and turns a launch error into the call's error.  The only other launches are the three handle-less wire
    entry points' kernels in spgroup.cu."""
    csrc = os.path.join(ROOT, "improved_body_parts_b200", "csrc")
    runtime = open(os.path.join(csrc, "runtime.cuh")).read()
    body = runtime.split("\nint launch(")[1].split("\n}\n")[0]
    assert body.count("<<<") == 1
    wire = ("int spg_wire_signal(", "int spg_wire_signal_many(", "int spg_wire_wait(")
    spgroup = open(os.path.join(csrc, "spgroup.cu")).read()
    for entry in wire:
        fn = spgroup.split(entry)[1].split("\n}\n")[0]
        assert fn.count("<<<") == 1, entry
        spgroup = spgroup.replace(fn, "")
    for name in os.listdir(csrc):
        if name.endswith((".cu", ".cuh")):
            txt = {"runtime.cuh": runtime.replace(body, ""), "spgroup.cu": spgroup}.get(name)
            assert "<<<" not in (txt if txt is not None else open(os.path.join(csrc, name)).read()), name
