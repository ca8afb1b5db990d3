"""CPU: the frame API's C declarations and the argument checks ``dropin.FrameStream`` and ``spg_reserve_frame`` make before
they touch a device."""
import ctypes
import os
import re

import pytest

from improved_body_parts_b200 import dropin, grouping

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "spgroup.h")


def test_capture_error_code_is_declared():
    src = open(HEADER).read()
    m = re.search(r"SPG_E_CAPTURE\s*=\s*(-?\d+)", src)
    assert m and int(m.group(1)) == grouping.E_CAPTURE
    codes = [int(v) for v in re.findall(r"SPG_E_\w+\s*=\s*(-\d+)", src)]
    assert len(codes) == len(set(codes)), "error codes must be distinct"


def test_reserve_frame_is_declared_and_bound():
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"int\s+spg_reserve_frame\s*\(([^)]*)\)\s*;", src)
    assert m, "spg_reserve_frame is not declared"
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    assert params == ["spg_handle *h", "int32_t height", "int32_t width", "int32_t max_downsample",
                      "const spg_prenet_item *items", "int32_t n_items", "int32_t stride", "int32_t *moved"]
    restype, argtypes = grouping._PROTOTYPES["spg_reserve_frame"]
    assert restype is ctypes.c_int and len(argtypes) == len(params)


def test_reserve_frame_without_a_handle_is_invalid():
    import __graft_entry__ as ge

    ge.build()
    lib = grouping.load_library()
    item = grouping._PrenetItem(1.0, 0, 0, grouping._matrix6(None), None, 0)
    moved = ctypes.c_int32(7)
    assert lib.spg_reserve_frame(None, 64, 64, 32, ctypes.byref(item), 1, 4, ctypes.byref(moved)) == -1


@pytest.mark.parametrize("kw,match", [(dict(model_params=dict(boxsize=160, stride=8, max_downsample=32, padValue=128)),
                                       "stride 4"),
                                      (dict(slots=0), "slots"),
                                      (dict(input_stage="gpu"), "input_stage")])
def test_frame_stream_arguments(kw, match):
    args = dict(model=lambda x: None, params=dict(scale_search=[1.0], rotation_search=[0.0]),
                model_params=dict(boxsize=160, stride=4, max_downsample=32, padValue=128))
    args.update({k: v for k, v in kw.items() if k in args})
    with pytest.raises(ValueError, match=match):
        dropin.FrameStream(args["model"], args["params"], args["model_params"],
                           **{k: v for k, v in kw.items() if k not in args})
