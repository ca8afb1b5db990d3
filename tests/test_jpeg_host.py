"""CPU: spg_jpeg_parse from the built library against the port's header parse, field for field, on every golden; its
record layout against include/spgroup.h; malformed headers refused without reading past the buffer."""
import ctypes
import json
import os
import struct
import subprocess

import numpy as np
import pytest

import make_jpeg_golden as mjg
from improved_body_parts_b200 import grouping
from oracle import jpeg_port as jp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "jpeg")
MANIFEST = json.load(open(os.path.join(GOLDEN, "MANIFEST.json")))["cases"]
PARSE_STATUS = {"corrupt": "ok", "range": "ok"}  # found by the decoder, not the parser


@pytest.fixture(scope="module", autouse=True)
def built():
    import __graft_entry__ as ge
    ge.build()


def _file(name: str) -> bytes:
    with open(os.path.join(GOLDEN, name + ".jpg"), "rb") as f:
        return f.read()


def _port_status(data: bytes) -> int:
    try:
        jp.parse(data)
    except jp.Refused as e:
        return e.status
    return jp.OK


def test_record_layout_matches_the_header(tmp_path):
    fields = [f for f in grouping.JPEG_RECORD.names]
    huff = [f for f in grouping.JPEG_HUFF.names]
    lines = ['printf("%zu %zu\\n", sizeof(spg_jpeg_record), sizeof(spg_jpeg_huff));']
    lines += [f'printf("%zu\\n", offsetof(spg_jpeg_record, {f}));' for f in fields]
    lines += [f'printf("%zu\\n", offsetof(spg_jpeg_huff, {f}));' for f in huff]
    probe, exe = tmp_path / "probe.c", tmp_path / "probe"
    probe.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "spgroup.h"\nint main(void){\n' + "\n".join(lines) +
                     "\nreturn 0;}\n")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(probe), "-o", str(exe)])
    out = subprocess.check_output([str(exe)], text=True).split()
    got = [int(v) for v in out]
    want = [grouping.JPEG_RECORD.itemsize, grouping.JPEG_HUFF.itemsize] + \
        [grouping.JPEG_RECORD.fields[f][1] for f in fields] + [grouping.JPEG_HUFF.fields[f][1] for f in huff]
    assert got == want


@pytest.mark.parametrize("name", sorted(MANIFEST))
def test_parse_matches_the_port(name):
    data = _file(name)
    rec = grouping.jpeg_parse(data)
    want = PARSE_STATUS.get(MANIFEST[name]["status"], MANIFEST[name]["status"])
    assert jp.REASONS[int(rec["status"])] == want
    if want != "ok":
        return
    h = jp.parse(data)
    for f in ("frame_height", "frame_width", "n_components", "h_samp", "v_samp", "mcus_x", "mcus_y", "blocks_per_mcu",
              "restart_interval", "n_intervals", "scan_offset", "scan_length", "orientation", "height", "width"):
        assert int(rec[f]) == getattr(h, f), f
    assert np.array_equal(rec["quant"], h.quant)
    for kind in ("dc", "ac"):
        for c in range(3):
            t, r = getattr(h, kind)[c], rec[kind][c]
            assert np.array_equal(r["lookup"], t.lookup) and np.array_equal(r["maxcode"][:18], t.maxcode)
            assert np.array_equal(r["valoff"][:17], t.valoff)
            assert np.array_equal(r["symbols"][:len(t.symbols)], t.symbols)


def _segment_at(data: bytes, marker: int) -> int:
    return next(p for p, m, _ in mjg.segments(data) if m == marker)


def _set_u16(data: bytes, at: int, value: int) -> bytes:
    return data[:at] + struct.pack(">H", value) + data[at + 2:]


def _malformed():
    base = _file("samp_420")
    sof, dht, dqt, sos = (_segment_at(base, m) for m in (0xC0, 0xC4, 0xDB, 0xDA))
    cases = {
        "empty": (b"", jp.NOT_JPEG),
        "soi_only": (b"\xff\xd8", jp.NOT_JPEG),
        "length_past_end": (_set_u16(base, dqt + 2, len(base)), jp.TRUNCATED),
        "cut_in_header": (base[:sof + 6], jp.TRUNCATED),
        "zero_height": (_set_u16(base, sof + 5, 0), jp.MALFORMED),
        "zero_width": (_set_u16(base, sof + 7, 0), jp.MALFORMED),
        "no_dht": (base[:dht] + base[dht + 2 + struct.unpack(">H", base[dht + 2:dht + 4])[0]:], jp.TABLES),
        "no_dqt": (base[:dqt] + base[dqt + 2 + struct.unpack(">H", base[dqt + 2:dqt + 4])[0]:], jp.TABLES),
        "no_eoi": (base[:-2], jp.TRUNCATED),
        "twelve_bit": (base[:sof + 4] + b"\x0c" + base[sof + 5:], jp.PRECISION),
        "four_components": (base[:sof + 9] + b"\x04" + base[sof + 10:], jp.COLOR),
    }
    # a Huffman table with more than 256 symbols: BITS that sum to 300
    bits = bytes([0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0])
    counts = bytearray(bits)
    counts[15] = 255
    counts[14] = 45
    seg = b"\xff\xc4" + struct.pack(">H", 2 + 17 + 300) + b"\x00" + bytes(counts) + bytes(300)
    cases["dht_300_symbols"] = (base[:dht] + seg + base[dht:], jp.TABLES)
    # a DHT whose symbol count runs past the segment
    seg = b"\xff\xc4" + struct.pack(">H", 2 + 17 + 4) + b"\x00" + bytes([0, 10] + [0] * 14) + bytes(4)
    cases["dht_symbols_past_segment"] = (base[:dht] + seg + base[dht:], jp.MALFORMED)
    cases["sos_components_reordered"] = (base[:sos + 5] + bytes([base[sos + 7]]) + base[sos + 6:sos + 7] +
                                         bytes([base[sos + 5]]) + base[sos + 8:], jp.SCAN)
    return cases


@pytest.mark.parametrize("name", sorted(_malformed()))
def test_malformed_headers_are_refused(name):
    data, status = _malformed()[name]
    assert _port_status(data) == status, jp.REASONS[_port_status(data)]
    assert int(grouping.jpeg_parse(data)["status"]) == status


def test_parse_reads_nothing_past_the_buffer():
    """Every prefix of a file parses inside its own bytes: a buffer mapped right before an inaccessible page."""
    import mmap
    data = _file("exif6_II")
    page = mmap.PAGESIZE
    lib = grouping.load_library()
    buf = mmap.mmap(-1, 2 * page, prot=mmap.PROT_READ | mmap.PROT_WRITE)
    libc = ctypes.CDLL(None)
    addr = ctypes.addressof(ctypes.c_char.from_buffer(buf))
    assert libc.mprotect(ctypes.c_void_p(addr + page), page, 0) == 0  # PROT_NONE: a read there faults
    rec = np.zeros(1, grouping.JPEG_RECORD)
    try:
        for n in range(0, len(data) + 1, 7):
            buf[page - n:page] = data[:n]
            assert lib.spg_jpeg_parse(addr + page - n, n, rec.ctypes.data) == 0
            assert int(rec[0]["status"]) == (jp.OK if n == len(data) else _port_status(data[:n]))
    finally:
        libc.mprotect(ctypes.c_void_p(addr + page), page, 3)
        del addr
        buf.close()


def test_parse_rejects_bad_arguments():
    lib = grouping.load_library()
    rec = np.zeros(1, grouping.JPEG_RECORD)
    assert lib.spg_jpeg_parse(None, 0, None) == -1
    assert lib.spg_jpeg_parse(None, 5, rec.ctypes.data) == -1
    assert lib.spg_jpeg_parse(None, -1, rec.ctypes.data) == -1


def test_device_decode_needs_the_device_input_stage():
    """configure(decode="device") and install(device_decode=True) refuse a setup whose predict_many would not feed the
    decoded CUDA images to the device input stage; the host decode stays the default."""
    import types

    from improved_body_parts_b200 import dropin
    assert dropin._decode == "host"
    with pytest.raises(ValueError):
        dropin.configure(input_stage="host", decode="device")
    with pytest.raises(ValueError):
        dropin.configure(decode="disk")
    mod = types.SimpleNamespace(limbSeq=dropin.LIMBS)
    for kw in (dict(device_predict=True, device_input=False, batch=4), dict(device_predict=True, device_input=True, batch=1),
               dict(device_predict=False, device_input=True, batch=4)):
        with pytest.raises(ValueError):
            dropin.install(mod, device_decode=True, **kw)
    assert dropin._decode == "host"


_LAUNCH = r'''
import json, os, sys
sys.path.insert(0, {root!r})
import importlib.util
spec = importlib.util.spec_from_file_location("run_evaluate_b200", os.path.join({root!r}, "tools", "run_evaluate_b200.py"))
L = importlib.util.module_from_spec(spec); spec.loader.exec_module(L)
try:
    L.prepare({ref!r}, batch=1, device_decode=True)
    refused = False
except ValueError:
    refused = True
ev = L.prepare({ref!r}, batch=4, device_decode=True)
from improved_body_parts_b200 import dropin
print("RESULT " + json.dumps(dict(refused=refused, decode=dropin._decode, stage=dropin._input_stage,
                                  many=ev.predict_many.__qualname__)))
'''


def test_launcher_device_decode(tmp_path):
    """prepare(..., device_decode=True) installs the batched predict_many with the device input stage and the device
    decode; with batch 1 it refuses."""
    import shutil
    import sys

    from test_launcher import _STAND_IN
    ref = tmp_path / "checkout"
    (ref / "utils").mkdir(parents=True)
    (ref / "evaluate.py").write_text(_STAND_IN)
    shutil.copy(os.path.join(ROOT, "tests", "golden", "reference_utils_config.ini"), ref / "utils" / "config")
    r = subprocess.run([sys.executable, "-c", _LAUNCH.format(root=ROOT, ref=str(ref))], capture_output=True, text=True,
                       timeout=300, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads(next(line for line in r.stdout.splitlines() if line.startswith("RESULT "))[7:])
    assert out == {"refused": True, "decode": "device", "stage": "device", "many": "install.<locals>._predict_many"}


@pytest.mark.parametrize("fill", [1, 2, 3])
def test_fill_bytes_before_a_stuffed_byte_are_refused(fill):
    """0xFF fill bytes before a stuffed pair (FF FF 00): libjpeg-turbo ends the data at FF FF, so the parser refuses the
    file for cv2, at every stuffed pair of a file; fill bytes before a marker stay accepted (the fill_ff golden)."""
    data = mjg.encode(mjg.content(10, 64, 96), "420", 97)
    rec = grouping.jpeg_parse(data)
    seg0 = int(rec["scan_offset"])
    pairs = [i for i in range(seg0, seg0 + int(rec["scan_length"]) - 1) if data[i] == 0xFF and data[i + 1] == 0x00]
    assert len(pairs) >= 3
    for i in pairs[:: max(1, len(pairs) // 8)]:
        bad = data[:i] + b"\xff" * fill + data[i:]
        assert _port_status(bad) == jp.MALFORMED
        assert int(grouping.jpeg_parse(bad)["status"]) == jp.MALFORMED


def test_imread_many_gives_none_for_a_missing_file(tmp_path):
    from improved_body_parts_b200 import dropin
    images, host = dropin.imread_many([str(tmp_path / "missing.jpg")])
    assert images == [None] and host == 1
