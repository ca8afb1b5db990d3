"""Regenerate tests/golden/jpeg/: small JPEG files made with cv2.imencode and by byte surgery, and cv2.imdecode's decode of
each (IMREAD_COLOR, EXIF orientation applied), for the device decoder's tests.  Usage: python tests/golden/make_jpeg_golden.py

- ``<name>.jpg``: the file; ``decoded.npz``: cv2's decode of every file that cv2 decodes, keyed by name;
- ``MANIFEST.json``: per file how it was made and the status spg_jpeg_parse / the decoder give it (``ok``, or the reason
  the file is left to cv2), with the cv2 and libjpeg-turbo versions that made the decodes.

The helpers below (``content``, ``encode`` and the segment surgery) are also what the tests use to make COCO-sized files
at run time.
"""
from __future__ import annotations

import json
import os
import struct
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "jpeg")
sys.path[:0] = [os.path.dirname(os.path.dirname(HERE))]


def content(seed: int, h: int, w: int, grey: bool = False) -> np.ndarray:
    """A seeded photo-like uint8 BGR (or grey) image (``synth.photo``)."""
    from improved_body_parts_b200 import synth
    return synth.photo(seed, h, w, grey)


SAMPLING = {"444": 0x111111, "422": 0x211111, "420": 0x221111, "440": 0x121111, "411": 0x411111}


def encode(img: np.ndarray, sampling: str = "420", quality: int = 95, restart: int = 0, optimize: bool = False,
           progressive: bool = False) -> bytes:
    import cv2
    params = [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_RST_INTERVAL, restart,
              cv2.IMWRITE_JPEG_OPTIMIZE, int(optimize), cv2.IMWRITE_JPEG_PROGRESSIVE, int(progressive)]
    if img.ndim == 3:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLING[sampling]]
    ok, buf = cv2.imencode(".jpg", img, params)
    assert ok
    return buf.tobytes()


def segments(data: bytes):
    """(offset of the marker, marker, length field) of every segment from SOI up to and including SOS."""
    p, out = 2, []
    while True:
        m = data[p + 1]
        length = struct.unpack(">H", data[p + 2:p + 4])[0]
        out.append((p, m, length))
        if m == 0xDA:
            return out
        p += 2 + length


def insert_segment(data: bytes, marker: int, payload: bytes, after: int = 0xE0) -> bytes:
    """A marker segment inserted after the first segment with marker `after` (else right after SOI)."""
    seg = bytes([0xFF, marker]) + struct.pack(">H", len(payload) + 2) + payload
    for p, m, length in segments(data):
        if m == after:
            q = p + 2 + length
            return data[:q] + seg + data[q:]
    return data[:2] + seg + data[2:]


def exif(orientation: int, order: str = "II") -> bytes:
    """An APP1 payload: Exif, a TIFF header in the byte order, IFD0 with one SHORT orientation entry."""
    e = "<" if order == "II" else ">"
    tiff = order.encode() + struct.pack(e + "HI", 42, 8) + struct.pack(e + "H", 1) + \
        struct.pack(e + "HHI", 0x0112, 3, 1) + struct.pack(e + "H", orientation) + b"\0\0" + struct.pack(e + "I", 0)
    return b"Exif\0\0" + tiff


def dqt16(data: bytes, scale: int = 1) -> bytes:
    """Every quantisation table rewritten with 16-bit entries (times `scale`, capped at 65535)."""
    out = bytearray(data[:2])
    segs = segments(data)
    for p, m, length in segs:
        seg = data[p:p + 2 + length]
        if m == 0xDB:
            body, o, nb = seg[4:], 0, bytearray()
            while o < len(body):
                tq, size = body[o] & 15, 128 if body[o] >> 4 else 64
                vals = np.frombuffer(body[o + 1:o + 1 + size], ">u2" if size == 128 else np.uint8).astype(np.int64)
                nb += bytes([0x10 | tq]) + np.minimum(vals * scale, 65535).astype(">u2").tobytes()
                o += 1 + size
            seg = b"\xff\xdb" + struct.pack(">H", len(nb) + 2) + bytes(nb)
        out += seg
    p, _, length = segs[-1]
    return bytes(out + data[p + 2 + length:])


def fill_bytes(data: bytes, n: int = 3) -> bytes:
    """n extra 0xFF fill bytes before the SOS marker, before every restart marker and before EOI."""
    p, _, length = segments(data)[-1]
    body = data[p:]
    head = data[:p] + b"\xff" * n
    scan_start = 2 + length
    ent = bytearray(body[:scan_start])
    i = scan_start
    while i < len(body):
        b = body[i]
        if b == 0xFF and i + 1 < len(body) and body[i + 1] != 0x00:
            ent += b"\xff" * n
        ent.append(b)
        i += 1
    return head + bytes(ent)


def fill_before_stuffing(data: bytes) -> bytes:
    """One 0xFF fill byte inserted before the first stuffed pair (0xFF 0x00) of the entropy-coded data."""
    p, _, length = segments(data)[-1]
    i = data.index(b"\xff\x00", p + 2 + length)
    return data[:i] + b"\xff" + data[i:]


def garbage_scan(data: bytes, seed: int) -> bytes:
    """The entropy-coded data replaced by seeded random bytes without 0xFF: a file that parses, whose data decodes to
    blocks no encoder makes."""
    p, _, length = segments(data)[-1]
    start = p + 2 + length
    rng = np.random.default_rng(seed)
    junk = rng.integers(0, 255, len(data) - 2 - start).astype(np.uint8).tobytes()
    return data[:start] + junk + b"\xff\xd9"


def cases():
    """name -> (file bytes, how it was made)."""
    out = {}
    base = content(1, 17, 33)
    for s in ("444", "422", "420", "440"):
        out[f"samp_{s}"] = (encode(base, s, 75), f"17x33 {s} q75")
    out["samp_411"] = (encode(base, "411", 75), "17x33 4:1:1 q75 (unsupported sampling)")
    out["grey"] = (encode(content(2, 17, 33, grey=True), quality=75), "17x33 grey q75")
    for q in (1, 50, 100):
        out[f"q{q}"] = (encode(content(3, 33, 47), "420", q), f"33x47 420 q{q}")
    out["optimized"] = (encode(content(4, 48, 64), "420", 90, optimize=True), "48x64 420 q90 optimised tables")
    out["optimized_444_q100"] = (encode(content(5, 40, 40), "444", 100, optimize=True), "40x40 444 q100 optimised tables")
    for r in (1, 3, 7):
        out[f"rst{r}"] = (encode(content(6, 40, 56), "420", 80, restart=r), f"40x56 420 q80, restart every {r} MCUs of 12")
    out["rst2_444"] = (encode(content(6, 40, 56), "444", 80, restart=2), "40x56 444 q80, restart every 2 MCUs")
    for h, w in ((1, 1), (7, 9), (97, 131)):
        out[f"size_{h}x{w}"] = (encode(content(7, h, w), "420", 85), f"{h}x{w} 420 q85")
    out["size_7x9_422"] = (encode(content(7, 7, 9), "422", 85), "7x9 422 q85")
    out["size_3x4_440"] = (encode(content(7, 3, 4), "440", 85), "3x4 440 q85")
    out["dqt16"] = (dqt16(encode(content(8, 24, 24), "420", 70)), "24x24 420 q70, DQT rewritten with 16-bit entries")
    out["dqt16_x8_range"] = (dqt16(encode(content(8, 24, 24), "420", 70), 8),
                             "24x24 420 q70, 16-bit DQT x8: blocks outside the SIMD/C agreement range")
    small = encode(content(9, 9, 13), "420", 80)
    for o in range(1, 9):
        for order in ("II", "MM"):
            out[f"exif{o}_{order}"] = (insert_segment(small, 0xE1, exif(o, order)), f"9x13 420, EXIF orientation {o} {order}")
    out["exif_9_ignored"] = (insert_segment(small, 0xE1, exif(9)), "9x13 420, EXIF orientation 9 (ignored)")
    out["adobe_com"] = (insert_segment(insert_segment(small, 0xEE, b"Adobe\x00\x64\x00\x00\x00\x00\x01"), 0xFE,
                                       b"a comment"), "9x13 420 with APP14 Adobe (transform 1) and COM")
    out["fill_ff"] = (fill_bytes(encode(content(10, 24, 40), "420", 80, restart=2)),
                      "24x40 420 q80 restart 2, 0xFF fill bytes before SOS, every RST and EOI")
    out["fill_before_stuffing"] = (fill_before_stuffing(encode(content(10, 64, 96), "420", 97)),
                                   "64x96 420 q97, a 0xFF fill byte before a stuffed 0xFF (FF FF 00)")
    out["progressive"] = (encode(content(11, 24, 32), "420", 80, progressive=True), "24x32 420 progressive")
    whole = encode(content(12, 32, 48), "420", 80)
    out["truncated"] = (whole[:len(whole) * 2 // 3], "32x48 420 cut at two thirds")
    out["garbage_scan"] = (garbage_scan(whole, 13), "32x48 420, entropy-coded data replaced by random bytes")
    cut = whole[:len(whole) * 2 // 3].rstrip(b"\xff")
    out["short_scan"] = (cut + b"\xff\xd9", "32x48 420 cut at two thirds and closed with EOI: too few blocks")
    return out


def main() -> None:
    import cv2
    from oracle import jpeg_port as jp
    os.makedirs(OUT, exist_ok=True)
    manifest, decoded = {}, {}
    for name, (data, how) in sorted(cases().items()):
        with open(os.path.join(OUT, name + ".jpg"), "wb") as f:
            f.write(data)
        img = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)
        if img is not None:
            decoded[name] = img
        manifest[name] = {"how": how, "bytes": len(data), "status": jp.REASONS[jp.classify(data)],
                          "cv2_shape": None if img is None else list(img.shape)}
    np.savez_compressed(os.path.join(OUT, "decoded.npz"), **decoded)
    build = [ln.strip() for ln in cv2.getBuildInformation().splitlines() if "JPEG:" in ln]
    with open(os.path.join(OUT, "MANIFEST.json"), "w") as f:
        json.dump({"cv2": cv2.__version__, "jpeg": build, "cases": manifest}, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
