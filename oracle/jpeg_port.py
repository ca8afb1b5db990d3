"""numpy restatement of what ``cv2.imread`` / ``cv2.imdecode(buf, IMREAD_COLOR)`` computes for a sequential Huffman JPEG.

Written from ITU-T T.81 and libjpeg's documented integer arithmetic (the decoder's defaults: the "islow" integer IDCT,
"fancy" triangle-filter chroma upsampling, the fixed-point YCbCr -> RGB tables), plus OpenCV's EXIF orientation.  Each
stage is exposed so that a mismatch can be localised:

    parse(data)            -> Header (or raises Refused(reason))
    coefficients(data, h)  -> per component int32 [rows][cols][64] quantised coefficients, natural order, DC undone
    planes(h, coefs)       -> per component uint8 planes of whole blocks (the islow IDCT of the dequantised blocks)
    bgr(h, planes)         -> uint8 [frame_h][frame_w][3] before orientation
    decode(data)           -> uint8 [H][W][3]: bgr() with the EXIF orientation applied

The refusal reasons are the status codes of ``spg_jpeg_parse`` (include/spgroup.h): a refused file is one the device
decoder leaves to cv2.imread.
"""
from __future__ import annotations

import dataclasses
import struct
from typing import List, Optional, Tuple

import numpy as np

# spg_jpeg_parse's status codes (include/spgroup.h SPG_JPEG_*)
OK = 0
NOT_JPEG = 1      # no SOI marker
TRUNCATED = 2     # a segment or the entropy-coded data runs past the end of the file, or no EOI
PROCESS = 3       # progressive, lossless, arithmetic-coded or hierarchical
PRECISION = 4     # not 8-bit samples
COLOR = 5         # not 1 or 3 components, or 3 components that libjpeg treats as RGB (Adobe transform 0, 'R','G','B' ids)
SAMPLING = 6      # sampling factors other than luma 1x1 / 2x1 / 1x2 / 2x2 with 1x1 chroma
SCAN = 7          # more than one scan, a non-interleaved or reordered scan, or spectral/approximation parameters
TABLES = 8        # a missing or invalid quantisation or Huffman table
MALFORMED = 9     # a length, count or marker that the decoder would reject or treat as corrupt
EXIF = 10         # an EXIF block whose orientation cannot be read the way OpenCV reads it
CORRUPT = 11      # (decoder only) the entropy-coded data is malformed: bad code, coefficient overrun, wrong block count
RANGE = 12        # (decoder only) a block leaves the range in which libjpeg's C and SIMD islow IDCTs agree (see idct_range_ok)

REASONS = {OK: "ok", NOT_JPEG: "not_jpeg", TRUNCATED: "truncated", PROCESS: "process", PRECISION: "precision",
           COLOR: "color", SAMPLING: "sampling", SCAN: "scan", TABLES: "tables", MALFORMED: "malformed", EXIF: "exif",
           CORRUPT: "corrupt", RANGE: "range"}


class Refused(Exception):
    def __init__(self, status: int, why: str = ""):
        super().__init__(f"{REASONS[status]}: {why}")
        self.status = status


# zigzag position -> natural (row-major) position
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
                   7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
                   39, 46, 53, 60, 61, 54, 47, 55, 62, 63], np.int32)


@dataclasses.dataclass
class Huffman:
    bits: np.ndarray      # [17]: bits[l] = number of codes of length l (1..16)
    symbols: np.ndarray   # [count] uint8
    maxcode: np.ndarray   # [18] int32: largest code of length l, -1 if none; maxcode[17] = 0x7fffffff
    valoff: np.ndarray    # [17] int32: symbol index = code + valoff[l]
    lookup: np.ndarray    # [512] uint16: 9-bit lookahead -> (length << 8) | symbol, 0 when the code is longer


@dataclasses.dataclass
class Header:
    frame_height: int
    frame_width: int
    n_components: int
    h_samp: int            # luma sampling factors; chroma is 1x1 (grey: 1x1)
    v_samp: int
    mcus_x: int
    mcus_y: int
    blocks_per_mcu: int
    restart_interval: int  # MCUs per interval, 0: none
    n_intervals: int
    scan_offset: int       # first byte of the entropy-coded data
    scan_length: int       # bytes up to the EOI marker
    quant: np.ndarray      # [3][64] uint16, natural order, per component
    dc: List[Huffman]      # per component
    ac: List[Huffman]
    orientation: int       # EXIF 1..8 (1 when absent)

    @property
    def height(self) -> int:
        return self.frame_width if self.orientation >= 5 else self.frame_height

    @property
    def width(self) -> int:
        return self.frame_height if self.orientation >= 5 else self.frame_width

    def comp_samp(self, c: int) -> Tuple[int, int]:
        return (self.h_samp, self.v_samp) if c == 0 else (1, 1)


def build_huffman(bits: np.ndarray, symbols: np.ndarray) -> Huffman:
    """libjpeg's derived decoding table (T.81 C.2 / F.2.2.3), with its checks: more than 256 codes, or a code that
    does not fit its length, is an invalid table."""
    if int(bits[1:].sum()) > 256:
        raise Refused(TABLES, "Huffman table with more than 256 codes")
    maxcode = np.full(18, -1, np.int32)
    maxcode[17] = 0x7fffffff
    valoff = np.zeros(17, np.int32)
    lookup = np.zeros(512, np.uint16)
    code, p = 0, 0
    longest = max([length for length in range(1, 17) if bits[length]], default=0)
    for length in range(1, longest + 1):
        n = int(bits[length])
        if n:
            valoff[length] = p - code
            for _ in range(n):
                if code < (1 << length) and length <= 9:
                    lo = code << (9 - length)
                    lookup[lo:lo + (1 << (9 - length))] = (length << 8) | int(symbols[p])
                code += 1
                p += 1
            maxcode[length] = code - 1
        # one more than the last code of this length must still fit it: no code is all ones
        if code >= (1 << length):
            raise Refused(TABLES, "Huffman code does not fit its length")
        code <<= 1
    return Huffman(bits=bits.astype(np.int32), symbols=symbols.astype(np.uint8), maxcode=maxcode, valoff=valoff,
                   lookup=lookup)


def _u16(data: bytes, o: int) -> int:
    return (data[o] << 8) | data[o + 1]


def _exif_orientation(seg: bytes) -> int:
    """OpenCV's ExifReader on the first APP1 segment: the TIFF header 6 bytes in, IFD0's first orientation entry (its
    16-bit value at entry + 8, whatever the entry's type), 1..8 applied and anything else ignored.  Reads outside the
    segment, which OpenCV handles by giving up part way, refuse the file."""
    if len(seg) <= 6:
        return 1
    t = seg[6:]
    if len(t) < 2:
        raise Refused(EXIF, "short TIFF header")
    if t[:2] == b"II":
        u16 = lambda o: struct.unpack_from("<H", t, o)[0]  # noqa: E731
        u32 = lambda o: struct.unpack_from("<I", t, o)[0]  # noqa: E731
    elif t[:2] == b"MM":
        u16 = lambda o: struct.unpack_from(">H", t, o)[0]  # noqa: E731
        u32 = lambda o: struct.unpack_from(">I", t, o)[0]  # noqa: E731
    else:
        raise Refused(EXIF, "APP1 without a TIFF byte order")
    if len(t) < 8:
        raise Refused(EXIF, "short TIFF header")
    if u16(2) != 0x2A:
        return 1
    off = u32(4)
    if off + 2 > len(t):
        raise Refused(EXIF, "IFD0 past the segment")
    n = u16(off)
    if off + 2 + 12 * n > len(t):
        raise Refused(EXIF, "IFD0 entries past the segment")
    for e in range(n):
        o = off + 2 + 12 * e
        if u16(o) == 0x0112:
            v = u16(o + 8)
            return v if 1 <= v <= 8 else 1
    return 1


def parse(data: bytes) -> Header:
    """The header of a JPEG file, or Refused(reason) for a file the device path does not decode."""
    data = bytes(data)
    n = len(data)
    if n < 4 or data[0] != 0xFF or data[1] != 0xD8:
        raise Refused(NOT_JPEG, "no SOI")
    p = 2
    qt: List[Optional[np.ndarray]] = [None] * 4
    dht = {}
    restart = 0
    frame = None
    jfif = adobe = False
    adobe_transform = -1
    orientation = None
    while True:
        # markers may be preceded by any number of 0xFF fill bytes
        if p >= n:
            raise Refused(TRUNCATED, "no SOS")
        if data[p] != 0xFF:
            raise Refused(MALFORMED, f"expected a marker at {p}")
        while p < n and data[p] == 0xFF:
            p += 1
        if p >= n:
            raise Refused(TRUNCATED, "marker at the end")
        m = data[p]
        p += 1
        if m == 0xD8 or m == 0xD9 or m == 0x01 or 0xD0 <= m <= 0xD7:
            raise Refused(MALFORMED, f"marker {m:#x} before the scan")
        if p + 2 > n:
            raise Refused(TRUNCATED, "segment length past the end")
        length = _u16(data, p)
        if length < 2 or p + length > n:
            raise Refused(TRUNCATED if length >= 2 else MALFORMED, "segment past the end")
        seg = data[p + 2:p + length]
        p += length
        if m in (0xC0, 0xC1):
            if frame is not None:
                raise Refused(MALFORMED, "second SOF")
            if len(seg) < 6:
                raise Refused(MALFORMED, "short SOF")
            prec, fh, fw, nc = seg[0], _u16(seg, 1), _u16(seg, 3), seg[5]
            if prec != 8:
                raise Refused(PRECISION, f"{prec}-bit samples")
            if fh == 0 or fw == 0:
                raise Refused(MALFORMED, "zero dimension")
            if nc not in (1, 3):
                raise Refused(COLOR, f"{nc} components")
            if len(seg) != 6 + 3 * nc:
                raise Refused(MALFORMED, "SOF length")
            comps = [(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i]) for i in range(nc)]
            for _, hs, vs, tq in comps:
                if not (1 <= hs <= 4 and 1 <= vs <= 4) or tq > 3:
                    raise Refused(MALFORMED, "component parameters")
            if len({c[0] for c in comps}) != nc:
                raise Refused(MALFORMED, "duplicate component ids")
            frame = (fh, fw, comps)
        elif 0xC2 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            raise Refused(PROCESS, f"SOF{m - 0xC0}")
        elif m == 0xCC:
            raise Refused(PROCESS, "arithmetic conditioning")
        elif m == 0xC4:
            o = 0
            while o < len(seg):
                if o + 17 > len(seg):
                    raise Refused(MALFORMED, "short DHT")
                tc, th = seg[o] >> 4, seg[o] & 15
                bits = np.zeros(17, np.int32)
                bits[1:] = np.frombuffer(seg[o + 1:o + 17], np.uint8)
                count = int(bits.sum())
                if tc > 1 or th > 3:
                    raise Refused(TABLES, "DHT class or id")
                if count > 256:
                    raise Refused(TABLES, "Huffman table with more than 256 codes")
                if o + 17 + count > len(seg):
                    raise Refused(MALFORMED, "DHT symbols past the segment")
                symbols = np.frombuffer(seg[o + 17:o + 17 + count], np.uint8).copy()
                dht[(tc, th)] = (bits, symbols)
                o += 17 + count
        elif m == 0xDB:
            o = 0
            while o < len(seg):
                pq, tq = seg[o] >> 4, seg[o] & 15
                if tq > 3 or pq > 1:
                    raise Refused(TABLES, "DQT precision or id")
                size = 128 if pq else 64
                if o + 1 + size > len(seg):
                    raise Refused(MALFORMED, "DQT past the segment")
                vals = np.frombuffer(seg[o + 1:o + 1 + size], ">u2" if pq else np.uint8).astype(np.int32)
                q = np.zeros(64, np.uint16)
                q[ZIGZAG] = vals
                qt[tq] = q
                o += 1 + size
        elif m == 0xDD:
            if len(seg) != 2:
                raise Refused(MALFORMED, "DRI length")
            restart = _u16(seg, 0)
        elif m == 0xE0:
            if len(seg) >= 14 and seg[:5] == b"JFIF\0":
                jfif = True
        elif m == 0xE1:
            if orientation is None:
                orientation = _exif_orientation(seg)
        elif m == 0xEE:
            if len(seg) >= 12 and seg[:5] == b"Adobe":
                adobe, adobe_transform = True, seg[11]
        elif m == 0xDA:
            break
        elif 0xE0 <= m <= 0xEF or m == 0xFE:
            pass
        else:
            raise Refused(MALFORMED, f"marker {m:#x}")
    # SOS
    if frame is None:
        raise Refused(MALFORMED, "SOS before SOF")
    fh, fw, comps = frame
    ns = seg[0] if len(seg) else 0
    if len(seg) != 4 + 2 * ns or ns == 0:
        raise Refused(MALFORMED, "SOS length")
    if ns != len(comps):
        raise Refused(SCAN, "scan does not hold every component")
    sel = [(seg[1 + 2 * i], seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15) for i in range(ns)]
    if [s[0] for s in sel] != [c[0] for c in comps]:
        raise Refused(SCAN, "scan components not in frame order")
    ss, se, ah, al = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns] >> 4, seg[3 + 2 * ns] & 15
    if (ss, se, ah, al) != (0, 63, 0, 0):
        raise Refused(SCAN, "spectral selection or successive approximation")
    nc = len(comps)
    if nc == 3:
        if jfif:
            rgb = False
        elif adobe:
            rgb = adobe_transform == 0
        else:
            rgb = [c[0] for c in comps] == [82, 71, 66]
        if rgb:
            raise Refused(COLOR, "RGB colour space")
        if adobe and not jfif and adobe_transform not in (0, 1):
            raise Refused(COLOR, "Adobe transform")
        hs, vs = comps[0][1], comps[0][2]
        if (hs, vs) not in ((1, 1), (2, 1), (1, 2), (2, 2)) or any((c[1], c[2]) != (1, 1) for c in comps[1:]):
            raise Refused(SAMPLING, "sampling factors")
    else:
        hs = vs = 1  # a single-component scan is one block per MCU whatever the factors
    quant = np.zeros((3, 64), np.uint16)
    dc, ac = [], []
    for c, (cid, h, v, tq) in enumerate(comps):
        if qt[tq] is None:
            raise Refused(TABLES, "missing quantisation table")
        quant[c] = qt[tq]
        _, td, ta = sel[c]
        if td > 3 or ta > 3 or (0, td) not in dht or (1, ta) not in dht:
            raise Refused(TABLES, "missing Huffman table")
        dbits, dsym = dht[(0, td)]
        if dsym.size and int(dsym.max()) > 15:
            raise Refused(TABLES, "DC symbol above 15")
        dc.append(build_huffman(dbits, dsym))
        ac.append(build_huffman(*dht[(1, ta)]))
    for c in range(nc, 3):
        quant[c] = quant[0]
        dc.append(dc[0])
        ac.append(ac[0])
    mcus_x, mcus_y = -(-fw // (8 * hs)), -(-fh // (8 * vs))
    bpm = hs * vs + (2 if nc == 3 else 0)
    n_intervals = -(-(mcus_x * mcus_y) // restart) if restart else 1
    # the entropy-coded data: up to EOI, with RST0..7 in order between the intervals and nothing else
    start = p
    expect_rst, found = 0, 0
    q = start
    while True:
        q = data.find(b"\xff", q)
        if q < 0 or q + 1 >= n:
            raise Refused(TRUNCATED, "no EOI after the scan")
        r = q + 1
        while r < n and data[r] == 0xFF:
            r += 1
        if r >= n:
            raise Refused(TRUNCATED, "no EOI after the scan")
        mk = data[r]
        if mk == 0x00:
            if r > q + 1:  # fill bytes before a stuffed 0xFF: libjpeg-turbo ends the data at the first FF FF
                raise Refused(MALFORMED, "0xFF fill bytes before a stuffed 0xFF")
            q = r + 1
            continue
        if 0xD0 <= mk <= 0xD7:
            if not restart or mk != 0xD0 + expect_rst or found + 1 >= n_intervals:
                raise Refused(MALFORMED, "unexpected restart marker")
            expect_rst = (expect_rst + 1) & 7
            found += 1
            q = r + 1
            continue
        if mk == 0xD9:
            end = q
            break
        raise Refused(SCAN, f"marker {mk:#x} after the scan")
    if found != n_intervals - 1:
        raise Refused(MALFORMED, "restart marker count")
    return Header(frame_height=fh, frame_width=fw, n_components=nc, h_samp=hs, v_samp=vs, mcus_x=mcus_x, mcus_y=mcus_y,
                  blocks_per_mcu=bpm, restart_interval=restart, n_intervals=n_intervals, scan_offset=start,
                  scan_length=end - start, quant=quant, dc=dc, ac=ac, orientation=orientation or 1)


def entropy_intervals(data: bytes, h: Header) -> List[bytes]:
    """The entropy-coded data of each restart interval with the stuffing removed (0xFF 0x00 -> 0xFF; fill bytes before a
    marker dropped)."""
    seg = bytes(data[h.scan_offset:h.scan_offset + h.scan_length])
    out, cur, i, n = [], bytearray(), 0, len(seg)
    while i < n:
        b = seg[i]
        if b != 0xFF:
            cur.append(b)
            i += 1
            continue
        j = i + 1
        while j < n and seg[j] == 0xFF:
            j += 1
        if j < n and seg[j] == 0x00:
            cur.append(0xFF)
            i = j + 1
        else:  # RSTn (the parser checked the order)
            out.append(bytes(cur))
            cur = bytearray()
            i = j + 1
    out.append(bytes(cur))
    return out


class CorruptData(Exception):
    pass


class _Bits:
    def __init__(self, buf: bytes):
        self.buf = buf + bytes(1024)  # a block reads at most 64 x 32 bits past the end: zeros, as libjpeg inserts
        self.nbits = 8 * len(buf)
        self.p = 0

    def peek16(self) -> int:
        o = self.p >> 3
        w = (self.buf[o] << 16) | (self.buf[o + 1] << 8) | self.buf[o + 2]
        return (w >> (8 - (self.p & 7))) & 0xFFFF

    def get(self, s: int) -> int:
        o = self.p >> 3
        w = int.from_bytes(self.buf[o:o + 4], "big")
        v = (w >> (32 - (self.p & 7) - s)) & ((1 << s) - 1)
        self.p += s
        return v

    def decode(self, t: Huffman) -> int:
        w = self.peek16()
        e = int(t.lookup[w >> 7])
        if e:
            self.p += e >> 8
            return e & 0xFF
        for length in range(10, 17):
            code = w >> (16 - length)
            if code <= t.maxcode[length]:
                self.p += length
                idx = code + int(t.valoff[length])
                if not 0 <= idx < len(t.symbols):
                    raise CorruptData("bad Huffman code")
                return int(t.symbols[idx])
        raise CorruptData("bad Huffman code")


def _extend(v: int, s: int) -> int:
    return v - (1 << s) + 1 if v < (1 << (s - 1)) else v


def block_layout(h: Header):
    """Per block of an MCU: (component, row offset, column offset) in that component's block grid."""
    lay = [(0, t // h.h_samp, t % h.h_samp) for t in range(h.h_samp * h.v_samp)]
    if h.n_components == 3:
        lay += [(1, 0, 0), (2, 0, 0)]
    return lay


def coefficients(data: bytes, h: Header) -> List[np.ndarray]:
    """Quantised coefficients (DC prediction undone, natural order) per component: int32 [rows][cols][64] with rows =
    mcus_y * v and cols = mcus_x * h of the component.  Raises CorruptData where the device decoder flags the image."""
    lay = block_layout(h)
    out = [np.zeros((h.mcus_y * h.comp_samp(c)[1], h.mcus_x * h.comp_samp(c)[0], 64), np.int32)
           for c in range(h.n_components)]
    total = h.mcus_x * h.mcus_y
    per = h.restart_interval or total
    for k, seg in enumerate(entropy_intervals(data, h)):
        bits = _Bits(seg)
        pred = [0, 0, 0]
        for m in range(k * per, min(total, (k + 1) * per)):
            my, mx = divmod(m, h.mcus_x)
            for c, ry, rx in lay:
                blk = out[c][my * h.comp_samp(c)[1] + ry, mx * h.comp_samp(c)[0] + rx]
                s = bits.decode(h.dc[c])
                diff = _extend(bits.get(s), s) if s else 0
                pred[c] = _wrap32(pred[c] + diff)  # libjpeg's int predictor, stored as a 16-bit coefficient
                blk[0] = ((pred[c] + 0x8000) & 0xFFFF) - 0x8000
                i = 1
                while i < 64:
                    rs = bits.decode(h.ac[c])
                    r, s = rs >> 4, rs & 15
                    if s:
                        i += r
                        if i > 63:
                            raise CorruptData("coefficient index past 63")
                        blk[ZIGZAG[i]] = _extend(bits.get(s), s)
                        i += 1
                    elif r == 15:
                        i += 16
                        if i > 64:
                            raise CorruptData("coefficient index past 63")
                    else:
                        break
                if bits.p > bits.nbits:
                    raise CorruptData("entropy-coded data ends inside a block")
    return out


# islow IDCT (13-bit constants, 2 extra bits of precision between the passes)
_CB, _P1 = 13, 2
F0_298, F0_390, F0_541, F0_765 = 2446, 3196, 4433, 6270
F0_899, F1_175, F1_501, F1_847 = 7373, 9633, 12299, 15137
F1_961, F2_053, F2_562, F3_072 = 16069, 16819, 20995, 25172


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _idct_1d(d0, d1, d2, d3, d4, d5, d6, d7, shift):
    """One 8-point pass on int64 arrays; returns the 8 outputs descaled by `shift`."""
    z1 = (d2 + d6) * F0_541
    tmp2 = z1 + d6 * (-F1_847)
    tmp3 = z1 + d2 * F0_765
    tmp0 = (d0 + d4) << _CB
    tmp1 = (d0 - d4) << _CB
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = d7, d5, d3, d1
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * F1_175
    t0, t1, t2, t3 = t0 * F0_298, t1 * F2_053, t2 * F3_072, t3 * F1_501
    z1, z2, z3, z4 = z1 * (-F0_899), z2 * (-F2_562), z3 * (-F1_961), z4 * (-F0_390)
    z3 = z3 + z5
    z4 = z4 + z5
    t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
    return [_descale(v, shift) for v in (tmp10 + t3, tmp11 + t2, tmp12 + t1, tmp13 + t0,
                                         tmp13 - t0, tmp12 - t1, tmp11 - t2, tmp10 - t3)]


def _wrap32(x):
    return ((x + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


#: libjpeg's post-IDCT range limit: index (x & 1023) of the level-shifted-out value x
RANGE_LIMIT = np.concatenate([np.arange(128, 256), np.full(384, 255), np.zeros(384), np.arange(0, 128)]).astype(np.uint8)


def idct_islow(coef: np.ndarray, quant: np.ndarray) -> np.ndarray:
    """[..., 64] quantised coefficients (natural order) and the [64] table -> [..., 8, 8] uint8 samples."""
    c = coef.astype(np.int64).reshape(-1, 8, 8) * quant.astype(np.int64).reshape(8, 8)
    c = _wrap32(c)
    # pass 1: columns (vertical frequencies), workspace kept as int
    ws = np.stack(_idct_1d(*[c[:, r, :] for r in range(8)], _CB - _P1), axis=1)
    ws = _wrap32(ws)
    # pass 2: rows
    out = np.stack(_idct_1d(*[ws[:, :, k] for k in range(8)], _CB + _P1 + 3), axis=2)
    return RANGE_LIMIT[(out & 1023)].reshape(coef.shape[:-1] + (8, 8))


#: the bounds inside which libjpeg-turbo's SIMD islow IDCT (16-bit products and sums, a saturating pack between the
#: passes and a plain clamp at the end) and its C one (int arithmetic and the range-limit table) give the same samples
DEQUANT_MAX, PASS1_MAX, OUT_MIN, OUT_MAX = 16383, 8191, -512, 511


def idct_range_ok(coef: np.ndarray, quant: np.ndarray) -> np.ndarray:
    """[..., 64] coefficients -> [...] bool: the block's dequantised coefficients, first-pass outputs and descaled
    outputs lie within the bounds above.  Real images stay far inside them (|dequantised| <= 1 100, |first pass| <= 4 300,
    |descaled outputs| <= 209 in seeded worst cases); a block outside them is left to cv2."""
    c = coef.astype(np.int64).reshape(-1, 8, 8) * quant.astype(np.int64).reshape(8, 8)
    ws = np.stack(_idct_1d(*[c[:, r, :] for r in range(8)], _CB - _P1), axis=1)
    out = np.stack(_idct_1d(*[ws[:, :, k] for k in range(8)], _CB + _P1 + 3), axis=2)
    ok = (np.abs(c) <= DEQUANT_MAX).all(axis=(1, 2)) & (np.abs(ws) <= PASS1_MAX).all(axis=(1, 2)) & \
        ((out >= OUT_MIN) & (out <= OUT_MAX)).all(axis=(1, 2))
    return ok.reshape(coef.shape[:-1])


def planes(h: Header, coefs: List[np.ndarray]) -> List[np.ndarray]:
    """The IDCT of every block: per component a uint8 plane of rows*8 x cols*8 samples."""
    out = []
    for c, co in enumerate(coefs):
        R, Cn = co.shape[:2]
        b = idct_islow(co, h.quant[c])  # [R, C, 8, 8]
        out.append(b.transpose(0, 2, 1, 3).reshape(R * 8, Cn * 8))
    return out


def _fancy_h2(row: np.ndarray, n: int) -> np.ndarray:
    """h2v1 fancy upsampling of the first n columns of int rows [..., >=n] -> [..., 2n] (n > 2)."""
    x = row[..., :n].astype(np.int32)
    out = np.empty(x.shape[:-1] + (2 * n,), np.int32)
    left = np.concatenate([x[..., :1], x[..., :-1]], axis=-1)
    right = np.concatenate([x[..., 1:], x[..., -1:]], axis=-1)
    out[..., 0::2] = (3 * x + left + 1) >> 2
    out[..., 1::2] = (3 * x + right + 2) >> 2
    out[..., 0] = x[..., 0]
    out[..., -1] = x[..., -1]
    return out


def _fancy_h2v2(p: np.ndarray, dh: int, dw: int) -> np.ndarray:
    """h2v2 fancy upsampling of the dh x dw downsampled plane p -> 2dh x 2dw (dw > 2)."""
    x = p[:dh, :dw].astype(np.int32)
    up = np.concatenate([x[:1], x[:-1]], axis=0)
    down = np.concatenate([x[1:], x[-1:]], axis=0)
    out = np.empty((2 * dh, 2 * dw), np.int32)
    for v, nb in ((0, up), (1, down)):
        cs = 3 * x + nb  # column sums
        left = np.concatenate([cs[:, :1], cs[:, :-1]], axis=1)
        right = np.concatenate([cs[:, 1:], cs[:, -1:]], axis=1)
        o = np.empty((dh, 2 * dw), np.int32)
        o[:, 0::2] = (3 * cs + left + 8) >> 4
        o[:, 1::2] = (3 * cs + right + 7) >> 4
        o[:, 0] = (4 * cs[:, 0] + 8) >> 4
        o[:, -1] = (4 * cs[:, -1] + 7) >> 4
        out[v::2] = o
    return out


def _fancy_h1v2(p: np.ndarray, dh: int, dw: int) -> np.ndarray:
    x = p[:dh, :dw].astype(np.int32)
    up = np.concatenate([x[:1], x[:-1]], axis=0)
    down = np.concatenate([x[1:], x[-1:]], axis=0)
    out = np.empty((2 * dh, dw), np.int32)
    out[0::2] = (3 * x + up + 1) >> 2
    out[1::2] = (3 * x + down + 2) >> 2
    return out


def upsample(h: Header, plane: np.ndarray) -> np.ndarray:
    """A chroma plane at the luma resolution (frame_height x frame_width), as libjpeg's default upsampler does it:
    fancy h2v1 / h2v2 when the downsampled width exceeds 2 (box replication otherwise), fancy h1v2 always."""
    H, W = h.frame_height, h.frame_width
    dh, dw = -(-H // h.v_samp), -(-W // h.h_samp)
    if (h.h_samp, h.v_samp) == (1, 1):
        out = plane[:H, :W].astype(np.int32)
    elif (h.h_samp, h.v_samp) == (2, 1):
        out = _fancy_h2(plane[:dh], dw) if dw > 2 else np.repeat(plane[:dh, :dw].astype(np.int32), 2, axis=1)
    elif (h.h_samp, h.v_samp) == (1, 2):
        out = _fancy_h1v2(plane, dh, dw)
    else:
        out = _fancy_h2v2(plane, dh, dw) if dw > 2 else \
            np.repeat(np.repeat(plane[:dh, :dw].astype(np.int32), 2, axis=0), 2, axis=1)
    return out[:H, :W]


def _fix(x: float) -> int:
    return int(x * 65536 + 0.5)


_X = np.arange(256, dtype=np.int64) - 128
CR_R = (_fix(1.40200) * _X + 32768) >> 16
CB_B = (_fix(1.77200) * _X + 32768) >> 16
CR_G = -_fix(0.71414) * _X
CB_G = -_fix(0.34414) * _X + 32768


def bgr(h: Header, pl: List[np.ndarray]) -> np.ndarray:
    """Colour conversion (libjpeg's fixed-point YCbCr -> RGB; grey replicated) at the frame size, in B, G, R order."""
    H, W = h.frame_height, h.frame_width
    y = pl[0][:H, :W].astype(np.int64)
    if h.n_components == 1:
        return np.repeat(y.astype(np.uint8)[:, :, None], 3, axis=2)
    cb, cr = upsample(h, pl[1]), upsample(h, pl[2])
    r = np.clip(y + CR_R[cr], 0, 255)
    g = np.clip(y + ((CB_G[cb] + CR_G[cr]) >> 16), 0, 255)
    b = np.clip(y + CB_B[cb], 0, 255)
    return np.stack([b, g, r], axis=2).astype(np.uint8)


def orient(img: np.ndarray, orientation: int) -> np.ndarray:
    """OpenCV's ApplyExifOrientation."""
    if orientation >= 5:
        img = img.transpose(1, 0, 2)
    flip = {1: None, 2: "h", 3: "hv", 4: "v", 5: None, 6: "h", 7: "hv", 8: "v"}[orientation]
    if flip and "h" in flip:
        img = img[:, ::-1]
    if flip and "v" in flip:
        img = img[::-1]
    return np.ascontiguousarray(img)


def decode(data: bytes) -> np.ndarray:
    """cv2.imdecode(data, IMREAD_COLOR) for a file parse() accepts; raises Refused / CorruptData otherwise."""
    h = parse(data)
    return orient(bgr(h, planes(h, coefficients(data, h))), h.orientation)


def classify(data: bytes) -> int:
    """The status the device path gives the file: OK, a parse refusal, or CORRUPT."""
    try:
        h = parse(data)
        co = coefficients(data, h)
    except Refused as e:
        return e.status
    except CorruptData:
        return CORRUPT
    return OK if all(idct_range_ok(c, h.quant[i]).all() for i, c in enumerate(co)) else RANGE
