"""JPEG headers on the host: the marker walk in front of the device decoder (csrc/jpeg.cu) and the route decision.

`parse(data)` walks SOI, APPn, DQT, DHT, SOF, DRI and SOS and returns a `JpegInfo`: the frame (size, components, sampling
factors), the quantisation tables in natural order, the Huffman tables as the lookup tables the device decoder copies into
shared memory, the restart interval, the EXIF orientation and the byte range of the one scan.  Its `device` flag says whether
the device decoder reproduces Pillow for the file; `reason` says why not.  The device takes (ITU-T T.81 names):

  * SOF0 / SOF1 (baseline and extended-sequential Huffman), 8-bit samples, one interleaved scan holding every component;
  * one component (grayscale, sampling 1x1), or three components in YCbCr with luma 1x1, 2x1 or 2x2 over chroma 1x1
    (4:4:4, 4:2:2, 4:2:0);
  * with or without restart markers.

Everything else (progressive, arithmetic coding, lossless, 12-bit, CMYK, Adobe-transformed RGB, other sampling ratios, several
scans, XMP-only orientation) takes the host route, `PIL.Image.open` as detectron2's `read_image` does today.  A file is either
decoded bit-exactly on the device or decoded on the host: nothing is approximated.
"""
from dataclasses import dataclass, field

import numpy as np

# T.81 Figure A.6: zig-zag index k -> natural (row-major) index
ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
    28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54,
    47, 55, 62, 63], dtype=np.int32)

LOOKAHEAD = 9            # bits resolved by one table read on the device; longer codes walk maxcode[]
TABLE_WORDS = 1024       # int32 words per uploaded Huffman table (layout below)
_LUT, _MAXCODE, _VALOFF, _VALS = 0, 512, 529, 546

EXIF_ORIENTATION = 0x0112
SUPPORTED_SAMPLING = {(1, 1): "4:4:4", (2, 1): "4:2:2", (2, 2): "4:2:0"}


class JpegError(ValueError):
    """The bytes are not a JPEG file the marker walk can follow (the host decoder then reports its own error)."""


@dataclass
class JpegInfo:
    height: int = 0
    width: int = 0
    precision: int = 8
    sof: int = 0                                   # 0xC0 .. 0xCF
    components: list = field(default_factory=list)  # [(id, h, v, tq)] in frame order
    qtables: dict = field(default_factory=dict)     # tq -> int32 [64] natural order
    huff: dict = field(default_factory=dict)        # (class 0=DC / 1=AC, id) -> (bits[17], huffval)
    scan_tables: list = field(default_factory=list)  # [(td, ta)] per component, frame order
    restart_interval: int = 0
    orientation: int = 1
    scan_start: int = 0                             # byte range of the entropy-coded data of the one scan
    scan_end: int = 0
    restart_markers: list = field(default_factory=list)  # offsets of the RSTn markers inside the scan
    jfif: bool = False
    exif_has_orientation: bool = False
    adobe: bool = False
    device: bool = False
    reason: str = ""

    @property
    def ncomp(self):
        return len(self.components)

    @property
    def hmax(self):
        return max(c[1] for c in self.components)

    @property
    def vmax(self):
        return max(c[2] for c in self.components)

    @property
    def oriented_hw(self):
        """(H, W) of the image after the EXIF transpose detectron2's `_apply_exif_orientation` applies."""
        return (self.width, self.height) if self.orientation in (5, 6, 7, 8) else (self.height, self.width)


def huffman_lut(bits, huffval):
    """The decoder table of one DHT entry (T.81 Annex C canonical codes, F.2.2.3 decoding procedure) as int32
    [TABLE_WORDS]: lut[0:512] = (length << 8) | symbol for every 9-bit prefix whose code has <= 9 bits, else 0;
    maxcode[l] (l = 0..16, -1 when no code has l bits); valoff[l] = index of the first length-l symbol minus its code;
    huffval[0:256].  Raises JpegError for a table whose code space overflows (libjpeg refuses it too)."""
    t = np.zeros(TABLE_WORDS, dtype=np.int32)
    t[_MAXCODE:_MAXCODE + 17] = -1
    code, k = 0, 0
    for l in range(1, 17):
        n = int(bits[l])
        if n:
            t[_VALOFF + l] = k - code
            for _ in range(n):
                if code >= (1 << l):
                    raise JpegError("bad Huffman table: code space overflow")
                if l <= LOOKAHEAD:
                    lo = code << (LOOKAHEAD - l)
                    t[_LUT + lo:_LUT + lo + (1 << (LOOKAHEAD - l))] = (l << 8) | int(huffval[k])
                code += 1
                k += 1
            t[_MAXCODE + l] = code - 1
        code <<= 1
    t[_VALS:_VALS + len(huffval)] = np.asarray(huffval, dtype=np.int32)
    return t


def _exif_orientation(seg):
    """Orientation tag of IFD0 of an `Exif\\0\\0` APP1 payload (TIFF 6.0 layout); None when the tag is absent."""
    tiff = seg[6:]
    if len(tiff) < 8 or tiff[:2] not in (b"II", b"MM"):
        raise JpegError("malformed Exif header")
    bo = "<" if tiff[:2] == b"II" else ">"
    u16 = np.dtype(bo + "u2")
    u32 = np.dtype(bo + "u4")
    if int(np.frombuffer(tiff, u16, 1, 2)[0]) != 42:
        raise JpegError("malformed Exif header")
    ifd = int(np.frombuffer(tiff, u32, 1, 4)[0])
    if ifd + 2 > len(tiff):
        raise JpegError("Exif IFD0 outside the segment")
    n = int(np.frombuffer(tiff, u16, 1, ifd)[0])
    if ifd + 2 + 12 * n > len(tiff):
        raise JpegError("Exif IFD0 outside the segment")
    for i in range(n):
        e = ifd + 2 + 12 * i
        tag, typ = int(np.frombuffer(tiff, u16, 1, e)[0]), int(np.frombuffer(tiff, u16, 1, e + 2)[0])
        cnt = int(np.frombuffer(tiff, u32, 1, e + 4)[0])
        if tag != EXIF_ORIENTATION:
            continue
        if cnt != 1 or typ not in (3, 4):
            raise JpegError("Exif orientation of an unexpected type")
        return int(np.frombuffer(tiff, u16 if typ == 3 else u32, 1, e + 8)[0])
    return None


def find_scan_end(buf, start):
    """Offset of the marker that ends the entropy-coded data at `start`: the first 0xFF not followed by a stuffed 0x00 or a
    restart marker (T.81 B.1.1.5: 0xFF data bytes are always followed by 0x00; fill 0xFF bytes may precede a marker).
    Returns (end, restart_marker_offsets)."""
    a = np.frombuffer(buf, dtype=np.uint8, offset=start)
    ff = np.flatnonzero(a[:-1] == 0xFF) if len(a) > 1 else np.zeros(0, np.int64)
    nxt = a[ff + 1] if len(ff) else ff
    is_rst = (nxt >= 0xD0) & (nxt <= 0xD7)
    is_marker = (nxt != 0x00) & ~is_rst & (nxt != 0xFF)
    m = np.flatnonzero(is_marker)
    if len(m):
        end = int(ff[m[0]])
        # fill bytes: a run of 0xFF in front of the marker belongs to the marker, not to the data
        while end > 0 and a[end - 1] == 0xFF:
            end -= 1
    else:
        end = len(a)  # truncated file: the data runs to the end of the bytes
    rst = ff[is_rst]
    rst = rst[rst < end]
    return start + end, [start + int(r) for r in rst]


def parse(data):
    """Walk the markers of a JPEG file (bytes-like) and decide the route.  Raises JpegError when the bytes are not a JPEG
    whose headers can be followed to the first scan; a returned info with device=False names the reason in `reason`."""
    buf = bytes(data) if not isinstance(data, (bytes, bytearray, memoryview)) else data
    buf = memoryview(buf).cast("B") if not isinstance(buf, bytes) else buf
    n = len(buf)
    if n < 4 or buf[0] != 0xFF or buf[1] != 0xD8:
        raise JpegError("not a JPEG file (no SOI)")
    info = JpegInfo()
    exif_segments, xmp = 0, False
    reasons = []
    p = 2
    while True:
        while p < n and buf[p] != 0xFF:  # tolerate garbage between segments as libjpeg does (with a warning)
            p += 1
        while p < n and buf[p] == 0xFF:
            p += 1
        if p >= n:
            raise JpegError("truncated file: no SOS")
        marker = 0xFF00 | buf[p]
        p += 1
        if marker in (0xFFD8, 0xFF01) or 0xFFD0 <= marker <= 0xFFD7:
            continue
        if marker == 0xFFD9:
            raise JpegError("EOI before the first scan")
        if p + 2 > n:
            raise JpegError("truncated file in a marker segment")
        L = (buf[p] << 8) | buf[p + 1]
        if L < 2 or p + L > n:
            raise JpegError("truncated file in a marker segment")
        seg = bytes(buf[p + 2:p + L])
        p += L
        if marker == 0xFFE0 and seg.startswith(b"JFIF\0"):
            info.jfif = True
        elif marker == 0xFFE1 and seg.startswith(b"Exif\0\0"):
            exif_segments += 1
            try:
                o = _exif_orientation(seg)
            except (JpegError, ValueError, IndexError):
                reasons.append("malformed Exif segment")
                o = None
            if o is not None:
                info.orientation = o
                info.exif_has_orientation = True
        elif marker == 0xFFE1 and seg.startswith(b"http://ns.adobe.com/xap/1.0/\x00"):
            xmp = True
        elif marker == 0xFFEE and seg.startswith(b"Adobe"):
            info.adobe = True
        elif marker == 0xFFDB:
            q = 0
            while q < len(seg):
                pq, tq = seg[q] >> 4, seg[q] & 15
                size = 128 if pq else 64
                if q + 1 + size > len(seg) or tq > 3:
                    raise JpegError("bad DQT segment")
                vals = np.frombuffer(seg, dtype=">u2" if pq else np.uint8, count=64, offset=q + 1).astype(np.int32)
                nat = np.zeros(64, np.int32)
                nat[ZIGZAG] = vals
                info.qtables[tq] = nat
                q += 1 + size
        elif marker == 0xFFC4:
            q = 0
            while q < len(seg):
                if q + 17 > len(seg):
                    raise JpegError("bad DHT segment")
                tc, th = seg[q] >> 4, seg[q] & 15
                bits = [0] + list(seg[q + 1:q + 17])
                cnt = sum(bits)
                if tc > 1 or th > 3 or cnt > 256 or q + 17 + cnt > len(seg):
                    raise JpegError("bad DHT segment")
                info.huff[(tc, th)] = (np.array(bits, np.int32), np.frombuffer(seg, np.uint8, cnt, q + 17).astype(np.int32))
                q += 17 + cnt
        elif marker == 0xFFDD:
            if len(seg) < 2:
                raise JpegError("bad DRI segment")
            info.restart_interval = (seg[0] << 8) | seg[1]
        elif 0xFFC0 <= marker <= 0xFFCF and marker not in (0xFFC4, 0xFFC8, 0xFFCC):
            if len(seg) < 6:
                raise JpegError("bad SOF segment")
            info.sof = marker & 0xFF
            info.precision = seg[0]
            info.height, info.width = (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4]
            nf = seg[5]
            if len(seg) < 6 + 3 * nf:
                raise JpegError("bad SOF segment")
            info.components = [(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i]) for i in range(nf)]
        elif marker == 0xFFDA:
            if not info.components:
                raise JpegError("SOS before SOF")
            ns = seg[0]
            if len(seg) < 1 + 2 * ns + 3:
                raise JpegError("bad SOS segment")
            ids = [seg[1 + 2 * i] for i in range(ns)]
            tabs = {seg[1 + 2 * i]: (seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15) for i in range(ns)}
            ss, se, ahal = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
            if sorted(ids) != sorted(c[0] for c in info.components):
                reasons.append("the first scan does not hold every component")
            else:
                info.scan_tables = [tabs[c[0]] for c in info.components]
            if (ss, se, ahal) != (0, 63, 0) and info.sof in (0xC0, 0xC1):
                reasons.append("sequential scan with spectral selection")
            info.scan_start = p
            info.scan_end, info.restart_markers = find_scan_end(buf, p)
            break
        # other APPn, COM, DAC, DNL...: skipped; they do not change Pillow's pixels (DNL-sized frames fail below)
    if exif_segments > 1:
        reasons.append("several Exif segments")
    if xmp and not info.exif_has_orientation:
        reasons.append("orientation possibly in XMP")
    _decide(info, reasons)
    return info


def _decide(info, reasons):
    if info.sof not in (0xC0, 0xC1):
        reasons.append({0xC2: "progressive", 0xC3: "lossless"}.get(info.sof, "arithmetic / hierarchical") + f" (SOF{info.sof - 0xC0})")
    if info.precision != 8:
        reasons.append(f"{info.precision}-bit samples")
    if info.height == 0 or info.width == 0:
        reasons.append("zero-sized frame (DNL)")
    if info.ncomp == 1:
        if info.components[0][1:3] != (1, 1):
            reasons.append("grayscale with sampling other than 1x1")
    elif info.ncomp == 3:
        ids = [c[0] for c in info.components]
        if info.adobe:
            reasons.append("Adobe colour transform marker")
        elif not info.jfif and ids == [82, 71, 66]:
            reasons.append("RGB components")
        y, cb, cr = info.components
        if (y[1], y[2]) not in SUPPORTED_SAMPLING or (cb[1], cb[2]) != (1, 1) or (cr[1], cr[2]) != (1, 1):
            reasons.append(f"sampling {y[1]}x{y[2]},{cb[1]}x{cb[2]},{cr[1]}x{cr[2]}")
    else:
        reasons.append(f"{info.ncomp} components")
    if not reasons:
        for c, (td, ta) in zip(info.components, info.scan_tables):
            if c[3] not in info.qtables:
                reasons.append("missing quantisation table")
            if (0, td) not in info.huff or (1, ta) not in info.huff:
                reasons.append("missing Huffman table")
            elif (info.huff[(0, td)][1] > 15).any():
                reasons.append("DC table with a symbol above 15")
        try:
            for key in {(0, td) for td, _ in info.scan_tables} | {(1, ta) for _, ta in info.scan_tables}:
                if key in info.huff:
                    huffman_lut(*info.huff[key])
        except JpegError as e:
            reasons.append(str(e))
    if not reasons and info.restart_interval:
        n_int = (mcu_count(info) + info.restart_interval - 1) // info.restart_interval
        if len(info.restart_markers) != n_int - 1:
            reasons.append("restart markers do not match the restart interval")
    info.device = not reasons
    info.reason = "; ".join(reasons)


def mcu_grid(info):
    """(mcus_x, mcus_y, blocks per MCU).  One component: a non-interleaved scan of ceil(W/8) x ceil(H/8) single blocks (T.81
    A.2.2); three components: interleaved MCUs of h*v luma blocks followed by one Cb and one Cr block (A.2.3)."""
    if info.ncomp == 1:
        return -(-info.width // 8), -(-info.height // 8), 1
    h, v = info.hmax, info.vmax
    return -(-info.width // (8 * h)), -(-info.height // (8 * v)), h * v + 2


def mcu_count(info):
    mx, my, _ = mcu_grid(info)
    return mx * my


def device_tables(info):
    """Arrays the device decoder takes: huff int32 [n_tables, TABLE_WORDS]; comp int32 [3, 4] rows of (dc table, ac table,
    quant table, h << 4 | v) per component; quant int32 [n_q, 64] natural order; restart offsets int32 (start of each interval after the
    first, i.e. two bytes past each RSTn marker, relative to the scan start)."""
    keys = sorted({(0, td) for td, _ in info.scan_tables} | {(1, ta) for _, ta in info.scan_tables})
    slot = {k: i for i, k in enumerate(keys)}
    huff = np.stack([huffman_lut(*info.huff[k]) for k in keys])
    qkeys = sorted({c[3] for c in info.components})
    qslot = {k: i for i, k in enumerate(qkeys)}
    quant = np.stack([info.qtables[k] for k in qkeys]).astype(np.int32)
    comp = np.zeros((3, 4), np.int32)
    for i, (c, (td, ta)) in enumerate(zip(info.components, info.scan_tables)):
        comp[i] = (slot[(0, td)], slot[(1, ta)], qslot[c[3]], (c[1] << 4) | c[2])
    rst = np.array([r + 2 - info.scan_start for r in info.restart_markers], np.int32)
    return huff, comp, quant, rst
