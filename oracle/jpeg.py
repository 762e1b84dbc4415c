"""Readable numpy restatement of the device JPEG decoder (ape_b200/csrc/jpeg.cu), stage by stage, pinned to Pillow bit for bit
by tests/test_jpeg_cpu.py.  Test infrastructure only: the Huffman decode is a plain Python loop.

Stages (each a function, so a device mismatch can be located):
  coefficients   sequential Huffman decode (ITU-T T.81 F.2.2), DC prediction reset at each restart, quantised int16
                 coefficients per component [rows of blocks, columns of blocks, 64] in natural order
  idct_islow     dequantise and the accurate integer IDCT Pillow's libjpeg uses by default (JDCT_ISLOW: the Loeffler-Ligtenberg-
                 Moschytz factorisation with 13-bit constants, 2 extra bits kept between the passes, round-half-up descaling,
                 the 1024-entry range-limit table)
  upsample       libjpeg's "fancy" chroma upsampling: triangle filters, 3/4 + 1/4 per axis, with the rounding bias alternating
                 between the two outputs of one input sample; plain replication when the chroma row is at most 2 samples wide
  ycc_to_rgb     JFIF YCbCr -> RGB in 16-bit fixed point (T.871 coefficients, tables rounded once, one rounding per channel)
  orient         detectron2's _apply_exif_orientation: the PIL transposes of EXIF orientations 2..8
"""
import numpy as np

from ape_b200 import jpeg as J


class BitReader:
    """MSB-first bits of one entropy-coded segment with the stuffed 0x00 after each 0xFF removed (T.81 F.1.2.3).  Reading past
    the end raises: a decoder that needs bits the file does not hold is decoding a truncated or corrupt scan."""

    def __init__(self, seg):
        a = np.frombuffer(seg, np.uint8)
        stuffed = np.zeros(len(a), bool)
        stuffed[1:] = (a[1:] == 0) & (a[:-1] == 0xFF)
        self.bits = np.unpackbits(a[~stuffed]).astype(np.int64)
        self.pos = 0

    def bit(self):
        if self.pos >= len(self.bits):
            raise ValueError("scan ends inside a code")
        b = int(self.bits[self.pos])
        self.pos += 1
        return b

    def get(self, n):
        v = 0
        for _ in range(n):
            v = (v << 1) | self.bit()
        return v


def _decode_symbol(r, table):
    """T.81 F.2.2.3 DECODE with MAXCODE / VALPTR: read bits until the code is not above the largest code of its length."""
    maxcode = table[J._MAXCODE:J._MAXCODE + 17]
    code = 0
    for l in range(1, 17):
        code = (code << 1) | r.bit()
        if code <= maxcode[l]:
            return int(table[J._VALS + table[J._VALOFF + l] + code])
    raise ValueError("invalid Huffman code")


def _extend(v, s):
    """T.81 F.2.2.1 EXTEND: an s-bit magnitude category value to a signed coefficient."""
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def coefficients(info, data):
    """Quantised coefficients of every component, [by, bx, 64] int16 in natural order, blocks covering whole MCUs."""
    huff, comp, _, rst = J.device_tables(info)
    mx, my, bpm = J.mcu_grid(info)
    layout = []  # (component, dy, dx) of each block of an MCU
    for ci, (_, h, v, _) in enumerate(info.components):
        hh, vv = (1, 1) if info.ncomp == 1 else (h, v)
        layout += [(ci, dy, dx) for dy in range(vv) for dx in range(hh)]
    out = []
    for ci, (_, h, v, _) in enumerate(info.components):
        hh, vv = (1, 1) if info.ncomp == 1 else (h, v)
        out.append(np.zeros((my * vv, mx * hh, 64), np.int16))
    starts = [0] + [int(o) for o in rst]
    ends = [int(o) - 2 for o in rst] + [info.scan_end - info.scan_start]
    ri = info.restart_interval or mx * my
    mcu = 0
    for s, e in zip(starts, ends):
        r = BitReader(bytes(data[info.scan_start + s:info.scan_start + e]))
        pred = [0, 0, 0]
        for _ in range(min(ri, mx * my - mcu)):
            mcux, mcuy = mcu % mx, mcu // mx
            for ci, dy, dx in layout:
                hh, vv = (1, 1) if info.ncomp == 1 else info.components[ci][1:3]
                blk = out[ci][mcuy * vv + dy, mcux * hh + dx]
                sym = _decode_symbol(r, huff[comp[ci, 0]])
                pred[ci] += _extend(r.get(sym), sym)
                blk[0] = np.int16(((pred[ci] + 32768) & 0xFFFF) - 32768)
                k = 1
                while k < 64:
                    rs = _decode_symbol(r, huff[comp[ci, 1]])
                    run, size = rs >> 4, rs & 15
                    if size:
                        k += run
                        blk[J.ZIGZAG[min(k, 63)]] = _extend(r.get(size), size)
                        k += 1
                    elif run == 15:
                        k += 16
                    else:
                        break
            mcu += 1
    return out


def _range_limit(x):
    """libjpeg's IDCT output table indexed by (value & 1023): value + 128 clamped to 0..255 for |value| < 512, and the table's
    wrap-around beyond (never reached by coefficients an encoder produces)."""
    i = x & 1023
    return np.where(i < 128, i + 128, np.where(i < 512, 255, np.where(i < 896, 0, i - 896))).astype(np.uint8)


def idct_islow(coef, quant):
    """coef int16 [..., 64] natural order, quant int [64] -> uint8 [..., 8, 8]."""
    c = coef.astype(np.int64) * quant.astype(np.int16).astype(np.int64)  # libjpeg keeps the multipliers as int16
    c = c.reshape(coef.shape[:-1] + (8, 8))

    def one_d(d0, d1, d2, d3, d4, d5, d6, d7):
        z1 = (d2 + d6) * 4433
        t2 = z1 - d6 * 15137
        t3 = z1 + d2 * 6270
        t0 = (d0 + d4) << 13
        t1 = (d0 - d4) << 13
        t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
        o0, o1, o2, o3 = d7, d5, d3, d1
        z1, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
        z5 = (z3 + z4) * 9633
        o0, o1, o2, o3 = o0 * 2446, o1 * 16819, o2 * 25172, o3 * 12299
        z1, z2, z3, z4 = z1 * -7373, z2 * -20995, z3 * -16069 + z5, z4 * -3196 + z5
        o0, o1, o2, o3 = o0 + z1 + z3, o1 + z2 + z4, o2 + z2 + z3, o3 + z1 + z4
        return [t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3]

    def descale(x, n):
        return (x + (1 << (n - 1))) >> n

    cols = one_d(*[c[..., r, :] for r in range(8)])  # pass 1 over columns: row r of the result
    ws = np.stack([descale(v, 13 - 2) for v in cols], axis=-2)
    rows = one_d(*[ws[..., :, k] for k in range(8)])  # pass 2 over rows
    out = np.stack([descale(v, 13 + 2 + 3) for v in rows], axis=-1)
    return _range_limit(out)


def planes(info, data):
    """Component sample planes (uint8, whole blocks) after the IDCT."""
    _, comp, quant, _ = J.device_tables(info)
    ps = []
    for ci, c in enumerate(coefficients(info, data)):
        px = idct_islow(c, quant[comp[ci, 2]])
        ps.append(px.transpose(0, 2, 1, 3).reshape(c.shape[0] * 8, c.shape[1] * 8))
    return ps


def upsample(plane, h, v, dw, dh, width, height):
    """A chroma plane (dw x dh real samples) to width x height with libjpeg's fancy upsampling (h, v in {1, 2})."""
    p = plane[:dh, :dw].astype(np.int64)
    if h == 1:
        return p[:height, :width]
    if dw <= 2:  # too narrow for the triangle filter: box replication
        return np.repeat(np.repeat(p, 2, 1), v, 0)[:height, :width]
    left = np.concatenate([p[:, :1], p[:, :-1]], 1)
    right = np.concatenate([p[:, 1:], p[:, -1:]], 1)
    if v == 1:
        even = (3 * p + left + 1) >> 2
        odd = (3 * p + right + 2) >> 2
        even[:, 0] = p[:, 0]
        odd[:, -1] = p[:, -1]
        out = np.stack([even, odd], -1).reshape(dh, 2 * dw)
        return out[:height, :width]
    up = np.concatenate([p[:1], p[:-1]], 0)
    down = np.concatenate([p[1:], p[-1:]], 0)
    rows = []
    for nb in (up, down):  # output row 2i: rows i and i-1; row 2i+1: rows i and i+1
        cs = 3 * p + nb
        cl = np.concatenate([cs[:, :1], cs[:, :-1]], 1)
        cr = np.concatenate([cs[:, 1:], cs[:, -1:]], 1)
        even = (3 * cs + cl + 8) >> 4
        odd = (3 * cs + cr + 7) >> 4
        even[:, 0] = (4 * cs[:, 0] + 8) >> 4
        odd[:, -1] = (4 * cs[:, -1] + 7) >> 4
        rows.append(np.stack([even, odd], -1).reshape(dh, 2 * dw))
    out = np.stack(rows, 1).reshape(2 * dh, 2 * dw)
    return out[:height, :width]


def ycc_to_rgb(y, cb, cr):
    """libjpeg's ycc_rgb_convert: R = Y + 1.402 Cr', G = Y - 0.34414 Cb' - 0.71414 Cr', B = Y + 1.772 Cb' with
    Cb' = Cb - 128, coefficients scaled by 2^16 and rounded (FIX), the R and B terms rounded per table entry, the G term
    rounded once after the sum (the +1/2 sits in the Cb table), arithmetic right shifts, results clamped to 0..255."""
    fix = lambda x: int(x * 65536 + 0.5)  # noqa: E731
    cb = cb.astype(np.int64) - 128
    cr = cr.astype(np.int64) - 128
    y = y.astype(np.int64)
    r = y + ((fix(1.40200) * cr + 32768) >> 16)
    g = y + ((-fix(0.34414) * cb + -fix(0.71414) * cr + 32768) >> 16)
    b = y + ((fix(1.77200) * cb + 32768) >> 16)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def orient(img, orientation):
    """PIL Image.transpose of detectron2's _apply_exif_orientation on an HWC array."""
    if orientation == 2:
        return img[:, ::-1]
    if orientation == 3:
        return img[::-1, ::-1]
    if orientation == 4:
        return img[::-1]
    if orientation == 5:
        return img.transpose(1, 0, 2)
    if orientation == 6:
        return img[::-1].transpose(1, 0, 2)
    if orientation == 7:
        return img[::-1, ::-1].transpose(1, 0, 2)
    if orientation == 8:
        return img[:, ::-1].transpose(1, 0, 2)
    return img


def decode(data, format="RGB", apply_orientation=True):
    """The uint8 [H, W, 3] image of detectron2's read_image(file, format) for a file the device route takes."""
    info = J.parse(data)
    assert info.device, info.reason
    ps = planes(info, data)
    H, W = info.height, info.width
    if info.ncomp == 1:
        g = ps[0][:H, :W]
        rgb = np.stack([g, g, g], -1)
    else:
        h, v = info.hmax, info.vmax
        dw, dh = -(-W // h), -(-H // v)
        cb = upsample(ps[1], h, v, dw, dh, W, H)
        cr = upsample(ps[2], h, v, dw, dh, W, H)
        rgb = ycc_to_rgb(ps[0][:H, :W], cb, cr)
    if apply_orientation:
        rgb = orient(rgb, info.orientation)
    if format == "BGR":
        rgb = rgb[:, :, ::-1]
    return np.ascontiguousarray(rgb)
