"""JPEG header walk, route decision and the numpy restatement of the device decoder (oracle/jpeg.py) pinned to Pillow.

The corpus is written by Pillow at test time from seeded numpy images; nothing is downloaded or committed."""
import io

import numpy as np
import pytest

Image = pytest.importorskip("PIL.Image")

from ape_b200 import jpeg as J  # noqa: E402
from ape_b200.engine.read import host_read_image  # noqa: E402
from oracle import jpeg as OJ  # noqa: E402

SAMPLING = {0: (1, 1), 1: (2, 1), 2: (2, 2)}


def make_image(h, w, seed, kind="noise"):
    g = np.random.default_rng(seed)
    if kind == "noise":
        return g.integers(0, 256, (h, w, 3), dtype=np.uint8)
    yy, xx = np.mgrid[:h, :w]
    base = np.stack([(xx * 5 + yy * 3) % 256, 128 + 0 * xx, (yy * 7) % 256], -1)
    return (base // 32 * 32).astype(np.uint8)  # flat patches: mostly end-of-block codes


def encode(img, gray=False, **kw):
    # Pillow's optimize / progressive writers hold the whole file in one buffer of at least ImageFile.MAXBLOCK bytes, sized
    # for photographs: noise at high quality needs more
    from PIL import ImageFile

    b = io.BytesIO()
    old = ImageFile.MAXBLOCK
    ImageFile.MAXBLOCK = max(old, 4 * img.shape[0] * img.shape[1] + (1 << 16))
    try:
        Image.fromarray(img[..., 0] if gray else img).save(b, "JPEG", **kw)
    finally:
        ImageFile.MAXBLOCK = old
    return b.getvalue()


def pillow_rgb(data):
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


@pytest.mark.parametrize("ss", [0, 1, 2])
def test_parse_colour_layouts(ss):
    data = encode(make_image(17, 9, 0), quality=90, subsampling=ss)
    info = J.parse(data)
    assert info.device, info.reason
    assert (info.height, info.width, info.ncomp) == (17, 9, 3)
    assert info.components[0][1:3] == SAMPLING[ss] and all(c[1:3] == (1, 1) for c in info.components[1:])
    assert info.restart_interval == 0 and info.orientation == 1
    assert data[info.scan_end:info.scan_end + 2] == b"\xff\xd9" and info.scan_start < info.scan_end
    h, v = SAMPLING[ss]
    assert J.mcu_grid(info) == (-(-9 // (8 * h)), -(-17 // (8 * v)), h * v + 2)
    huff, comp, quant, rst = J.device_tables(info)
    assert huff.shape[1] == J.TABLE_WORDS and quant.shape[1] == 64 and rst.size == 0
    assert comp[0, 3] == (h << 4) | v


def test_parse_grayscale_and_quant_natural_order():
    data = encode(make_image(7, 13, 1), gray=True, quality=50)
    info = J.parse(data)
    assert info.device and info.ncomp == 1 and J.mcu_grid(info) == (2, 1, 1)
    # Pillow's quality-50 luma table is the T.81 Annex K table: natural order starts 16 11 10 16 24
    assert list(info.qtables[info.components[0][3]][:5]) == [16, 11, 10, 16, 24]


def test_huffman_lut_resolves_every_code():
    data = encode(make_image(16, 16, 2), quality=75, optimize=True)
    info = J.parse(data)
    for bits, vals in info.huff.values():
        t = J.huffman_lut(bits, vals)
        code, k = 0, 0
        for l in range(1, 17):
            for _ in range(int(bits[l])):
                if l <= J.LOOKAHEAD:
                    e = t[code << (J.LOOKAHEAD - l)]
                    assert (e >> 8, e & 255) == (l, vals[k])
                else:
                    assert t[J._MAXCODE + l] >= code and t[J._VALS + t[J._VALOFF + l] + code] == vals[k]
                code += 1
                k += 1
            code <<= 1


@pytest.mark.parametrize("kw", [dict(restart_marker_blocks=1), dict(restart_marker_blocks=5), dict(restart_marker_rows=1)])
def test_parse_restart_markers(kw):
    data = encode(make_image(48, 40, 3), quality=80, subsampling=2, **kw)
    info = J.parse(data)
    assert info.device, info.reason
    assert info.restart_interval > 0
    _, _, _, rst = J.device_tables(info)
    assert len(rst) == -(-J.mcu_count(info) // info.restart_interval) - 1 > 0
    for off in rst:  # two bytes past each RSTn, numbered 0..7 in turn
        assert data[info.scan_start + off - 2] == 0xFF and 0xD0 <= data[info.scan_start + off - 1] <= 0xD7


@pytest.mark.parametrize("orientation", range(1, 9))
def test_parse_exif_orientation(orientation):
    ex = Image.Exif()
    ex[J.EXIF_ORIENTATION] = orientation
    info = J.parse(encode(make_image(9, 14, 4), exif=ex))
    assert info.device and info.orientation == orientation
    assert info.oriented_hw == ((14, 9) if orientation >= 5 else (9, 14))


def test_host_route_progressive_cmyk_and_440():
    img = make_image(16, 16, 5)
    prog = J.parse(encode(img, progressive=True))
    assert not prog.device and "progressive" in prog.reason
    b = io.BytesIO()
    Image.fromarray(img).convert("CMYK").save(b, "JPEG")
    cmyk = J.parse(b.getvalue())
    assert not cmyk.device and "4 components" in cmyk.reason
    # 4:4:0 (luma 1x2): Pillow cannot write it, so patch the SOF0 of a 4:4:4 file (only the route decision is tested)
    data = bytearray(encode(img, subsampling=0))
    sof = data.index(b"\xff\xc0")
    assert data[sof + 11] == 0x11  # component 1's sampling byte
    data[sof + 11] = 0x12
    v440 = J.parse(bytes(data))
    assert not v440.device and "sampling 1x2" in v440.reason


def test_parse_rejects_non_jpeg_and_truncated_headers():
    with pytest.raises(J.JpegError):
        J.parse(b"\x89PNG\r\n\x1a\n")
    data = encode(make_image(8, 8, 6))
    with pytest.raises(J.JpegError):
        J.parse(data[:100])  # ends inside the header segments


CASES = [(h, w, ss, q, kind) for (h, w) in [(1, 1), (7, 13), (17, 9), (33, 40)] for ss in (0, 1, 2, "gray")
         for q in (5, 50, 95, 100) for kind in ("noise", "flat")]


@pytest.mark.parametrize("h,w,ss,q,kind", CASES)
def test_oracle_equals_pillow(h, w, ss, q, kind):
    img = make_image(h, w, 7 + h * w, kind)
    data = encode(img, gray=True, quality=q) if ss == "gray" else encode(img, quality=q, subsampling=ss)
    assert J.parse(data).device
    np.testing.assert_array_equal(OJ.decode(data), pillow_rgb(data))


@pytest.mark.parametrize("kw", [dict(optimize=True), dict(restart_marker_blocks=2), dict(restart_marker_rows=1),
                                dict(restart_marker_blocks=7, optimize=True)])
@pytest.mark.parametrize("ss", [0, 1, 2])
def test_oracle_equals_pillow_optimized_and_restarts(kw, ss):
    data = encode(make_image(35, 50, 8), quality=90, subsampling=ss, **kw)
    assert J.parse(data).device
    np.testing.assert_array_equal(OJ.decode(data), pillow_rgb(data))


@pytest.mark.parametrize("orientation", range(1, 9))
@pytest.mark.parametrize("fmt", ["BGR", "RGB"])
def test_oracle_equals_read_image_semantics(orientation, fmt):
    ex = Image.Exif()
    ex[J.EXIF_ORIENTATION] = orientation
    data = encode(make_image(11, 19, 9), quality=85, subsampling=2, exif=ex)
    want = host_read_image(data, fmt)
    assert want.shape[:2] == J.parse(data).oriented_hw
    np.testing.assert_array_equal(OJ.decode(data, fmt), want)


def test_orientations_are_pil_transposes():
    """oracle.orient(o) equals PIL's transpose of detectron2's table for every orientation."""
    img = make_image(5, 7, 10)
    table = {2: "FLIP_LEFT_RIGHT", 3: "ROTATE_180", 4: "FLIP_TOP_BOTTOM", 5: "TRANSPOSE", 6: "ROTATE_270", 7: "TRANSVERSE",
             8: "ROTATE_90"}
    for o, name in table.items():
        want = np.asarray(Image.fromarray(img).transpose(getattr(Image.Transpose, name)))
        np.testing.assert_array_equal(OJ.orient(img, o), want)


def test_oracle_stages_locate_the_arithmetic():
    """The stages compose to the decode: IDCT planes, then upsampling and colour."""
    data = encode(make_image(16, 24, 11), quality=70, subsampling=2)
    info = J.parse(data)
    ps = OJ.planes(info, data)
    assert [p.shape for p in ps] == [(16, 32), (8, 16), (8, 16)]
    cb = OJ.upsample(ps[1], 2, 2, 12, 8, 24, 16)
    cr = OJ.upsample(ps[2], 2, 2, 12, 8, 24, 16)
    np.testing.assert_array_equal(OJ.ycc_to_rgb(ps[0][:16, :24], cb, cr), pillow_rgb(data))


def test_oracle_rejects_a_truncated_scan():
    data = encode(make_image(32, 32, 12), quality=95)
    info = J.parse(data)
    cut = data[:info.scan_start + (info.scan_end - info.scan_start) // 2]
    tinfo = J.parse(cut)
    assert tinfo.device and tinfo.scan_end == len(cut)  # the headers are intact: the device route takes it and must fail
    with pytest.raises(ValueError):
        OJ.decode(cut)
