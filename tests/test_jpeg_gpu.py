"""Device JPEG decode (csrc/jpeg.cu) against Pillow, bit for bit, and the predictor taking JPEG files."""
import io

import numpy as np
import pytest
import torch

from test_jpeg_cpu import encode, make_image, pillow_rgb

Image = pytest.importorskip("PIL.Image")

pytestmark = pytest.mark.gpu


def device_rgb(data, fmt="RGB"):
    from ape_b200.engine import read_image

    img, route = read_image(data, format=fmt, with_route=True)
    assert route == "device"
    assert img.is_cuda and img.dtype == torch.uint8
    return img.cpu().numpy()


SIZES = [(1, 1), (7, 13), (17, 9), (480, 640), (769, 1023), (3024, 4032)]


@pytest.mark.parametrize("h,w", SIZES)
@pytest.mark.parametrize("ss", [0, 1, 2, "gray"])
def test_device_decode_equals_pillow_sizes(built, h, w, ss):
    img = make_image(h, w, h + w, "noise" if h * w < 1 << 20 else "flat")
    if h * w >= 1 << 20:  # photo-like: smooth gradients plus mild noise
        img = np.clip(img.astype(np.int16) + np.random.default_rng(1).integers(-12, 13, img.shape), 0, 255).astype(np.uint8)
    data = encode(img, gray=True, quality=95) if ss == "gray" else encode(img, quality=95, subsampling=ss)
    np.testing.assert_array_equal(device_rgb(data), pillow_rgb(data))


@pytest.mark.parametrize("q", [5, 50, 95, 100])
@pytest.mark.parametrize("ss", [0, 1, 2, "gray"])
@pytest.mark.parametrize("kind", ["noise", "flat"])
def test_device_decode_equals_pillow_quality(built, q, ss, kind):
    img = make_image(123, 201, q, kind)
    data = encode(img, gray=True, quality=q) if ss == "gray" else encode(img, quality=q, subsampling=ss)
    np.testing.assert_array_equal(device_rgb(data), pillow_rgb(data))


@pytest.mark.parametrize("kw", [dict(optimize=True), dict(restart_marker_blocks=1), dict(restart_marker_blocks=5),
                                dict(restart_marker_rows=1), dict(restart_marker_rows=3, optimize=True)])
@pytest.mark.parametrize("ss", [0, 1, 2])
def test_device_decode_equals_pillow_tables_and_restarts(built, kw, ss):
    data = encode(make_image(301, 257, 3), quality=90, subsampling=ss, **kw)
    np.testing.assert_array_equal(device_rgb(data), pillow_rgb(data))


def test_noise_scan_is_long_and_stuffed(built):
    """Noise at quality 100: long codes and many stuffed 0xFF 0x00 pairs across hundreds of subsequences."""
    data = encode(make_image(512, 768, 4), quality=100, subsampling=0)
    from ape_b200 import jpeg as J

    info = J.parse(data)
    scan = np.frombuffer(data, np.uint8)[info.scan_start:info.scan_end]
    assert int(((scan[:-1] == 0xFF) & (scan[1:] == 0)).sum()) > 1000
    np.testing.assert_array_equal(device_rgb(data), pillow_rgb(data))


@pytest.mark.parametrize("orientation", range(1, 9))
@pytest.mark.parametrize("fmt", ["BGR", "RGB"])
def test_device_read_image_orientation_and_format(built, orientation, fmt):
    from ape_b200.engine.read import host_read_image

    ex = Image.Exif()
    ex[0x0112] = orientation
    data = encode(make_image(37, 61, 5), quality=90, subsampling=2, exif=ex)
    np.testing.assert_array_equal(device_rgb(data, fmt), host_read_image(data, fmt))


def test_host_route_for_progressive(built, tmp_path):
    from ape_b200.engine import read_image
    from ape_b200.engine.read import host_read_image

    data = encode(make_image(40, 30, 6), quality=90, progressive=True)
    p = tmp_path / "p.jpg"
    p.write_bytes(data)
    img, route = read_image(str(p), with_route=True)
    assert route == "host" and img.is_cuda
    np.testing.assert_array_equal(img.cpu().numpy(), host_read_image(data, "BGR"))


def test_corrupt_scans_raise(built):
    """Input validation: a truncated file and a scan with an invalid Huffman code each return an error status (decoded once
    each)."""
    from ape_b200 import jpeg as J
    from ape_b200.engine import read_image

    data = encode(make_image(64, 96, 7), quality=95, subsampling=2)
    info = J.parse(data)
    cut = data[:info.scan_start + (info.scan_end - info.scan_start) // 2]
    with pytest.raises(RuntimeError, match="corrupt scan"):
        read_image(cut)
    # sixteen 1 bits are no code of any JPEG Huffman table (the all-ones code is reserved, T.81 C): 0xFF 0x00 0xFF 0x00
    # written at the start of the scan (stuffed, so the marker structure stays intact)
    bad = bytearray(data)
    bad[info.scan_start:info.scan_start + 4] = b"\xff\x00\xff\x00"
    with pytest.raises(RuntimeError, match="invalid Huffman code"):
        read_image(bytes(bad))


def _model(masks):
    from ape_b200 import configs
    from ape_b200.modeling import build_model
    from oracle import synth

    model = build_model(configs.MINI)
    synth.fill_state_dict(model)
    model = model.cuda().eval()
    model.test_mask_on = masks
    return model


@pytest.mark.parametrize("masks", [False, True])
def test_predictor_on_paths_equals_predictor_on_arrays(built, tmp_path, masks):
    from ape_b200.engine import DefaultPredictor, ResizeShortestEdge, read_image

    model = _model(masks)
    pred = DefaultPredictor(model, ResizeShortestEdge(48, 64), input_format="RGB")
    paths = []
    for i, (h, w, o) in enumerate([(45, 60, 1), (60, 45, 6), (50, 50, 3)]):
        ex = Image.Exif()
        ex[0x0112] = o
        p = tmp_path / f"{i}.jpg"
        p.write_bytes(encode(make_image(h, w, 20 + i, "flat"), quality=90, subsampling=2, exif=ex))
        paths.append(str(p))
    for p in paths:
        arr = read_image(p).cpu().numpy()
        inp = pred.preprocess(p)
        assert (inp["height"], inp["width"]) == arr.shape[:2]
        assert torch.equal(inp["image"], pred.preprocess(arr)["image"])
        a, b = pred(p)["instances"], pred(arr)["instances"]
        assert len(a) == len(b) > 0
        assert torch.equal(a.pred_boxes.tensor, b.pred_boxes.tensor) and torch.equal(a.scores, b.scores)
        assert torch.equal(a.pred_classes, b.pred_classes)
        if masks:
            assert torch.equal(a.pred_masks, b.pred_masks)
    arrays = [read_image(p).cpu().numpy() for p in paths]
    by_path = pred.predict_batch(paths + [open(paths[0], "rb").read()])
    by_array = pred.predict_batch(arrays + [arrays[0]])
    for a, b in zip(by_path, by_array):
        a, b = a["instances"], b["instances"]
        assert torch.equal(a.pred_boxes.tensor, b.pred_boxes.tensor) and torch.equal(a.scores, b.scores)
