"""`read_image` on the device: detectron2's `detectron2.data.detection_utils.read_image(file_name, format)` for JPEG files
(PIL decode, `_apply_exif_orientation`, `convert("RGB")`, the channel flip of format="BGR"), with the decode in the engine's
own kernels (csrc/jpeg.cu) and only the compressed bytes uploaded.  Files the device decoder does not reproduce bit for bit
(see `ape_b200.jpeg`) take the host route: Pillow, then an upload of the decoded array."""
import io
import os

import numpy as np
import torch

from .. import jpeg as J
from .. import ops

_EXIF_TRANSPOSE = {2: "FLIP_LEFT_RIGHT", 3: "ROTATE_180", 4: "FLIP_TOP_BOTTOM", 5: "TRANSPOSE", 6: "ROTATE_270",
                   7: "TRANSVERSE", 8: "ROTATE_90"}


def file_bytes(path_or_bytes):
    """The bytes of a file given by path (str / os.PathLike) or as bytes-like."""
    if isinstance(path_or_bytes, (bytes, bytearray, memoryview)):
        return bytes(path_or_bytes)
    with open(os.fspath(path_or_bytes), "rb") as f:
        return f.read()


def is_encoded(x):
    """True for the inputs the predictor decodes itself: a path or the bytes of a file."""
    return isinstance(x, (str, bytes, bytearray, memoryview, os.PathLike))


def host_read_image(data, format="BGR"):
    """detectron2 read_image(file, format) for format "BGR" / "RGB" on the host: Pillow decode, EXIF transpose, RGB."""
    from PIL import Image

    img = Image.open(io.BytesIO(data))
    try:
        exif = img.getexif()
    except Exception:  # detectron2 ignores unreadable EXIF blocks
        exif = None
    method = _EXIF_TRANSPOSE.get(exif.get(J.EXIF_ORIENTATION)) if exif is not None else None
    if method is not None:
        img = img.transpose(getattr(Image.Transpose, method))
    a = np.asarray(img.convert("RGB"))
    return np.ascontiguousarray(a[:, :, ::-1]) if format == "BGR" else a


def decode(data, format="BGR", device="cuda", host=None):
    """Start the decode of one file's bytes on the current stream.  Returns (image, status, route): on the device route
    `status` is the decoder's device status word (check it with ops.jpeg_check); on the host route it is None and the image
    is the uploaded host decode."""
    assert format in ("BGR", "RGB"), f"read_image: format {format!r} (BGR or RGB)"
    try:
        info = J.parse(data)
    except J.JpegError:
        info = None
    if info is not None and info.device:
        img, status = ops.jpeg_decode(info, data, format=format, device=device, host=host)
        return img, status, "device"
    return torch.from_numpy(host_read_image(data, format)).to(device), None, "host"


def read_image(path_or_bytes, format="BGR", device="cuda", with_route=False):
    """The uint8 [H, W, 3] device tensor that detectron2's read_image(path, format) returns, bit for bit (format "BGR" or
    "RGB").  Supported JPEGs are decoded on the device from their compressed bytes; anything else is decoded by Pillow on the
    host and uploaded.  with_route=True returns (image, route) with route "device" or "host".  A corrupt scan on the device
    route raises RuntimeError."""
    img, status, route = decode(file_bytes(path_or_bytes), format, device)
    if status is not None:
        ops.jpeg_check(status)
    return (img, route) if with_route else img
