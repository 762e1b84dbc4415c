#!/usr/bin/env python
"""Device JPEG decode against detectron2-style host decode (development aid; numbers in DESIGN.md §5 and the README).

One run prints: the card and its power limit; per image (640x480 COCO-like and 4032x3024 photo-like, quality 95, Pillow's
default 4:2:0) the device decode time (CUDA events around ops.jpeg_decode, warmed: upload of the compressed bytes + kernels),
the end-to-end read_image time (header walk + upload + decode + status check), the host read_image time (Pillow decode +
EXIF + convert) and its upload, and the bytes uploaded on each route; then DefaultPredictor.predict_batch throughput over 64
files against the same 64 images as decoded arrays (APE-L_D spec of bench.py at 1024^2, boxes)."""
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ape_b200 import jpeg as J  # noqa: E402
from ape_b200 import ops  # noqa: E402
from ape_b200.engine import read as R  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def photo(h, w, seed):
    """Smooth colour gradients + blobs + mild sensor-like noise: compresses like a photograph at quality 95."""
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[:h, :w].astype(np.float32)
    img = np.stack([128 + 100 * np.sin(xx / (37 + 11 * c) + yy / (53 + 7 * c) + c) for c in range(3)], -1)
    for _ in range(12):
        cy, cx, r = g.uniform(0, h), g.uniform(0, w), g.uniform(0.05, 0.2) * min(h, w)
        img += g.uniform(-60, 60, 3) * np.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * r * r))[..., None]
    img += g.normal(0, 4, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


def encode(img, q=95):
    import io

    from PIL import Image

    b = io.BytesIO()
    Image.fromarray(img).save(b, "JPEG", quality=q)
    return b.getvalue()


def time_events(fn, n):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / n


def time_host(fn, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n * 1e3


def decode_table():
    rows = []
    for name, (h, w) in (("640x480", (480, 640)), ("4032x3024", (3024, 4032))):
        data = encode(photo(h, w, 0))
        info = J.parse(data)
        assert info.device, info.reason
        host_buf = torch.empty((3 * len(data) + (1 << 16),), dtype=torch.uint8, pin_memory=True)
        n = 50 if h < 1000 else 10
        for _ in range(3):
            ops.jpeg_decode(info, data, "BGR", "cuda", host=host_buf)
        torch.cuda.synchronize()
        dev_ms = time_events(lambda: ops.jpeg_decode(info, data, "BGR", "cuda", host=host_buf), n)
        e2e_ms = time_host(lambda: R.read_image(data), n)
        host_ms = time_host(lambda: R.host_read_image(data, "BGR"), n)
        arr = R.host_read_image(data, "BGR")
        up_ms = time_host(lambda: torch.from_numpy(arr).to("cuda"), n)
        got = R.read_image(data).cpu().numpy()
        assert np.array_equal(got, arr), "device decode differs from the host decode"
        scan = info.scan_end - info.scan_start
        rows.append(dict(image=name, file_bytes=len(data), device_upload_bytes=scan, host_upload_bytes=arr.nbytes,
                         device_decode_ms=round(dev_ms, 3), device_read_image_ms=round(e2e_ms, 3),
                         host_decode_ms=round(host_ms, 3), host_upload_ms=round(up_ms, 3)))
    return rows


def predictor_throughput(tmpdir, n_files=64):
    import bench
    from ape_b200.engine import DefaultPredictor, ResizeShortestEdge
    from ape_b200.modeling import build_model

    model = bench.bench_weights(build_model(bench.bench_spec(), num_text=1203)).to("cuda")
    model.engine_dtype = torch.float16
    model.use_cuda_graphs = True
    pred = DefaultPredictor(model, ResizeShortestEdge(1024, 1024), "RGB")
    paths = []
    for i in range(n_files):
        p = os.path.join(tmpdir, f"{i}.jpg")
        with open(p, "wb") as f:
            f.write(encode(photo(480, 640, i)))
        paths.append(p)
    arrays = [R.host_read_image(R.file_bytes(p), "BGR") for p in paths]
    pred.predict_batch(arrays[:4])  # captures the packed-forward graph
    pred.predict_batch(paths[:4])
    t_arr = time_host(lambda: pred.predict_batch(arrays), 2) / n_files
    t_path = time_host(lambda: pred.predict_batch(paths), 2) / n_files
    t_read = time_host(lambda: pred.predict_batch([R.host_read_image(R.file_bytes(p), "BGR") for p in paths]), 2) / n_files
    return dict(images=n_files, size="640x480 q95 -> 1024", ms_per_image_arrays_predecoded=round(t_arr, 3),
                ms_per_image_paths_device_decode=round(t_path, 3), ms_per_image_paths_host_read_image=round(t_read, 3))


if __name__ == "__main__":
    import json
    import tempfile

    print(json.dumps(dict(card=card(), torch=torch.__version__)))
    for r in decode_table():
        print(json.dumps(r))
    with tempfile.TemporaryDirectory() as d:
        print(json.dumps(predictor_throughput(d)))
