#!/usr/bin/env python
"""CUDA graphs over a stream of mixed image sizes.  Development aid.

    python tests/perf_graph_sizes.py [--rounds 5] [--images 64]

APE-L_D at 1024^2, 1203 names, fp16, boxes only, bench.py's weights and score threshold.  The stream: a seeded list of photo sizes
between 320 and 640 pixels a side, passed through ResizeShortestEdge(1024, 1024), one image per call.  Records:
  eager_ms         the eager step (use_cuda_graphs off) at the stream's first size
  replay_fixed_ms  the graph replay step at that one size (bench.py's condition)
  replay_stream_ms the graph step averaged over the mixed stream, once per round
  capture_ms       the first call at a new key (two eager warm-up passes, capture, instantiate, replay)
  old_key_captures the captures a key holding the image sizes with an 8-entry LRU would make on the stream (replayed on the host)
  graphs           the "forward" graphs held after the stream; peak_mib the peak device memory after it
  pad_geometry_ms  ops.pad_geometry at B = 1 (CUDA events over 50 launches) against the torch geometry it replaces
Times are the median and [min, max] in ms of host clocks around work that ends in a synchronise; the first line is the card."""
import argparse
import collections
import copy
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from perf_ape_ti import card  # noqa: E402

SCORE_THRESH = 0.0123  # bench.py's BENCH_SCORE_THRESH


def stat(ts, digits=3):
    return {"median": round(statistics.median(ts), digits), "min": round(min(ts), digits), "max": round(max(ts), digits)}


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def stream_sizes(n, seed=0):
    from ape_b200.engine import ResizeShortestEdge

    g = np.random.default_rng(seed)
    orig = [(int(g.integers(320, 641)), int(g.integers(320, 641))) for _ in range(n)]
    return [ResizeShortestEdge.get_output_shape(h, w, 1024, 1024) for h, w in orig]


def old_key_captures(sizes, capacity=8):
    lru, n = collections.OrderedDict(), 0
    for s in sizes:
        if s in lru:
            lru.move_to_end(s)
            continue
        n += 1
        while len(lru) >= capacity:
            lru.popitem(last=False)
        lru[s] = True
    return n


def geometry_kernel(model, rounds):
    """ops.pad_geometry (what every CUDA forward now runs) against the torch geometry of the parent's _geometry."""
    from ape_b200 import ops

    h, w = 1024, 768
    pgeo = model._padded_geometry((1, 3, 1024, 1024))
    sizes = torch.tensor([[h, w]], dtype=torch.int32, device="cuda")
    tr, pe = model.transformer, model.position_embedding

    def kernel():
        ops.pad_geometry(sizes, (1024, 1024), pgeo["shapes"], pgeo["dim_t"], tr.level_embeds, torch.float16, pe.offset, pe.eps, pe.scale)

    def torch_geometry():
        m = torch.ones((1, 1024, 1024), device="cuda")
        m[0, :h, :w] = 0
        masks = [F.interpolate(m[None], size=sh).to(torch.bool).squeeze(0) for sh in pgeo["shapes"]]
        geo = tr.geometry(pgeo["shapes"], masks, [pe(x).to(torch.float32) for x in masks])
        lvl = torch.cat([tr.level_embeds[i].view(1, 1, -1).expand(1, a * b, -1) for i, (a, b) in enumerate(pgeo["shapes"])], 1)
        (geo["pos_flatten"] + lvl.float()).to(torch.float16)

    out = {}
    with torch.no_grad():
        for name, fn, n in (("kernel", kernel, 50), ("torch", torch_geometry, 10)):
            for _ in range(3):
                fn()
            ts = []
            for _ in range(rounds):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(n):
                    fn()
                b.record()
                torch.cuda.synchronize()
                ts.append(a.elapsed_time(b) / n)
            out[name] = stat(ts, 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--images", type=int, default=64)
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)

    from ape_b200 import configs, synthetic
    from ape_b200.modeling import build_model

    spec = copy.deepcopy(configs.APE_L_D)
    spec["test_score_thresh"] = SCORE_THRESH
    model = build_model(spec, num_text=1203)
    synthetic.fill_state_dict(model)
    synthetic.suppress_invalid_anchor_logits(model)
    model = model.to("cuda").eval()
    model.engine_dtype = torch.float16
    model.test_mask_on = False

    sizes = stream_sizes(args.images)
    g = torch.Generator().manual_seed(0)
    imgs = {s: torch.randint(0, 256, (3, *s), generator=g).float().cuda() for s in set(sizes)}

    def call(s):
        return model([{"image": imgs[s], "height": s[0], "width": s[1]}])

    first = sizes[0]
    model.use_cuda_graphs = False
    for _ in range(2):
        call(first)
    eager = [timed(lambda: call(first)) for _ in range(args.rounds * 2)]

    model.use_cuda_graphs = True
    model._graph_cache.clear()
    capture = timed(lambda: call(first))
    for _ in range(2):
        call(first)
    fixed = [timed(lambda: call(first)) for _ in range(args.rounds * 2)]
    for s in sizes:  # warm: allocator and text cache settle; no further capture may happen below
        call(s)
    n_graphs = sum(1 for k in model._graph_cache if k[0][0] == "forward")
    mixed = [timed(lambda: [call(s) for s in sizes]) / len(sizes) for _ in range(args.rounds)]
    fixed_after = [timed(lambda: call(first)) for _ in range(args.rounds * 2)]
    assert sum(1 for k in model._graph_cache if k[0][0] == "forward") == n_graphs
    print(json.dumps({"model": "APE-L_D", "names": 1203, "dtype": "float16", "pad": 1024, "images": len(sizes),
                      "distinct_sizes": len(set(sizes)), "first_size": list(first),
                      "eager_ms": stat(eager), "replay_fixed_ms": stat(fixed + fixed_after), "replay_stream_ms": stat(mixed),
                      "capture_ms": round(capture, 1), "old_key_captures": old_key_captures(sizes), "graphs": n_graphs,
                      "peak_mib": round(torch.cuda.max_memory_allocated() / 2 ** 20, 1)}), flush=True)
    print(json.dumps({"pad_geometry_ms": geometry_kernel(model, args.rounds)}), flush=True)


if __name__ == "__main__":
    main()
