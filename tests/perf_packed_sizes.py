#!/usr/bin/env python
"""`forward_packed` with masks, semantic and panoptic maps over a stream of mixed sizes: `packed_output_capacity` against the
per-size graph key.  Development aid.

    python tests/perf_packed_sizes.py [--rounds 3] [--images 64] [--capacity 1024]

APE-L_D at 1024^2, 1203 names (80 thing and 53 stuff classes for the panoptic merge), fp16, bench.py's weights and score threshold,
instance masks as run-length codes.  The stream: a seeded list of photo sizes between 320 and 640 pixels a side, passed through
ResizeShortestEdge(1024, 1024), one image per call, each asking for its photo's size as the output (COCO-like).  Records:
  captures          "forward" graphs captured over the stream in capacity mode (one is the goal)
  stream_ms         the capacity-mode graph step averaged over the stream, once per round
  replay_fixed_ms   the per-size graph (capacity None) replayed at the stream's first size: today's best case
  eager_ms          the eager step (use_cuda_graphs off, capacity None) at that size
  stages_ms         device times of the packed stages in one eager step at that size, exact sizes against capacity mode (CUDA
                    events around each ops call, summed per stage; median and [min, max] over rounds)
  peak_mib          peak device memory after the stream
Step times are the median and [min, max] in ms of host clocks around work that ends in a synchronise; the first line is the card.
The multi-GPU gather is not measured here (one GPU)."""
import argparse
import collections
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from perf_ape_ti import card  # noqa: E402
from perf_graph_sizes import stat, stream_sizes, timed  # noqa: E402


def stage_times(model, call, size, cap, rounds):
    """Device ms per packed stage of one eager forward_packed, from ops' CUDA events (tags summed per stage name)."""
    from ape_b200 import ops

    model.use_cuda_graphs, model.packed_output_capacity = False, cap
    per = collections.defaultdict(list)
    for _ in range(rounds):
        ops.PROFILE_EVENTS = []
        call(size)
        torch.cuda.synchronize()
        acc = collections.defaultdict(float)
        for tag, a, b in ops.PROFILE_EVENTS:
            name = tag[0].replace("_dev", "")
            if name in ("mask_pack", "semseg_label", "semseg_pack", "panoptic_winners", "panoptic_pack"):
                acc[name] += a.elapsed_time(b)
        ops.PROFILE_EVENTS = None
        for k, v in acc.items():
            per[k].append(v)
    return {k: stat(v) for k, v in sorted(per.items())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--capacity", type=int, default=1024)
    args = ap.parse_args()
    print(json.dumps({"card": card(), "gpus": torch.cuda.device_count()}), flush=True)

    import bench
    from ape_b200.modeling import build_model

    model = bench.bench_weights(build_model(bench.bench_spec(), num_text=1203)).to("cuda").eval()
    model.engine_dtype = torch.float16
    model.test_mask_on, model.semantic_on, model.panoptic_on = True, True, True
    model.mask_format = "rle"
    name = model.dataset_names[0]
    vocab = list(model.vocabulary[name])
    model.dataset_stuff[name] = (vocab[:80], vocab[80:133], "thing+stuff")
    model.set_eval_dataset(name)

    sizes = stream_sizes(args.images)  # ResizeShortestEdge(1024, 1024) of the photo sizes below (the same seed and draws)
    g = np.random.default_rng(0)
    photos = [(int(g.integers(320, 641)), int(g.integers(320, 641))) for _ in range(args.images)]  # the requested outputs
    gen = torch.Generator().manual_seed(0)
    imgs = {s: torch.randint(0, 256, (3, *s), generator=gen).float().cuda() for s in set(sizes)}

    def call(i):
        s = sizes[i]
        return model.forward_packed([{"image": imgs[s], "height": photos[i][0], "width": photos[i][1]}])

    model.use_cuda_graphs, model.packed_output_capacity = False, None
    for _ in range(2):
        call(0)
    eager = [timed(lambda: call(0)) for _ in range(args.rounds * 2)]

    model.use_cuda_graphs = True
    model._graph_cache.clear()
    for _ in range(3):
        call(0)
    fixed = [timed(lambda: call(0)) for _ in range(args.rounds * 2)]

    model._graph_cache.clear()
    model.packed_output_capacity = args.capacity
    torch.cuda.reset_peak_memory_stats()
    for i in range(len(sizes)):  # first pass: captures happen here
        call(i)
    captures = sum(1 for k in model._graph_cache if k[0][0] == "forward")
    stream = [timed(lambda: [call(i) for i in range(len(sizes))]) / len(sizes) for _ in range(args.rounds)]
    assert sum(1 for k in model._graph_cache if k[0][0] == "forward") == captures
    peak = torch.cuda.max_memory_allocated() / 2 ** 20

    print(json.dumps({"model": "APE-L_D", "names": 1203, "dtype": "float16", "pad": 1024, "capacity": args.capacity,
                      "images": len(sizes), "distinct_pairs": len(set(zip(sizes, photos))), "first_size": list(sizes[0]),
                      "first_output": list(photos[0]), "captures": captures, "stream_ms": stat(stream),
                      "replay_fixed_ms": stat(fixed), "eager_ms": stat(eager), "peak_mib": round(peak, 1)}), flush=True)
    print(json.dumps({"stages_ms": {"exact": stage_times(model, lambda i: call(i), 0, None, args.rounds * 2),
                                    "capacity": stage_times(model, lambda i: call(i), 0, args.capacity, args.rounds * 2)}}),
          flush=True)
    if torch.cuda.device_count() < 2:
        print(json.dumps({"multi_gpu": "not measured: one GPU"}), flush=True)


if __name__ == "__main__":
    main()
