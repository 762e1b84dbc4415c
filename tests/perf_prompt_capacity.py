#!/usr/bin/env python
"""`model.prompt_capacity` on a demo-like stream of changing prompts.  Development aid.

    python tests/perf_prompt_capacity.py [--calls 24] [--caps 256 1536] [--reps 20]

APE-L_D at 1024^2, synthetic weights, fp16, use_cuda_graphs, boxes only.  In one process, for the parent behaviour
(prompt_capacity None) and each capacity C:
  names    a stream of `calls` name prompts ("a,b,c": one fusion token), a new count of 1 to 60 names on every call
  phrases  a stream of `calls` phrase prompts of 1 to 16 phrases (the folded fusion over the text), a new count on most calls
per stream: per-call median and max latency (host clock around each call, which ends in a device synchronise), the "forward"
graphs captured, and the peak device memory after the stream (torch.cuda.max_memory_allocated, reset before it).
Then the cost of padding: the replay step at C against the exact-n replay (prompt_capacity None, same prompt repeated) for
n = 3 and n = 1203 name prompts (n = 1203 only where it fits C).  The first line is the card and its power limit."""
import argparse
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

from perf_ape_ti import card  # noqa: E402

SCORE_THRESH = 0.0123  # bench.py's BENCH_SCORE_THRESH


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def stat(ts):
    return {"median": round(statistics.median(ts), 2), "max": round(max(ts), 2), "min": round(min(ts), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=24)
    ap.add_argument("--caps", type=int, nargs="+", default=[256, 1536])
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_prompt_capacity.py needs a GPU"
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
    model.use_cuda_graphs = True
    g = torch.Generator().manual_seed(0)
    img = torch.randint(0, 256, (3, 1024, 1024), generator=g).float().cuda()
    rng = np.random.default_rng(0)
    name_counts = [int(c) for c in rng.choice(np.arange(1, 61), size=args.calls, replace=False)]
    phrase_counts = [int(c) for c in rng.integers(1, 17, size=args.calls)]

    def inputs(text):
        return [{"image": img, "height": 1024, "width": 1024, "prompt": "text", "text_prompt": text}]

    def names(n, tag):
        return ",".join(f"n{tag}_{i}" for i in range(n))

    def phrases(n, tag):
        return ",".join(f"object {tag} {i}" for i in range(n))

    model(inputs(names(3, "w")))  # module loads, weight packing
    for cap in [None] + args.caps:
        model.prompt_capacity = cap
        for kind, counts, make in (("names", name_counts, names), ("phrases", phrase_counts, phrases)):
            model._graph_cache.clear()
            model.__dict__.pop("_graph_seen_keys", None)
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            ts = [timed(lambda: model(inputs(make(n, f"{kind}{i}")))) for i, n in enumerate(counts)]
            row = {"C": cap, "stream": kind, "calls": len(ts), "per_call_ms": stat(ts),
                   "graphs": sum(1 for k in model._graph_cache if k[0][0] == "forward"),
                   "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}
            print(json.dumps(row), flush=True)
    for n in (3, 1203):
        text = names(n, "pad")
        model._graph_cache.clear()
        model.prompt_capacity = None
        model(inputs(text))
        exact = stat([timed(lambda: model(inputs(text))) for _ in range(args.reps)])
        row = {"n": n, "exact_replay_ms": exact}
        for cap in args.caps:
            if n > cap:
                continue
            model._graph_cache.clear()
            model.prompt_capacity = cap
            model(inputs(text))
            row[f"replay_ms_C{cap}"] = stat([timed(lambda: model(inputs(text))) for _ in range(args.reps)])
        model.prompt_capacity = None
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
