#!/usr/bin/env python
"""Region prompts (`mask_prompt`) on the device and on the captured step.  Development aid.

    python tests/perf_region_prompt.py [--reps 20]

APE-L_D at 1024^2, synthetic weights, fp16, boxes only.  Records, in one process:
  kernel_ms       ops.region_prompt alone (ape_region_prompt_empty + ape_region_prompt) at the 1024^2 pad (S = 87 296 tokens),
                  CUDA events over `reps` calls
  torch_ms        the torch path it replaces, as the engine ran it before: the prompt padded into fp32, `sum() == 0` (a host
                  synchronisation), five F.interpolate + `.to(bool)`, the concatenation and the two masked_fill of the anchors
  then, for a 1024 x 768 image with a region prompt, per prompt (1203 names; a repeated 3-phrase prompt):
  eager_ms        the step with use_cuda_graphs off (what every region prompt ran before)
  replay_ms       the graph replay step with use_cuda_graphs on, after capture
Step times are the median and [min, max] in ms of host clocks around work that ends in a synchronise; the first line is the card
(name and power limit, read in the same run)."""
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


def event_ms(fn, reps):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_region_prompt.py needs a GPU"
    print(json.dumps({"card": card()}), flush=True)

    from ape_b200 import configs, ops, synthetic
    from ape_b200.modeling import build_model

    spec = copy.deepcopy(configs.APE_L_D)
    spec["test_score_thresh"] = SCORE_THRESH
    H = W = spec["backbone"]["square_pad"]
    shapes = configs.level_shapes(spec)
    S = sum(h * w for h, w in shapes)
    g = torch.Generator().manual_seed(0)
    h, w = 768, 1024
    prompt = torch.zeros((h, w), device="cuda")
    prompt[200:520, 300:800] = 255.0

    # 1. the kernel alone against the torch path it replaces
    with torch.no_grad():
        props = torch.randn((1, S, 4), generator=g).cuda()
        inv = (torch.rand((1, S, 1), generator=g) < 0.1).cuda()
        rmap = torch.zeros((1, H, W), dtype=torch.uint8, device="cuda")
        rmap[0, :h, :w] = prompt != 0

        def kernel():
            return ops.region_prompt(rmap, shapes, props, inv)

        def torch_path():
            mp = torch.zeros((1, H, W), device="cuda")
            mp[0, :h, :w] = prompt
            if mp.sum() == 0:
                mp[...] = 255
            r = torch.cat([F.interpolate(mp[None], size=sh, mode="bilinear").to(torch.bool).squeeze(0).flatten(1) for sh in shapes], 1)
            return props.masked_fill(~r.unsqueeze(-1), float("inf")), inv | ~r.unsqueeze(-1)

        kp, ki, _ = kernel()
        tp, ti = torch_path()
        row = {"S": S, "kernel_ms": round(event_ms(kernel, 200), 4), "torch_ms": round(event_ms(torch_path, 200), 4),
               "bit_exact": bool(torch.equal(kp, tp) and torch.equal(ki, ti))}
    print(json.dumps(row), flush=True)

    # 2. the step with a region prompt, graphed against eager
    model = build_model(spec, num_text=1203)
    synthetic.fill_state_dict(model)
    synthetic.suppress_invalid_anchor_logits(model)
    model = model.to("cuda").eval()
    model.engine_dtype = torch.float16
    model.test_mask_on = False
    img = torch.randint(0, 256, (3, h, w), generator=g).float().cuda()
    base = {"image": img, "height": h, "width": w, "mask_prompt": prompt}
    for name, extra in (("names_1203", {}), ("phrases_3", {"prompt": "text", "text_prompt": "red car,a person walking,traffic light"})):
        inputs = [dict(base, **extra)]
        row = {"prompt": name}
        with torch.no_grad():
            model.use_cuda_graphs = False
            model(inputs)
            row["eager_ms"] = stat([timed(lambda: model(inputs)) for _ in range(5)])
            model.use_cuda_graphs = True
            model._graph_cache.clear()
            model.__dict__.pop("_graph_seen_keys", None)
            for _ in range(3):  # a repeated multi-token prompt is captured on its second call
                model(inputs)
            row["replay_ms"] = stat([timed(lambda: model(inputs)) for _ in range(args.reps)])
            row["region_graphs"] = sum(1 for k in model._graph_cache if k[0][0] == "forward" and k[0][-1] is True)
            model._graph_cache.clear()
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
