#!/usr/bin/env python
"""Multi-token prompts through the folded vision-language fusion.  Development aid.

    python tests/perf_prompt_graph.py [--tokens 3 80 256 1203] [--reps 20]

APE-L_D at 1024^2 (S = 87 296 vision tokens), synthetic weights, fp16, a phrase prompt of N free-text phrases, boxes only.
Records per N, in one process:
  fusion_folded_ms   one fusion layer on the folded path (BiAttentionBlock.folded: language GEMM, ape_vlf_fold_vision,
                     ape_vlf_fold_pool, the Delta-l GEMM), CUDA events over `reps` calls
  fusion_engine_ms   the same layer through BiMultiHeadAttention.forward_engine (six projections, two ape_attn_cross_fwd
                     passes), the sequence the folded path replaces
  eager_ms           the whole step with use_cuda_graphs off
  first_call_ms      the first call of a new N with use_cuda_graphs on (one eager pass, nothing captured)
  capture_ms         the second call (two eager warm-ups, capture, replay)
  replay_ms          the graph replay step
  fusion_share       6 x fusion_folded_ms / replay_ms (six encoder layers)
Step times are the median and [min, max] in ms of host clocks around work that ends in a synchronise; the first line is the card."""
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
    ap.add_argument("--tokens", type=int, nargs="+", default=[3, 80, 256, 1203])
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_prompt_graph.py needs a GPU"
    print(json.dumps({"card": card()}), flush=True)

    from ape_b200 import configs, ops, synthetic
    from ape_b200.modeling import build_model

    spec = copy.deepcopy(configs.APE_L_D)
    spec["test_score_thresh"] = SCORE_THRESH
    model = build_model(spec, num_text=1203)
    synthetic.fill_state_dict(model)
    synthetic.suppress_invalid_anchor_logits(model)
    model = model.to("cuda").eval()
    model.engine_dtype = torch.float16
    model.test_mask_on = False
    blk = model.transformer.encoder.vl_layers[0].b_attn
    g = torch.Generator().manual_seed(0)
    img = torch.randint(0, 256, (3, 1024, 1024), generator=g).float().cuda()
    S = 87296

    for N in args.tokens:
        row = {"N": N}
        with torch.no_grad():
            v = torch.randn(1, S, 256, generator=g).cuda().half()
            l = torch.randn(1, N, spec["lang_dim"], generator=g).cuda()
            vn = ops.layernorm_module(blk.layer_norm_v, v)
            ln = blk.layer_norm_l(l)

            def engine():
                dv, dl = blk.attn.forward_engine(vn, ln)
                return vn + blk.gamma_v.to(vn.dtype) * dv, ln + blk.gamma_l.float() * dl

            row["fusion_folded_ms"] = round(event_ms(lambda: blk.folded(vn, ln), args.reps), 3)
            row["fusion_engine_ms"] = round(event_ms(engine, args.reps), 3)
            fv, fl = blk.folded(vn, ln)
            ev, el = engine()
            row["folded_vs_engine_max_abs"] = [round((fv.float() - ev.float()).abs().max().item(), 5),
                                               round((fl - el).abs().max().item(), 5)]
        text = ",".join(f"object number {i}" for i in range(N))  # spaces: a phrase prompt
        inputs = [{"image": img, "height": 1024, "width": 1024, "prompt": "text", "text_prompt": text}]
        model.use_cuda_graphs = False
        model(inputs)
        row["eager_ms"] = stat([timed(lambda: model(inputs)) for _ in range(5)])
        model.use_cuda_graphs = True
        model._graph_cache.clear()
        model.__dict__.pop("_graph_seen_keys", None)
        row["first_call_ms"] = round(timed(lambda: model(inputs)), 2)
        row["capture_ms"] = round(timed(lambda: model(inputs)), 2)
        row["replay_ms"] = stat([timed(lambda: model(inputs)) for _ in range(args.reps)])
        row["fusion_share"] = round(6 * row["fusion_folded_ms"] / row["replay_ms"]["median"], 3)
        row["graphs"] = sum(1 for k in model._graph_cache if k[0][0] == "forward")
        model._graph_cache.clear()
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
