#!/usr/bin/env python
"""The opt-in FP8 ViT-L path (`ViT(fp8_linears=True)`) against fp16.  Development aid.

    python tests/perf_vit_fp8.py [--rounds 5] [--iters 20] > vit_fp8.jsonl

1. Per GEMM, at the ViT-L shapes of APE-L_D at 1024^2: qkv (4096 x 3072 x 1024, bias) and w12 (4096 x 5460 x 1024, SwiGLU +
   slab statistics), each with the LayerNorm that feeds it: fp16 LayerNorm + fp16 GEMM against e4m3 LayerNorm + e4m3 GEMM.
   Each arm is a CUDA graph of 20 (LayerNorm, GEMM) pairs over rotating fp32 inputs that together exceed L2; the arms are
   replayed in turn, round after round.
2. The APE-L_D backbone + pyramid graph replay and the whole detection step (1024 x 768 padded to 1024^2, 1203 names,
   B = 1, CUDA graphs), fp16 against fp16 + FP8, alternated round by round.
Each record gives the median and [min, max] over the rounds; GEMM records also give TFLOP/s (2 M N K over the pair's time and
over the GEMM's alone) against the data-sheet dense peaks, 989 (fp16) and 1,979 (FP8) TFLOP/s.  The first line is the card."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from perf_ape_ti import card, graphed, time_ms  # noqa: E402

DEV = "cuda:0"
LAUNCHES = 20
PEAK = {"fp16": 989.0, "fp8": 1979.0}
SHAPES = [("vit_qkv", 4096, 3072, 1024, None), ("vit_w12", 4096, 5460, 1024, "swiglu")]


def gemm_arms(M, N, K, act):
    from ape_b200 import ops

    g = torch.Generator(device=DEV).manual_seed(N)
    w = torch.randn(N, K, device=DEV, generator=g) * K ** -0.5
    bias = torch.randn(N, device=DEV, generator=g) * 0.5
    lw = torch.randn(K, device=DEV, generator=g) * 0.2 + 1
    lb = torch.randn(K, device=DEV, generator=g) * 0.1
    n_sets = max(2, -(-150_000_000 // (M * K * 4)))  # fp32 LayerNorm inputs: more than L2 in all
    xs = [torch.randn(M, K, device=DEV, generator=g) for _ in range(n_sets)]
    w16 = w.half()
    wq, sw = ops.quantize_rows_e4m3(w)
    stats = act == "swiglu"

    def fp16(i):
        h = ops.layernorm(xs[i % n_sets], lw, lb, eps=1e-6, out_dtype=torch.float16)
        return ops.linear_tc(h, w16, bias, act=act, stats_out=stats)

    def fp8(i):
        hq, hs = ops.layernorm(xs[i % n_sets], lw, lb, eps=1e-6, out_dtype=torch.float8_e4m3fn)
        return ops.linear_fp8(hq, hs, wq, sw, bias, act=act, stats_out=stats)

    def gemm16(i):
        return ops.linear_tc(h16[i % n_sets], w16, bias, act=act, stats_out=stats)

    def gemm8(i):
        return ops.linear_fp8(hq8[i % n_sets][0], hq8[i % n_sets][1], wq, sw, bias, act=act, stats_out=stats)

    h16 = [ops.layernorm(x, lw, lb, eps=1e-6, out_dtype=torch.float16) for x in xs]
    hq8 = [ops.layernorm(x, lw, lb, eps=1e-6, out_dtype=torch.float8_e4m3fn) for x in xs]
    return {"fp16": fp16, "fp8": fp8, "gemm_fp16": gemm16, "gemm_fp8": gemm8}


def capture(fn):
    def many(_):
        for i in range(LAUNCHES):
            fn(i)
    replay, _ = graphed(many, None)
    return replay


def gemm_records(rounds, iters):
    for name, M, N, K, act in SHAPES:
        arms = gemm_arms(M, N, K, act)
        replays = {k: capture(f) for k, f in arms.items()}
        times = {k: [] for k in replays}
        for _ in range(rounds):
            for k, r in replays.items():
                times[k].append(time_ms(r, iters) * 1e3 / LAUNCHES)
        flop = 2.0 * M * N * K
        rec = {"shape": name, "M": M, "N": N, "K": K, "act": act or "bias"}
        for k, ts in times.items():
            med = statistics.median(ts)
            peak = PEAK["fp8" if k.endswith("fp8") else "fp16"]
            rec[k] = {"us_median": round(med, 2), "us_min": round(min(ts), 2), "us_max": round(max(ts), 2),
                      "tflops": round(flop / med / 1e6, 1), "share_of_peak": round(flop / med / 1e6 / peak, 3)}
        print(json.dumps(rec), flush=True)
        del replays, arms
        torch.cuda.empty_cache()


def model_records(rounds, iters):
    from ape_b200 import configs, synthetic
    from ape_b200.modeling import build_model

    m = build_model(configs.APE_L_D, num_text=1203)
    synthetic.fill_state_dict(m)
    synthetic.suppress_invalid_anchor_logits(m)
    m = m.to("cuda")
    m.engine_dtype, m.use_cuda_graphs = torch.float16, True
    img = synthetic.image(1024, 768, seed=0).float().cuda()
    inputs = [{"image": img, "height": 1024, "width": 768}]
    x = torch.zeros(1, 3, 1024, 1024, device="cuda")
    x[0, :, :, :768] = (img - m.pixel_mean) / m.pixel_std
    x = x.half()

    def backbone(t):
        with torch.no_grad():
            return m.backbone(t)

    replay = {}
    for mode in ("fp16", "fp8"):
        m.backbone.net.fp8_linears = mode == "fp8"
        replay[mode], _ = graphed(backbone, x)
        for _ in range(3):  # capture this mode's graph of the whole step, then warm it
            m(inputs)
    res = {mode: {"backbone_pyramid_ms": [], "step_ms": []} for mode in replay}
    for _ in range(rounds):
        for mode in replay:
            m.backbone.net.fp8_linears = mode == "fp8"
            res[mode]["backbone_pyramid_ms"].append(time_ms(replay[mode], iters))
            res[mode]["step_ms"].append(time_ms(lambda: m(inputs), iters))
    m.backbone.net.fp8_linears = False
    out = {"model": "APE-L_D", "workload": "1024 x 768 padded to 1024^2, 1203 names, boxes, B=1, fp16, CUDA graphs",
           "rounds": rounds, "iters": iters}
    for mode, r in res.items():
        out[mode] = {k: {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}
                     for k, v in r.items()}
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--no-model", action="store_true", help="GEMM records only")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_vit_fp8.py needs a GPU"
    print(json.dumps({"card": card(), "sms": torch.cuda.get_device_properties(0).multi_processor_count}), flush=True)
    gemm_records(args.rounds, args.iters)
    if not args.no_model:
        model_records(args.rounds, args.iters)


if __name__ == "__main__":
    main()
