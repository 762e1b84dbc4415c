#!/usr/bin/env python
"""The ping-pong GEMM kernel against the cooperative one at the APE-L_D step's GEMM shapes (BN = 128, the model's
epilogues).  Development aid.

    python tests/perf_gemm_pingpong.py > gemm_pingpong.jsonl

tile_n bit 0x8000 forces the ping-pong kernel, 0x10000 the cooperative one.  Each arm is a CUDA graph of 20 launches over
rotating operand sets that together exceed L2; the arms are replayed in turn, round after round, and each record gives
the median and [min, max] over the rounds of us per launch, TFLOP/s (2 M N K flop) and GB/s against the bytes the GEMM
must move to and from HBM at the least (A, W, the output and the residual once)."""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ape_b200 import ops  # noqa: E402

DEV = "cuda:0"
PP, COOP = 0x8000, 0x10000
LAUNCHES, ROUNDS, REPS = 20, 7, 3
ENC = 87296  # encoder tokens of APE-L_D at 1024² (p2..p6 of one image)
# name, M, N, K, epilogue: "f16" (16-bit out), "relu", "f32", "f32_res_ln" (LayerNorm fold + fp32 residual), "swiglu_stats"
SHAPES = [
    ("vit_qkv", 4096, 3072, 1024, "f16"),
    ("vit_proj", 4096, 1024, 1024, "f32_res_ln"),
    ("vit_w12", 4096, 5460, 1024, "swiglu_stats"),
    ("enc_256x256", ENC, 256, 256, "f16"),
    ("enc_offsets_logits", ENC, 480, 256, "f16"),
    ("enc_output", ENC, 256, 256, "f32"),
    ("proposal_mlp", ENC, 256, 256, "relu"),
    ("proposal_class", ENC, 256, 256, "f32"),
    ("pyramid_deconv1", 4096, 2048, 1024, "f16"),
    ("pyramid_deconv2", 16384, 1024, 512, "f16"),
    ("pyramid_1x1_p2", 16384, 256, 256, "f16"),
    ("pyramid_1x1_p4", 4096, 256, 1024, "f16"),
    ("decoder_900", 900, 256, 256, "f16"),
]


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), (v.strip() for v in r.stdout.splitlines()[0].split(","))))
    except Exception as ex:  # noqa: BLE001
        return {"error": str(ex)[:200]}


def least_bytes(M, N, K, epi):
    out_n, out_e = (N // 2, 2) if epi == "swiglu_stats" else (N, 4 if epi.startswith("f32") else 2)
    b = M * K * 2 + N * K * 2 + M * out_n * out_e
    if epi == "f32_res_ln":
        b += M * N * 4
    return b


def make(M, N, K, epi, dtype, n_sets):
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    w = (torch.randn(N, K, device=DEV, generator=g) * K ** -0.5).to(dtype)
    b = torch.randn(N, device=DEV, generator=g) * 0.5
    colsum = w.float().sum(1)
    sets = []
    for _ in range(n_sets):
        x = torch.randn(M, K, device=DEV, generator=g).to(dtype)
        res = torch.randn(M, N, device=DEV, generator=g) if epi == "f32_res_ln" else None
        part = torch.rand(M, 4, 2, device=DEV, generator=g) if epi == "f32_res_ln" else None
        sets.append((x, res, part))

    def run(i, tile_n):
        x, res, part = sets[i % len(sets)]
        if epi == "swiglu_stats":
            return ops.linear_tc(x, w, b, act="swiglu", stats_out=True, tile_n=tile_n)
        if epi == "f32_res_ln":
            return ops.linear_tc(x, w, b, residual=res, out_dtype=torch.float32, ln_fold=(part, colsum, K, 1e-6), tile_n=tile_n)
        return ops.linear_tc(x, w, b, act="relu" if epi == "relu" else None,
                             out_dtype=torch.float32 if epi == "f32" else None, tile_n=tile_n)

    return run


def capture(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for i in range(LAUNCHES):
            fn(i)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(LAUNCHES):
            fn(i)
    g.replay()
    torch.cuda.synchronize()
    return g


def time_graph(g):
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(REPS):
        g.replay()
    e.record()
    torch.cuda.synchronize()
    return a.elapsed_time(e) / (REPS * LAUNCHES) * 1e3


def main():
    print(json.dumps({"card": card(), "sms": torch.cuda.get_device_properties(0).multi_processor_count,
                      "launches_per_graph": LAUNCHES, "rounds": ROUNDS}), flush=True)
    dtype = torch.float16
    for name, M, N, K, epi in SHAPES:
        per_set = M * K * 2 + (M * N * 4 if epi == "f32_res_ln" else 0)
        run = make(M, N, K, epi, dtype, max(2, min(LAUNCHES, -(-150_000_000 // per_set))))
        a, b = run(0, PP), run(0, COOP)
        a, b = (a if isinstance(a, tuple) else (a,)), (b if isinstance(b, tuple) else (b,))
        same = all(torch.equal(u, v) for u, v in zip(a, b))
        graphs = {"coop": capture(lambda i: run(i, COOP)), "pingpong": capture(lambda i: run(i, PP))}
        times = {arm: [] for arm in graphs}
        for _ in range(ROUNDS):
            for arm, g in graphs.items():
                times[arm].append(time_graph(g))
        flop, hbm = 2.0 * M * N * K, least_bytes(M, N, K, epi)
        rec = {"shape": name, "M": M, "N": N, "K": K, "epilogue": epi, "tiles": -(-M // 128) * -(-N // 128),
               "least_hbm_bytes": hbm, "bit_identical": same}
        for arm, ts in times.items():
            ts = sorted(ts)
            med = ts[len(ts) // 2]
            rec[arm] = {"us_median": round(med, 2), "us_min": round(ts[0], 2), "us_max": round(ts[-1], 2),
                        "tflops": round(flop / med / 1e6, 1), "GBps": round(hbm / med / 1e3, 1)}
        print(json.dumps(rec), flush=True)
        del graphs, run
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
