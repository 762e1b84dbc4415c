#!/usr/bin/env python
"""GEMM shape sweep of the APE-L_D step (development aid): TFLOP/s of ape_gemm_tn per model shape and kernel
variant (CUDA events, warm L2, 30 iterations).  python tests/perf_gemm.py > gpurun_out/gemm_sweep.jsonl"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ape_b200  # noqa: E402
from ape_b200 import ops  # noqa: E402

SHAPES = [  # (M, N, K, act, count per step, what)
    (4096, 5460, 1024, "swiglu", 24, "vit w12"),
    (4096, 1024, 2730, None, 24, "vit w3"),
    (4096, 3072, 1024, None, 24, "vit qkv"),
    (4096, 1024, 1024, None, 24, "vit proj"),
    (87296, 2048, 256, "relu", 6, "enc ffn1"),
    (87296, 256, 2048, None, 6, "enc ffn2"),
    (87296, 256, 256, None, 21, "enc/dec 256x256"),
    (87296, 480, 256, None, 6, "enc qo"),
    (87296, 512, 256, "relu", 1, "heads h0"),
    (65536, 256, 256, None, 2, "p2 1x1"),
    (900, 256, 256, None, 31, "dec small"),
]
VARIANTS = {"mc256": 256 | 0x4000, "mc128": 128 | 0x4000, "single256": 256 | 0x1000, "single128": 128 | 0x1000}


def main():
    dev = "cuda:0"
    for (M, N, K, act, cnt, what) in SHAPES:
        Kp = (K + 7) // 8 * 8
        x = torch.randn(M, Kp, device=dev, dtype=torch.float16)[:, :K]
        w = (torch.randn(N, Kp, device=dev, dtype=torch.float16) * K ** -0.5)[:, :K]
        b = torch.randn(N, device=dev)
        n_out = N // 2 if act == "swiglu" else N
        out = torch.empty(M, (n_out + 7) // 8 * 8, device=dev, dtype=torch.float16)[:, :n_out]
        ref = None
        for name, tile in VARIANTS.items():
            try:
                for _ in range(3):
                    ops.linear_tc(x, w, b, act=act, tile_n=tile, out=out)
                torch.cuda.synchronize()
                a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(30):
                    ops.linear_tc(x, w, b, act=act, tile_n=tile, out=out)
                e.record()
                torch.cuda.synchronize()
                us = a.elapsed_time(e) / 30 * 1e3
                if ref is None:
                    ref = out.clone()
                diff = (out.float() - ref.float()).abs().max().item()
                print(json.dumps({"what": what, "M": M, "N": N, "K": K, "variant": name, "us": round(us, 2),
                                  "tflops": round(2 * M * N * K / us / 1e6, 1), "max_diff_vs_first": diff,
                                  "ms_per_step": round(us * cnt / 1e3, 3)}), flush=True)
            except Exception as ex:  # noqa: BLE001
                print(json.dumps({"what": what, "variant": name, "error": str(ex)[:200]}), flush=True)


if __name__ == "__main__":
    main()
