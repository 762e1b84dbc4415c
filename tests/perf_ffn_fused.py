#!/usr/bin/env python
"""The fused FFN kernel (ops.ffn_fused) against the two-GEMM pair it replaces (ops.linear_tc relu, then bias + residual with
an fp32 output) at the APE-L_D encoder (87 296 tokens) and decoder (900 queries) shapes.  Development aid.

    python tests/perf_ffn_fused.py > ffn_fused.jsonl

Each arm is a CUDA graph of 20 launches over rotating operand sets that together exceed L2 (at the encoder shape); the arms
are replayed in turn, round after round, and each record gives the median and [min, max] over the rounds of us per launch,
TFLOP/s (4 M 256 F flop) and the bytes the arm must move to and from HBM at the least: x once (the residual re-read is an L2
hit), both weights once, the fp32 output, and for the pair the 16-bit hidden activation written and read back."""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ape_b200 import ops  # noqa: E402

DEV = "cuda:0"
E = 256
SHAPES = [("encoder", 87296, 2048), ("decoder", 900, 2048)]
LAUNCHES, ROUNDS, REPS = 20, 7, 3


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), (v.strip() for v in r.stdout.splitlines()[0].split(","))))
    except Exception as ex:  # noqa: BLE001
        return {"error": str(ex)[:200]}


def make_sets(M, F, dtype, n):
    g = torch.Generator(device=DEV).manual_seed(M + F)
    w1 = (torch.randn(F, E, device=DEV, generator=g) * E ** -0.5).to(dtype)
    b1 = torch.randn(F, device=DEV, generator=g) * 0.5
    w2 = (torch.randn(E, F, device=DEV, generator=g) * F ** -0.5).to(dtype)
    b2 = torch.randn(E, device=DEV, generator=g) * 0.5
    h = torch.empty(M, F, device=DEV, dtype=dtype)  # the pair's hidden activation (one buffer: it streams through HBM anyway)
    sets = [(torch.randn(M, E, device=DEV, generator=g).to(dtype), torch.empty(M, E, device=DEV)) for _ in range(n)]
    return (w1, b1, w2, b2, h), sets


def arms(weights, sets):
    w1, b1, w2, b2, h = weights

    def pair(i):
        x, out = sets[i % len(sets)]
        ops.linear_tc(x, w1, b1, act="relu", out=h)
        ops.linear_tc(h, w2, b2, residual=x, out=out)

    def fused(variant):
        def f(i):
            x, out = sets[i % len(sets)]
            ops.ffn_fused(x, w1, b1, w2, b2, out=out, variant=variant)
        return f

    return {"two_gemm": pair, "fused_single": fused(1), "fused_cluster": fused(2)}


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
    print(json.dumps({"card": card(), "launches_per_graph": LAUNCHES, "rounds": ROUNDS}), flush=True)
    for dtype in (torch.float16, torch.bfloat16):
        for what, M, F in SHAPES:
            per_set = M * E * (2 + 4)
            weights, sets = make_sets(M, F, dtype, max(2, min(LAUNCHES, -(-150_000_000 // per_set))))
            fns = arms(weights, sets)
            # the arms compute the same bits: check on the first set before timing
            fns["two_gemm"](0)
            ref = sets[0][1].clone()
            same = {}
            for name in ("fused_single", "fused_cluster"):
                fns[name](0)
                same[name] = bool(torch.equal(sets[0][1], ref))
            graphs = {name: capture(fn) for name, fn in fns.items()}
            times = {name: [] for name in graphs}
            for _ in range(ROUNDS):
                for name, g in graphs.items():
                    times[name].append(time_graph(g))
            flop = 4.0 * M * E * F
            w_bytes = 2 * F * E * 2
            for name, ts in times.items():
                ts = sorted(ts)
                med = ts[len(ts) // 2]
                hbm = M * E * 2 + w_bytes + M * E * 4 + (2 * M * F * 2 if name == "two_gemm" else 0)
                print(json.dumps({
                    "shape": what, "M": M, "E": E, "F": F, "dtype": str(dtype).replace("torch.", ""), "arm": name,
                    "us_median": round(med, 2), "us_min": round(ts[0], 2), "us_max": round(ts[-1], 2),
                    "tflops_median": round(flop / med / 1e6, 1), "hbm_bytes_min": hbm,
                    "hbm_GBps_at_median": round(hbm / med / 1e3, 1), "operand_sets": len(sets),
                    "bit_identical_to_two_gemm": same.get(name, True)}), flush=True)
            del graphs, fns, sets, weights, ref
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
