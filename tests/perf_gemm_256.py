#!/usr/bin/env python
"""128 x 256 GEMM tiles (single CTA and cluster of two) against the 128 x 128 kernel each shape ran before they existed,
at the ViT-L and pyramid GEMM shapes of the APE-L_D step with the model's epilogues, fp16.  Development aid.

    python tests/perf_gemm_256.py > gemm_256.jsonl

Arms, pinned by tile_n bits: "base" is the 128 x 128 kernel that the tile count and K used to select (ping-pong 0x8000
from 2 x SM-count tiles up, else cooperative 0x10000, which takes the cluster of two at K >= 2048), "w256_cl1" is
256 | 0x1000 and "w256_cl2" is 256 | 0x4000.  Each arm is a CUDA graph of 20 launches over rotating operand sets that
together exceed L2; the arms are replayed in turn, round after round, and each record gives the median and [min, max]
over the rounds of us per launch and TFLOP/s (2 M N K flop).  "l2_bytes" is the operand traffic from L2 into shared
memory that the tiling implies (every CTA loads its 128-row A tile for each k-block, a weight tile is loaded once per
cluster), and "l2_TBps" that traffic over the median time.  "issue" and "tail" are the kernel's own clock64 phases
(ape_gemm_set_trace), median over CTAs of one eager launch, in cycles: first operands landed -> last MMA issued (every
tile of the CTA but the last one's epilogue), and last accumulator complete -> epilogue drained (the exposed epilogue)."""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ape_b200 import _lib, ops  # noqa: E402

DEV = "cuda:0"
PP, COOP, SINGLE, CLUSTER = 0x8000, 0x10000, 0x1000, 0x4000
LAUNCHES, ROUNDS, REPS = 20, 7, 3
# name, M, N, K, epilogue: "f16" (16-bit out), "f32_res" (fp32 out + fp32 residual), "f32_res_ln" (LayerNorm fold + fp32
# residual), "swiglu_stats"
SHAPES = [
    ("vit_qkv", 4096, 3072, 1024, "f16"),
    ("vit_proj", 4096, 1024, 1024, "f32_res_ln"),
    ("vit_w12", 4096, 5460, 1024, "swiglu_stats"),
    ("vit_w3", 4096, 1024, 2730, "f32_res_ln"),
    ("vit_patch_embed", 4096, 1024, 768, "f32_res"),
    ("pyramid_deconv1", 4096, 2048, 1024, "f16"),
    ("pyramid_deconv2", 16384, 1024, 512, "f16"),
]


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), (v.strip() for v in r.stdout.splitlines()[0].split(","))))
    except Exception as ex:  # noqa: BLE001
        return {"error": str(ex)[:200]}


def arms(M, N, K, sms):
    tiles = -(-M // 128) * -(-N // 128)
    base = COOP if K >= 2048 or tiles < 2 * sms else PP
    # (tile_n bits, tile width, cluster size)
    return {"base": (base, 128, 2 if base == COOP and K >= 2048 else 1), "w256_cl1": (256 | SINGLE, 256, 1),
            "w256_cl2": (256 | CLUSTER, 256, 2)}


def l2_bytes(M, N, K, bn, cl):
    kp = -(-K // 64) * 64
    m_blocks = -(-(-(-M // 128)) // cl) * cl  # a cluster's second CTA loads its (empty) A tile too
    n_blocks = -(-N // bn)
    ctas = m_blocks * n_blocks
    return ctas * 128 * kp * 2 + ctas // cl * bn * kp * 2


def pitched(t):
    """t [rows, K] with its rows 16-byte aligned (w3's K = 2730 runs on such views of padded buffers in the model)."""
    kp = -(-t.shape[1] // 8) * 8
    out = torch.zeros(t.shape[0], kp, dtype=t.dtype, device=t.device)[:, : t.shape[1]]
    out.copy_(t)
    return out


def make(M, N, K, epi, dtype, n_sets):
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    w = pitched((torch.randn(N, K, device=DEV, generator=g) * K ** -0.5).to(dtype))
    b = torch.randn(N, device=DEV, generator=g) * 0.5
    colsum = w.float().sum(1)
    sets = []
    for _ in range(n_sets):
        x = pitched(torch.randn(M, K, device=DEV, generator=g).to(dtype))
        res = torch.randn(M, N, device=DEV, generator=g) if epi.startswith("f32_res") else None
        part = torch.rand(M, 4, 2, device=DEV, generator=g) if epi == "f32_res_ln" else None
        sets.append((x, res, part))

    def run(i, tile_n):
        x, res, part = sets[i % len(sets)]
        if epi == "swiglu_stats":
            return ops.linear_tc(x, w, b, act="swiglu", stats_out=True, tile_n=tile_n)
        if epi == "f32_res_ln":
            return ops.linear_tc(x, w, b, residual=res, out_dtype=torch.float32, ln_fold=(part, colsum, K, 1e-6), tile_n=tile_n)
        if epi == "f32_res":
            return ops.linear_tc(x, w, b, residual=res, out_dtype=torch.float32, tile_n=tile_n)
        return ops.linear_tc(x, w, b, tile_n=tile_n)

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


def phases(run, tile_n, sms):
    buf = torch.zeros(sms * 8, dtype=torch.int64, device=DEV)
    torch.cuda.synchronize()
    _lib.lib.ape_gemm_set_trace(buf.data_ptr())
    try:
        run(0, tile_n)
        torch.cuda.synchronize()
    finally:
        _lib.lib.ape_gemm_set_trace(None)
    t = buf.view(-1, 8).cpu()
    t = t[t[:, 0] != 0].double()
    med = lambda v: int(v.median().item())  # noqa: E731
    return {"issue": med(t[:, 3] - t[:, 2]), "tail": med(t[:, 6] - t[:, 5])}


def main():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(json.dumps({"card": card(), "sms": sms, "launches_per_graph": LAUNCHES, "rounds": ROUNDS}), flush=True)
    dtype = torch.float16
    for name, M, N, K, epi in SHAPES:
        per_set = M * K * 2 + (M * N * 4 if epi.startswith("f32_res") else 0)
        run = make(M, N, K, epi, dtype, max(2, min(LAUNCHES, -(-150_000_000 // per_set))))
        cfg = arms(M, N, K, sms)
        outs = {}
        for arm, (bits, _, _) in cfg.items():
            o = run(0, bits)
            outs[arm] = o if isinstance(o, tuple) else (o,)
        same = all(all(torch.equal(u, v) for u, v in zip(outs["base"], o)) for o in outs.values())
        trace = {arm: phases(run, bits, sms) for arm, (bits, _, _) in cfg.items()}
        graphs = {arm: capture(lambda i, bits=bits: run(i, bits)) for arm, (bits, _, _) in cfg.items()}
        times = {arm: [] for arm in graphs}
        for _ in range(ROUNDS):
            for arm, g in graphs.items():
                times[arm].append(time_graph(g))
        flop = 2.0 * M * N * K
        rec = {"shape": name, "M": M, "N": N, "K": K, "epilogue": epi, "bit_identical": same}
        for arm, ts in times.items():
            bits, bn, cl = cfg[arm]
            ts = sorted(ts)
            med = ts[len(ts) // 2]
            l2 = l2_bytes(M, N, K, bn, cl)
            rec[arm] = {"tile_n": hex(bits), "us_median": round(med, 2), "us_min": round(ts[0], 2), "us_max": round(ts[-1], 2),
                        "tflops": round(flop / med / 1e6, 1), "l2_bytes": l2, "l2_TBps": round(l2 / med / 1e6, 2), **trace[arm]}
        print(json.dumps(rec), flush=True)
        del graphs, run
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
