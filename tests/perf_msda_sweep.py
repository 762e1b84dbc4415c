"""GPU microbench sweep for ms_deform_attn forward (BASELINE.json config 5) — run on the GPU:

    python tests/perf_msda_sweep.py [--quick] > gpurun_out/msda_sweep.jsonl

For every (shape, dtype, loc distribution) it times each kernel variant of libape_b200 and the
reference's own CUDA kernel (oracle/_ref, recompiled for sm_90a) on identical tensors, with an
L2 flush before every timed launch, and prints one JSON line per measurement.
Lives under tests/ because it uses the oracle (reference kernel) as comparison."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import ape_b200  # noqa: E402
from ape_b200 import ops  # noqa: E402
from oracle import msda as O  # noqa: E402

DEV = "cuda:0"
H, D, P = 8, 32, 4
SHAPES = {
    "L5_1024": [(256, 256), (128, 128), (64, 64), (32, 32), (16, 16)],
    "L5_1536": [(384, 384), (192, 192), (96, 96), (48, 48), (24, 24)],
    "L4": [(128, 128), (64, 64), (32, 32), (16, 16)],
}


def nbytes(B, S, Q, L, e):
    return e * (B * S * H * D + B * Q * H * L * P * 3 + B * Q * H * D) + 24 * L


def encoder_like_loc(B, shapes, gen, noise=0.5):
    """Sampling locations as the encoder produces them at initialisation: reference point = the
    query pixel's own centre (deformable_transformer_vl.py:371-400), offsets = the grid_init bias
    (multi_scale_deform_attn.py:195-207: head direction x (p+1) pixels) + N(0, noise) pixels."""
    import math
    refs = []
    for (h, w) in shapes:
        ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float32) + 0.5, torch.arange(w, dtype=torch.float32) + 0.5,
                                indexing="ij")
        refs.append(torch.stack([xs.reshape(-1) / w, ys.reshape(-1) / h], -1))
    ref = torch.cat(refs, 0)  # [S,2]
    S, L = ref.shape[0], len(shapes)
    th = torch.arange(H, dtype=torch.float32) * (2 * math.pi / H)
    g = torch.stack([th.cos(), th.sin()], -1)
    g = g / g.abs().max(-1, keepdim=True)[0]  # [H,2]
    pts = torch.arange(1, P + 1, dtype=torch.float32)
    off = g[:, None, None, :] * pts[None, None, :, None]  # [H,1,P,2]
    off = off.expand(H, L, P, 2)
    norm = torch.tensor([[w, h] for h, w in shapes], dtype=torch.float32)  # [L,2] (W,H)
    loc = ref[None, :, None, None, None, :] + (off[None, None] + noise * torch.randn(B, S, H, L, P, 2, generator=gen)) \
        / norm[None, None, None, :, None, :]
    return loc


def time_fn(fn, flush, iters):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--iters", type=int, default=15)
    args = ap.parse_args()
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=DEV)
    peak = 6576.4
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        peak = json.load(open(p))["hbm_gbs"]

    cases = [  # (name, shapes key, B, Q or None(=S), loc kind)
        ("enc1024_uniform", "L5_1024", 1, None, "uniform"),
        ("enc1024_model", "L5_1024", 1, None, "model"),
        ("dec1024_uniform", "L5_1024", 1, 900, "uniform"),
        ("L4_q300", "L4", 1, 300, "uniform"),
        ("L4_q900", "L4", 1, 900, "uniform"),
        ("L4_qS", "L4", 1, None, "uniform"),
        ("L4_qS_model", "L4", 1, None, "model"),
        ("L4_q900_b8", "L4", 8, 900, "uniform"),
        ("dec1024_b8", "L5_1024", 8, 900, "uniform"),
        ("enc1536_model", "L5_1536", 1, None, "model"),
    ]
    if args.quick:
        cases = cases[:3]
    variants = [("ht1_u4", 1 | (4 << 8)), ("ht1_u2", 1 | (2 << 8)), ("ht1_u1", 1 | (1 << 8)), ("ht2_u4", 2 | (4 << 8)),
                ("ht8_u4", 8 | (4 << 8)), ("ht8_u2", 8 | (2 << 8)), ("scalar", 0x1000), ("default", -1)]
    for name, sk, B, Q, kind in cases:
        shapes = SHAPES[sk]
        ss = torch.tensor(shapes, dtype=torch.int64)
        S = int((ss[:, 0] * ss[:, 1]).sum())
        L = len(shapes)
        q = S if Q is None else Q
        gen = torch.Generator().manual_seed(3)
        value = torch.randn(B, S, H, D, generator=gen)
        if kind == "model" and Q is None:
            loc = encoder_like_loc(B, shapes, gen)
        else:
            loc = torch.rand(B, q, H, L, P, 2, generator=gen)
        attn = torch.randn(B, q, H, L * P, generator=gen).softmax(-1).view(B, q, H, L, P)
        st = O.level_start_index(ss)
        for dname, dt, e in (("fp32", torch.float32, 4), ("fp16", torch.float16, 2), ("bf16", torch.bfloat16, 2)):
            v, lo, at = (t.to(DEV, dt) for t in (value, loc, attn))
            ssd, std = ss.to(DEV), st.to(DEV)
            nb = nbytes(B, S, q, L, e)
            rows = []
            if O.have_ref_cuda() and dt != torch.bfloat16:
                rows.append(("reference_kernel_sm100a", lambda: O.ref_cuda(v, ssd, std, lo, at)))
            for vn, vc in variants:
                rows.append((vn, lambda vc=vc: ops.ms_deform_attn_forward(v, ssd, std, lo, at, 64, variant=vc)))
            base = None
            for vn, fn in rows:
                out = fn()
                if base is None:
                    base = out
                err = (out.float() - base.float()).abs().max().item()
                med, best = time_fn(fn, flush, args.iters)
                print(json.dumps({"case": name, "dtype": dname, "variant": vn, "B": B, "Q": q, "S": S, "L": L,
                                  "ms_median": round(med, 5), "ms_min": round(best, 5), "alg_MB": round(nb / 1e6, 2),
                                  "alg_GBps": round(nb / med / 1e6, 1), "frac_hbm_peak": round(nb / med / 1e6 / peak, 4),
                                  "gathered_MB": round(B * q * H * L * P * 4 * D * e / 1e6, 1),
                                  "max_abs_diff_vs_first": err}), flush=True)
            del v, lo, at


if __name__ == "__main__":
    main()
