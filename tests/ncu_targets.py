"""Launches ONE kernel family a few times at the APE-L_D model shapes, for `ncu --set full` captures:

    ncu --set full --import-source on -k regex:attn_fwd -s 1 -c 1 -o gpurun_out/r02_attn_window python tests/ncu_targets.py attn_window

Targets: attn_window (4 x 1024 tokens x 16 heads), attn_global (4096 x 16), gemm_qkv (4096x3072x1024), gemm_proj (4096x1024x1024,
fp32 out + residual + LayerNorm fold), gemm_ffn1 (87296x2048x256, ReLU), msda_pair (encoder, 1024^2), msda_generic, xattn (256-wide heads)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import ape_b200  # noqa: E402,F401
from ape_b200 import ops  # noqa: E402

DEV = "cuda:0"
dt = torch.float16


def main():
    which = sys.argv[1]
    g = torch.Generator().manual_seed(0)
    if which in ("attn_window", "attn_global"):
        nseq, n = (4, 1024) if which == "attn_window" else (1, 4096)
        qkv = torch.randn(nseq * n, 3 * 1024, generator=g).to(DEV, dt)
        fn = lambda: ops.attention_qkv(qkv, nseq, n, 16, 64, 0.125, stats_out=True)
    elif which == "gemm_qkv":
        a, w, b = torch.randn(4096, 1024, generator=g).to(DEV, dt), torch.randn(3072, 1024, generator=g).to(DEV, dt), torch.zeros(3072, device=DEV)
        fn = lambda: ops.linear_tc(a, w, b)
    elif which == "gemm_proj":
        a, w, b = torch.randn(4096, 1024, generator=g).to(DEV, dt), torch.randn(1024, 1024, generator=g).to(DEV, dt), torch.zeros(1024, device=DEV)
        res = torch.randn(4096, 1024, device=DEV)
        part = torch.stack([a.float().view(4096, 16, 64).sum(-1), (a.float() ** 2).view(4096, 16, 64).sum(-1)], -1).contiguous()
        cs = w.float().sum(1).contiguous()
        fn = lambda: ops.linear_tc(a, w, b, residual=res, out_dtype=torch.float32, ln_fold=(part, cs, 1024, 1e-6))
    elif which == "gemm_ffn1":
        a, w, b = torch.randn(87296, 256, generator=g).to(DEV, dt), torch.randn(2048, 256, generator=g).to(DEV, dt), torch.zeros(2048, device=DEV)
        fn = lambda: ops.linear_tc(a, w, b, act="relu")
    elif which in ("msda_pair", "msda_generic"):
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import perf_msda_pair as P

        shapes = [(256, 256), (128, 128), (64, 64), (32, 32), (16, 16)]
        value, ss, st, qo, ref, S = P.case(shapes, dt)
        n_off = 8 * 5 * 4 * 2
        if which == "msda_pair":
            v2 = ops.msda_pair_values(value, 8)
            fn = lambda: ops.ms_deform_attn_pair_fused_forward(v2, ss, st, shapes, qo[..., :n_off], qo[..., n_off:], ref, 4)
        else:
            v4 = value.view(1, S, 8, 32)
            fn = lambda: ops.ms_deform_attn_fused_forward(v4, ss, st, qo[..., :n_off], qo[..., n_off:], ref, 4)
    elif which == "xattn":
        q = torch.randn(8192, 2048, generator=g).to(DEV, dt)
        k = torch.randn(1216, 2048, generator=g).to(DEV, dt)
        v = torch.randn(1216, 2048, generator=g).to(DEV, dt)
        fn = lambda: ops.attention_cross(q, k, v, 1, 8192, 1216, 1203, 8, 256, 256 ** -0.5)
    else:
        raise SystemExit(f"unknown target {which}")
    for _ in range(3):
        fn()
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()
