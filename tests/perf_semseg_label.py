"""Semantic branch per image, sem_seg_format "maps" against "label", alternated round by round on identical inputs: 300 kept
queries, 1203 classes, 256^2 mask logits, a 1024 x 768 image padded to 1024^2, outputs of 1024 x 768, 480 x 640 and 2048 x 1536.
Reports the median ms per image and the peak memory above the inputs for each, with the card and its power limit.

    python tests/perf_semseg_label.py [--rounds 7] [--dtype fp16|bf16]
"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ape_b200 import configs  # noqa: E402
from ape_b200.modeling import build_model  # noqa: E402

DEV = "cuda:0"


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        q = torch.cuda.get_device_name(0) + ", power limit unknown"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--dtype", default="fp16", choices=("fp16", "bf16"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dt = torch.float16 if args.dtype == "fp16" else torch.bfloat16
    model = build_model(configs.MINI).to(DEV)
    model.engine_dtype, model.semantic_post_nms = dt, False  # all 300 queries kept
    Q, N = 300, 1203
    g = torch.Generator().manual_seed(0)
    box_cls = (torch.randn((1, Q, N), generator=g) * 2).to(DEV)
    box_pred = (torch.rand((1, Q, 4), generator=g) * 0.5 + 0.25).to(DEV)
    mask_pred = (torch.randn((1, Q, 256, 256), generator=g) * 4).to(DEV)
    print(f"card: {card()}; operands {args.dtype}; {Q} queries x {N} classes, 256^2 logits, 1024^2 padded, 1024 x 768 image")
    for out_hw in ((1024, 768), (480, 640), (2048, 1536)):
        call = (box_cls, box_pred, mask_pred, [(1024, 768)], (1024, 1024), [{"height": out_hw[0], "width": out_hw[1]}])
        times = {"maps": [], "label": []}
        peak = {}
        for r in range(args.rounds + 1):  # round 0 warms up both
            for fmt in ("maps", "label"):
                model.sem_seg_format = fmt
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                res = model._semantic(*call)
                b.record()
                torch.cuda.synchronize()
                if r > 0:
                    times[fmt].append(a.elapsed_time(b))
                    peak[fmt] = (torch.cuda.max_memory_allocated() - base) / 2**30
                del res
        line = ", ".join(f"{fmt} {statistics.median(times[fmt]):.2f} ms (min {min(times[fmt]):.2f}) / {peak[fmt]:.2f} GiB peak"
                         for fmt in ("maps", "label"))
        print(f"output {out_hw[0]} x {out_hw[1]}: {line}")
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
