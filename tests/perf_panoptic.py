"""Panoptic branch per image, the library-op path (engine_dtype fp32: upsample, crop-resize, sigmoid and argmax over [K, H, W]
stacks, postprocess.postprocess_panoptic) against the device path (engine_dtype fp16: csrc/panoptic.cu,
postprocess.postprocess_panoptic_winners), alternated round by round on identical inputs: K = 100 and 300 kept queries
(panoptic_post_nms off), 256^2 fp16 mask logits (overlapping blobs), a 1024 x 768 image padded to 1024^2, outputs of 1024 x 768, 480 x 640 and
2048 x 1536.  Both arms include the device->host copy and the segment bookkeeping.  Reports the median ms per image [min, max]
over the rounds, the peak memory above the inputs, and the time of the ape_panoptic_winners call alone, with the card and its
power limit.

    python tests/perf_panoptic.py [--rounds 5]
"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ape_b200 import configs, ops  # noqa: E402
from ape_b200.modeling import build_model  # noqa: E402

DEV = "cuda:0"


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        q = torch.cuda.get_device_name(0) + ", power limit unknown"
    return q


def timed(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    res = fn()
    b.record()
    torch.cuda.synchronize()
    return res, a.elapsed_time(b), (torch.cuda.max_memory_allocated() - base) / 2**30


def stat(xs):
    return f"{statistics.median(xs):.2f} [{min(xs):.2f}, {max(xs):.2f}]"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    model = build_model(configs.MINI).to(DEV)
    name = model.dataset_names[0]
    n_cls = 133  # COCO-panoptic: 80 things + 53 stuff
    model.dataset_stuff[name] = ([f"t{i}" for i in range(80)], [f"s{i}" for i in range(53)], "thing+stuff")
    model.set_eval_dataset(name)
    model.panoptic_post_nms = False  # every query is kept: K = Q
    print(f"card: {card()}; 256^2 fp16 mask logits, 1024^2 padded, 1024 x 768 image, {n_cls} classes; "
          f"median ms per image [min, max] over {args.rounds} rounds")
    g = torch.Generator().manual_seed(0)
    for K in (100, 300):
        box_cls = (torch.randn((1, K, n_cls), generator=g) * 2).to(DEV)
        box_pred = (torch.rand((1, K, 4), generator=g) * 0.5 + 0.25).to(DEV)
        # overlapping blobs with noise, so that queries compete and segments survive the overlap test
        yy, xx = torch.meshgrid(torch.arange(256.0), torch.arange(256.0), indexing="ij")
        c, r = torch.rand(K, 2, generator=g) * 256, torch.rand(K, generator=g) * 50 + 8
        d = ((yy[None] - c[:, 0, None, None]) ** 2 + (xx[None] - c[:, 1, None, None]) ** 2).sqrt()
        mask_pred = ((r[:, None, None] - d) * 0.3 + torch.randn(d.shape, generator=g) * 0.3)[None].to(DEV, torch.float16)
        qi = torch.arange(K, device=DEV)
        for out_hw in ((1024, 768), (480, 640), (2048, 1536)):
            call = (box_cls, box_pred, mask_pred, [(1024, 768)], (1024, 1024), [{"height": out_hw[0], "width": out_hw[1]}])
            times = {"old": [], "new": [], "kernel": []}
            peak = {}
            res = {}
            for r in range(args.rounds + 1):  # round 0 warms up both
                for arm, dt in (("old", torch.float32), ("new", torch.float16)):
                    model.engine_dtype = dt
                    res[arm], t, pk = timed(lambda: model._panoptic(*call))
                    if r > 0:
                        times[arm].append(t)
                        peak[arm] = pk
                scores = torch.rand(K, device=DEV)
                _, t, _ = timed(lambda: ops.panoptic_winners(mask_pred[0], qi, scores, (1024, 1024), (1024, 768), out_hw, 0.1))
                if r > 0:
                    times["kernel"].append(t)
            model.engine_dtype = torch.float32
            (seg_o, info_o), (seg_n, info_n) = res["old"][0], res["new"][0]
            same = "same segments" if info_o == info_n else "DIFFERENT segments"
            frac = (seg_o != seg_n).float().mean().item()
            print(f"K={K} output {out_hw[0]} x {out_hw[1]}: old {stat(times['old'])} ms / {peak['old']:.2f} GiB peak, "
                  f"new {stat(times['new'])} ms / {peak['new'] * 1024:.1f} MiB peak "
                  f"(ape_panoptic_winners alone {stat(times['kernel'])} ms); {len(info_n)} segments, {same}, "
                  f"{frac:.1e} of the pixels differ")
            del res
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
