#!/usr/bin/env python
"""Instance masks through `forward_packed` (run-length codes built on the device in fixed-size slots) against `model(inputs)`
with `mask_format = "rle"` (the same codes, with a host synchronisation per image).  Development aid.

    python tests/perf_mask_pack.py [--rounds 5] [--calls 5]
    torchrun --nproc-per-node N tests/perf_mask_pack.py --gpus N

APE-L_D, 1203 names, bench.py's score threshold and synthetic weights, instance masks, fp16, CUDA graphs, one image per call
(1024 x 768 and 1024^2, on the device).  Arms, alternated round by round, host clock around calls that end with the results on
the host: `model` = model(inputs); `packed` = parallel.unpack_packed(model.forward_packed(inputs)).  With --gpus N > 1 the step
of each arm is what a multi-GPU evaluation runs: model(inputs) + gather_detections (boxes only: the masks stay on their rank)
against forward_packed + gather_packed (masks included); rank 0 prints.  Also: the mask stage alone (ops.mask_pack, CUDA events
over 20 launches), the bytes per image of the gather, and the share of slots that hold bits.  Synthetic-weight masks are noisy
blobs, so their codes are longer than a trained model's: the bits share here is not representative.  Every record gives the
median and [min, max]; the first line is the card, its power limit and maximal SM clock."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--gpus", type=int, default=1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_mask_pack.py needs a GPU"
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    assert world == args.gpus, f"--gpus {args.gpus} needs as many processes (torchrun --nproc-per-node {args.gpus})"
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        import torch.distributed as dist

        dist.init_process_group("nccl", device_id=dev)
    from ape_b200 import configs, ops, parallel, synthetic
    from ape_b200.modeling import build_model

    spec = copy.deepcopy(configs.APE_L_D)
    spec["test_score_thresh"] = SCORE_THRESH
    model = build_model(spec, num_text=1203)
    synthetic.fill_state_dict(model)
    synthetic.suppress_invalid_anchor_logits(model)
    model = model.to(dev).eval()
    model.engine_dtype, model.use_cuda_graphs = torch.float16, True
    model.test_mask_on, model.mask_format = True, "rle"
    if rank == 0:
        print(json.dumps({"card": card(), "gpus": world, "model": "APE-L_D", "names": 1203, "dtype": "float16", "graphs": True,
                          "score_thresh": SCORE_THRESH, "mask_slot_bytes": model.mask_slot_bytes}), flush=True)
    g = torch.Generator().manual_seed(rank)
    for (h, w) in ((1024, 768), (1024, 1024)):
        imgs = [torch.randint(0, 256, (3, h, w), generator=g).float().to(dev) for _ in range(3)]

        def inputs(i):
            return [{"image": imgs[i % len(imgs)], "height": h, "width": w}]

        def arm_model(i):
            out = model(inputs(i))
            if world > 1:
                parallel.gather_detections([o["instances"] for o in out], 300, dev, dst=0)
            return out

        def arm_packed(i):
            if world > 1:
                out = parallel.gather_packed(model.forward_packed(inputs(i)), dst=0)
                if out is None:
                    torch.cuda.current_stream().synchronize()
                return out
            return parallel.unpack_packed(model.forward_packed(inputs(i)))

        arms = {"model": arm_model, "packed": arm_packed}
        for i in range(3):  # warm-up: graphs captured, caches filled
            for fn in arms.values():
                fn(i)
        want, got = model(inputs(0)), parallel.unpack_packed(model.forward_packed(inputs(0)))
        same = all([r["counts"] for r in a["instances"].pred_masks_rle] == [r["counts"] for r in b["instances"].pred_masks_rle]
                   and torch.equal(a["instances"].pred_boxes.tensor, b["instances"].pred_boxes.tensor) for a, b in zip(want, got))
        times = {k: [] for k in arms}
        for r in range(args.rounds):
            for k, fn in arms.items():
                if world > 1:
                    torch.distributed.barrier()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for c in range(args.calls):
                    fn(r * args.calls + c)
                torch.cuda.synchronize()
                times[k].append((time.perf_counter() - t0) * 1e3 / args.calls)
        # the mask stage alone, on this image's selection rows and mask logits
        packed = model.forward_packed(inputs(0))
        rows = packed[..., :52].contiguous().view(torch.float32)
        logits = model.last_outputs["pred_masks"].contiguous()
        padded = (1024, 1024)
        ops.mask_pack(logits, rows, [(h, w)], padded, model.mask_slot_bytes)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(20):
            ops.mask_pack(logits, rows, [(h, w)], padded, model.mask_slot_bytes)
        b.record()
        torch.cuda.synchronize()
        kinds = packed[..., 52:56].contiguous().view(torch.int32)[..., 0].flatten().tolist()
        live = [k for k in kinds if k != 0]
        rec = {"image": [h, w], "rounds": args.rounds, "calls_per_round": args.calls,
               "model_rle_ms": stat(times["model"]), "packed_ms": stat(times["packed"]),
               "speedup": round(statistics.median(times["model"]) / statistics.median(times["packed"]), 3),
               "mask_stage_ms": round(a.elapsed_time(b) / 20, 4), "detections": len(live),
               "bits_share": round(sum(k == ops.MASK_SLOT_BITS for k in live) / max(len(live), 1), 4),
               "gather_bytes_per_image": int(packed[0].numel()), "boxes_only_gather_bytes_per_image": int(packed.shape[1] * 13 * 4),
               "outputs_identical": bool(same)}
        if rank == 0:
            print(json.dumps(rec), flush=True)
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    with torch.no_grad():
        main()
