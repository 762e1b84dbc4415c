#!/usr/bin/env python
"""Panoptic maps in the packed device results: the per-image stage alone and the packed results end to end.  Development aid.

    python tests/perf_panoptic_pack.py [--rounds 7] [--calls 3]

(a) The per-image stage at K in {100, 300} and outputs 480 x 640, 1024 x 768 and 2048 x 1536 on the blob logits of
    test_panoptic_merge_gpu.py (fp16): postprocess_panoptic_winners (the winners kernel, one device->host copy of the counts, the
    segment bookkeeping on the host, the painting by lookup) against ops.panoptic_winners + ops.panoptic_pack (no host work), each
    timed with a host clock around calls that end in a synchronise; and ops.panoptic_pack alone (CUDA events over 20 launches).
(b) APE-L_D, synthetic weights, 133 names (80 things + 53 stuff, the COCO panoptic configuration: instance, masks, semantic and
    panoptic branches), fp16, CUDA graphs, one 1024 x 768 image per call: model(inputs) (mask_format and sem_seg_format "rle")
    against parallel.unpack_packed(model.forward_packed(inputs)), alternated; and whether both give the same panoptic_seg.
(c) The gathered bytes per image.
Records give the median and [min, max] in ms; the first line is the card, its power limit and maximal SM clock."""
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


def host_clock(fn, rounds):
    ts = []
    for _ in range(rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return ts


def stage(args):
    from ape_b200 import ops
    from ape_b200.modeling.postprocess import _query_scores, postprocess_panoptic_winners
    from test_panoptic_merge_gpu import CFG, N_CLS, N_THING, PADDED, _inputs

    for K in (100, 300):
        logits, qi, mask_cls = _inputs(K, torch.float16, seed=K)
        img = (1000, 760)
        for out in ((480, 640), (1024, 768), (2048, 1536)):
            slot = torch.empty((ops.panoptic_slot_bytes_needed(K, out),), dtype=torch.uint8, device="cuda")

            def host_path():
                return postprocess_panoptic_winners(mask_cls, logits, qi, PADDED, img, out[0], out[1], range(N_THING), N_THING, False,
                                                    CFG)

            def device_path():
                scores, labels, keep = _query_scores(mask_cls, CFG)
                ids, counts = ops.panoptic_winners(logits, qi, torch.where(keep, scores, float("-inf")), PADDED, img, out, CFG["prob"])
                ops.panoptic_pack(ids, counts, labels.to(torch.int32), N_CLS, N_THING, False, CFG["overlap_threshold"], slot)
                return ids, counts, labels

            for _ in range(3):
                host_path()
                ids, counts, labels = device_path()
            t_host, t_dev = [], []
            for _ in range(args.rounds):  # alternated
                t_host += host_clock(host_path, 1)
                t_dev += host_clock(device_path, 1)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            cls = labels.to(torch.int32)
            a.record()
            for _ in range(20):
                ops.panoptic_pack(ids, counts, cls, N_CLS, N_THING, False, CFG["overlap_threshold"], slot)
            b.record()
            torch.cuda.synchronize()
            print(json.dumps({"arm": "stage", "K": K, "output": list(out), "postprocess_panoptic_winners_ms": stat(t_host),
                              "winners_plus_pack_ms": stat(t_dev), "panoptic_pack_kernels_ms": round(a.elapsed_time(b) / 20, 4),
                              "slot_bytes": slot.numel()}), flush=True)


def end_to_end(args):
    from ape_b200 import configs, parallel, synthetic
    from ape_b200.modeling import build_model

    spec = copy.deepcopy(configs.APE_L_D)
    spec["test_score_thresh"] = SCORE_THRESH
    model = build_model(spec, num_text=133)
    synthetic.fill_state_dict(model)
    synthetic.suppress_invalid_anchor_logits(model)
    model = model.to("cuda").eval()
    model.engine_dtype, model.use_cuda_graphs = torch.float16, True
    model.instance_on, model.test_mask_on, model.semantic_on, model.panoptic_on = True, True, True, True
    model.mask_format, model.sem_seg_format = "rle", "rle"
    name = model.dataset_names[0]
    names = [f"class{i}" for i in range(133)]
    model.dataset_stuff[name] = (names[:80], names[80:], "thing+stuff")
    model.set_eval_dataset(name)
    h, w = 1024, 768
    g = torch.Generator().manual_seed(0)
    imgs = [torch.randint(0, 256, (3, h, w), generator=g).float().cuda() for _ in range(3)]

    def inputs(i):
        return [{"image": imgs[i % len(imgs)], "height": h, "width": w}]

    arms = {"model": lambda i: model(inputs(i)), "packed": lambda i: parallel.unpack_packed(model.forward_packed(inputs(i)))}
    for i in range(2):
        for fn in arms.values():
            fn(i)
    want, got = arms["model"](0)[0], arms["packed"](0)[0]
    same = torch.equal(want["panoptic_seg"][0].cpu(), got["panoptic_seg"][0]) and want["panoptic_seg"][1] == got["panoptic_seg"][1]
    times = {k: [] for k in arms}
    for r in range(args.rounds):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for c in range(args.calls):
                fn(r * args.calls + c)
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3 / args.calls)
    packed = model.forward_packed(inputs(0))
    print(json.dumps({"arm": "end_to_end", "model": "APE-L_D", "names": 133, "image": [h, w], "rounds": args.rounds,
                      "calls_per_round": args.calls, "model_ms": stat(times["model"]), "packed_ms": stat(times["packed"]),
                      "gather_bytes_per_image": int(packed[0].numel()), "panoptic_slot_bytes": model.panoptic_slot_bytes,
                      "segments": len(got["panoptic_seg"][1]), "panoptic_identical": bool(same)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--skip-model", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_panoptic_pack.py needs a GPU"
    print(json.dumps({"card": card(), "gpus": 1, "multi_gpu_step": "not measured"}), flush=True)
    stage(args)
    if not args.skip_model:
        end_to_end(args)


if __name__ == "__main__":
    with torch.no_grad():
        main()
