#!/usr/bin/env python
"""Semantic label maps as run-length codes: the encoder alone and the packed semantic results end to end.  Development aid.

    python tests/perf_semseg_pack.py [--rounds 5] [--calls 3]
    torchrun --nproc-per-node N tests/perf_semseg_pack.py --gpus N

(a) The encoder alone (ops.semseg_pack with a slot that always holds the codes: CUDA events over 20 launches; and
    ops.label_map_rle, host clock, codes on the host) at 1024 x 768 and 2048 x 1024, on the engine's own label map (APE-L_D, synthetic
    weights, 1203 names) and on a smooth map (Voronoi cells of 30 seeds), against the host work of encode_json_sem_seg on the same
    map: np.unique, then per label the mask in Fortran order and its runs (numpy; cocoapi's C string coding is not counted, so
    the host figure is a lower bound).
(b) APE-L_D, 1203 names, boxes + masks + semantic, fp16, CUDA graphs, one image per call: parallel.unpack_packed(forward_packed)
    against model(inputs) with sem_seg_format = "label" plus the host encoding of (a).  With --gpus N > 1 each arm's step is what a
    multi-GPU evaluation runs: model(inputs) + gather_detections (boxes only) against forward_packed + gather_packed.
(c) Gather bytes per image and the share of slot kinds (1 codes, 2 map as uint16, 3 nothing fits).
Synthetic-weight label maps are noisy, so their codes are longer than a trained model's: the kind shares here are not
representative.  Records give the median and [min, max]; the first line is the card, its power limit and maximal SM clock."""
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

from perf_ape_ti import card  # noqa: E402

SCORE_THRESH = 0.0123  # bench.py's BENCH_SCORE_THRESH


def stat(ts, digits=3):
    return {"median": round(statistics.median(ts), digits), "min": round(min(ts), digits), "max": round(max(ts), digits)}


def voronoi(h, w, n, seed):
    rng = np.random.default_rng(seed)
    seeds = rng.random((n, 2)) * [h, w]
    labels = rng.integers(0, 1203, n)
    out = np.empty((h, w), np.int64)
    xx = np.arange(w)
    for y in range(h):  # row by row: [n, w] distances, not [n, h, w]
        d = (y - seeds[:, 0, None]) ** 2 + (xx[None] - seeds[:, 1, None]) ** 2
        out[y] = labels[d.argmin(0)]
    return out


def host_encode(L):
    """The array work of encode_json_sem_seg: per label present, its mask in Fortran order and the run boundaries."""
    runs = []
    for c in np.unique(L):
        v = np.asfortranarray(L == c).reshape(-1, order="F")
        runs.append(np.flatnonzero(v[1:] != v[:-1]))
    return runs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--gpus", type=int, default=1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_semseg_pack.py needs a GPU"
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
    model.test_mask_on, model.mask_format, model.semantic_on = True, "rle", True
    if rank == 0:
        print(json.dumps({"card": card(), "gpus": world, "model": "APE-L_D", "names": 1203, "dtype": "float16", "graphs": True,
                          "score_thresh": SCORE_THRESH, "mask_slot_bytes": model.mask_slot_bytes,
                          "sem_seg_slot_bytes": model.sem_seg_slot_bytes}), flush=True)
    g = torch.Generator().manual_seed(rank)
    for (h, w) in ((1024, 768), (1024, 2048)):
        imgs = [torch.randint(0, 256, (3, h, w), generator=g).float().to(dev) for _ in range(3)]
        scale = 1024 / max(h, w)  # the model's input is at most 1024 on its long side; the output is the full size
        small = [torch.nn.functional.interpolate(im[None], scale_factor=scale, mode="bilinear")[0] for im in imgs]

        def inputs(i):
            return [{"image": small[i % len(small)], "height": h, "width": w}]

        # (a) the encoder alone
        model.sem_seg_format = "label"
        engine_map = model(inputs(0))[0]["sem_seg_label"]
        maps = {"engine": engine_map, "voronoi30": torch.from_numpy(voronoi(h, w, 30, 7)).to(dev)}
        for name, L in maps.items():
            L = L.contiguous()
            slot = int(ops._lib.lib.ape_label_rle_out_bytes(min(L.numel(), 65536), L.numel())) // 4 * 4 + 4
            slot = min(slot, 1 << 30)
            slots = torch.empty((1, slot), dtype=torch.uint8, device=dev)
            info = torch.empty((1, 3), dtype=torch.int32, device=dev)
            ops.semseg_pack([L], 1203, slots, info)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(20):
                ops.semseg_pack([L], 1203, slots, info)
            b.record()
            torch.cuda.synchronize()
            kind, nbytes, P = info[0].tolist()
            host = L.cpu().numpy()
            t_dev, t_host = [], []
            for _ in range(args.rounds):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                ops.label_map_rle(L)
                t_dev.append((time.perf_counter() - t0) * 1e3)
                t0 = time.perf_counter()
                host_encode(host)
                t_host.append((time.perf_counter() - t0) * 1e3)
            if rank == 0:
                print(json.dumps({"arm": "encoder", "map": name, "size": [h, w], "labels": P, "kind": kind, "code_bytes": nbytes,
                                  "device_encode_ms": round(a.elapsed_time(b) / 20, 4), "label_map_rle_ms": stat(t_dev),
                                  "host_encode_lower_bound_ms": stat(t_host)}), flush=True)

        # (b) end to end, (c) gather bytes and slot kinds
        def arm_model(i):
            model.sem_seg_format = "label"
            out = model(inputs(i))
            for o in out:
                host_encode(o["sem_seg_label"].cpu().numpy())
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
        for i in range(2):
            for fn in arms.values():
                fn(i)
        model.sem_seg_format = "rle"
        want, got = model(inputs(0)), parallel.unpack_packed(model.forward_packed(inputs(0)))
        same = all([(e["label"], e["segmentation"]["counts"]) for e in a["sem_seg_rle"]] ==
                   [(e["label"], e["segmentation"]["counts"]) for e in b["sem_seg_rle"]] for a, b in zip(want, got))
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
        kinds = []
        for i in range(len(imgs)):
            packed = model.forward_packed(inputs(i))
            kinds.append(int(packed[0, :32].view(torch.int32)[2]))
        rec = {"arm": "end_to_end", "image": [h, w], "rounds": args.rounds, "calls_per_round": args.calls,
               "model_label_plus_host_encode_ms": stat(times["model"]), "packed_ms": stat(times["packed"]),
               "gather_bytes_per_image": int(packed[0].numel()), "slot_kinds": {k: kinds.count(k) / len(kinds) for k in (1, 2, 3)},
               "sem_seg_rle_identical": bool(same)}
        if rank == 0:
            print(json.dumps(rec), flush=True)
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    with torch.no_grad():
        main()
