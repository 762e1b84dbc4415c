#!/usr/bin/env python
"""The text tower's length-packed mode (`pack_prompts=True`) against the padded engine path.  Development aid.

    python tests/perf_text_pack.py [--rounds 5] [--layers 32] > text_pack.jsonl

EVA02-CLIP-bigE-14-plus text tower (32 layers, width 1280, 20 heads x 64, 77-token context), fp16, synthetic weights, one
model in one process.  Prompt sets (random word ids; only the lengths matter to the time):
  names        1203 prompts, lengths uniform in 3..8 including the start and end-of-text tokens
  phrases      5000 prompts, lengths uniform in 4..16
  expressions  3 prompts of 11, 12 and 13 tokens (referring expressions: a latency-bound call)
  full         256 prompts of 77 tokens (packing gains nothing: one prompt per 128-row tile against 80 rows padded, so the
               mode runs such a chunk padded; the attention records below show the packed kernel at this shape)
Arms of `forward_text`, fed host tokens as a tokenizer returns them, alternated round by round over rotating token sets,
host clock around calls that end in a device synchronise: `padded` (pack_prompts=False), `packed` (pack_prompts=True,
need_hidden=False: what the detector asks for) and `packed_hidden` (pack_prompts=True with `last_hidden_state`).  Then the
attention kernel alone at each set's shape: a CUDA graph of 20 launches over rotating qkv buffers, ape_attn_fwd_ex (causal,
77 of 80 rows, chunks of max_batch_size prompts) against ape_attn_fwd_seg over the packed tiles.  Every record gives the median
and [min, max] over the rounds; the first line is the card, its power limit and maximal SM clock."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from perf_ape_ti import card, graphed, time_ms  # noqa: E402

DEV = "cuda:0"
CTX, VOCAB, LAUNCHES, SETS = 77, 49408, 20, 4
CASES = {  # name: (prompts, shortest, longest, calls per round)
    "names": (1203, 3, 8, 3),
    "phrases": (5000, 4, 16, 2),
    "expressions": (3, 11, 13, 20),
    "full": (256, 77, 77, 3),
}


def tokens(n, lo, hi, seed):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(lo, hi + 1, (n,), generator=g)
    tok = torch.randint(1, VOCAB - 2, (n, CTX), generator=g)
    tok[torch.arange(CTX)[None] >= lens[:, None]] = 0
    tok[:, 0] = VOCAB - 2
    tok[torch.arange(n), lens - 1] = VOCAB - 1
    return tok, lens


def stat(ts, digits=3):
    return {"median": round(statistics.median(ts), digits), "min": round(min(ts), digits), "max": round(max(ts), digits)}


def tower_records(clip, rounds):
    from ape_b200.modeling.text import pack_layout

    arms = {"padded": (False, True), "packed": (True, False), "packed_hidden": (True, True)}
    for name, (n, lo, hi, calls) in CASES.items():
        sets = [tokens(n, lo, hi, seed=s) for s in range(SETS)]

        def run(arm, i):
            clip.pack_prompts, need_hidden = arms[arm]
            return clip.forward_text(sets[i % SETS][0], need_hidden=need_hidden)

        outs = {arm: run(arm, 0)["last_hidden_state_eot"] for arm in arms}  # warm-up of every shape, and the results compared
        for arm in arms:
            run(arm, 1)
        times = {arm: [] for arm in arms}
        for r in range(rounds):
            for arm in arms:
                k = iter(range(r * calls, (r + 1) * calls))
                times[arm].append(time_ms(lambda: run(arm, next(k)), calls))
        lens = sets[0][1].tolist()
        mbs = clip.max_batch_size
        packed_rows = sum(pack_layout(lens[i:i + mbs], CTX)["tiles"] * 128 for i in range(0, n, mbs))
        rec = {"case": name, "prompts": n, "lengths": [lo, hi], "tokens": int(sum(lens)), "rows_padded": 80 * n,
               "rows_packed": packed_rows, "rounds": rounds, "calls_per_round": calls,
               "max_abs_diff_packed_vs_padded": (outs["packed"] - outs["padded"]).abs().max().item(),
               "output_rms": outs["padded"].pow(2).mean().sqrt().item()}
        for arm, ts in times.items():
            rec[arm + "_ms"] = stat(ts)
        rec["speedup_packed"] = round(rec["padded_ms"]["median"] / rec["packed_ms"]["median"], 2)
        print(json.dumps(rec), flush=True)
        del outs
        torch.cuda.empty_cache()


def attention_records(clip, rounds, iters=10):
    from ape_b200 import ops
    from ape_b200.modeling.text import pack_layout

    H, mbs = clip.net.text.heads, clip.max_batch_size
    g = torch.Generator(device=DEV).manual_seed(0)
    for name, (n, lo, hi, _) in CASES.items():
        lens = tokens(n, lo, hi, seed=0)[1].tolist()
        chunks = [lens[i:i + mbs] for i in range(0, n, mbs)]
        lays = [pack_layout(c, CTX) for c in chunks]
        segs = [torch.from_numpy(lay["seg_start"]).to(DEV) for lay in lays]
        nbuf = 2 if 80 * n * 3 * H * 64 * 2 > 100_000_000 else SETS
        padded_qkv = [[torch.randn(80 * len(c), 3 * H * 64, device=DEV, generator=g).half() for c in chunks] for _ in range(nbuf)]
        packed_qkv = [[torch.randn(128 * lay["tiles"], 3 * H * 64, device=DEV, generator=g).half() for lay in lays] for _ in range(nbuf)]

        def padded(_):
            for i in range(LAUNCHES):
                for c, q in zip(chunks, padded_qkv[i % nbuf]):
                    ops.attention_qkv(q, len(c), 128, H, 64, 0.125, n_valid=CTX, seq_stride=80, causal=True)

        def packed(_):
            for i in range(LAUNCHES):
                for lay, seg, q in zip(lays, segs, packed_qkv[i % nbuf]):
                    ops.attention_qkv(q, lay["tiles"], 128, H, 64, 0.125, causal=True, seg_start=seg)

        replays = {"padded": graphed(padded, None)[0], "packed": graphed(packed, None)[0]}
        times = {k: [] for k in replays}
        for _ in range(rounds):
            for k, r in replays.items():
                times[k].append(time_ms(r, iters) * 1e3 / LAUNCHES)
        rec = {"attention": name, "heads": H, "launches_per_layer": len(chunks), "tiles_padded": n, "tiles_packed": sum(lay["tiles"] for lay in lays)}
        for k, ts in times.items():
            rec[k + "_us_per_layer"] = stat(ts, 1)
        print(json.dumps(rec), flush=True)
        del replays, padded_qkv, packed_qkv
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--layers", type=int, default=32, help="fewer layers for a quick look (the records say how many)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_text_pack.py needs a GPU"
    from ape_b200 import synthetic
    from ape_b200.modeling import EVA02CLIP

    print(json.dumps({"card": card(), "sms": torch.cuda.get_device_properties(0).multi_processor_count, "layers": args.layers,
                      "width": 1280, "dtype": "float16"}), flush=True)
    cfg = dict(EVA02CLIP.CONFIGS["EVA02-CLIP-bigE-14-plus"]["text_cfg"], layers=args.layers)
    clip = EVA02CLIP(dtype="float16", text_cfg=cfg)
    synthetic.fill_state_dict(clip.net.text)
    clip = clip.to(DEV)
    with torch.no_grad():
        tower_records(clip, args.rounds)
        attention_records(clip, args.rounds)


if __name__ == "__main__":
    main()
