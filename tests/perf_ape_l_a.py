"""APE-L_A against APE-L_B at 1024^2 (1203 names, boxes, B = 1, fp16, CUDA graphs), in one process, alternated round by
round: the whole detection step, and the backbone + pyramid replay alone (one captured graph each).  The two share the
backbone and the neck-less feature path; APE-L_A's encoder has no vision-language fusion layers, so the difference in the
step is what the six fusion layers (and their row kernels) cost.

    python tests/perf_ape_l_a.py [--rounds 5] [--iters 20]

Prints the card name and power limit, then one JSON line with the median and [min, max] per step (ms)."""
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


def build(spec):
    from ape_b200 import synthetic
    from ape_b200.modeling import build_model

    m = build_model(spec, num_text=1203)
    synthetic.fill_state_dict(m)
    synthetic.suppress_invalid_anchor_logits(m)
    m = m.to("cuda")
    m.engine_dtype, m.use_cuda_graphs = torch.float16, True
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_ape_l_a.py needs a GPU"
    from ape_b200 import configs, synthetic

    models = {"APE-L_A": build(configs.APE_L_A), "APE-L_B": build(configs.APE_L_B)}
    img = synthetic.image(1024, 768, seed=0).float().cuda()
    inputs = [{"image": img, "height": 1024, "width": 768}]

    def backbone_fn(m):
        def fn(t):
            with torch.autocast("cuda", dtype=torch.float16), torch.no_grad():
                return m.backbone(t)
        return fn

    replay = {}
    for k, m in models.items():
        x = torch.zeros(1, 3, 1024, 1024, device="cuda")
        x[0, :, :, :768] = (img - m.pixel_mean) / m.pixel_std
        replay[k], _ = graphed(backbone_fn(m), x.half())
        for _ in range(3):  # capture the per-geometry graph of the whole step, then warm it
            m(inputs)
    res = {k: {"backbone_pyramid": [], "step": []} for k in models}
    for _ in range(args.rounds):
        for k, m in models.items():
            res[k]["backbone_pyramid"].append(time_ms(replay[k], args.iters))
            res[k]["step"].append(time_ms(lambda: m(inputs), args.iters))
    print(f"card: {card()}")
    out = {k: {s: round(statistics.median(v), 3) for s, v in r.items()} for k, r in res.items()}
    out["spread"] = {k: {s: [round(min(v), 3), round(max(v), 3)] for s, v in r.items()} for k, r in res.items()}
    out.update(workload="1024 x 768 padded to 1024^2, 1203 names, boxes, B=1, fp16, CUDA graphs", rounds=args.rounds,
               iters=args.iters)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
