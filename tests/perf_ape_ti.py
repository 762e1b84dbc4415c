"""APE-Ti at 1024^2 (BASELINE.json configs[0], 80 names, fp16, CUDA graphs): the ViT backbone + feature pyramid and the whole
detection step, on the engine's raster token path against the library path (cuBLAS / cuDNN / SDPA under autocast, what the
16-bit mode ran before the engine covered APE-Ti).  Both run in one process on two copies of the same model, alternated
round by round; the library copy has ViT._engine_ok patched to refuse.

    python tests/perf_ape_ti.py [--rounds 5] [--iters 20]

Prints the card name and power limit, then one JSON line with the median times (ms)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def build(engine):
    from ape_b200 import configs, synthetic
    from ape_b200.modeling import build_model

    m = build_model(configs.APE_TI, num_text=80)
    synthetic.fill_state_dict(m)
    m = m.to("cuda")
    m.engine_dtype, m.use_cuda_graphs = torch.float16, True
    if not engine:
        m.backbone.net._engine_ok = lambda x: False
    return m


def graphed(fn, x):
    """fn(x) captured once (after two warm-up calls on a side stream); returns the replay callable."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            fn(x)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn(x)
    return g.replay, out


def time_ms(run, iters):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        run()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_ape_ti.py needs a GPU"
    from ape_b200 import synthetic

    models = {"engine": build(True), "library": build(False)}
    img = synthetic.image(1024, 1024, seed=0).float().cuda()
    x = ((img - models["engine"].pixel_mean) / models["engine"].pixel_std)[None].half()

    def backbone_fn(m):
        def fn(t):
            with torch.autocast("cuda", dtype=torch.float16), torch.no_grad():
                return m.backbone(t)
        return fn

    replay, feats = {}, {}
    for k, m in models.items():
        replay[k], feats[k] = graphed(backbone_fn(m), x)
    replay["engine"]()
    replay["library"]()
    torch.cuda.synchronize()
    diff = max((feats["engine"][f].float() - feats["library"][f].float()).abs().max().item() for f in feats["engine"])
    inputs = [{"image": img, "height": 1024, "width": 1024}]
    for m in models.values():  # capture the per-geometry graph of the whole step, then warm it
        for _ in range(3):
            m(inputs)
    res = {k: {"backbone_pyramid": [], "step": []} for k in models}
    for _ in range(args.rounds):
        for k, m in models.items():
            res[k]["backbone_pyramid"].append(time_ms(replay[k], args.iters))
            res[k]["step"].append(time_ms(lambda: m(inputs), args.iters))
    print(f"card: {card()}")
    out = {k: {s: round(statistics.median(v), 3) for s, v in r.items()} for k, r in res.items()}
    out["spread"] = {k: {s: [round(min(v), 3), round(max(v), 3)] for s, v in r.items()} for k, r in res.items()}
    out["backbone_pyramid_max_abs_diff_engine_vs_library"] = diff
    out.update(workload="APE-Ti 1024^2, 80 names, B=1, fp16, CUDA graphs", rounds=args.rounds, iters=args.iters)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
