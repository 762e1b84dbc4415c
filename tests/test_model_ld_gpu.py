"""GPU parity of the BENCHMARKED configuration against the reference itself: APE-L_D (ViT-L 24 blocks, 6+6 deformable
layers, 900 queries), one 1024 x 768 image padded to 1024^2, 1203-name vocabulary, boxes only.

`tests/golden/model_ld_1024.npz` was recorded by running the reference's own files on the CPU (fp32, pytorch_attn=True;
tests/golden/gen_model_golden.py ld).  The engine is compared with it stage by stage in three numeric modes:
  float32           library GEMMs + the repo's MSDA / NMS kernels (strict mode)
  float16 + graphs  the SHIPPED path of bench.py: wgmma GEMMs / attention, fused MSDA, one CUDA graph
  bfloat16 + graphs same kernels, bf16 operands
Each stage prints max |err|, the RMS of the golden tensor and the max / median error relative to that RMS."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from ape_b200 import configs
from oracle import synth

pytestmark = [pytest.mark.gpu, pytest.mark.slow]
DEV = "cuda:0"
N_TEXT = 1203

# median|err| / rms(golden) allowed per stage and mode; the maximum may be 5x that.
# The decoder amplifies encoder-output differences about 100x with these untrained weights (fp32 GPU vs fp32 CPU: memory
# 2e-5 -> logits 2e-3), so north_star's 1e-3 on the logits is met by the median of the fp32 mode only; see DESIGN.md.
TOL = {
    "float32": dict(backbone=1e-4, neck=1e-4, encoder=2e-4, memory=2e-4, logits=6e-3, boxes=8e-3),
    "float16": dict(backbone=2e-3, neck=2.5e-3, encoder=2.5e-3, memory=2.5e-3, logits=1e-1, boxes=2e-1),
    "bfloat16": dict(backbone=1.5e-2, neck=2e-2, encoder=2e-2, memory=2e-2, logits=1.5e-1, boxes=3e-1),
}


def err(name, got, want, report):
    got, want = got.float().cpu(), want.float()
    assert got.shape == want.shape, (name, got.shape, want.shape)
    d = (got - want).abs()
    rms = want.pow(2).mean().sqrt().item() + 1e-12
    rel = d / want.abs().clamp_min(1e-6)
    rec = dict(max_abs=d.max().item(), rms=rms, max_over_rms=d.max().item() / rms, median_over_rms=d.median().item() / rms,
               median_rel=rel.median().item())
    report[name] = rec
    print(f"  {name:24s} max|err| {rec['max_abs']:.3e}  rms(ref) {rms:.3e}  max/rms {rec['max_over_rms']:.3e}  "
          f"median/rms {rec['median_over_rms']:.3e}  median rel {rec['median_rel']:.3e}")
    return rec


@pytest.fixture(scope="module")
def setup():
    from ape_b200.modeling import build_model

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    model = build_model(configs.APE_L_D, num_text=N_TEXT)
    synth.fill_state_dict(model)
    synth.suppress_invalid_anchor_logits(model)
    model = model.to(DEV)
    return model, load_golden("model_ld_1024.npz")


def run(model, mode, thresh=0.0):
    dt = getattr(torch, mode)
    model.engine_dtype = dt
    model.use_cuda_graphs = dt != torch.float32
    model.test_score_thresh = thresh
    model.transformer.encoder.record_taps = True
    try:
        inp = [{"image": synth.image(1024, 768, seed=0), "height": 1024, "width": 768}]
        out = model(inp)
        if model.use_cuda_graphs:  # second call = graph REPLAY (the first captured); results must come from the replay
            out = model(inp)
        lo = dict(model.last_outputs)
        lo["topk"] = model.transformer.last_topk_proposals.clone()
        lo["taps"] = {k: v.clone() for k, v in getattr(model.transformer.encoder, "taps", {}).items()}
        lo["enc_class"] = lo.get("enc_class")
        return out, lo
    finally:
        model.engine_dtype, model.use_cuda_graphs = torch.float32, False
        model.transformer.encoder.record_taps = False


@pytest.mark.parametrize("mode", ["float32", "float16", "bfloat16"])
def test_ld_1024_stagewise_vs_reference_golden(setup, mode):
    model, g = setup
    tol = TOL[mode]
    report = {}
    print(f"\n== APE-L_D 1024^2 / 1203 names, engine mode {mode}" + (" + CUDA graph replay" if mode != "float32" else ""))
    out, lo = run(model, mode)
    for k in ("p2", "p3", "p4", "p5", "p6"):
        r = err(f"backbone.{k}", lo["features"][k][:, ::16, ::8, ::8], g[f"backbone.{k}"], report)
        assert r["max_over_rms"] < tol["backbone"] * 5 and r["median_over_rms"] < tol["backbone"]
    for i in range(5):
        r = err(f"neck.{i}", lo["neck"][i][:, ::16, ::8, ::8], g[f"neck.{i}"], report)
        assert r["max_over_rms"] < tol["neck"] * 5 and r["median_over_rms"] < tol["neck"]
    for k, v in sorted(lo["taps"].items()):  # per-layer fusion / encoder-layer outputs (engine schedule exposes them as taps)
        r = err(k, v[:, ::2048, ::4], g[k], report)
        assert r["max_over_rms"] < tol["encoder"] * 5 and r["median_over_rms"] < tol["encoder"]
    r = err("memory", lo["memory"][:, ::512, ::4], g["memory"], report)
    assert r["max_over_rms"] < tol["memory"] * 5 and r["median_over_rms"] < tol["memory"]
    # two-stage selection: proposal indices.  Bit-exactness of the selection CODE on identical inputs is asserted in
    # tests/test_model_gpu.py (oracle inputs); end to end the 16-bit encoder output perturbs near-ties of top-k / NMS(0.9)
    sel, want = lo["topk"][0].cpu().tolist(), g["topk_proposals"][0].tolist()
    common = sorted(set(sel) & set(want))
    frac = len(common) / len(want)
    same_slot = sum(int(a == b) for a, b in zip(sel, want)) / len(want)
    print(f"  selected proposals: {len(common)}/{len(want)} in common ({frac:.4f}), {same_slot:.4f} at the same slot")
    assert frac > (0.99 if mode == "float32" else 0.95 if mode == "float16" else 0.9)
    ia = torch.tensor([sel.index(i) for i in common])
    ib = torch.tensor([want.index(i) for i in common])
    r = err("pred_logits (common q)", lo["pred_logits"][0][ia][:, ::32], g["pred_logits"][0][ib], report)
    logit_rel = ((lo["pred_logits"][0][ia][:, ::32].float().cpu() - g["pred_logits"][0][ib]).abs() / g["pred_logits"][0][ib].abs()).max().item()
    print(f"  pred_logits max RELATIVE error on commonly selected queries: {logit_rel:.3e} (north_star: 1e-3)")
    assert r["max_over_rms"] < tol["logits"]
    r = err("pred_boxes (common q)", lo["pred_boxes"][0][ia], g["pred_boxes"][0][ib], report)
    assert r["max_over_rms"] < tol["boxes"]
    # final detections at the config's own test_score_thresh = 0.0: 1.08 M (query, class) candidates -> per-class NMS -> top 300
    inst = out[0]["instances"]
    assert len(inst) == len(g["det0.scores"]) == 300
    k = 50
    torch.testing.assert_close(inst.scores[:k], g["det0.scores"][:k], rtol=1e-1 if mode != "float32" else 5e-3, atol=2e-3 if mode != "float32" else 1e-4)
    got_pairs = {(sel[q], c) for q, c in zip(inst.query_index.tolist(), inst.pred_classes.tolist())}
    want_classes = g["det0.classes"].tolist()
    agree = len(set(inst.pred_classes.tolist()) & set(want_classes)) / len(set(want_classes))
    top_agree = len(set(inst.pred_classes[:k].tolist()) & set(want_classes[:k])) / len(set(want_classes[:k]))
    print(f"  final detections (thresh 0.0, top-300): class-set agreement {agree:.3f} (top-{k}: {top_agree:.3f}), "
          f"{len(got_pairs)} distinct (proposal, class) pairs")
    if mode == "float32":
        assert top_agree > 0.9 and agree > 0.9


@pytest.mark.parametrize("mode", ["float32", "float16"])
def test_ld_1024_thresholded_detections_vs_reference_golden(setup, mode):
    """Selection load of the bench: a score threshold that ~500 of the 1.08 M pairs pass (coordinate-trick NMS path)."""
    model, g = setup
    thr = float(g["det_thr.thresh"])
    out, lo = run(model, mode, thresh=thr)
    inst = out[0]["instances"]
    sel = lo["topk"][0].cpu().tolist()
    want_prop = g["topk_proposals"][0][g["det_thr.query_index"]].tolist()
    want = set(zip(want_prop, g["det_thr.classes"].tolist()))
    got = set(zip([sel[q] for q in inst.query_index.tolist()], inst.pred_classes.tolist()))
    inter = len(want & got) / max(1, len(want))
    print(f"\n== thresholded selection ({mode}): {len(got)} kept, {len(want)} in the golden, {inter:.3f} of the golden's (proposal, class) pairs reproduced")
    assert abs(len(got) - len(want)) <= (2 if mode == "float32" else 30)
    assert inter > (0.98 if mode == "float32" else 0.80)
    if mode == "float32":  # scores by rank; boxes of the pairs both sides kept (near-equal scores may swap ranks)
        k = min(len(inst), len(g["det_thr.scores"]), 100)
        torch.testing.assert_close(inst.scores[:k], g["det_thr.scores"][:k], rtol=5e-3, atol=1e-4)
        gpairs = list(zip([sel[q] for q in inst.query_index.tolist()], inst.pred_classes.tolist()))
        wpairs = list(zip(want_prop, g["det_thr.classes"].tolist()))
        widx = {p: i for i, p in enumerate(wpairs)}
        ia = [i for i, p in enumerate(gpairs) if p in widx]
        ib = [widx[gpairs[i]] for i in ia]
        torch.testing.assert_close(inst.pred_boxes.tensor[ia], g["det_thr.boxes"][ib], rtol=5e-3, atol=2.0)
