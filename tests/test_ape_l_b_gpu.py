"""GPU: APE-L_B / APE-L_C on the engine — the vit_eva02.py sub-LN ViT-L (16 x 16 windows, global blocks 5 / 11 / 17 / 23, no
inner_attn_ln) and the neck-less feature path.

* The 16-bit ViT engine path against its fp32 library path at 1024^2, batch 1 and 2, fp16 and bf16.
* The 16-bit backbone + pyramid launch no library linear, matmul, convolution or SDPA.
* Without a neck the pyramid's last LayerNorms (and p6) write into one [B, S, 256] buffer: p2..p6 are views of it, the encoder
  consumes it, and it matches the fp32 path's concatenated levels.
* MINI_EVA02L against tests/golden/model_mini_lb.npz (reference files, CPU, fp32).
* APE-L_B at 1024^2, 1203 names against tests/golden/model_lb_1024.npz, stage by stage in fp32, fp16 + graphs and
  bf16 + graphs; graph replay equals eager bit for bit.
Weights: name-derived synthetic (oracle/synth.py); TF32 off.  Each comparison prints the errors it measured."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden
from ape_b200 import configs
from oracle import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
N_TEXT = 1203

# median|err| / rms(golden) allowed per stage and mode (the maximum may be 5x that); the bounds of test_model_ld_gpu.py
TOL = {
    "float32": dict(backbone=1e-4, encoder=2e-4, memory=2e-4, logits=6e-3, boxes=8e-3),
    "float16": dict(backbone=2e-3, encoder=2.5e-3, memory=2.5e-3, logits=1e-1, boxes=2e-1),
    "bfloat16": dict(backbone=1.5e-2, encoder=2e-2, memory=2e-2, logits=1.5e-1, boxes=3e-1),
}


def err(name, got, want):
    got, want = got.float().cpu(), want.float().cpu()
    assert got.shape == want.shape, (name, got.shape, want.shape)
    d = (got - want).abs()
    rms = want.pow(2).mean().sqrt().item() + 1e-12
    rec = dict(max_abs=d.max().item(), rms=rms, max_over_rms=d.max().item() / rms, median_over_rms=d.median().item() / rms)
    print(f"  {name:24s} max|err| {rec['max_abs']:.3e}  rms(ref) {rms:.3e}  max/rms {rec['max_over_rms']:.3e}  "
          f"median/rms {rec['median_over_rms']:.3e}")
    return rec


def _build(spec, num_text=None, suppress=True):
    from ape_b200.modeling import build_model

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    m = build_model(spec, num_text=num_text)
    synth.fill_state_dict(m)
    if suppress:  # as the golden generator did (model_lb_1024.npz: yes; model_mini_lb.npz: no)
        synth.suppress_invalid_anchor_logits(m)
    return m.to(DEV)


@pytest.fixture(scope="module")
def lb():
    return _build(configs.APE_L_B, num_text=N_TEXT)


# -- ViT engine path ------------------------------------------------------------------------------------------------------
@pytest.mark.slow
@pytest.mark.parametrize("B,dtype,tol", [(1, torch.float16, (3e-3, 3e-2)), (2, torch.float16, (3e-3, 3e-2)),
                                         (1, torch.bfloat16, (2.5e-2, 2.5e-1)), (2, torch.bfloat16, (2.5e-2, 2.5e-1))])
def test_lb_vit_engine_path_matches_fp32_library_path(lb, B, dtype, tol):
    net = lb.backbone.net
    assert net._flavour == "eva02_subln"
    img = torch.randn(B, 3, 1024, 1024, generator=torch.Generator().manual_seed(5)).to(DEV)
    assert net._engine_ok(img)
    want = net(img)["last_feat"]
    got = net(img.to(dtype))["last_feat"]
    assert got.dtype == dtype and got.shape == want.shape == (B, 1024, 64, 64)
    r = err(f"ViT-L eva02 B={B} {str(dtype)[6:]}", got, want)
    assert r["median_over_rms"] < tol[0] and r["max_over_rms"] < tol[1]


@pytest.mark.slow
def test_lb_backbone_runs_no_library_kernels(lb, monkeypatch):
    import ape_b200

    def forbidden(*a, **k):
        raise AssertionError("library kernel called on the APE-L_B engine path")

    for mod, name in ((F, "linear"), (F, "conv2d"), (F, "conv_transpose2d"), (F, "scaled_dot_product_attention"),
                      (torch, "matmul")):
        monkeypatch.setattr(mod, name, forbidden)
    img = torch.randn(1, 3, 1024, 1024, generator=torch.Generator().manual_seed(8)).to(DEV, torch.float16)
    n0 = ape_b200._lib.launch_count()
    feats = lb.backbone(img)
    torch.cuda.synchronize()
    assert sorted(feats) == ["p2", "p3", "p4", "p5", "p6"]
    assert ape_b200._lib.launch_count() - n0 > 24 * 8


@pytest.mark.slow
@pytest.mark.parametrize("B", [1, 2])
def test_lb_levels_are_views_of_the_encoder_input(lb, B):
    """No neck: p2..p6 share storage with the flat [B, S, 256] buffer, which matches the fp32 path's concatenated levels."""
    img = torch.randn(B, 3, 1024, 1024, generator=torch.Generator().manual_seed(6)).to(DEV)
    want = lb.backbone(img)
    assert lb.backbone.last_flat is None
    want_flat = torch.cat([want[k].flatten(2).transpose(1, 2) for k in ("p2", "p3", "p4", "p5", "p6")], 1)
    got = lb.backbone(img.half())
    flat = lb.backbone.last_flat
    assert flat is not None and flat.shape == want_flat.shape == (B, 256 * 256 + 128 * 128 + 64 * 64 + 32 * 32 + 16 * 16, 256)
    base = flat.untyped_storage().data_ptr()
    for k in ("p2", "p3", "p4", "p5", "p6"):
        assert got[k].untyped_storage().data_ptr() == base, f"{k} is a copy"
        assert got[k].shape == want[k].shape
    r = err(f"flat levels B={B} fp16", flat, want_flat)
    assert r["median_over_rms"] < TOL["float16"]["backbone"] and r["max_over_rms"] < 2e-2
    # p6 is p5 subsampled (LastLevelMaxPool: kernel 1, stride 2), bit for bit
    assert torch.equal(got["p6"], got["p5"][:, :, ::2, ::2])
    # the encoder consumes that buffer: the model's levels are the same views
    lb.engine_dtype = torch.float16
    try:
        lb([{"image": synth.image(1024, 768, seed=0), "height": 1024, "width": 768}] * B)
        feats = lb.last_outputs["neck"]
        assert len(feats) == 5 and all(f.untyped_storage().data_ptr() == lb.backbone.last_flat.untyped_storage().data_ptr()
                                       for f in feats)
    finally:
        lb.engine_dtype = torch.float32


# -- MINI_EVA02L against the reference -------------------------------------------------------------------------------------
def test_mini_lb_matches_reference_golden():
    model = _build(configs.MINI_EVA02L, suppress=False)
    g = load_golden("model_mini_lb.npz")
    model.test_mask_on, model.semantic_on = True, True
    out = model([{"image": synth.image(48, 64, seed=0), "height": 96, "width": 128}])
    lo = model.last_outputs
    tol = dict(rtol=2e-3, atol=2e-3)
    for k in ("p2", "p3", "p4", "p5", "p6"):
        err(f"backbone.{k}", lo["features"][k][:, ::4], g[f"backbone.{k}"])
        torch.testing.assert_close(lo["features"][k][:, ::4].cpu(), g[f"backbone.{k}"], **tol)
    err("memory", lo["memory"][:, ::4], g["memory"])
    torch.testing.assert_close(lo["memory"][:, ::4].cpu(), g["memory"], rtol=5e-3, atol=5e-3)
    sel, want = model.transformer.last_topk_proposals.cpu(), g["topk_proposals"]
    valid = torch.isfinite(g["init_reference"]).all(-1) & (g["init_reference"] < 1).all(-1)
    assert sel.shape == want.shape and torch.equal(sel[valid], want[valid])
    torch.testing.assert_close(lo["init_reference"].cpu(), g["init_reference"], **tol)
    torch.testing.assert_close(lo["inter_states"].cpu(), g["inter_states"], rtol=5e-3, atol=5e-3)
    torch.testing.assert_close(lo["inter_references"].cpu(), g["inter_references"], **tol)
    err("pred_masks", lo["pred_masks"], g["pred_masks"])
    torch.testing.assert_close(lo["pred_masks"].cpu(), g["pred_masks"], rtol=5e-3, atol=5e-3)
    inst = out[0]["instances"]
    assert torch.equal(inst.pred_classes, g["det0.classes"])  # kept (query, class) pairs
    torch.testing.assert_close(inst.scores, g["det0.scores"], rtol=1e-3, atol=1e-5)
    torch.testing.assert_close(inst.pred_boxes.tensor, g["det0.boxes"], rtol=1e-3, atol=2e-2)
    want_m = torch.from_numpy(np.unpackbits(g["det0.masks_packed"].numpy(), axis=-1)).bool()[..., : int(g["det0.masks_shape"][2])]
    assert inst.pred_masks.dtype == torch.bool and tuple(inst.pred_masks.shape) == tuple(want_m.shape)
    flips = (inst.pred_masks != want_m).float().mean().item()
    print(f"  instance mask pixels that differ: {flips:.2e}")
    assert flips < 2e-3
    err("sem_seg", out[0]["sem_seg"], g["sem_seg"])
    torch.testing.assert_close(out[0]["sem_seg"].cpu(), g["sem_seg"], rtol=2e-3, atol=2e-3)


# -- APE-L_B at 1024^2 against the reference -------------------------------------------------------------------------------
def _run(model, mode):
    dt = getattr(torch, mode)
    model.engine_dtype = dt
    model.use_cuda_graphs = dt != torch.float32
    model.transformer.encoder.record_taps = True
    try:
        inp = [{"image": synth.image(1024, 768, seed=0), "height": 1024, "width": 768}]
        out = model(inp)
        if model.use_cuda_graphs:  # second call = graph replay
            out = model(inp)
        lo = dict(model.last_outputs)
        lo["topk"] = model.transformer.last_topk_proposals.clone()
        lo["taps"] = {k: v.clone() for k, v in getattr(model.transformer.encoder, "taps", {}).items()}
        lo["pred_logits"] = lo["pred_logits"].clone()
        lo["features"] = {k: v.clone() for k, v in lo["features"].items()}
        return out, lo
    finally:
        model.engine_dtype, model.use_cuda_graphs = torch.float32, False
        model.transformer.encoder.record_taps = False


@pytest.mark.slow
@pytest.mark.parametrize("mode", ["float32", "float16", "bfloat16"])
def test_lb_1024_stagewise_vs_reference_golden(lb, mode):
    g = load_golden("model_lb_1024.npz")
    tol = TOL[mode]
    print(f"\n== APE-L_B 1024^2 / {N_TEXT} names, engine mode {mode}" + (" + CUDA graph replay" if mode != "float32" else ""))
    out, lo = _run(lb, mode)
    for k in ("p2", "p3", "p4", "p5", "p6"):
        r = err(f"backbone.{k}", lo["features"][k][:, ::16, ::8, ::8], g[f"backbone.{k}"])
        assert r["max_over_rms"] < tol["backbone"] * 5 and r["median_over_rms"] < tol["backbone"]
    for k, v in sorted(lo["taps"].items()):
        r = err(k, v[:, ::2048, ::4], g[k])
        assert r["max_over_rms"] < tol["encoder"] * 5 and r["median_over_rms"] < tol["encoder"]
    r = err("memory", lo["memory"][:, ::512, ::4], g["memory"])
    assert r["max_over_rms"] < tol["memory"] * 5 and r["median_over_rms"] < tol["memory"]
    sel, want = lo["topk"][0].cpu().tolist(), g["topk_proposals"][0].tolist()
    common = sorted(set(sel) & set(want))
    frac = len(common) / len(want)
    same_slot = sum(int(a == b) for a, b in zip(sel, want)) / len(want)
    print(f"  selected proposals: {len(common)}/{len(want)} in common ({frac:.4f}), {same_slot:.4f} at the same slot")
    assert frac > (0.99 if mode == "float32" else 0.95 if mode == "float16" else 0.9)
    ia = torch.tensor([sel.index(i) for i in common])
    ib = torch.tensor([want.index(i) for i in common])
    r = err("pred_logits (common q)", lo["pred_logits"][0][ia][:, ::32], g["pred_logits"][0][ib])
    assert r["max_over_rms"] < tol["logits"]
    r = err("pred_boxes (common q)", lo["pred_boxes"][0][ia], g["pred_boxes"][0][ib])
    assert r["max_over_rms"] < tol["boxes"]
    inst = out[0]["instances"]
    assert len(inst) == len(g["det0.scores"]) == 300
    k = 50
    torch.testing.assert_close(inst.scores[:k], g["det0.scores"][:k], rtol=1e-1 if mode != "float32" else 5e-3,
                               atol=2e-3 if mode != "float32" else 1e-4)
    want_classes = g["det0.classes"].tolist()
    agree = len(set(inst.pred_classes.tolist()) & set(want_classes)) / len(set(want_classes))
    top_agree = len(set(inst.pred_classes[:k].tolist()) & set(want_classes[:k])) / len(set(want_classes[:k]))
    print(f"  final detections (thresh 0.0, top-300): class-set agreement {agree:.3f} (top-{k}: {top_agree:.3f})")
    if mode == "float32":
        assert top_agree > 0.9 and agree > 0.9


@pytest.mark.slow
def test_lb_1024_graph_replay_equals_eager(lb):
    inp = [{"image": synth.image(1024, 768, seed=0), "height": 1024, "width": 768}]
    lb.engine_dtype = torch.float16
    try:
        eager = lb(inp)
        eager_logits = lb.last_outputs["pred_logits"].clone()
        lb.use_cuda_graphs = True
        for seed in (0, 3, 0):  # capture, then replays with a different image in between
            out = lb([{"image": synth.image(1024, 768, seed=seed), "height": 1024, "width": 768}])
        graph_logits = lb.last_outputs["pred_logits"].clone()
    finally:
        lb.engine_dtype, lb.use_cuda_graphs = torch.float32, False
    assert torch.equal(graph_logits, eager_logits), "CUDA graph replay differs from eager"
    assert torch.equal(out[0]["instances"].pred_classes, eager[0]["instances"].pred_classes)
    assert torch.equal(out[0]["instances"].scores, eager[0]["instances"].scores)
