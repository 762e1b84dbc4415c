"""GPU: APE-L_A on the engine — APE-L_B's backbone and neck-less feature path under the model classes without vision-language
fusion (DeformableDETRSegm over DeformableDetrTransformer), and its EVA01-CLIP text tower.

* MINI_L_A against tests/golden/model_mini_la.npz (reference files, CPU, fp32): identical selected proposal indices.
* APE-L_A at 1024^2, 1203 names against tests/golden/model_la_1024.npz, stage by stage in fp32, fp16 + graphs and
  bf16 + graphs (the bounds of tests/test_ape_l_b_gpu.py); graph replay equals eager bit for bit.
* The 16-bit encoder launches only libape_b200 kernels (torch.profiler), and its fused row-kernel schedule equals the
  layer-by-layer loop.
* EVA01CLIP's engine path in fp16 / bf16 against tests/golden/text_eva01.npz (the bounds of tests/test_text_gpu.py).
Weights: name-derived synthetic (oracle/synth.py); TF32 off.  Each comparison prints the errors it measured."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from ape_b200 import configs
from oracle import synth
from test_ape_l_b_gpu import TOL, _build, _run, err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
N_TEXT = 1203


@pytest.fixture(scope="module")
def la():
    return _build(configs.APE_L_A, num_text=N_TEXT)


# -- MINI_L_A against the reference -----------------------------------------------------------------------------------------
def test_mini_la_matches_reference_golden():
    model = _build(configs.MINI_L_A, suppress=False)
    g = load_golden("model_mini_la.npz")
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
    assert sel.shape == want.shape and valid.any() and torch.equal(sel[valid], want[valid])
    torch.testing.assert_close(lo["init_reference"].cpu(), g["init_reference"], **tol)
    torch.testing.assert_close(lo["inter_states"].cpu(), g["inter_states"], rtol=5e-3, atol=5e-3)
    torch.testing.assert_close(lo["inter_references"].cpu(), g["inter_references"], **tol)
    err("pred_masks", lo["pred_masks"], g["pred_masks"])
    torch.testing.assert_close(lo["pred_masks"].cpu(), g["pred_masks"], rtol=5e-3, atol=5e-3)
    inst = out[0]["instances"]
    assert torch.equal(inst.pred_classes, g["det0.classes"])
    torch.testing.assert_close(inst.scores, g["det0.scores"], rtol=1e-3, atol=1e-5)
    torch.testing.assert_close(inst.pred_boxes.tensor, g["det0.boxes"], rtol=1e-3, atol=2e-2)
    want_m = torch.from_numpy(np.unpackbits(g["det0.masks_packed"].numpy(), axis=-1)).bool()[..., : int(g["det0.masks_shape"][2])]
    assert inst.pred_masks.dtype == torch.bool and tuple(inst.pred_masks.shape) == tuple(want_m.shape)
    flips = (inst.pred_masks != want_m).float().mean().item()
    print(f"  instance mask pixels that differ: {flips:.2e}")
    assert flips < 2e-3
    err("sem_seg", out[0]["sem_seg"], g["sem_seg"])
    torch.testing.assert_close(out[0]["sem_seg"].cpu(), g["sem_seg"], rtol=2e-3, atol=2e-3)


# -- APE-L_A at 1024^2 against the reference -------------------------------------------------------------------------------
@pytest.mark.slow
@pytest.mark.parametrize("mode", ["float32", "float16", "bfloat16"])
def test_la_1024_stagewise_vs_reference_golden(la, mode):
    g = load_golden("model_la_1024.npz")
    tol = TOL[mode]
    print(f"\n== APE-L_A 1024^2 / {N_TEXT} names, engine mode {mode}" + (" + CUDA graph replay" if mode != "float32" else ""))
    out, lo = _run(la, mode)
    if mode != "float32":  # the fusion-free model is captured for "name" prompts too
        assert any(k[0][0] == "forward" for k in la._graph_cache)
    for k in ("p2", "p3", "p4", "p5", "p6"):
        r = err(f"backbone.{k}", lo["features"][k][:, ::16, ::8, ::8], g[f"backbone.{k}"])
        assert r["max_over_rms"] < tol["backbone"] * 5 and r["median_over_rms"] < tol["backbone"]
    assert sorted(lo["taps"]) == [f"enc{i}" for i in range(6)]
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
def test_la_1024_graph_replay_equals_eager(la):
    inp = [{"image": synth.image(1024, 768, seed=0), "height": 1024, "width": 768}]
    la.engine_dtype = torch.float16
    try:
        eager = la(inp)
        eager_logits = la.last_outputs["pred_logits"].clone()
        la.use_cuda_graphs = True
        for seed in (0, 3, 0):  # capture, then replays with a different image in between
            out = la([{"image": synth.image(1024, 768, seed=seed), "height": 1024, "width": 768}])
        graph_logits = la.last_outputs["pred_logits"].clone()
    finally:
        la.engine_dtype, la.use_cuda_graphs = torch.float32, False
    assert torch.equal(graph_logits, eager_logits), "CUDA graph replay differs from eager"
    assert torch.equal(out[0]["instances"].pred_classes, eager[0]["instances"].pred_classes)
    assert torch.equal(out[0]["instances"].scores, eager[0]["instances"].scores)


def _encoder_inputs(model, dt, seed=7):
    """The encoder's inputs for an unpadded 1024^2 image (stage_encode's call), in the engine dtype."""
    tr = model.transformer
    shapes = configs.level_shapes(configs.APE_L_A)
    g = torch.Generator().manual_seed(seed)
    S = sum(h * w for h, w in shapes)
    feat = torch.randn(1, S, 256, generator=g).to(DEV, dt)
    masks = [torch.zeros(1, h, w, dtype=torch.bool, device=DEV) for h, w in shapes]
    pos = [torch.randn(1, 256, h, w, generator=g).to(DEV) for h, w in shapes]
    geo = tr.geometry(shapes, masks, pos)
    kw = dict(query_key_padding_mask=None, spatial_shapes=geo["spatial_shapes"], reference_points=geo["reference_points"],
              level_start_index=geo["level_start_index"], valid_ratios=geo["valid_ratios"], host_shapes=geo["shapes"])
    return feat, geo["pos_flatten"].to(dt).contiguous(), kw


@pytest.mark.slow
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_la_encoder_schedule_equals_layer_loop_and_runs_no_library_kernels(la, dtype):
    """The 16-bit encoder: every layer's last norm fused with the next layer's `query + pos`, the first layer's sum from the
    same row kernel, against the plain loop over the layers (the norm and the add unfused); and a profiler run of the
    schedule that lists only the engine's kernels.  Unpadded input: with padding, the value projection's masked_fill
    (multi_scale_deform_attn.py) is a library kernel, in the VL encoder as well."""
    import ape_b200

    enc = la.transformer.encoder
    feat, pos, kw = _encoder_inputs(la, dtype)
    with torch.no_grad(), torch.autocast("cuda", dtype=dtype):
        got = enc(feat, None, None, query_pos=pos, **kw)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            n0 = ape_b200._lib.launch_count()
            again = enc(feat, None, None, query_pos=pos, **kw)
            torch.cuda.synchronize()
            launched = ape_b200._lib.launch_count() - n0
    want = feat
    with torch.no_grad():
        for layer in enc.layers:  # the generic loop: each layer normalises its own output, MSDA adds query + pos
            want = layer(want, pos, None, kw["reference_points"], kw["spatial_shapes"], kw["level_start_index"], kw["host_shapes"])
    assert got.dtype == dtype and got.shape == feat.shape
    assert torch.equal(again, got)
    # same functions in the same precision; only the LayerNorm kernels' summation order differs
    r = err(f"encoder schedule vs loop {str(dtype)[6:]}", got, want)
    tol = TOL[str(dtype)[6:]]["encoder"]
    assert r["median_over_rms"] < tol and r["max_over_rms"] < 5 * tol
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    print(f"  {len(names)} kernels, {launched} launched by libape_b200")
    assert names and launched > 0
    library = [n for n in names if "ape::" not in n]
    assert not library, sorted(set(library))[:5]
    assert sum("layernorm_ex_kernel" in n for n in names) == 6  # first layer's sum + five fused norms


# -- EVA01-CLIP text tower --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_eva01_engine_matches_reference_golden(dtype):
    from ape_b200.modeling import EVA01CLIP

    g = load_golden("text_eva01.npz")
    clip = EVA01CLIP("EVA_CLIP_g_14_X", cache_dir=None, dtype=dtype)
    synth.fill_state_dict(clip.net.text)
    clip = clip.to(DEV)
    out = clip.forward_text(g["tokens"])
    eot, xx = out["last_hidden_state_eot"].float().cpu(), out["last_hidden_state"].float().cpu()
    rms = g["eot"].pow(2).mean().sqrt().item()
    e = (eot - g["eot"]).abs().max().item()
    print(f"EVA01 text tower {dtype} engine vs reference golden: max|err| {e:.3e} on rms {rms:.3e}")
    tol = 4e-3 if dtype == "float16" else 3e-2  # test_text_gpu.py's bounds at the bigE geometry
    assert e < tol * max(rms, 1.0)
    ends = out["end_token_idx"].cpu()
    keep = (torch.arange(77)[None] <= ends[:, None])[:, ::7]  # positions after the end-of-text token are unconstrained padding
    assert ((xx[:, ::7] - g["all"]).abs() * keep[..., None]).max().item() < tol * max(rms, 1.0)
