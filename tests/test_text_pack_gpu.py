"""GPU: the text tower's length-packed mode (`pack_prompts=True`: prompts laid back to back in 128-row tiles, segment-causal
attention, packed embedding, end-of-text readout) against the padded engine path and against the goldens recorded from the
reference's text towers, with the bounds tests/test_text_gpu.py and tests/test_ape_l_a_gpu.py hold the padded path to.
Synthetic name-derived weights (oracle/synth.py)."""
import pytest
import torch

from conftest import load_golden
from oracle import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CTX = 77
TOL = {"float16": 4e-3, "bfloat16": 3e-2}  # of max(rms, 1): the padded engine path's bounds against fp32


def _tokens(lengths, vocab, seed=0):
    """int64 [N, 77]: start token, random words, the end-of-text token (the largest id) at lengths[i] - 1, zeros after it."""
    g = torch.Generator().manual_seed(seed)
    tok = torch.zeros(len(lengths), CTX, dtype=torch.int64)
    for i, n in enumerate(lengths):
        tok[i, :n] = torch.randint(1, vocab - 2, (n,), generator=g)
        tok[i, 0], tok[i, n - 1] = vocab - 2, vocab - 1
    return tok


def _lengths(kind, seed=0):
    g = torch.Generator().manual_seed(seed)
    if kind == "short":
        return torch.randint(3, 9, (150,), generator=g).tolist()
    if kind == "full":
        return [CTX] * 5
    if kind == "mixed":
        return torch.randint(2, CTX + 1, (60,), generator=g).tolist()
    return [6]  # "one"


def _tower(kind, dtype, **kw):
    from ape_b200.modeling import EVA01CLIP, EVA02CLIP

    if kind == "eva02":  # EVA02-CLIP-bigE width and heads, two layers
        clip = EVA02CLIP(dtype=dtype, text_cfg=dict(context_length=CTX, vocab_size=2000, width=1280, heads=20, layers=2),
                         embed_dim=1024, **kw)
    else:                # EVA01-CLIP width and heads, two layers
        clip = EVA01CLIP(cache_dir=None, dtype=dtype, text_cfg=dict(context_length=CTX, vocab_size=2000, width=768, heads=12, layers=2),
                         embed_dim=1024, **kw)
    synth.fill_state_dict(clip.net.text)
    return clip.to(DEV)


def _compare(packed, padded, tokens, tol, what):
    end = tokens.argmax(-1).to(DEV)
    assert torch.equal(packed["end_token_idx"], padded["end_token_idx"]) and torch.equal(packed["end_token_idx"], end)
    assert torch.equal(packed["attention_mask"], padded["attention_mask"])
    a, b = packed["last_hidden_state_eot"], padded["last_hidden_state_eot"]
    assert a.shape == b.shape and a.dtype == b.dtype
    scale = max(b.pow(2).mean().sqrt().item(), 1.0)
    e = (a - b).abs().max().item()
    keep = torch.arange(CTX, device=DEV)[None] <= end[:, None]
    ha, hb = packed["last_hidden_state"], padded["last_hidden_state"]
    assert ha.shape == hb.shape and ha.dtype == hb.dtype
    eh = ((ha - hb).abs() * keep[..., None]).max().item()
    print(f"  {what}: packed vs padded engine path max|diff| {e:.3e} (end of text), {eh:.3e} (every valid token), scale {scale:.3f}")
    assert e < tol * scale and eh < tol * scale
    assert not ha[~keep].any()  # zeros after the end-of-text token
    assert torch.equal(ha[torch.arange(len(end), device=DEV), end], a)


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
@pytest.mark.parametrize("tower", ["eva02", "eva01"])
@pytest.mark.parametrize("prompts", ["short", "full", "mixed", "one"])
def test_packed_matches_padded_and_literal(tower, dtype, prompts):
    import ape_b200

    clip = _tower(tower, dtype)
    tokens = _tokens(_lengths(prompts, seed=3), 2000, seed=len(prompts))
    padded = clip.forward_text(tokens)
    clip.pack_prompts = True
    n0 = ape_b200._lib.launch_count()
    packed = clip.forward_text(tokens)
    launched = ape_b200._lib.launch_count() - n0
    assert launched >= 2 * 7 + 2  # 7 kernels per block and the readout; nothing but the attention differs when the chunk runs padded
    _compare(packed, padded, tokens, TOL[dtype], f"{tower} {dtype} {prompts}")
    lean = clip.forward_text(tokens, need_hidden=False)
    assert lean["last_hidden_state"] is None and torch.equal(lean["last_hidden_state_eot"], packed["last_hidden_state_eot"])
    # against the fp32 literal path of the same module
    clip.pack_prompts, clip.net.text.engine_dtype = False, None
    want = clip.forward_text(tokens)["last_hidden_state_eot"]
    scale = max(want.pow(2).mean().sqrt().item(), 1.0)
    e = (packed["last_hidden_state_eot"] - want).abs().max().item()
    print(f"  {tower} {dtype} {prompts}: packed vs literal fp32 max|err| {e:.3e}, scale {scale:.3f}")
    assert e < TOL[dtype] * scale


def test_long_prompts_run_padded_and_short_ones_packed():
    """The row count decides per chunk: 77-token prompts (128 rows each packed, 80 padded) and a single prompt take the padded
    layout, whose launches the mode then repeats; lists of short prompts take the packed kernels."""
    import ape_b200

    clip = _tower("eva01", "float16", pack_prompts=True)
    counts = {}
    for kind in ("full", "one", "short"):
        tokens = _tokens(_lengths(kind, seed=3), 2000, seed=2)
        n0 = ape_b200._lib.launch_count()
        clip.forward_text(tokens, need_hidden=False)
        counts[kind] = ape_b200._lib.launch_count() - n0
    assert counts["full"] == counts["one"] == 2 * 7 + 2   # blocks, ln_final, projection
    assert counts["short"] == 1 + 2 * 7 + 3               # + packed embedding and the end-of-text gather


def test_packed_chunks_by_max_batch_size():
    """N that crosses max_batch_size: each chunk is packed on its own; rows do not depend on their neighbours in a launch except
    through the attention's key-block partition, so the chunked result stays within the same bound of the unchunked one."""
    lengths = _lengths("short", seed=8)[:70]
    tokens = _tokens(lengths, 2000, seed=8)
    whole = _tower("eva01", "float16", pack_prompts=True)
    a = whole.forward_text(tokens)
    whole.max_batch_size = 32  # 70 prompts: chunks of 32, 32, 6
    b = whole.forward_text(tokens)
    _compare(b, a, tokens, TOL["float16"], "chunks of 32 vs one chunk")
    whole.pack_prompts = False
    _compare(b, whole.forward_text(tokens), tokens, TOL["float16"], "chunks of 32 vs padded")


def test_flag_off_is_the_padded_path_unchanged():
    """pack_prompts=False: the launches and the bits of the engine path as it was — restated here from the module sequence
    of the padded layout (stride 80, causal attention with n_valid = 77) — and of the fp32 literal path."""
    from ape_b200 import ops

    clip = _tower("eva01", "float16")
    assert clip.pack_prompts is False
    tokens = _tokens(_lengths("mixed", seed=1)[:9], 2000, seed=1).to(DEV)
    got = clip.forward_text(tokens)
    m, dt = clip.net.text, torch.float16
    N, L, D, stride = tokens.shape[0], CTX, m.width, 80
    with torch.no_grad():
        xs = torch.zeros((N, stride, D), dtype=torch.float32, device=DEV)
        xs[:, :L] = (m.token_embedding(tokens) + m.positional_embedding).float()
        x = xs.view(N * stride, D)
        for blk in m.transformer.resblocks:
            h = ops.layernorm_module(blk.ln_1, x, out_dtype=dt)
            qkv = ops.linear_tc(h, blk.attn.in_proj_weight.to(dt), blk.attn.in_proj_bias.float())
            o = ops.attention_qkv(qkv, N, 128, m.heads, 64, 0.125, n_valid=L, seq_stride=stride, causal=True)
            x = ops.linear_module_tc(blk.attn.out_proj, o, residual=x, out_dtype=torch.float32)
            u = ops.linear_module_tc(blk.mlp.c_fc, ops.layernorm_module(blk.ln_2, x, out_dtype=dt), act="gelu")
            x = ops.linear_module_tc(blk.mlp.c_proj, u, residual=x, out_dtype=torch.float32)
        xn = ops.layernorm_module(m.ln_final, x, out_dtype=dt)
        xx = ops.linear_tc(xn, m.text_projection.t().to(dt).contiguous(), None, out_dtype=torch.float32).view(N, stride, -1)[:, :L]
    assert torch.equal(got["last_hidden_state"], xx)
    assert torch.equal(got["last_hidden_state_eot"], xx[torch.arange(N, device=DEV), tokens.argmax(-1)])


def test_packed_small_tower_matches_reference_golden(dtype=torch.float16):
    """tests/golden/text_tower_small.npz (the reference's TextTransformer, fp32), bound of tests/test_text_gpu.py (fp16)."""
    from ape_b200.modeling.text import TextTransformer

    g = load_golden("text_tower_small.npz")
    m = TextTransformer(context_length=77, vocab_size=1000, width=128, heads=2, layers=3, output_dim=64).eval()
    synth.fill_state_dict(m)
    m = m.to(DEV)
    m.engine_dtype, m.pack_prompts = dtype, True
    with torch.no_grad():
        eot, xx = m.encode(g["tokens"].to(DEV))
    rms = g["eot"].pow(2).mean().sqrt().item()
    err = (eot.cpu() - g["eot"]).abs().max().item()
    print(f"  packed text tower {dtype} vs reference golden: max|err| {err:.3e} on rms {rms:.3e}")
    bound = 5e-3 * max(rms, 1e-3) + 1e-4
    assert err < bound
    keep = (torch.arange(77)[None] <= g["tokens"].argmax(-1)[:, None])[:, ::7]
    assert ((xx.cpu()[:, ::7] - g["all"]).abs() * keep[..., None]).max().item() < bound


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_packed_eva01_matches_reference_golden(dtype):
    """tests/golden/text_eva01.npz (the reference's EVA01-CLIP text tower at full size), bounds of tests/test_ape_l_a_gpu.py."""
    from ape_b200.modeling import EVA01CLIP

    g = load_golden("text_eva01.npz")
    clip = EVA01CLIP("EVA_CLIP_g_14_X", cache_dir=None, dtype=dtype, pack_prompts=True)
    synth.fill_state_dict(clip.net.text)
    clip = clip.to(DEV)
    out = clip.forward_text(g["tokens"])
    eot, xx = out["last_hidden_state_eot"].float().cpu(), out["last_hidden_state"].float().cpu()
    rms = g["eot"].pow(2).mean().sqrt().item()
    e = (eot - g["eot"]).abs().max().item()
    print(f"  packed EVA01 text tower {dtype} vs reference golden: max|err| {e:.3e} on rms {rms:.3e}")
    assert e < TOL[dtype] * max(rms, 1.0)
    keep = (torch.arange(77)[None] <= out["end_token_idx"].cpu()[:, None])[:, ::7]
    assert ((xx[:, ::7] - g["all"]).abs() * keep[..., None]).max().item() < TOL[dtype] * max(rms, 1.0)


def test_model_keeps_the_same_detections_with_packed_prompts():
    """An APE-L_D MINI forward with a `text_prompt` of phrases through a text tower with 64-channel heads: the same kept
    (query, class) pairs with the mode on and off."""
    from ape_b200 import configs
    from ape_b200.modeling import EVA02CLIP, build_model

    def tokenizer(texts):  # stand-in: one token per word, ids from the characters
        tok = torch.zeros(len(texts), CTX, dtype=torch.int64)
        for i, t in enumerate(texts):
            ids = [498] + [1 + sum(map(ord, w)) % 490 for w in t.split()][: CTX - 2] + [499]
            tok[i, : len(ids)] = torch.tensor(ids)
        return tok

    spec = configs.MINI
    model = build_model(spec)
    synth.fill_state_dict(model)
    clip = EVA02CLIP(dtype="float16", tokenizer=tokenizer, embed_dim=spec["lang_dim"],
                     text_cfg=dict(context_length=CTX, vocab_size=500, width=128, heads=2, layers=2))
    synth.fill_state_dict(clip.net.text)
    model, clip = model.to(DEV), clip.to(DEV)
    model.set_model_language(clip)
    inp = {"image": synth.image(64, 56, seed=0), "height": 128, "width": 112, "prompt": "text",
           "text_prompt": "the red apple on the left, a dog, two people walking, a small white boat on the water, "
                          "a man riding a brown horse, the tallest tree, green traffic light, a cup of coffee on a wooden table, "
                          "an open laptop, the child in the yellow raincoat, parked cars, a bird in flight over the sea, "
                          "the second window from the right, a stack of old books"}  # 14 phrases, 95 tokens: both key blocks
    outs = {}
    for on in (False, True):
        clip.pack_prompts = on
        inst = model([dict(inp)])[0]["instances"]
        outs[on] = (inst.pred_classes.clone(), inst.scores.clone(), inst.pred_boxes.tensor.clone(), model.last_outputs["pred_logits"].clone())
    assert len(outs[True][0]) > 0 and torch.equal(outs[True][0], outs[False][0])
    torch.testing.assert_close(outs[True][1], outs[False][1], rtol=2e-2, atol=1e-4)
    torch.testing.assert_close(outs[True][2], outs[False][2], rtol=1e-2, atol=0.5)
    print(f"  MINI phrase forward: {len(outs[True][0])} detections, max|logit diff| {(outs[True][3] - outs[False][3]).abs().max().item():.3e}")
