"""GPU: the APE-Ti backbone (vit_eva02.py: fused qkv, packed SwiGLU, 14x14 windows over a grid they need not tile) and its
feature pyramid on the engine's kernels, against the fp32 library path of the same modules; the row-mapped attention
output those windows use (ape_attn_fwd_mapped) against a torch reference."""
import copy

import pytest
import torch
import torch.nn.functional as F

from ape_b200 import configs
from oracle import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _build(img_size=1024):
    from ape_b200.modeling import build_model

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    spec = copy.deepcopy(configs.APE_TI)
    spec["backbone"].update(img_size=img_size, square_pad=img_size)
    m = build_model(spec, num_text=80)
    synth.fill_state_dict(m)
    return m.to(DEV)


@pytest.fixture(scope="module")
def ti():
    return _build()


def _window_maps(B, g, ws):
    """raster row -> padded window-major row (window_partition order), and its inverse with -1 on pad rows."""
    nw = -(-g // ws)
    b, y, x = torch.meshgrid(torch.arange(B), torch.arange(g), torch.arange(g), indexing="ij")
    row = (((b * nw + y // ws) * nw + x // ws) * (ws * ws) + (y % ws) * ws + x % ws).reshape(-1)
    inv = torch.full((B * nw * nw * ws * ws,), -1, dtype=torch.int32)
    inv[row] = torch.arange(B * g * g, dtype=torch.int32)
    return row, inv, B * nw * nw


@pytest.fixture(params=[0, 1], ids=["smemP", "regP"])
def variant(request):
    import ape_b200

    prev = ape_b200._lib.lib.ape_attn_variant(-1)
    ape_b200._lib.lib.ape_attn_variant(request.param)
    yield request.param
    ape_b200._lib.lib.ape_attn_variant(prev)


@pytest.mark.parametrize("dtype,tol", [(torch.float16, 2e-3), (torch.bfloat16, 1.6e-2)])
def test_row_mapped_attention_matches_reference(variant, dtype, tol):
    """Padded 14x14 windows over a 20x20 grid (4 windows per image, 2 images): each window is a 196-row sequence at a
    196-row stride inside 256-row kernel tiles; query rows come back in raster order, pad rows are not stored."""
    from ape_b200 import ops

    B, g, ws, heads, hd = 2, 20, 14, 3, 64
    C = heads * hd
    row, inv, nwin = _window_maps(B, g, ws)
    qkv = torch.randn(nwin * ws * ws, 3 * C, generator=torch.Generator().manual_seed(7)).to(DEV, dtype)
    canary = 7.0
    extra = 8  # canary rows before and after `out`, and rows of `out` no query maps to
    buf = torch.full((B * g * g + 3 * extra, C), canary, dtype=dtype, device=DEV)
    out = buf[extra:-extra]
    got, st = ops.attention_qkv(qkv, nwin, 256, heads, hd, hd ** -0.5, n_valid=ws * ws, seq_stride=ws * ws,
                                out_row_map=inv.to(DEV), out=out, stats_out=True)
    assert got is out and st.shape == (out.shape[0], heads, 2)
    q, k, v = qkv.float().view(nwin, ws * ws, 3, heads, hd).permute(2, 0, 3, 1, 4)
    want = (torch.softmax(q @ k.transpose(-1, -2) * hd ** -0.5, -1) @ v).permute(0, 2, 1, 3).reshape(-1, C)
    torch.testing.assert_close(out[: B * g * g].float(), want[row.to(DEV)], rtol=tol, atol=tol)
    assert (buf[:extra] == canary).all() and (buf[extra + B * g * g:] == canary).all(), \
        "a row mapped to -1 (a pad token) was written"
    o = out[: B * g * g].float().view(-1, heads, hd)
    torch.testing.assert_close(st[: B * g * g, :, 0], o.sum(-1), rtol=1e-5, atol=1e-4)
    torch.testing.assert_close(st[: B * g * g, :, 1], (o ** 2).sum(-1), rtol=1e-5, atol=1e-4)


def test_row_mapped_attention_rejects_bad_arguments():
    import ape_b200
    from ape_b200 import ops

    C = 3 * 64
    qkv = torch.zeros(4 * 196, 3 * C, dtype=torch.float16, device=DEV)
    good_map = torch.arange(4 * 196, dtype=torch.int32, device=DEV)
    out = torch.zeros(4 * 196, C, dtype=torch.float16, device=DEV)
    kw = dict(n_valid=196, seq_stride=196)
    ok = ops.attention_qkv(qkv, 4, 256, 3, 64, 0.125, out_row_map=good_map, out=out, **kw)
    assert ok is out
    bad = [
        dict(out_row_map=good_map.long(), out=out),                           # int64 map
        dict(out_row_map=good_map[:-1], out=out),                             # one entry short
        dict(out_row_map=good_map.cpu(), out=out),                            # host memory
        dict(out_row_map=good_map),                                           # no destination
        dict(out_row_map=good_map, out=out.float()),                          # wrong output dtype
        dict(out_row_map=good_map, out=out[:, :128]),                         # wrong width
        dict(out=out),                                                        # `out` without a map
    ]
    for b in bad:
        with pytest.raises(RuntimeError):
            ops.attention_qkv(qkv, 4, 256, 3, 64, 0.125, **kw, **b)
    lib = ape_b200._lib.lib
    rc = lib.ape_attn_fwd_mapped(qkv.data_ptr(), 3 * C, out.data_ptr(), C, 4, 256, 196, 3, 64, 0.125, 1, None, 196, 0,
                                 qkv.shape[0], None, None)
    assert rc == -3 and b"out_row_map" in lib.ape_last_error()
    rc = lib.ape_attn_fwd_mapped(qkv.data_ptr(), 3 * C, out.data_ptr(), C, 4, 200, 196, 3, 64, 0.125, 1, None, 196, 0,
                                 qkv.shape[0], good_map.data_ptr(), None)
    assert rc == -2  # n must be a multiple of 128


@pytest.mark.parametrize("img_size,B,dtype,tol", [
    (1024, 1, torch.float16, 5e-2),   # 64x64 grid: 14x14 windows over the 70x70 padded grid
    (1024, 2, torch.float16, 5e-2),
    (448, 1, torch.float16, 5e-2),    # 28x28 grid: the windows tile it exactly
    (1024, 1, torch.bfloat16, 2e-1),
])
def test_ti_vit_engine_path_matches_fp32_library_path(ti, img_size, B, dtype, tol):
    """The APE-Ti ViT on the engine (raster-order fp32 residual stream, padded windows by row maps) against the fp32
    library path of the same module (which test_ape_ti_1024_matches_reference_golden pins to the reference)."""
    net = (ti if img_size == 1024 else _build(img_size)).backbone.net
    img = torch.randn(B, 3, img_size, img_size, generator=torch.Generator().manual_seed(5)).to(DEV)
    assert net._engine_ok(img)
    want = net(img)["last_feat"]
    got = net(img.to(dtype))["last_feat"]
    assert got.dtype == dtype and got.shape == want.shape
    err = (got.float() - want).abs().max().item()
    print(f"APE-Ti ViT {img_size}^2 B={B} {dtype}: max|err| {err:.3e} on max|ref| {want.abs().max().item():.3e}")
    torch.testing.assert_close(got.float(), want, rtol=tol, atol=tol)


def test_ti_pyramid_and_neck_engine_paths_match_fp32_library_path(ti):
    """SimpleFeaturePyramid at Ti's widths (192 -> 96 -> 48 channels, 1x1 GEMMs with K = 48 / 96) + ChannelMapper."""
    img = torch.randn(1, 3, 1024, 1024, generator=torch.Generator().manual_seed(6)).to(DEV)
    want = ti.backbone(img)
    want_neck = ti.neck(want)
    got = ti.backbone(img.half())
    got_neck = ti.neck(got)
    for k in want:
        assert got[k].shape == want[k].shape
        err = (got[k].float() - want[k]).abs().max().item()
        print(f"APE-Ti pyramid {k}: max|err| {err:.3e}")
        torch.testing.assert_close(got[k].float(), want[k], rtol=5e-2, atol=5e-2)
    for a, b in zip(got_neck, want_neck):
        torch.testing.assert_close(a.float(), b, rtol=5e-2, atol=5e-2)


def test_ti_backbone_runs_no_library_kernels(ti, monkeypatch):
    """The 16-bit APE-Ti backbone + pyramid launch the engine's kernels only: no cuBLAS linear / matmul, no cuDNN
    convolution, no PyTorch SDPA."""
    import ape_b200

    def forbidden(*a, **k):
        raise AssertionError("library kernel called on the APE-Ti engine path")

    for mod, name in ((F, "linear"), (F, "conv2d"), (F, "conv_transpose2d"), (F, "scaled_dot_product_attention"),
                      (torch, "matmul")):
        monkeypatch.setattr(mod, name, forbidden)
    img = torch.randn(1, 3, 1024, 1024, generator=torch.Generator().manual_seed(8)).to(DEV, torch.float16)
    n0 = ape_b200._lib.launch_count()
    feats = ti.backbone(img)
    torch.cuda.synchronize()
    assert sorted(feats) == ["p2", "p3", "p4", "p5", "p6"]
    assert ape_b200._lib.launch_count() - n0 > 12 * 8


@pytest.mark.slow
def test_ape_ti_1024_fp16_graphs_close_to_fp32():
    """Whole APE-Ti at 1024^2, 80 names: fp16 engine mode with CUDA graphs against the fp32 run of the same model (which
    test_ape_ti_1024_matches_reference_golden pins to the reference); graph replay equals eager bit for bit."""
    model = _build()
    inp = [{"image": synth.image(768, 1024, seed=11), "height": 384, "width": 512}]
    ref = model(inp)
    ref_feats = {k: v.float().clone() for k, v in model.last_outputs["features"].items()}
    ref_sel = model.transformer.last_topk_proposals[0].tolist()
    model.engine_dtype = torch.float16
    try:
        eager = model(inp)
        eager_logits = model.last_outputs["pred_logits"].clone()
        feats = {k: v.float().clone() for k, v in model.last_outputs["features"].items()}
        sel = model.transformer.last_topk_proposals[0].tolist()
        model.use_cuda_graphs = True
        for seed in (11, 12, 11):  # capture, then replays with a different image in between
            out = model([{"image": synth.image(768, 1024, seed=seed), "height": 384, "width": 512}])
        graph_logits = model.last_outputs["pred_logits"].clone()
    finally:
        model.engine_dtype, model.use_cuda_graphs = torch.float32, False
    assert torch.equal(graph_logits, eager_logits), "CUDA graph replay differs from eager"
    assert torch.equal(out[0]["instances"].pred_classes, eager[0]["instances"].pred_classes)
    for k in ("p2", "p3", "p4", "p5", "p6"):
        err = (feats[k] - ref_feats[k]).abs().max().item()
        print(f"APE-Ti {k} fp16 engine vs fp32: max|err| {err:.3e}")
        torch.testing.assert_close(feats[k], ref_feats[k], rtol=5e-2, atol=5e-2)
    frac = len(set(sel) & set(ref_sel)) / len(ref_sel)
    print(f"APE-Ti fp16 vs fp32 proposal set agreement: {frac:.4f}")
    assert frac > 0.85
    gi, ri = eager[0]["instances"], ref[0]["instances"]
    assert abs(len(gi) - len(ri)) <= max(3, len(ri) // 10)
    k = min(20, len(gi), len(ri))
    print(f"APE-Ti top-{k} scores fp16 vs fp32: max|diff| {(gi.scores[:k] - ri.scores[:k]).abs().max().item():.3e}")
    torch.testing.assert_close(gi.scores[:k], ri.scores[:k], rtol=2e-2, atol=1e-3)
