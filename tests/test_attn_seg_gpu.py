"""GPU: segment-causal flash attention (ape_attn_fwd_seg) — 128-row tiles that hold several short sequences each, as the text
tower's length-packed mode lays its prompts out — against an fp32 PyTorch reference with the explicit block-diagonal causal
mask on the same 16-bit inputs; and the packed embedding / row gather kernels of that mode against indexing."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TILE, HD = 128, 64


@pytest.fixture(scope="module", params=[0, 1], ids=["smemP", "regP"])
def ops(request):
    """Both structures of the attention kernel (ape_attn_variant): P read by the P.V MMA from shared memory or from registers."""
    import ape_b200

    prev = ape_b200._lib.lib.ape_attn_variant(-1)
    ape_b200._lib.lib.ape_attn_variant(request.param)
    yield ape_b200.ops
    ape_b200._lib.lib.ape_attn_variant(prev)


def _segments(kind, T, seed):
    """seg_start [T * 128] int32 (row, within the tile, where the row's segment starts) and the pad-row mask."""
    g = torch.Generator().manual_seed(seed)
    seg = torch.arange(TILE).repeat(T, 1)  # every row its own segment: what a pad row carries
    pad = torch.zeros(T, TILE, dtype=torch.bool)
    for t in range(T):
        if kind == "one":
            lens = [TILE]
        elif kind == "rows":
            lens = [1] * TILE
        elif kind == "mixed":  # segments of 1..77 rows up to the end of the tile
            lens, left = [], TILE
            while left:
                lens.append(min(left, int(torch.randint(1, 78, (1,), generator=g))))
                left -= lens[-1]
        else:  # "tails": short segments, then pad rows (up to a whole half tile of them)
            fill = int(torch.randint(2, TILE - 1, (1,), generator=g))
            lens, left = [], fill
            while left:
                lens.append(min(left, int(torch.randint(2, 17, (1,), generator=g))))
                left -= lens[-1]
            pad[t, fill:] = True
        r = 0
        for n in lens:
            seg[t, r:r + n] = r
            r += n
    return seg.reshape(-1).to(torch.int32), pad.reshape(-1)


def _reference(qkv, seg, T, heads, scale):
    q, k, v = qkv.float().view(T, TILE, 3, heads, HD).permute(2, 0, 3, 1, 4)  # [3][t, h, 128, d]
    r = torch.arange(TILE, device=qkv.device)
    lo = seg.view(T, TILE).to(qkv.device).long()
    allow = (r[None, None, :] <= r[None, :, None]) & (r[None, None, :] >= lo[:, :, None])  # [t, query, key]
    s = (q @ k.transpose(-1, -2) * scale).masked_fill(~allow[:, None], float("-inf"))
    return (torch.softmax(s, dim=-1) @ v).permute(0, 2, 1, 3).reshape(T * TILE, heads * HD)


@pytest.mark.parametrize("dtype,tol", [(torch.float16, 2e-3), (torch.bfloat16, 1.6e-2)])
@pytest.mark.parametrize("kind", ["one", "rows", "mixed", "tails"])
@pytest.mark.parametrize("T,heads", [(1, 12), (3, 20), (64, 12), (17, 20)])
def test_segment_causal_matches_fp32_reference(ops, dtype, tol, kind, T, heads):
    g = torch.Generator().manual_seed(T * 31 + heads)
    qkv = torch.randn(T * TILE, 3 * heads * HD, generator=g).to(DEV, dtype)
    seg, pad = _segments(kind, T, seed=T + heads)
    got = ops.attention_qkv(qkv, T, TILE, heads, HD, 0.125, causal=True, seg_start=seg.to(DEV))
    want = _reference(qkv, seg, T, heads, 0.125)
    assert torch.isfinite(got).all()  # pad rows attend themselves
    torch.testing.assert_close(got.float(), want, rtol=tol, atol=tol)
    if kind == "one":  # the same mask in the same order as the causal kernel: the same bits
        assert torch.equal(got, ops.attention_qkv(qkv, T, TILE, heads, HD, 0.125, causal=True))
    if kind == "rows":  # a row that sees only itself returns its own value row
        assert torch.equal(got, qkv[:, 2 * heads * HD:])
    if pad.any():
        assert torch.equal(got[pad.to(DEV)], qkv[:, 2 * heads * HD:][pad.to(DEV)])


def test_segments_do_not_leak(ops):
    """Changing one segment's rows leaves every other segment's output as it was, bit for bit."""
    T, heads = 2, 2
    g = torch.Generator().manual_seed(5)
    qkv = torch.randn(T * TILE, 3 * heads * HD, generator=g).to(DEV, torch.float16)
    seg, _ = _segments("mixed", T, seed=9)
    segd = seg.to(DEV)
    a = ops.attention_qkv(qkv, T, TILE, heads, HD, 0.125, causal=True, seg_start=segd)
    first = (seg[:TILE] == 0)  # the first segment of the first tile
    qkv2 = qkv.clone()
    qkv2[:TILE][first.to(DEV)] = 7.0
    b = ops.attention_qkv(qkv2, T, TILE, heads, HD, 0.125, causal=True, seg_start=segd)
    others = torch.ones(T * TILE, dtype=torch.bool)
    others[:TILE] = ~first
    assert torch.equal(a[others.to(DEV)], b[others.to(DEV)]) and not torch.equal(a, b)


def test_invalid_arguments_are_reported():
    import ape_b200

    lib = ape_b200._lib.lib
    T, heads = 1, 2
    qkv = torch.zeros(T * TILE, 3 * heads * HD, dtype=torch.float16, device=DEV)
    out = torch.zeros(T * TILE, heads * HD, dtype=torch.float16, device=DEV)
    seg = torch.zeros(T * TILE, dtype=torch.int32, device=DEV)

    def call(n=TILE, n_valid=TILE, head_dim=HD, stride=0, causal=1, seg_ptr=seg.data_ptr(), dtype=1):
        return lib.ape_attn_fwd_seg(qkv.data_ptr(), qkv.stride(0), out.data_ptr(), out.stride(0), T, n, n_valid, heads, head_dim,
                                    ctypes.c_float(0.125), dtype, None, stride, causal, 0, seg_ptr, None)

    assert call(seg_ptr=None) == -3 and b"seg_start" in lib.ape_last_error()
    for kw in (dict(n=256, n_valid=256), dict(n_valid=77), dict(stride=80), dict(causal=0), dict(head_dim=32), dict(dtype=0)):
        assert call(**kw) < 0 and lib.ape_last_error() != b"", kw
    torch.cuda.synchronize()
    assert not out.any()  # nothing was launched
    with pytest.raises(RuntimeError, match="seg_start"):
        ape_b200.ops.attention_qkv(qkv, T, TILE, heads, HD, 0.125, causal=True, seg_start=seg[:-1])
    with pytest.raises(RuntimeError, match="128"):
        ape_b200.ops.attention_qkv(torch.cat([qkv, qkv]), 1, 256, heads, HD, 0.125, causal=True,
                                   seg_start=torch.zeros(256, dtype=torch.int32, device=DEV))


@pytest.mark.parametrize("D", [128, 768, 1280])
def test_text_embed_packed_is_the_fp32_sum(D):
    import ape_b200

    g = torch.Generator().manual_seed(D)
    vocab, ctx, M = 500, 77, 384
    table = torch.randn(vocab, D, generator=g).to(DEV)
    posemb = torch.randn(ctx, D, generator=g).to(DEV)
    tok = torch.randint(0, vocab, (M,), generator=g).to(DEV, torch.int32)
    pos = torch.randint(0, ctx, (M,), generator=g).to(DEV, torch.int32)
    pad = torch.rand(M, generator=g).to(DEV) < 0.2
    pos[pad] = -1
    tok[0], pos[0] = 0, 0  # token id 0 is a token like any other; only pos < 0 marks a pad row
    pad[0] = False
    n0 = ape_b200._lib.launch_count()
    x = ape_b200.ops.text_embed_packed(table, posemb, tok, pos)
    assert ape_b200._lib.launch_count() == n0 + 1
    want = table[tok.long()] + posemb[pos.clamp(min=0).long()]
    assert x.dtype == torch.float32 and x.shape == (M, D)
    assert torch.equal(x[~pad], want[~pad]) and not x[pad].any()
    tok[5], pos[7] = vocab, ctx  # outside their tables: zeros, nothing read out of bounds
    x = ape_b200.ops.text_embed_packed(table, posemb, tok, pos)
    assert not x[5].any() and not x[7].any() and torch.equal(x[8:][~pad[8:]], want[8:][~pad[8:]])
    lib = ape_b200._lib.lib
    assert lib.ape_text_embed_packed(table.data_ptr(), posemb.data_ptr(), None, pos.data_ptr(), x.data_ptr(), M, D, vocab, ctx, None) == -3
    assert lib.ape_text_embed_packed(table.data_ptr(), posemb.data_ptr(), tok.data_ptr(), pos.data_ptr(), x.data_ptr(), M, 6, vocab, ctx, None) == -1
    assert b"text_embed_packed" in lib.ape_last_error()


def test_rows_gather():
    import ape_b200

    g = torch.Generator().manual_seed(1)
    buf = torch.randn(300, 1280 + 8, generator=g).to(DEV)
    x = buf[:, :1280]  # a padded row pitch
    rows = torch.randint(0, 300, (57,), generator=g).to(DEV)
    assert torch.equal(ape_b200.ops.rows_gather(x, rows), x[rows])
    assert ape_b200.ops.rows_gather(x, rows[:0]).shape == (0, 1280)
    lib = ape_b200._lib.lib
    assert lib.ape_rows_gather(x.data_ptr(), x.stride(0), None, x.data_ptr(), x.stride(0), 4, 1280, None) == -3
    assert lib.ape_rows_gather(x.data_ptr(), 100, rows.data_ptr(), x.data_ptr(), x.stride(0), 4, 1280, None) == -1
    assert b"rows_gather" in lib.ape_last_error()
