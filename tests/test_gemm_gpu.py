"""GPU: the TMA/wgmma linear layer (ape_gemm_tn) against a plain PyTorch fp32 reference of
the same op on the same (16-bit rounded) operands.  Tolerance: fp32 accumulation over K terms of
16-bit products -> relative 2e-3 on fp16/bf16 outputs (output rounding), 1e-4 on fp32 outputs."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def ops():
    import ape_b200

    return ape_b200.ops


def ref_linear(x, w, b=None, act=None, residual=None):
    y = F.linear(x.float(), w.float(), b)
    if act == "relu":
        y = F.relu(y)
    elif act == "gelu":
        y = F.gelu(y)
    elif act == "swiglu":
        y = F.silu(y[..., 0::2]) * y[..., 1::2]
    if residual is not None:
        y = y + residual.float()
    return y


def rnd(*shape, dtype, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).to(DEV)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M,N,K,tile", [
    (128, 128, 64, 128), (128, 256, 64, 256), (256, 256, 128, 0), (384, 512, 1024, 128),
    (4096, 3072, 1024, 256),   # ViT-L fused q/k/v projection
    (4096, 1024, 1024, 128),   # ViT-L attention output projection
    (900, 256, 256, 0),        # decoder tokens: M not a multiple of 128
    (1000, 1203, 256, 0),      # LVIS vocabulary: N not a multiple of the tile
    (300, 96, 200, 128),       # K not a multiple of 64 (TMA zero-fills the tail)
])
def test_plain_gemm(ops, dtype, M, N, K, tile):
    x = rnd(M, K, dtype=dtype, seed=1)
    w = rnd(N, K, dtype=dtype, seed=2, scale=K ** -0.5)
    y = ops.linear_tc(x, w, tile_n=tile)
    assert y.dtype == dtype and y.shape == (M, N)
    torch.testing.assert_close(y.float(), ref_linear(x, w), rtol=1e-2, atol=1e-2 if dtype == torch.bfloat16 else 2e-3)
    y32 = ops.linear_tc(x, w, out_dtype=torch.float32, tile_n=tile)
    torch.testing.assert_close(y32, ref_linear(x, w), rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("act", [None, "relu", "gelu", "swiglu"])
def test_epilogues(ops, act):
    M, N, K = 640, 512, 320
    dtype = torch.float16
    x = rnd(M, K, dtype=dtype, seed=3)
    w = rnd(N, K, dtype=dtype, seed=4, scale=K ** -0.5)
    b = rnd(N, dtype=torch.float32, seed=5)
    y = ops.linear_tc(x, w, b, act=act, out_dtype=torch.float32)
    torch.testing.assert_close(y, ref_linear(x, w, b, act), rtol=2e-4, atol=2e-4)
    if act != "swiglu":
        res = rnd(M, N, dtype=dtype, seed=6)
        y = ops.linear_tc(x, w, b, act=act, residual=res)
        torch.testing.assert_close(y.float(), ref_linear(x, w, b, act, res), rtol=2e-3, atol=4e-3)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_vit_swiglu_shape_16bit_out(ops, dtype):
    """ViT-L SwiGLU up-projection: interleaved (w1_j, w2_j) rows, N = 2*2730, 16-bit output through the
    shared-memory + TMA-store epilogue into a 2752-pitch buffer (N/2 = 2730 is not a multiple of 8)."""
    M, K, hid = 4096, 1024, 2730
    x = rnd(M, K, dtype=dtype, seed=11)
    w = rnd(2 * hid, K, dtype=dtype, seed=12, scale=K ** -0.5)
    b = rnd(2 * hid, dtype=torch.float32, seed=13)
    buf = torch.full((M, 2752), 9.0, dtype=dtype, device=DEV)
    y = ops.linear_tc(x, w, b, act="swiglu", out=buf[:, :hid])
    tol = 4e-3 if dtype == torch.float16 else 3e-2
    torch.testing.assert_close(y.float(), ref_linear(x, w, b, "swiglu"), rtol=tol, atol=tol)
    # the TMA store clips at N/2 = 2730; the tail of the last 16-byte unit of a row (2730..2735) may be
    # zero-filled, nothing beyond it is touched
    assert (buf[:, 2736:] == 9.0).all()
    pad = buf[:, hid:2736]
    assert ((pad == 9.0) | (pad == 0.0)).all()


@pytest.mark.parametrize("tile", [128, 256, 128 | 0x1000, 256 | 0x1000, 128 | 0x4000, 256 | 0x4000])  # default: per-shape policy; 0x1000: single CTA; 0x4000: cluster of 2 (TMA multicast)
def test_tma_store_epilogue_edges(ops, tile):
    # M and N both ragged, bias + relu + residual, 16-bit output with an aligned pitch
    M, N, K = 777, 840, 192
    dtype = torch.float16
    x = rnd(M, K, dtype=dtype, seed=21)
    w = rnd(N, K, dtype=dtype, seed=22, scale=K ** -0.5)
    b = rnd(N, dtype=torch.float32, seed=23)
    res = rnd(M, N, dtype=dtype, seed=24)
    y = ops.linear_tc(x, w, b, act="relu", residual=res, tile_n=tile)
    torch.testing.assert_close(y.float(), ref_linear(x, w, b, "relu", res), rtol=4e-3, atol=4e-3)


@pytest.mark.parametrize("M", [129, 256, 383, 640, 4096])
@pytest.mark.parametrize("tile", [128, 256])
def test_cluster_pairs_with_odd_row_block_counts(ops, M, tile):
    """Clusters of two CTAs share the weight tile by TMA multicast; an odd number of 128-row blocks leaves the
    second CTA of the last cluster with an all-out-of-range tile that must still take part in the protocol."""
    N, K = 512, 512
    x = rnd(M, K, dtype=torch.bfloat16, seed=41)
    w = rnd(N, K, dtype=torch.bfloat16, seed=42, scale=K ** -0.5)
    b = rnd(N, dtype=torch.float32, seed=43)
    y = ops.linear_tc(x, w, b, out_dtype=torch.float32, tile_n=tile)
    torch.testing.assert_close(y, ref_linear(x, w, b), rtol=2e-4, atol=2e-4)
    y1 = ops.linear_tc(x, w, b, out_dtype=torch.float32, tile_n=tile | 0x1000)
    assert torch.equal(y, y1)  # same accumulation order with and without the cluster
    assert torch.equal(y, ops.linear_tc(x, w, b, out_dtype=torch.float32, tile_n=tile | 0x4000))  # the multicast cluster of 2
    with pytest.raises(RuntimeError):  # the CTA-pair MMA flag names an instruction sm_90a lacks: rejected, not ignored
        ops.linear_tc(x, w, b, out_dtype=torch.float32, tile_n=tile | 0x2000)


def test_many_tiles_per_cta_ring_wraparound(ops):
    # 87 296 encoder tokens x FFN: 682 x 8 tiles over 132 persistent CTAs, K = 2048 (32 k-blocks)
    M, N, K = 87296, 256, 2048
    x = rnd(M, K, dtype=torch.float16, seed=31, scale=0.5)
    w = rnd(N, K, dtype=torch.float16, seed=32, scale=K ** -0.5)
    y = ops.linear_tc(x, w)
    idx = torch.randint(0, M, (2048,), device=DEV)
    torch.testing.assert_close(y[idx].float(), ref_linear(x[idx], w), rtol=4e-3, atol=4e-3)


def test_padded_pitch_and_batched_input(ops):
    # K = 2730 (SwiGLU hidden of ViT-L) stored with a 2752-element pitch; leading batch dims are flattened
    K, Kp, N = 2730, 2752, 1024
    buf = torch.zeros(2, 64, Kp, dtype=torch.bfloat16, device=DEV)
    buf[..., :K] = rnd(2, 64, K, dtype=torch.bfloat16, seed=7)
    wbuf = torch.zeros(N, Kp, dtype=torch.bfloat16, device=DEV)
    wbuf[:, :K] = rnd(N, K, dtype=torch.bfloat16, seed=8, scale=K ** -0.5)
    y = ops.linear_tc(buf[..., :K], wbuf[:, :K], out_dtype=torch.float32)
    assert y.shape == (2, 64, N)
    torch.testing.assert_close(y, ref_linear(buf[..., :K], wbuf[:, :K]), rtol=1e-4, atol=1e-4)


def test_rejects_bad_arguments(ops):
    x = rnd(128, 64, dtype=torch.float32, seed=1)
    with pytest.raises(RuntimeError):
        ops.linear_tc(x, x)  # fp32 operands are not a tensor-core format here
    with pytest.raises(RuntimeError):
        ops.linear_tc(x.cpu().half(), x.cpu().half())  # no CPU path


@pytest.mark.parametrize("dtype,tol", [(torch.float16, 4e-3), (torch.bfloat16, 3e-2)])
@pytest.mark.parametrize("use_map", [False, True])
def test_qkv_projection_with_fused_rope(ops, dtype, tol, use_map):
    """ape_gemm_tn_rope = ape_gemm_tn followed by the 2-D rotary embedding on the q and k thirds (the separate
    ape_rope_qk kernel and the reference formula, utils_eva02.py:248-252,346), single rounding."""
    M, C, heads, hd, K, npos = 640, 256, 4, 64, 192, 160
    x = rnd(M, K, dtype=dtype, seed=51)
    w = rnd(3 * C, K, dtype=dtype, seed=52, scale=K ** -0.5)
    b = rnd(3 * C, dtype=torch.float32, seed=53)
    g = torch.Generator().manual_seed(54)
    ang = torch.randn(npos, hd, generator=g)
    cos, sin = ang.cos().to(DEV), ang.sin().to(DEV)
    pos = torch.randint(0, npos, (M,), generator=g).to(torch.int32).to(DEV) if use_map else None
    got = ops.linear_rope_tc(x, w, b, cos, sin, C, hd, pos_map=pos)
    y = ref_linear(x, w, b)
    pidx = pos.long() if use_map else torch.arange(M, device=DEV) % npos

    def rope(t):
        t = t.view(M, heads, hd)
        pr = t.reshape(M, heads, hd // 2, 2)
        rot = torch.stack((-pr[..., 1], pr[..., 0]), -1).flatten(-2)
        return (t * cos[pidx][:, None] + rot * sin[pidx][:, None]).reshape(M, C)

    want = torch.cat([rope(y[:, :C]), rope(y[:, C:2 * C]), y[:, 2 * C:]], 1)
    torch.testing.assert_close(got.float(), want, rtol=tol, atol=tol)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,N,K,nparts", [(256, 256, 256, 4), (4096, 1024, 1024, 16), (4096, 1024, 2730, 43), (300, 96, 200, 4)])
def test_fp32_output_residual_dtypes_and_layernorm_fold(ops, dtype, M, N, K, nparts):
    """fp32 output through the TMA epilogue with a 16-bit / fp32 residual, and a LayerNorm folded around the GEMM
    (ape_gemm_tn_fused): rstd * (a (gamma .* W)^T - mean * colsum) + (beta W^T + b) == Linear(LayerNorm(a))."""
    Kp = (K + 7) // 8 * 8
    a = torch.zeros(M, Kp, dtype=dtype, device=DEV)
    a[:, :K] = rnd(M, K, dtype=dtype, seed=1, scale=2.0) + 0.7      # non-zero mean rows
    w = rnd(N, K, dtype=torch.float32, seed=2, scale=K ** -0.5)
    b = rnd(N, dtype=torch.float32, seed=3)
    gamma = 1.0 + 0.1 * rnd(K, dtype=torch.float32, seed=4)
    beta = 0.1 * rnd(K, dtype=torch.float32, seed=5)
    res16 = rnd(M, N, dtype=dtype, seed=6)
    res32 = rnd(M, N, dtype=torch.float32, seed=7)
    # plain fp32-out paths
    w16 = torch.zeros(N, Kp, dtype=dtype, device=DEV)
    w16[:, :K] = w.to(dtype)
    for res in (None, res16, res32):
        got = ops.linear_tc(a[:, :K], w16[:, :K], b, residual=res, out_dtype=torch.float32)
        want = ref_linear(a[:, :K], w16[:, :K], b, residual=res)
        torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-3)
    # LayerNorm fold: partial statistics in `nparts` chunks, as a producer kernel would leave them
    af = a[:, :K].float()
    edges = torch.linspace(0, K, nparts + 1).round().long().tolist()
    part = torch.stack([torch.stack([af[:, s:e].sum(1), (af[:, s:e] ** 2).sum(1)], -1) for s, e in zip(edges[:-1], edges[1:])], 1).contiguous()
    wl = torch.zeros(N, Kp, dtype=dtype, device=DEV)
    wl[:, :K] = (w * gamma[None, :]).to(dtype)
    colsum = wl.float().sum(1).contiguous()
    bias = (w @ beta + b).contiguous()
    got = ops.linear_tc(a[:, :K], wl[:, :K], bias, residual=res32, out_dtype=torch.float32, ln_fold=(part, colsum, K, 1e-6))
    want = F.linear(F.layer_norm(af, (K,), gamma, beta, 1e-6), wl[:, :K].float() / gamma[None, :], b) + res32
    # the reference applies gamma after normalising, the fold before rounding W: identical up to the 16-bit rounding of W'
    torch.testing.assert_close(got, want, rtol=2e-3, atol=2e-2 if dtype == torch.bfloat16 else 4e-3)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_swiglu_epilogue_row_statistics(ops, dtype):
    M, K, hid = 300, 256, 2730
    x = rnd(M, K, dtype=dtype, seed=11)
    w = rnd(2 * hid, K, dtype=dtype, seed=12, scale=K ** -0.5)
    b = rnd(2 * hid, dtype=torch.float32, seed=13)
    hp = (hid + 7) // 8 * 8
    buf = torch.zeros(M, hp, dtype=dtype, device=DEV)
    out, st = ops.linear_tc(x, w, b, act="swiglu", out=buf[:, :hid], stats_out=True)
    nslab = (hid + 63) // 64
    assert st.shape == (M, nslab, 2)
    of = out.float()
    for sidx in (0, 1, nslab // 2, nslab - 1):
        sl = of[:, sidx * 64: min(hid, sidx * 64 + 64)]
        torch.testing.assert_close(st[:, sidx, 0], sl.sum(1), rtol=1e-4, atol=1e-3)
        torch.testing.assert_close(st[:, sidx, 1], (sl ** 2).sum(1), rtol=1e-4, atol=1e-3)
    torch.testing.assert_close(st[..., 0].sum(1), of.sum(1), rtol=1e-4, atol=1e-2)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("B,H,W,Cin,Cout", [(1, 32, 32, 256, 256), (2, 64, 64, 256, 256), (1, 16, 16, 64, 128), (1, 256, 256, 256, 256),
                                            (1, 16, 8, 128, 64), (1, 48, 96, 64, 256)])
def test_conv3x3_implicit_gemm_matches_conv2d(ops, dtype, B, H, W, Cin, Cout):
    """ape_conv3x3_nhwc (implicit GEMM: 4-D TMA boxes at shifted positions, zero fill = zero padding) vs F.conv2d in fp32."""
    assert ops.conv3x3_supported(H, W, Cin, Cout, dtype)
    assert not ops.conv3x3_supported(8, 8, Cin, Cout, dtype)  # a 128-pixel tile does not fit an 8 x 8 map: callers fall back
    g = torch.Generator().manual_seed(H + Cin)
    x = torch.randn(B, H, W, Cin, generator=g).to(DEV, dtype)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) * (9 * Cin) ** -0.5).to(DEV, dtype)
    got = ops.conv3x3_nhwc(x, w.permute(0, 2, 3, 1).contiguous())
    want = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), padding=1).permute(0, 2, 3, 1)
    tol = 4e-3 if dtype == torch.float16 else 3e-2
    torch.testing.assert_close(got.float(), want, rtol=tol, atol=tol)


@pytest.mark.parametrize("M,N,K,act,out32", [
    (19100, 256, 256, None, False),     # 150 row tiles: more tiles than the 132 persistent CTAs
    (40000, 256, 192, "relu", False),   # 3 k blocks, several tiles per CTA, ragged last tile
    (25000, 200, 256, None, True),      # N < tile, fp32 output + residual
    (19000, 2048, 256, "relu", False),  # 149 row blocks x 8 column blocks (encoder FFN1 geometry)
    (30000, 480, 256, None, False),     # ragged second column block (stacked offsets / logits projection)
    (20000, 1024, 200, None, True),     # K not a multiple of 64, fp32 output + residual
])
def test_short_k_many_tiles_per_cta(ops, M, N, K, act, out32):
    """K <= 256 with tens of tiles per CTA (the encoder's GEMMs): main loops of 2-4 k blocks back to back with the lean epilogues,
    every row block written exactly once with its own rows."""
    dtype = torch.float16
    x = rnd(M, K + (-K) % 8, dtype=dtype, seed=11)[:, :K]
    w = rnd(N, K + (-K) % 8, dtype=dtype, seed=12, scale=K ** -0.5)[:, :K]
    b = rnd(N, dtype=torch.float32, seed=13)
    res = rnd(M, N, dtype=torch.float32, seed=14) if out32 else None
    y = ops.linear_tc(x, w, b, act=act, residual=res, out_dtype=torch.float32 if out32 else None)
    want = ref_linear(x, w, b, act=act, residual=res)
    if out32:
        torch.testing.assert_close(y, want, rtol=1e-4, atol=1e-4)
    else:
        torch.testing.assert_close(y.float(), want, rtol=1e-2, atol=2e-3)
    # every row block was written exactly once with its own rows: compare a shuffled-row run
    perm = torch.randperm(M, device=DEV)
    y2 = ops.linear_tc(x[perm].contiguous(), w, b, act=act, residual=res[perm].contiguous() if out32 else None,
                       out_dtype=torch.float32 if out32 else None)
    assert torch.equal(y2, y[perm])
