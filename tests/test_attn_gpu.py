"""GPU: the wgmma flash-attention kernel (ape_attn_fwd) against a plain PyTorch fp32 reference of the same op
(softmax(q k^T * scale) v per head) on the same 16-bit inputs."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module", params=[0, 1], ids=["smemP", "tmemP"])
def ops(request):
    """Every test of this file runs against both structures of the ViT attention kernel (ape_attn_variant): P read by the
    P.V MMA from shared memory ("smemP") or kept on-chip in registers as its A operand (id "tmemP", kept from earlier
    hardware where it lived in tensor memory)."""
    import ape_b200

    prev = ape_b200._lib.lib.ape_attn_variant(-1)
    ape_b200._lib.lib.ape_attn_variant(request.param)
    yield ape_b200.ops
    ape_b200._lib.lib.ape_attn_variant(prev)


def ref_attention(qkv, num_seq, n, heads, hd, scale):
    q, k, v = qkv.float().view(num_seq, n, 3, heads, hd).permute(2, 0, 3, 1, 4)  # [3][s, h, n, d]
    p = torch.softmax(q @ k.transpose(-1, -2) * scale, dim=-1)
    return (p @ v).permute(0, 2, 1, 3).reshape(num_seq * n, heads * hd)


@pytest.mark.parametrize("dtype,tol", [(torch.float16, 2e-3), (torch.bfloat16, 1.6e-2)])
@pytest.mark.parametrize("num_seq,n,heads", [(1, 128, 1), (2, 256, 3), (4, 1024, 16), (1, 4096, 16)])
def test_attention_matches_fp32_reference(ops, dtype, tol, num_seq, n, heads):
    hd = 64
    g = torch.Generator().manual_seed(n + heads)
    qkv = torch.randn(num_seq * n, 3 * heads * hd, generator=g).to(DEV, dtype)
    scale = hd ** -0.5
    got = ops.attention_qkv(qkv, num_seq, n, heads, hd, scale)
    want = ref_attention(qkv, num_seq, n, heads, hd, scale)
    torch.testing.assert_close(got.float(), want, rtol=tol, atol=tol)


def test_attention_large_logits_and_pitch(ops):
    """Peaked softmax (scores of +-40) and a qkv buffer with a padded row pitch."""
    num_seq, n, heads, hd = 2, 384, 2, 64
    g = torch.Generator().manual_seed(3)
    buf = torch.zeros(num_seq * n, 3 * heads * hd + 64, dtype=torch.float16, device=DEV)
    qkv = buf[:, : 3 * heads * hd]
    qkv.copy_((torch.randn(num_seq * n, 3 * heads * hd, generator=g) * 3).to(DEV))
    got = ops.attention_qkv(qkv, num_seq, n, heads, hd, 0.5)
    want = ref_attention(qkv, num_seq, n, heads, hd, 0.5)
    torch.testing.assert_close(got.float(), want, rtol=4e-3, atol=4e-3)


def test_attention_rejects_unsupported(ops):
    with pytest.raises(RuntimeError):
        ops.attention_qkv(torch.zeros(100, 192, dtype=torch.float16, device=DEV), 1, 100, 1, 64, 1.0)  # n % 128 != 0


@pytest.mark.parametrize("num_seq,n,n_valid,heads", [(1, 1024, 900, 8), (2, 128, 20, 4), (1, 256, 129, 2), (3, 384, 64, 1)])
def test_attention_padded_sequences_mask_keys(ops, num_seq, n, n_valid, heads):
    """Sequences padded to a multiple of 128 rows: only the first n_valid keys count (decoder self-attention over 900
    queries, deformable_transformer_vl.py:142-147); the padded rows hold zeros."""
    hd = 64
    g = torch.Generator().manual_seed(n_valid)
    qkv = torch.zeros(num_seq, n, 3 * heads * hd, dtype=torch.float16)
    qkv[:, :n_valid] = torch.randn(num_seq, n_valid, 3 * heads * hd, generator=g).to(torch.float16)
    qkv = qkv.to(DEV)
    got = ops.attention_qkv(qkv.view(num_seq * n, -1), num_seq, n, heads, hd, 0.2, n_valid=n_valid).view(num_seq, n, -1)
    want = ref_attention(qkv[:, :n_valid].reshape(num_seq * n_valid, -1), num_seq, n_valid, heads, hd, 0.2).view(num_seq, n_valid, -1)
    torch.testing.assert_close(got[:, :n_valid].float(), want, rtol=2e-3, atol=2e-3)
    assert torch.isfinite(got).all()


def test_attention_row_statistics_output(ops):
    """stats_out: per (row, head) sum and sum of squares of the stored 16-bit outputs (for the LayerNorm folded into proj)."""
    num_seq, n, heads, hd = 2, 256, 4, 64
    qkv = torch.randn(num_seq * n, 3 * heads * hd, generator=torch.Generator().manual_seed(5)).to(DEV, torch.float16)
    out, st = ops.attention_qkv(qkv, num_seq, n, heads, hd, 0.125, stats_out=True)
    assert st.shape == (num_seq * n, heads, 2)
    o = out.float().view(num_seq * n, heads, hd)
    torch.testing.assert_close(st[..., 0], o.sum(-1), rtol=1e-5, atol=1e-4)
    torch.testing.assert_close(st[..., 1], (o ** 2).sum(-1), rtol=1e-5, atol=1e-4)


@pytest.mark.parametrize("dtype,tol", [(torch.float16, 3e-3), (torch.bfloat16, 2e-2)])
@pytest.mark.parametrize("num_seq,nq,nk,heads,hd", [(1, 128, 64, 1, 256), (2, 256, 200, 8, 256), (1, 384, 1203, 2, 256),
                                                    (1, 128, 5000, 1, 256), (2, 256, 130, 3, 64)])
def test_cross_attention_wide_heads(ops, dtype, tol, num_seq, nq, nk, heads, hd):
    """ape_attn_cross_fwd (separate Q / K / V, 256-channel heads, padded + masked keys) against fp32 softmax attention."""
    g = torch.Generator().manual_seed(nk + heads)
    C = heads * hd
    nkp = (nk + 63) // 64 * 64
    q = torch.randn(num_seq, nq, C, generator=g).to(DEV, dtype)
    k = torch.zeros(num_seq, nkp, C, dtype=dtype, device=DEV)
    v = torch.zeros(num_seq, nkp, C, dtype=dtype, device=DEV)
    k[:, :nk] = torch.randn(num_seq, nk, C, generator=g).to(DEV, dtype)
    v[:, :nk] = torch.randn(num_seq, nk, C, generator=g).to(DEV, dtype)
    scale = hd ** -0.5
    got = ops.attention_cross(q.view(-1, C), k.view(-1, C), v.view(-1, C), num_seq, nq, nkp, nk, heads, hd, scale).view(num_seq, nq, C)
    qh = q.float().view(num_seq, nq, heads, hd).transpose(1, 2)
    kh = k[:, :nk].float().view(num_seq, nk, heads, hd).transpose(1, 2)
    vh = v[:, :nk].float().view(num_seq, nk, heads, hd).transpose(1, 2)
    want = (torch.softmax(qh @ kh.transpose(-1, -2) * scale, -1) @ vh).transpose(1, 2).reshape(num_seq, nq, C)
    torch.testing.assert_close(got.float(), want, rtol=tol, atol=tol)


@pytest.mark.parametrize("num_seq,n_valid,stride,heads", [(5, 77, 80, 20), (3, 128, 128, 2), (4, 200, 200, 3), (2, 77, 128, 1)])
def test_attention_causal_and_packed_sequences(ops, num_seq, n_valid, stride, heads):
    """Causal attention over sequences packed at a row stride smaller than the 128-row tile (EVA02-CLIP text tower: 77-token
    prompts, 20 heads x 64, eva02_clip/transformer.py:714-720): rows past a sequence are neither attended nor overwritten."""
    hd = 64
    n = (n_valid + 127) // 128 * 128
    g = torch.Generator().manual_seed(stride + heads)
    rows = (num_seq - 1) * stride + max(stride, n_valid)
    qkv = torch.randn(rows, 3 * heads * hd, generator=g).to(DEV, torch.float16)
    out = ops.attention_qkv(qkv, num_seq, n, heads, hd, 0.125, n_valid=n_valid, seq_stride=stride, causal=True)
    assert out.shape[0] == rows
    for s_ in range(num_seq):
        x = qkv[s_ * stride: s_ * stride + n_valid].float().view(n_valid, 3, heads, hd).permute(1, 2, 0, 3)
        sc = x[0] @ x[1].transpose(-1, -2) * 0.125
        sc = sc.masked_fill(torch.triu(torch.ones(n_valid, n_valid, dtype=torch.bool, device=DEV), 1), float("-inf"))
        want = (torch.softmax(sc, -1) @ x[2]).permute(1, 0, 2).reshape(n_valid, heads * hd)
        torch.testing.assert_close(out[s_ * stride: s_ * stride + n_valid].float(), want, rtol=2e-3, atol=2e-3)
