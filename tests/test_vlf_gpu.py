"""GPU: VisionLanguageFusion with one language token ("name" prompts): the restructured path with the
ape_vlf_pool kernels against the literal BiMultiHeadAttention op sequence (fuse_helper.py:67-166) in fp32."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("S", [77, 2048, 87296])
@pytest.mark.parametrize("dtype,tol", [(torch.float32, 2e-5), (torch.float16, 3e-3)])
def test_single_token_path_matches_literal_attention(S, dtype, tol):
    from ape_b200.layers.vision_language_fusion import BiAttentionBlock

    torch.manual_seed(0)
    blk = BiAttentionBlock(256, 1024, 2048, 8, init_values=1 / 6, stable_softmax_2d=True).eval().to(DEV)
    with torch.no_grad():
        for p in blk.parameters():
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.05)
        B = 2
        v = torch.randn(B, S, 256, device=DEV)
        l = torch.randn(B, 1, 1024, device=DEV)
        vn, ln = blk.layer_norm_v(v), blk.layer_norm_l(l)
        dv0, dl0 = blk.attn(vn, ln)                      # literal: three S x 256 x 2048 projections
        dv1, dl1 = blk.single_token(vn.to(dtype), ln)    # restructured + pooling kernels
    torch.testing.assert_close(dv1.float().expand_as(dv0), dv0, rtol=tol, atol=tol)
    torch.testing.assert_close(dl1.float(), dl0, rtol=tol, atol=tol)


def test_vlf_pool_extreme_scores_follow_reference_clamps():
    import ape_b200

    B, S, C, NH = 1, 300, 256, 8
    g = torch.Generator().manual_seed(1)
    v = torch.randn(B, S, C, generator=g).to(DEV)
    qa = (torch.randn(B, NH, C, generator=g) * 1e4).to(DEV)  # scores far beyond +-5e4: the clamps bite
    qc = torch.zeros(B, NH, device=DEV)
    got = ape_b200.ops.vlf_pool(v, qa, qc, True)
    w = torch.einsum("bsc,bhc->bhs", v, qa)
    w = torch.clamp(torch.clamp(w - w.max(), min=-50000), max=50000)
    wl = torch.clamp(torch.clamp(w - w.max(-1, keepdim=True)[0], min=-50000), max=50000).softmax(-1)
    want = torch.einsum("bhs,bsc->bhc", wl, v)
    torch.testing.assert_close(got, want, rtol=1e-3, atol=1e-4)


@pytest.mark.parametrize("S,N,dtype,tol", [(500, 3, torch.float16, 4e-3), (2048, 256, torch.float16, 4e-3),
                                           (5000, 1203, torch.float16, 4e-3), (1000, 77, torch.bfloat16, 3e-2)])
def test_multi_token_engine_path_matches_literal_attention(S, N, dtype, tol):
    """Phrase / text prompts (N_t > 1): BiAttentionBlock's engine path (LayerNorm kernel, wgmma GEMMs, two
    ape_attn_cross_fwd passes over 256-channel heads) against the literal op sequence of fuse_helper.py:67-166 in fp32
    (score matrix, global-max shift, clamps, two softmaxes) at N_t = 3, 77, 256 and 1203."""
    from ape_b200.layers.vision_language_fusion import BiAttentionBlock

    torch.manual_seed(1)
    blk = BiAttentionBlock(256, 1024, 2048, 8, init_values=1 / 6, stable_softmax_2d=True).eval().to(DEV)
    with torch.no_grad():
        for p in blk.parameters():
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.05)
        B = 2
        v = torch.randn(B, S, 256, device=DEV)
        l = torch.randn(B, N, 1024, device=DEV)
        want_v, want_l = blk(v, l)                                   # fp32: literal path
        got_v, got_l = blk(v.to(dtype), l)                           # 16-bit vision tokens: engine path
    assert got_v.dtype == dtype and got_l.dtype == torch.float32
    torch.testing.assert_close(got_v.float(), want_v, rtol=tol, atol=tol)
    torch.testing.assert_close(got_l, want_l, rtol=tol, atol=tol)
