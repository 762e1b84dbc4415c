"""CPU: the folded form of VisionLanguageFusion (BiAttentionBlock.fold_maps, evaluated by BiAttentionBlock.folded and the
ape_vlf_fold_* kernels on the GPU) is the same function as the literal BiMultiHeadAttention.forward (fuse_helper.py:67-166)
for any number of language tokens and any head dimension: checked in fp64 with random weights and non-zero biases."""
import pytest
import torch

from ape_b200.layers.vision_language_fusion import BiAttentionBlock


def _block(head_dim, l_dim, seed):
    torch.manual_seed(seed)
    blk = BiAttentionBlock(256, l_dim, 8 * head_dim, 8, init_values=1 / 6, stable_softmax_2d=True).double().eval()
    with torch.no_grad():
        for p in blk.parameters():
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.05)
    return blk


def _folded(blk, vn, ln):
    """The folded mathematics restated: [qa | U | qc] = ln Gm^T + gm0; the vision side softmaxes over the tokens n of each
    head, the language side over the S vision tokens (qc cancels), delta_l = E pooled + e0."""
    _, _, E, e0, Gm, gm0 = blk.fold_maps()
    nh, C = blk.attn.num_heads, vn.shape[-1]
    B, N, _ = ln.shape
    y = ln @ Gm.T + gm0
    qa = y[..., : nh * C].view(B, N, nh, C)
    u = y[..., nh * C: 2 * nh * C].view(B, N, nh, C)
    qc = y[..., 2 * nh * C:]                                                   # [B,N,nh]
    t = torch.einsum("bsc,bnhc->bhsn", vn, qa)
    dv = torch.einsum("bhsn,bnhc->bsc", (t + qc.transpose(1, 2)[:, :, None, :]).softmax(-1), u) + blk.attn.out_v_proj.bias
    pooled = torch.einsum("bhsn,bsc->bnhc", t.softmax(2), vn)
    dl = pooled.reshape(B, N, nh * C) @ E.T + e0
    return dv, dl


@pytest.mark.parametrize("head_dim", [32, 256])
@pytest.mark.parametrize("N", [1, 2, 77, 300])
def test_fold_matches_literal_attention(head_dim, N):
    blk = _block(head_dim, 64, seed=N + head_dim)
    B, S = 2, 37
    g = torch.Generator().manual_seed(N)
    with torch.no_grad():
        vn = blk.layer_norm_v(torch.randn(B, S, 256, generator=g, dtype=torch.float64))
        ln = blk.layer_norm_l(torch.randn(B, N, 64, generator=g, dtype=torch.float64))
        want_v, want_l = blk.attn(vn, ln)                                       # literal: projections, score matrix, clamps
        got_v, got_l = _folded(blk, vn, ln)
    torch.testing.assert_close(got_v, want_v, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(got_l, want_l, rtol=1e-10, atol=1e-10)


def test_one_token_map_is_the_multi_token_map_summed_over_heads():
    """fold_maps' one-token G ([qa | qc | delta_v]) and the N-token Gm ([qa | U | qc]) share qa and qc, and delta_v is U summed
    over the heads: the softmax over a single key is 1."""
    blk = _block(256, 64, seed=5)
    G, g0, _, _, Gm, gm0 = blk.fold_maps()
    nh, C = 8, 256
    torch.testing.assert_close(G[: nh * C], Gm[: nh * C], rtol=0, atol=0)
    torch.testing.assert_close(G[nh * C: nh * C + nh], Gm[2 * nh * C:], rtol=0, atol=0)
    torch.testing.assert_close(G[nh * C + nh:], Gm[nh * C: 2 * nh * C].view(nh, C, -1).sum(0), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(g0[nh * C + nh:], gm0[nh * C: 2 * nh * C].view(nh, C).sum(0) + blk.attn.out_v_proj.bias.double(),
                               rtol=1e-12, atol=1e-12)


def test_folded_path_selection():
    """The folded path takes 256-channel vision tokens, unmasked fusion and up to fold_max_tokens tokens; the rest keep
    forward_engine (longer prompts) or the literal path."""
    blk = _block(256, 64, seed=1)
    assert blk.folds(256, 64, 2) and blk.folds(256, 64, blk.fold_max_tokens)
    assert not blk.folds(256, 64, blk.fold_max_tokens + 1)
    assert not blk.folds(128, 64, 2)
    assert not _block(32, 64, seed=1).folds(256, 64, 2)
    blk.attn.use_attention_mask_v = True
    assert not blk.folds(256, 64, 2) and blk.folds(256, 64, 2, masked_v=False)
