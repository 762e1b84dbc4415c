"""GPU: VisionLanguageFusion for N > 1 language tokens through the folded path (BiAttentionBlock.folded: one language GEMM,
ape_vlf_fold_vision, ape_vlf_fold_pool) against the literal BiMultiHeadAttention op sequence (fuse_helper.py:67-166) in fp32,
and the two kernels directly: keys past N ignored, S split into chunks and combined deterministically."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHAPES = [(500, 2), (2048, 77), (5000, 256), (5000, 1203), (87296, 3), (87296, 80)]
DTYPES = [(torch.float16, 4e-3), (torch.bfloat16, 3e-2)]


def _block(seed):
    from ape_b200.layers.vision_language_fusion import BiAttentionBlock

    torch.manual_seed(seed)
    blk = BiAttentionBlock(256, 1024, 2048, 8, init_values=1 / 6, stable_softmax_2d=True).eval().to(DEV)
    with torch.no_grad():
        for p in blk.parameters():
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.05)
    return blk


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("S,N", SHAPES)
@pytest.mark.parametrize("dtype,tol", DTYPES)
def test_folded_block_matches_literal_attention(S, N, B, dtype, tol):
    blk = _block(S + N)
    with torch.no_grad():
        v = torch.randn(B, S, 256, device=DEV)
        l = torch.randn(B, N, 1024, device=DEV)
        want_v, want_l = blk(v, l)                              # fp32: the literal path
        launches = _launches()
        got_v, got_l = blk(v.to(dtype), l)                      # 16-bit: the folded path
        assert _launches() - launches >= 3                      # language GEMM + vision kernel + pooling kernels at least
    assert got_v.dtype == dtype and got_l.dtype == torch.float32
    torch.testing.assert_close(got_v.float(), want_v, rtol=tol, atol=tol)
    torch.testing.assert_close(got_l, want_l, rtol=tol, atol=tol)


def _launches():
    import ape_b200

    torch.cuda.synchronize()
    return ape_b200._lib.launch_count()


def _operands(B, S, N, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    v = torch.nn.functional.layer_norm(torch.randn(B, S, 256, generator=g), (256,)).to(DEV, dtype)
    # keys of head h scaled by 1 + h: a block read past head h's N keys reaches head h+1's much larger keys
    qa = (torch.randn(B, 8, N, 256, generator=g) * 0.05 * (1 + torch.arange(8.0))[None, :, None, None]).to(DEV, dtype)
    u = torch.randn(B, 8, N, 256, generator=g).to(DEV, dtype)
    qc = torch.randn(B, 8, N, generator=g).to(DEV)
    gamma, bias = torch.rand(256, generator=g).to(DEV), torch.randn(256, generator=g).to(DEV)
    return v, qa, u, qc, gamma, bias


@pytest.mark.parametrize("S,N", [(333, 1), (1000, 65), (4133, 130), (70001, 7)])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_kernels_match_fp32_reference(S, N, dtype):
    """N not a multiple of 64 (keys past N: the next head's rows or the tensor's end), S not a multiple of 128 or of the chunk."""
    from ape_b200 import ops

    B = 2
    v, qa, u, qc, gamma, bias = _operands(B, S, N, dtype, seed=S + N)
    vf, qf, uf = v.float(), qa.float(), u.float()
    t = torch.einsum("bsc,bhnc->bhsn", vf, qf)
    want_v = vf + gamma * (torch.einsum("bhsn,bhnc->bsc", (t + qc[:, :, None, :]).softmax(-1), uf) + bias)
    want_p = torch.einsum("bhsn,bsc->bnhc", t.softmax(2), vf).reshape(B * N, 8 * 256)
    got_v = ops.vlf_fold_vision(v, qa, u, qc, gamma, bias)
    got_p = ops.vlf_fold_pool(v, qa)
    tol = 2e-2 if dtype == torch.bfloat16 else 3e-3
    torch.testing.assert_close(got_v.float(), want_v, rtol=tol, atol=tol)
    torch.testing.assert_close(got_p.float(), want_p, rtol=tol, atol=tol)


def test_pool_combine_is_deterministic():
    from ape_b200 import ops

    v, qa, *_ = _operands(2, 87296, 3, torch.float16, seed=3)
    a = ops.vlf_fold_pool(v, qa)
    b = ops.vlf_fold_pool(v, qa)
    assert torch.equal(a, b)


def test_vision_kernel_writes_in_place():
    from ape_b200 import ops

    v, qa, u, qc, gamma, bias = _operands(1, 1000, 5, torch.float16, seed=9)
    want = ops.vlf_fold_vision(v, qa, u, qc, gamma, bias)
    ops.vlf_fold_vision(v, qa, u, qc, gamma, bias, out=v)
    assert torch.equal(v, want)
