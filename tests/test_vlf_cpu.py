"""CPU: the streaming evaluation of BiMultiHeadAttention (two attention calls, no S x N_t score tensor; used above
`stream_threshold_bytes`, i.e. for phrase prompts at scale) against the literal op sequence of the reference
(ape/layers/fuse_helper.py:67-166) as restated in the same module, and against outputs recorded from the reference module itself."""
import pytest
import torch

from ape_b200.layers.vision_language_fusion import BiAttentionBlock


@pytest.mark.parametrize("S,N", [(300, 7), (1000, 64), (64, 200)])
def test_streaming_equals_literal(S, N):
    torch.manual_seed(0)
    blk = BiAttentionBlock(256, 128, 512, 8, init_values=1 / 6, stable_softmax_2d=True).eval()
    with torch.no_grad():
        for p in blk.parameters():
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.05)
        v, l = torch.randn(2, S, 256), torch.randn(2, N, 128)
        blk.attn.stream_threshold_bytes = 1 << 60
        v0, l0 = blk(v, l)
        blk.attn.stream_threshold_bytes = 0
        v1, l1 = blk(v, l)
    torch.testing.assert_close(v1, v0, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(l1, l0, rtol=1e-5, atol=1e-5)


def test_streaming_is_skipped_when_the_clamps_could_bind():
    torch.manual_seed(1)
    blk = BiAttentionBlock(256, 128, 512, 8, init_values=1 / 6, stable_softmax_2d=True).eval()
    with torch.no_grad():
        blk.attn.l_proj.weight.mul_(1e5)  # scores far beyond +-5e4: the literal path (with its clamps) must be taken
        v, l = torch.randn(1, 50, 256), torch.randn(1, 5, 128)
        blk.attn.stream_threshold_bytes = 1 << 60
        v0, l0 = blk(v, l)
        blk.attn.stream_threshold_bytes = 0
        v1, l1 = blk(v, l)
    assert torch.equal(v1, v0) and torch.equal(l1, l0)


def make_block_and_inputs():
    """Seeded weights and inputs of test_literal_path_equals_reference_module (also used by tests/golden/gen_cpu_golden.py)."""
    torch.manual_seed(2)
    mine = BiAttentionBlock(256, 128, 512, 8, init_values=1 / 6, stable_softmax_2d=True).eval()
    with torch.no_grad():
        for p in mine.parameters():
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.05)
    return mine, torch.randn(2, 100, 256), torch.randn(2, 9, 128)


def test_literal_path_equals_reference_module():
    """The restated literal path against the reference's own BiAttentionBlock (fuse_helper.py) on the same weights and
    inputs, recorded in tests/golden/vlf_block_ref.npz by tests/golden/gen_cpu_golden.py."""
    from conftest import load_golden

    g = load_golden("vlf_block_ref.npz")
    mine, v, l = make_block_and_inputs()
    with torch.no_grad():
        mine.attn.stream_threshold_bytes = 1 << 60
        mv, ml = mine(v, l)
        mine.attn.stream_threshold_bytes = 0
        sv, sl = mine(v, l)
    torch.testing.assert_close(mv, g["v"], rtol=1e-6, atol=1e-6)
    torch.testing.assert_close(ml, g["l"], rtol=1e-6, atol=1e-6)
    torch.testing.assert_close(sv, g["v"], rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(sl, g["l"], rtol=1e-5, atol=1e-5)
