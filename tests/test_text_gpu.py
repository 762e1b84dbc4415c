"""GPU: the text tower's engine path (wgmma GEMMs, causal flash attention over packed 77-token prompts, LayerNorm kernels,
fp32 residual stream) against the golden recorded from the reference's TextTransformer and, at EVA02-CLIP-bigE geometry
(width 1280, 20 heads x 64), against the literal fp32 path of the same module."""
import pytest
import torch

from conftest import load_golden
from oracle import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def test_engine_matches_reference_golden():
    from ape_b200.modeling.text import TextTransformer

    g = load_golden("text_tower_small.npz")
    m = TextTransformer(context_length=77, vocab_size=1000, width=128, heads=2, layers=3, output_dim=64).eval()
    synth.fill_state_dict(m)
    m = m.to(DEV)
    with torch.no_grad():
        eot, xx = m.encode(g["tokens"].to(DEV))
    rms = g["eot"].pow(2).mean().sqrt().item()
    err = (eot.cpu() - g["eot"]).abs().max().item()
    print(f"text tower fp16 engine vs reference golden: max|err| {err:.3e} on rms {rms:.3e}")
    assert err < 5e-3 * max(rms, 1e-3) + 1e-4
    assert (xx.cpu()[:, ::7] - g["all"]).abs().max().item() < 5e-3 * max(rms, 1e-3) + 1e-4


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_engine_at_bigE_geometry_matches_literal_fp32(dtype):
    from ape_b200.modeling.text import TextTransformer

    m = TextTransformer(context_length=77, vocab_size=2000, width=1280, heads=20, layers=2, output_dim=1024).eval()
    synth.fill_state_dict(m)
    m = m.to(DEV)
    g = torch.Generator().manual_seed(0)
    tok = torch.randint(1, 1998, (33, 77), generator=g)
    tok[:, 50:] = 0
    tok[torch.arange(33), torch.randint(2, 50, (33,), generator=g)] = 1999
    tok = tok.to(DEV)
    with torch.no_grad():
        m.engine_dtype = None
        want, want_all = m.encode(tok)
        m.engine_dtype = dtype
        got, got_all = m.encode(tok)
    tol = 4e-3 if dtype == torch.float16 else 3e-2
    rms = want.pow(2).mean().sqrt().item()
    assert (got - want).abs().max().item() < tol * max(rms, 1.0)
    end = tok.argmax(-1)
    keep = torch.arange(77, device=DEV)[None] <= end[:, None]  # positions after the end-of-text token are unconstrained padding
    assert ((got_all - want_all).abs() * keep[..., None]).max().item() < tol * max(rms, 1.0)
