"""GPU: the LayerNorm with an e4m3 output and a scale per row (ape_layernorm_e4m3 / ops.layernorm(out_dtype=float8_e4m3fn))
against torch's fp32 F.layer_norm: s = max|row| / 448, and q * s within half an e4m3 ulp of the LayerNorm output
(plus the fp32 difference between the two LayerNorms, at most 1e-5 of the row maximum)."""
import pytest
import torch
import torch.nn.functional as F

from ape_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
E4M3 = torch.float8_e4m3fn


def _inputs(rows, C, dtype, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = (torch.randn(rows, C, device=DEV, generator=g) * 3 + torch.randn(rows, 1, device=DEV, generator=g)).to(dtype)
    w = torch.randn(C, device=DEV, generator=g) * 0.5 + 1
    b = torch.randn(C, device=DEV, generator=g) * 0.2
    return x, w, b


def _check(q, s, y):
    """q e4m3 [rows, C], s fp32 [rows] against the fp32 LayerNorm output y [rows, C]."""
    amax = y.abs().amax(1)
    want_s = amax / 448
    assert ((s - want_s).abs() <= 1e-6 * want_s).all(), (s - want_s).abs().max().item()
    t = torch.where(s[:, None] > 0, y / s[:, None].clamp_min(1e-30), torch.zeros_like(y))  # the exact e4m3-domain value
    exp = torch.floor(torch.log2(t.abs().clamp_min(2.0 ** -9))).clamp_min(-6)  # e4m3: 3 mantissa bits, min normal 2^-6
    half_ulp = 2.0 ** (exp - 4)
    # slack: t is formed from torch's LayerNorm, whose fp32 rounding differs from the kernel's by a few ulps of the row
    # maximum (448 in this domain), so a value near a rounding midpoint may round to the other neighbour
    err = (q.float() - t).abs()
    excess = (err - half_ulp).clamp_min(0).max().item()
    assert excess <= 1e-5 * 448, excess
    assert (q.float().abs() <= 448).all()


@pytest.mark.parametrize("C", [64, 256, 1000, 1024])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=["f32", "f16", "bf16"])
def test_scale_and_values_match_torch(dtype, C):
    x, w, b = _inputs(4099, C, dtype, seed=C)
    q, s = ops.layernorm(x, w, b, eps=1e-6, out_dtype=E4M3)
    torch.cuda.synchronize()
    assert q.dtype == E4M3 and q.shape == (4099, C) and s.shape == (4099,) and s.dtype == torch.float32
    _check(q, s, F.layer_norm(x.float(), (C,), w, b, 1e-6))


def test_all_zero_row_has_zero_scale_and_values():
    C = 1024
    x, w, b = _inputs(64, C, torch.float32, seed=1)
    x[5] = 2.5  # constant row: LN(x) = bias, which is zero here
    x[9] = 0.0
    b = torch.zeros_like(b)
    q, s = ops.layernorm(x, w, b, eps=1e-6, out_dtype=E4M3)
    torch.cuda.synchronize()
    assert s[5].item() == 0.0 and s[9].item() == 0.0
    assert (q[5].float() == 0).all() and (q[9].float() == 0).all()
    y = F.layer_norm(x, (C,), w, b, 1e-6)
    keep = torch.ones(64, dtype=torch.bool, device=DEV)
    keep[[5, 9]] = False
    _check(q[keep], s[keep], y[keep])


def test_row_map_scatters_values_and_scales():
    rows, C = 1000, 1024
    x, w, b = _inputs(rows, C, torch.float32, seed=2)
    perm = torch.randperm(rows + 24, generator=torch.Generator().manual_seed(0))[:rows].to(DEV, torch.int32)
    out = torch.full((rows + 24, C), 1.0, device=DEV).to(E4M3)
    sc = torch.full((rows + 24,), -1.0, device=DEV)
    q, s = ops.layernorm(x, w, b, eps=1e-6, row_map=perm, out=out, scale_out=sc)
    torch.cuda.synchronize()
    assert q is out and s is sc
    pl = perm.long()
    _check(out[pl], sc[pl], F.layer_norm(x, (C,), w, b, 1e-6))
    untouched = torch.ones(rows + 24, dtype=torch.bool, device=DEV)
    untouched[pl] = False
    assert (sc[untouched] == -1).all() and (out[untouched].float() == 1).all()
    # the plain form writes the same bytes, in input order
    q2, s2 = ops.layernorm(x, w, b, eps=1e-6, out_dtype=E4M3)
    assert torch.equal(q2.view(torch.uint8), out[pl].view(torch.uint8)) and torch.equal(s2, sc[pl])


def test_padding_columns_are_written_as_zero():
    rows, C = 300, 1001  # pitch 1008 bytes: the last 8-byte vector holds 7 padding bytes
    x, w, b = _inputs(rows, 1008, torch.float32, seed=3)
    x, w, b = x[:, :C], w[:C].contiguous(), b[:C].contiguous()  # input rows padded to 1008 elements as well
    buf = torch.full((rows, 1008), 3.0, device=DEV).to(E4M3)
    ops.layernorm(x, w, b, eps=1e-6, out=buf[:, :C])
    torch.cuda.synchronize()
    assert (buf[:, C:].float() == 0).all()
    _check(buf[:, :C], ops.layernorm(x, w, b, eps=1e-6, out_dtype=E4M3)[1], F.layer_norm(x, (C,), w, b, 1e-6))
