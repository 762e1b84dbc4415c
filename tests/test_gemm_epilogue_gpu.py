"""GPU: every compile-time epilogue variant of the wgmma GEMM (ape_b200/csrc/gemm_tc.cu, APE_GEMM_EPILOGUES) against a
PyTorch fp32 reference, on interior-only tiles (the unguarded epilogue), ragged M / N (the guarded one), many tiles per
CTA (the grouped tile order), a padded output pitch and an output without paired stores; combinations without a kernel
are rejected."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def ops():
    import ape_b200

    return ape_b200.ops


def rnd(*shape, dtype, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).to(DEV)


def ref(x, w, b, act, res):
    y = F.linear(x.float(), w.float(), b)
    if act == "relu":
        y = F.relu(y)
    elif act == "gelu":
        y = F.gelu(y)
    elif act == "clamp":
        y = y.clamp(-50000.0, 50000.0)
    elif act == "swiglu":
        y = F.silu(y[..., 0::2]) * y[..., 1::2]
    return y if res is None else y + res.float()


# (16-bit output?, act, residual: None / "f32" / "16"): the variants without LayerNorm fold or rotary embedding
VARIANTS = [
    (True, None, None), (True, "relu", None), (True, "gelu", None), (True, None, "f32"), (True, None, "16"),
    (True, "relu", "16"), (True, "gelu", "16"), (True, "swiglu", None),
    (False, None, None), (False, "relu", None), (False, "gelu", None), (False, "swiglu", None), (False, "clamp", None),
    (False, None, "f32"), (False, None, "16"),
]
SHAPES = [(512, 384, 192), (777, 840, 200), (20000, 1024, 128)]  # interior only; ragged M and N; many tiles per CTA


def check(got, want, out16, dtype):
    tol = (3e-2 if dtype == torch.bfloat16 else 4e-3) if out16 else 2e-4
    torch.testing.assert_close(got.float(), want, rtol=tol, atol=tol)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("out16,act,res", VARIANTS)
def test_epilogue_variant(ops, dtype, M, N, K, out16, act, res):
    x = rnd(M, K, dtype=dtype, seed=1)
    w = rnd(N, K, dtype=dtype, seed=2, scale=K ** -0.5)
    b = rnd(N, dtype=torch.float32, seed=3)
    n_out = N // 2 if act == "swiglu" else N
    r = None if res is None else rnd(M, n_out, dtype=torch.float32 if res == "f32" else dtype, seed=4)
    y = ops.linear_tc(x, w, b, act=act, residual=r, out_dtype=None if out16 else torch.float32)
    check(y, ref(x, w, b, act, r), out16, dtype)
    # without bias, into a padded-pitch view: the columns past n_out stay untouched
    buf = torch.full((M, n_out + 24), 7.0, dtype=dtype if out16 else torch.float32, device=DEV)
    y = ops.linear_tc(x, w, None, act=act, residual=r, out=buf[:, :n_out])
    check(y, ref(x, w, None, act, r), out16, dtype)
    assert (buf[:, n_out:] == 7.0).all()


@pytest.mark.parametrize("out16", [True, False])
def test_output_without_paired_stores(ops, out16):
    """An odd output pitch and a base one element off alignment: every tile takes the guarded epilogue, same values."""
    M, N, K = 640, 384, 256
    dtype = torch.float16
    x = rnd(M, K, dtype=dtype, seed=5)
    w = rnd(N, K, dtype=dtype, seed=6, scale=K ** -0.5)
    b = rnd(N, dtype=torch.float32, seed=7)
    odt = dtype if out16 else torch.float32
    aligned = ops.linear_tc(x, w, b, act="relu", out_dtype=odt)
    flat = torch.zeros(1 + M * (N + 1), dtype=odt, device=DEV)
    out = flat[1:].view(M, N + 1)[:, :N]
    ops.linear_tc(x, w, b, act="relu", out=out)
    assert torch.equal(out, aligned)


def test_residual_without_paired_loads(ops):
    M, N, K = 512, 256, 128
    x = rnd(M, K, dtype=torch.float16, seed=8)
    w = rnd(N, K, dtype=torch.float16, seed=9, scale=K ** -0.5)
    r = rnd(M, N + 1, dtype=torch.float32, seed=10)[:, 1:]  # odd pitch and offset
    y = ops.linear_tc(x, w, None, residual=r, out_dtype=torch.float32)
    torch.testing.assert_close(y, ref(x, w, None, None, r), rtol=2e-4, atol=2e-4)


def test_combinations_without_kernel_are_rejected(ops):
    x = rnd(256, 128, dtype=torch.float16, seed=11)
    w = rnd(256, 128, dtype=torch.float16, seed=12)
    with pytest.raises(RuntimeError):  # residual of the other 16-bit type
        ops.linear_tc(x, w, residual=rnd(256, 256, dtype=torch.bfloat16, seed=13))
    with pytest.raises(RuntimeError):  # 16-bit output of the other 16-bit type
        ops.linear_tc(x, w, out_dtype=torch.bfloat16)
    with pytest.raises(RuntimeError):  # activation and residual together under an fp32 output
        ops.linear_tc(x, w, act="gelu", residual=rnd(256, 256, dtype=torch.float32, seed=14), out_dtype=torch.float32)
