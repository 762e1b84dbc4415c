"""GPU: 128 x 256 GEMM tiles (gemm_tc_kernel with BN = 256, single CTA and cluster of two) compute the same bits as the
128 x 128 cooperative kernel.

tile_n 256 | 0x1000 pins the wide tile on one CTA, 256 | 0x4000 in a cluster of two along M that multicasts the weight
tile, and 0x10000 | 0x1000 the 128-wide cooperative kernel on one CTA.  Every output element is the same k-ordered wgmma
chain whatever the MMA's N, the SwiGLU statistics are per 64-column slab and the LayerNorm fold reads its partials in a
fixed order, so every output must be equal bit for bit.  Covered: every epilogue of APE_GEMM_EPILOGUES in fp16 and bf16;
an odd number of 128-row blocks (the second CTA of the last cluster has no rows); N = 5460 and N = 300; K not a multiple
of 64; RoPE with and without a row -> position map; SwiGLU statistics; the LayerNorm fold; fp32 output with a 16-bit
residual; an output pitch without paired stores; the shape rule's default dispatch; and a CUDA graph replay."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REF = 0x10000 | 0x1000
WIDE = {"cl1": 256 | 0x1000, "cl2": 256 | 0x4000}


@pytest.fixture(scope="module")
def ops():
    import ape_b200

    return ape_b200.ops


def rnd(*shape, dtype, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).to(DEV)


def rnd_pitched(rows, K, dtype, seed, scale=1.0):
    """rnd(rows, K) as a view with a 16-byte row pitch, as the ViT's w3 operands (K = 2730) have."""
    kp = -(-K // 8) * 8
    t = torch.zeros(rows, kp, dtype=dtype, device=DEV)[:, :K]
    t.copy_(rnd(rows, K, dtype=dtype, seed=seed, scale=scale))
    return t


def same_as_ref(fn):
    """fn(tile_n) under the 128-wide cooperative kernel and both wide arms; every returned tensor equal."""
    ref = fn(REF)
    ref = ref if isinstance(ref, tuple) else (ref,)
    for bits in WIDE.values():
        got = fn(bits)
        got = got if isinstance(got, tuple) else (got,)
        torch.cuda.synchronize()
        for x, y in zip(ref, got):
            assert torch.equal(x, y), hex(bits)
    return ref


# (16-bit output?, act, residual) of APE_GEMM_EPILOGUES without LayerNorm fold, RoPE or statistics
PLAIN = [
    (True, None, None), (True, "relu", None), (True, "gelu", None), (True, None, "f32"), (True, None, "16"),
    (True, "relu", "16"), (True, "gelu", "16"), (True, "swiglu", None),
    (False, None, None), (False, "relu", None), (False, "gelu", None), (False, "swiglu", None), (False, "clamp", None),
    (False, None, "f32"), (False, None, "16"),
]
# interior tiles (unguarded epilogue); 5 row blocks with N = 5460 and K = 1000; 5 row blocks with N = 300 and K = 200
SHAPES = [(2048, 1024, 512), (603, 5460, 1000), (600, 300, 200)]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("out16,act,res", PLAIN)
def test_plain_epilogues(ops, dtype, M, N, K, out16, act, res):
    x = rnd(M, K, dtype=dtype, seed=1)
    w = rnd(N, K, dtype=dtype, seed=2, scale=K ** -0.5)
    b = rnd(N, dtype=torch.float32, seed=3)
    n_out = N // 2 if act == "swiglu" else N
    r = None if res is None else rnd(M, n_out, dtype=torch.float32 if res == "f32" else dtype, seed=4)
    same_as_ref(lambda t: ops.linear_tc(x, w, b, act=act, residual=r, out_dtype=None if out16 else torch.float32, tile_n=t))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_swiglu_stats(ops, dtype, M, N, K):
    x = rnd(M, K, dtype=dtype, seed=5)
    w = rnd(N, K, dtype=dtype, seed=6, scale=K ** -0.5)
    b = rnd(N, dtype=torch.float32, seed=7)
    same_as_ref(lambda t: ops.linear_tc(x, w, b, act="swiglu", stats_out=True, tile_n=t))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,N,K", SHAPES + [(4096, 1024, 2730)])
def test_layernorm_fold(ops, dtype, M, N, K):
    x = rnd_pitched(M, K, dtype, seed=8)
    w = rnd_pitched(N, K, dtype, seed=9, scale=K ** -0.5)
    b = rnd(N, dtype=torch.float32, seed=10)
    part = torch.rand(M, 4, 2, device=DEV)  # (sum, sum of squares) partials: any non-negative values exercise the fold
    colsum = w.float().sum(1)
    r = rnd(M, N, dtype=torch.float32, seed=11)
    same_as_ref(lambda t: ops.linear_tc(x, w, b, residual=r, out_dtype=torch.float32, ln_fold=(part, colsum, K, 1e-6), tile_n=t))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("with_pos", [False, True])
def test_rope(ops, dtype, with_pos):
    from ape_b200 import _lib

    M, C, K, npos = 603, 512, 320, 1024
    N = 3 * C
    x = rnd(M, K, dtype=dtype, seed=12)
    w = rnd(N, K, dtype=dtype, seed=13, scale=K ** -0.5)
    b = rnd(N, dtype=torch.float32, seed=14)
    ang = torch.rand(npos, 64, device=DEV) * 6.3
    cos, sin = ang.cos().contiguous(), ang.sin().contiguous()
    pos = torch.randint(0, npos, (M,), device=DEV, dtype=torch.int32) if with_pos else None

    def run(t):
        out = torch.empty(M, N, dtype=dtype, device=DEV)
        rc = _lib.lib.ape_gemm_tn_rope(x.data_ptr(), K, w.data_ptr(), K, out.data_ptr(), N, b.data_ptr(), M, N, K,
                                       _lib.dtype_code(dtype), _lib.dtype_code(dtype), cos.data_ptr(), sin.data_ptr(),
                                       pos.data_ptr() if pos is not None else None, npos, 64, 2 * C, t,
                                       _lib.current_stream_ptr())
        _lib.check(rc, "ape_gemm_tn_rope")
        return out

    same_as_ref(run)


@pytest.mark.parametrize("out16", [True, False])
def test_output_without_paired_stores(ops, out16):
    M, N, K = 1000, 1100, 512
    x = rnd(M, K, dtype=torch.float16, seed=15)
    w = rnd(N, K, dtype=torch.float16, seed=16, scale=K ** -0.5)
    b = rnd(N, dtype=torch.float32, seed=17)
    odt = torch.float16 if out16 else torch.float32

    def run(t):
        flat = torch.zeros(1 + M * (N + 1), dtype=odt, device=DEV)
        out = flat[1:].view(M, N + 1)[:, :N]
        ops.linear_tc(x, w, b, act="relu", out=out, tile_n=t)
        return flat

    flat = same_as_ref(run)[0]
    assert torch.equal(flat[1:].view(M, N + 1)[:, :N], ops.linear_tc(x, w, b, act="relu", out_dtype=odt, tile_n=REF))


@pytest.mark.parametrize("M,N,K", [(4096, 3072, 1024), (4096, 1024, 2730), (603, 2048, 2048), (900, 256, 2048),
                                   (87296, 256, 256)])
def test_default_dispatch(ops, M, N, K):
    """Without flags the shape rule picks the tile (128 x 256 on one CTA for N >= 1024, K >= 2048); the result is the
    128-wide cooperative kernel's."""
    x = rnd_pitched(M, K, torch.float16, seed=18)
    w = rnd_pitched(N, K, torch.float16, seed=19, scale=K ** -0.5)
    b = rnd(N, dtype=torch.float32, seed=20)
    assert torch.equal(ops.linear_tc(x, w, b), ops.linear_tc(x, w, b, tile_n=REF))


def test_graph_replay_equals_eager(ops):
    M, N, K = 4096, 1024, 2730  # the ViT w3 shape: 128 x 256 tiles by default
    x = rnd_pitched(M, K, torch.float16, seed=21)
    w = rnd_pitched(N, K, torch.float16, seed=22, scale=K ** -0.5)
    b = rnd(N, dtype=torch.float32, seed=23)
    out = torch.empty(M, N, dtype=torch.float16, device=DEV)
    eager = ops.linear_tc(x, w, b, tile_n=REF)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.linear_tc(x, w, b, out=out)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.linear_tc(x, w, b, out=out)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
