"""GPU: the ping-pong GEMM kernel (gemm_pp_kernel, ape_b200/csrc/gemm_tc.cu) computes the same bits as the cooperative one.

tile_n bit 0x8000 forces the ping-pong kernel and 0x10000 the cooperative one.  Both run the same MMAs in the same k
order and the same epilogue code, so every output — including the SwiGLU row statistics and the class-argmax keys — must
be equal bit for bit.  Covered: every epilogue of APE_GEMM_EPILOGUES in fp16 and bf16, k-block counts that do and do
not divide the 6-stage ring (the stage / phase of a warpgroup's k-block comes from the CTA's running k-block index),
one tile (warpgroup 1 idle), odd and many tiles per CTA, ragged M / N, an output without paired stores, and a CUDA graph
replay."""
import threading

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PP, COOP = 0x8000, 0x10000


@pytest.fixture(scope="module")
def ops():
    import ape_b200

    return ape_b200.ops


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def rnd(*shape, dtype, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).to(DEV)


def both(fn):
    """fn(tile_n) under the forced ping-pong and the forced cooperative kernel; every returned tensor equal."""
    a, b = fn(PP), fn(COOP)
    torch.cuda.synchronize()
    a = a if isinstance(a, tuple) else (a,)
    b = b if isinstance(b, tuple) else (b,)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    return a


# (16-bit output?, act, residual) of APE_GEMM_EPILOGUES without LayerNorm fold, RoPE or statistics
PLAIN = [
    (True, None, None), (True, "relu", None), (True, "gelu", None), (True, None, "f32"), (True, None, "16"),
    (True, "relu", "16"), (True, "gelu", "16"), (True, "swiglu", None),
    (False, None, None), (False, "relu", None), (False, "gelu", None), (False, "swiglu", None), (False, "clamp", None),
    (False, None, "f32"), (False, None, "16"),
]
# interior tiles, many per CTA; ragged M and N
SHAPES = [(4096, 1024, 256), (3001, 904, 320)]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("out16,act,res", PLAIN)
def test_plain_epilogues(ops, dtype, M, N, K, out16, act, res):
    x = rnd(M, K, dtype=dtype, seed=1)
    w = rnd(N, K, dtype=dtype, seed=2, scale=K ** -0.5)
    b = rnd(N, dtype=torch.float32, seed=3)
    n_out = N // 2 if act == "swiglu" else N
    r = None if res is None else rnd(M, n_out, dtype=torch.float32 if res == "f32" else dtype, seed=4)
    both(lambda t: ops.linear_tc(x, w, b, act=act, residual=r, out_dtype=None if out16 else torch.float32, tile_n=t))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_swiglu_stats(ops, dtype, M, N, K):
    x = rnd(M, K, dtype=dtype, seed=5)
    w = rnd(N, K, dtype=dtype, seed=6, scale=K ** -0.5)
    b = rnd(N, dtype=torch.float32, seed=7)
    both(lambda t: ops.linear_tc(x, w, b, act="swiglu", stats_out=True, tile_n=t))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_layernorm_fold(ops, dtype, M, N, K):
    x = rnd(M, K, dtype=dtype, seed=8)
    w = rnd(N, K, dtype=dtype, seed=9, scale=K ** -0.5)
    b = rnd(N, dtype=torch.float32, seed=10)
    part = torch.rand(M, 3, 2, device=DEV)  # (sum, sum of squares) partials: any non-negative values exercise the fold
    colsum = w.float().sum(1)
    r = rnd(M, N, dtype=torch.float32, seed=11)
    both(lambda t: ops.linear_tc(x, w, b, residual=r, out_dtype=torch.float32, ln_fold=(part, colsum, K, 1e-6), tile_n=t))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("with_pos", [False, True])
def test_rope(ops, dtype, with_pos):
    from ape_b200 import _lib

    M, C, K, npos = 4096, 256, 256, 1024
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

    both(run)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_argmax_keys(ops, dtype):
    """ape_gemm_tn_argmax picks the kernel by tile count: one call over all rows (ping-pong) against row chunks of 8 row
    blocks (the cooperative kernel), into the same kind of key buffer."""
    from ape_b200 import _lib

    M, N, K, col_base = 40000, 1203, 320, 5
    x = rnd(M, K, dtype=dtype, seed=15)
    w = rnd(N, K, dtype=dtype, seed=16, scale=K ** -0.5)
    st = _lib.current_stream_ptr()

    def call(keys, r0, nr):
        rc = _lib.lib.ape_gemm_tn_argmax(x[r0:].data_ptr(), K, w.data_ptr(), K, keys[r0:].data_ptr(), nr, N, K, col_base,
                                         _lib.dtype_code(dtype), st)
        _lib.check(rc, "ape_gemm_tn_argmax")

    whole = torch.zeros(M, dtype=torch.int64, device=DEV)
    call(whole, 0, M)
    chunked = torch.zeros(M, dtype=torch.int64, device=DEV)
    for r0 in range(0, M, 1024):
        call(chunked, r0, min(1024, M - r0))
    torch.cuda.synchronize()
    assert torch.equal(whole, chunked)
    # and the keys name the class torch.argmax finds on the fp32 product (first maximum)
    y = ops.linear_tc(x, w, out_dtype=torch.float32, tile_n=COOP)
    assert torch.equal((0xFFFFFFFF - (whole & 0xFFFFFFFF)) - col_base, y.argmax(1))


@pytest.mark.parametrize("k_blocks", [1, 2, 3, 4, 5, 7, 16])
def test_k_blocks(ops, k_blocks):
    M, N = 4096, 768  # 32 x 6 = 192 tiles: one or two per CTA
    K = 64 * k_blocks
    x = rnd(M, K, dtype=torch.float16, seed=17)
    w = rnd(N, K, dtype=torch.float16, seed=18, scale=K ** -0.5)
    b = rnd(N, dtype=torch.float32, seed=19)
    both(lambda t: ops.linear_tc(x, w, b, act="relu", tile_n=t))
    # K not a multiple of 64: the last k-block is partly TMA zero fill
    x2, w2 = x[:, : K - 24].contiguous(), w[:, : K - 24].contiguous()
    both(lambda t: ops.linear_tc(x2, w2, b, out_dtype=torch.float32, tile_n=t))


@pytest.mark.parametrize("tiles_per_cta", ["one_tile", 1, 2, 3, 7, "many"])
def test_tiles_per_cta(ops, sms, tiles_per_cta):
    N, K = 256, 320  # 2 column blocks, 5 k-blocks (not a divisor of the 6 stages)
    if tiles_per_cta == "one_tile":
        M = 100  # a single tile: warpgroup 1 has none
    elif tiles_per_cta == "many":
        M = 87296
    else:
        M = 128 * sms * tiles_per_cta // 2 - 77  # ragged last row block
    x = rnd(M, K, dtype=torch.bfloat16, seed=20)
    w = rnd(N, K, dtype=torch.bfloat16, seed=21, scale=K ** -0.5)
    r = rnd(M, N, dtype=torch.bfloat16, seed=22)
    both(lambda t: ops.linear_tc(x, w, None, act="gelu", residual=r, tile_n=t))


@pytest.mark.parametrize("out16", [True, False])
def test_output_without_paired_stores(ops, out16):
    M, N, K = 5000, 384, 256
    x = rnd(M, K, dtype=torch.float16, seed=23)
    w = rnd(N, K, dtype=torch.float16, seed=24, scale=K ** -0.5)
    b = rnd(N, dtype=torch.float32, seed=25)
    odt = torch.float16 if out16 else torch.float32

    def run(t):
        flat = torch.zeros(1 + M * (N + 1), dtype=odt, device=DEV)
        out = flat[1:].view(M, N + 1)[:, :N]
        ops.linear_tc(x, w, b, act="relu", out=out, tile_n=t)
        return flat

    flat = both(run)[0]
    assert torch.equal(flat[1:].view(M, N + 1)[:, :N], ops.linear_tc(x, w, b, act="relu", out_dtype=odt, tile_n=COOP))


def test_default_dispatch_and_flags(ops, sms):
    """Without flags the kernel is chosen by tile count; either way the result is the cooperative kernel's."""
    K = 256
    w = rnd(256, K, dtype=torch.float16, seed=26, scale=K ** -0.5)
    for M in (900, 128 * sms, 4 * 128 * sms):
        x = rnd(M, K, dtype=torch.float16, seed=27)
        assert torch.equal(ops.linear_tc(x, w), ops.linear_tc(x, w, tile_n=COOP))
    x = rnd(512, K, dtype=torch.float16, seed=28)
    rejected = []

    def bad_flags():  # on a thread of its own: the per-thread ape_last_error() text of the test process stays empty
        for bad in (PP | COOP, PP | 256, PP | 0x4000):
            try:
                ops.linear_tc(x, w, tile_n=bad)
            except RuntimeError:
                rejected.append(bad)

    t = threading.Thread(target=bad_flags)
    t.start()
    t.join()
    assert rejected == [PP | COOP, PP | 256, PP | 0x4000]


def test_graph_replay_equals_eager(ops):
    M, N, K = 20000, 512, 256
    x = rnd(M, K, dtype=torch.float16, seed=29)
    w = rnd(N, K, dtype=torch.float16, seed=30, scale=K ** -0.5)
    b = rnd(N, dtype=torch.float32, seed=31)
    out = torch.empty(M, N, dtype=torch.float16, device=DEV)
    eager = ops.linear_tc(x, w, b, act="relu", tile_n=PP)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.linear_tc(x, w, b, act="relu", out=out, tile_n=PP)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.linear_tc(x, w, b, act="relu", out=out, tile_n=PP)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
