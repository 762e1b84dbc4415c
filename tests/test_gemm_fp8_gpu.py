"""GPU: the FP8 GEMM (ape_gemm_tn_e4m3 / ops.linear_fp8) against a float64 emulation.

The emulation is (A_q s_a)(W_q s_w)^T followed by the same epilogue in float64.  Products of e4m3 values are exact, so what
is left is how the sum is formed and the final rounding to 16 bit.  Within a 128-wide k-block the sum is the tensor cores'
FP8 accumulation, which keeps only about 13 to 14 bits of the running sum (not fp32); the kernel promotes it into an fp32
register accumulator after every k-block, so that error does not grow with K.  Per element:
    |got - ref| <= half an ulp of the 16-bit output at |ref|  +  C_SUM * 2^-24 * sum_k |a_k w_k|   (scaled values)
Each case prints the measured factor (the excess over the output rounding, in units of 2^-24 sum_k |a_k w_k|)."""
import threading

import pytest
import torch

from ape_b200 import _lib, ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS32 = 2.0 ** -24
# Bound on the summation error in units of 2^-24 sum_k |a_k w_k| (2^-11 of it).  On an H100 80GB HBM3 the largest factor over
# the 116 cases of this file was 5277 (4096 x 5460 x 128, fp16 output), about 2^-11.6 of sum_k |a_k w_k|: the tensor cores'
# FP8 accumulation inside one k-block.  With K = 1024 (8 promotions) no case exceeded 1000.
C_SUM = 8192.0
HALF_ULP = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
SUBNORMAL = {torch.float16: 2.0 ** -25, torch.bfloat16: 2.0 ** -134}


def _operands(M, N, K, seed, swiglu=False):
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = torch.randn(M, K, device=DEV, generator=g) * torch.rand(M, 1, device=DEV, generator=g) * 4
    w = torch.randn(N, K, device=DEV, generator=g) * K ** -0.5
    bias = torch.randn(N, device=DEV, generator=g) * 0.5
    aq, sa = ops.quantize_rows_e4m3(a)
    wq, sw = ops.quantize_rows_e4m3(w)
    return aq, sa, wq, sw, bias


def _emulate(aq, sa, wq, sw, bias):
    """float64 (A_q s_a)(W_q s_w)^T + bias, and sum_k |a_k w_k| of the scaled operands."""
    a = aq.double() * sa.double()[:, None]
    w = wq.double() * sw.double()[:, None]
    return a @ w.T + bias.double()[None, :], a.abs() @ w.abs().T


def _excess(got, ref, mag, dtype, extra=0.0):
    """max over elements of (|got - ref| - output rounding) / (2^-24 sum_k |a_k w_k|)."""
    rounding = HALF_ULP[dtype] * ref.abs() + SUBNORMAL[dtype] + extra
    ex = ((got.double() - ref).abs() - rounding).clamp_min(0) / (EPS32 * mag + 1e-30)
    return ex.max().item()


MEASURED = []

SHAPES = [(M, N, K) for M in (1, 127, 4096, 8192) for N in (128, 3072, 5460) for K in (128, 1024)]


@pytest.mark.parametrize("M,N,K", SHAPES, ids=[f"{m}x{n}x{k}" for m, n, k in SHAPES])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_bias_epilogue_matches_float64(dtype, M, N, K):
    aq, sa, wq, sw, bias = _operands(M, N, K, seed=M + N + K)
    got = ops.linear_fp8(aq, sa, wq, sw, bias, out_dtype=dtype)
    torch.cuda.synchronize()
    ref, mag = _emulate(aq, sa, wq, sw, bias)
    assert got.dtype == dtype and got.shape == (M, N) and torch.isfinite(got).all()
    ex = _excess(got, ref, mag, dtype)
    MEASURED.append(ex)
    print(f"  {M}x{N}x{K} {dtype}: summation error <= {ex:.2f} x 2^-24 sum|a w|")
    assert ex <= C_SUM


@pytest.mark.parametrize("M,N,K", [s for s in SHAPES if s[1] != 128] + [(4096, 128, 1024)],
                         ids=[f"{m}x{n}x{k}" for m, n, k in [s for s in SHAPES if s[1] != 128] + [(4096, 128, 1024)]])
@pytest.mark.parametrize("stats", [False, True], ids=["plain", "stats"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_swiglu_epilogue_matches_float64(dtype, stats, M, N, K):
    aq, sa, wq, sw, bias = _operands(M, N, K, seed=7 * M + N + K)
    res = ops.linear_fp8(aq, sa, wq, sw, bias, act="swiglu", stats_out=stats, out_dtype=dtype)
    got, st = res if stats else (res, None)
    torch.cuda.synchronize()
    ref, mag = _emulate(aq, sa, wq, sw, bias)
    gate, up = ref[:, 0::2], ref[:, 1::2]
    sig = torch.sigmoid(gate)
    y = gate * sig * up
    # first-order propagation of the gate / up errors through silu(gate) * up, plus the fast exp of the epilogue
    dsilu = (sig * (1 + gate * (1 - sig))).abs()
    mag_y = dsilu * up.abs() * mag[:, 0::2] + (gate * sig).abs() * mag[:, 1::2]
    assert got.shape == (M, N // 2) and torch.isfinite(got).all()
    ex = _excess(got, y, mag_y, dtype, extra=1e-5 * y.abs())
    MEASURED.append(ex)
    print(f"  swiglu {M}x{N}x{K} {dtype} stats={stats}: summation error <= {ex:.2f} x 2^-24 sum|a w|")
    assert ex <= C_SUM
    if stats:
        # the slab statistics of the values as stored, as the 16-bit kernel forms them from its output
        n_out = N // 2
        nslab = (n_out + 63) // 64
        v = torch.zeros(M, nslab * 64, dtype=torch.float64, device=DEV)
        v[:, :n_out] = got.double()
        v = v.view(M, nslab, 64)
        want = torch.stack([v.sum(-1), (v * v).sum(-1)], -1)
        scale = torch.stack([v.abs().sum(-1), (v * v).sum(-1)], -1)
        assert st.shape == (M, nslab, 2)
        assert ((st.double() - want).abs() <= 1e-5 * scale + 1e-30).all()


def test_sum_error_within_bound():
    if MEASURED:
        print(f"\n  largest summation error over {len(MEASURED)} cases: {max(MEASURED):.2f} x 2^-24 sum|a w| (bound {C_SUM})")


@pytest.mark.parametrize("act", [None, "swiglu"])
@pytest.mark.parametrize("M", [1, 127, 200])
def test_rows_and_columns_outside_the_output_are_not_written(M, act):
    N, K = 3072, 1024
    aq, sa, wq, sw, bias = _operands(M, N, K, seed=3)
    n_out = N // 2 if act else N
    buf = torch.full((M + 130, n_out + 8), 7.0, dtype=torch.float16, device=DEV)
    ops.linear_fp8(aq, sa, wq, sw, bias, act=act, out=buf[:M, :n_out])
    want = ops.linear_fp8(aq, sa, wq, sw, bias, act=act)
    torch.cuda.synchronize()
    assert torch.equal(buf[:M, :n_out], want)
    assert (buf[M:] == 7.0).all() and (buf[:, n_out:] == 7.0).all()


def test_cuda_graph_replay_equals_eager():
    aq, sa, wq, sw, bias = _operands(4096, 5460, 1024, seed=11)
    out = torch.empty(4096, 2730, dtype=torch.bfloat16, device=DEV)
    eager, st = ops.linear_fp8(aq, sa, wq, sw, bias, act="swiglu", stats_out=True, out_dtype=torch.bfloat16)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.linear_fp8(aq, sa, wq, sw, bias, act="swiglu", out=out)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.linear_fp8(aq, sa, wq, sw, bias, act="swiglu", out=out)
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)


def test_bad_arguments_are_rejected():
    lib = _lib.lib
    M, N, K = 256, 256, 128
    a = torch.zeros(M, K + 16, dtype=torch.float8_e4m3fn, device=DEV)
    w = torch.zeros(N, K, dtype=torch.float8_e4m3fn, device=DEV)
    sa = torch.ones(M, device=DEV)
    sw = torch.ones(N, device=DEV)
    c = torch.empty(M, N, dtype=torch.float16, device=DEV)
    stats = torch.empty(M, 2, 2, device=DEV)
    F16, F32 = _lib.APE_DTYPE_F16, _lib.APE_DTYPE_F32
    base = dict(A=a.data_ptr(), lda=K + 16, W=w.data_ptr(), ldw=K, sa=sa.data_ptr(), sw=sw.data_ptr(), C=c.data_ptr(), ldc=N,
                bias=None, M=M, N=N, K=K, out=F16, act=0, stats=None, nslab=0)
    cases = [  # (changes, status, text in ape_last_error())
        (dict(K=120), -1, "multiple of 16"),
        (dict(lda=K + 8), -1, "16-byte aligned"),
        (dict(A=a.data_ptr() + 8), -1, "16-byte aligned"),
        (dict(sa=None), -3, "null scale"),
        (dict(sw=None), -3, "null scale"),
        (dict(out=F32), -2, "fp16 or bf16"),
        (dict(act=1), -2, "activation 1"),
        (dict(stats=stats.data_ptr(), nslab=2), -1, "stats"),
        (dict(act=3, stats=stats.data_ptr(), nslab=1), -1, "stats"),
        (dict(A=None), -3, "null pointer"),
    ]
    results = []

    def reject_all():  # on a thread of its own: ape_last_error() is per thread, and this one's text dies with it
        for change, _, _ in cases:
            q = dict(base, **change)
            rc = lib.ape_gemm_tn_e4m3(q["A"], q["lda"], q["W"], q["ldw"], q["sa"], q["sw"], q["C"], q["ldc"], q["bias"], q["M"],
                                      q["N"], q["K"], q["out"], q["act"], q["stats"], q["nslab"], None)
            results.append((rc, lib.ape_last_error().decode()))

    t = threading.Thread(target=reject_all)
    t.start()
    t.join()
    for (change, status, text), (rc, msg) in zip(cases, results):
        assert rc == status and text in msg, (change, rc, msg)
    with pytest.raises(RuntimeError, match="e4m3 operands"):
        ops.linear_fp8(a[:, :K].to(torch.float16), sa, w, sw)
