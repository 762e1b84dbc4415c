"""GPU: every online / split softmax kernel against a literal float64 softmax on adversarial scores (the constructors of
tests/test_softmax_edges_cpu.py design the scores exactly in the 16-bit operands): a maximum that rises in every key block,
a maximum only in the last (partial) block, one dominant key, exact ties, 1e3..1e4-nat magnitudes, whole blocks or chunks
120 nats below the maximum, masked keys holding +-6e4, and rows with a single key.

Bounds, from their causes (u = unit roundoff: 2^-11 for fp16, 2^-8 for bf16):
  * P rounded to 16 bit before the P.V MMA: u relative per weight, i.e. u * sum_k p_k |v_k|; in fp16 a weight below 2^-14
    is subnormal and rounds to a step of 2^-24, at most 2^-25 * |v_k| per key;
  * the output's own rounding: u * |out|;
  * fp32 arithmetic (ex2.approx, fp32 accumulation and rescales): 2^-20 * sum_k p_k |v_k|, far below the 16-bit terms.
A row with a single key returns its value row within 2 u, not exactly: the key's weight is 2^r with r the fp32 rounding
residual of the row maximum in the exp2 domain (up to 2^-11 at 1e4 nats), rounded to 16 bit for the P.V MMA while the
row sum keeps it in fp32 (P rounding), and then the output is rounded.
Cases that are bit-exact by construction use torch.equal: a masked key's content never reaches the result, and a row of
exact ties over 2^k keys with values of a representable mean returns that mean."""
import pytest
import torch

from test_softmax_edges_cpu import (KB, PATTERNS, MSDA_PATTERNS, U16, attn_qkv_case, cross_case, fold_pool_case,
                                    fold_vision_case, msda_case, msda_reference, pool_shapes, vlf_pool_case,
                                    vlf_pool_reference, vlf_pool_strip)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = [torch.float16, torch.bfloat16]
F32_SLOP = 2.0 ** -20


@pytest.fixture(scope="module", params=[0, 1], ids=["smemP", "tmemP"])
def ops(request):
    """attention_qkv cases run against both structures of the attention kernel (ape_attn_variant): P read by the P.V MMA
    from shared memory, or kept in registers as its A operand."""
    import ape_b200

    prev = ape_b200._lib.lib.ape_attn_variant(-1)
    ape_b200._lib.lib.ape_attn_variant(request.param)
    yield ape_b200.ops
    ape_b200._lib.lib.ape_attn_variant(prev)


@pytest.fixture(scope="module")
def plain_ops():
    import ape_b200

    return ape_b200.ops


def softmax_bound(p, av, out, dtype, n_keys, vmax):
    """Bound on |kernel - float64| for a 16-bit P.V softmax: av = sum_k p_k |v_k|, out = the float64 result, vmax = max |v|
    over the keys (for fp16's subnormal weights)."""
    u = U16[dtype]
    tol = (u + F32_SLOP) * av + u * out.abs() + 2.0 ** -24
    if dtype == torch.float16:
        tol = tol + n_keys * 2.0 ** -25 * vmax
    return tol


def assert_within(got, want, tol, what):
    err = (got.double() - want).abs()
    bad = ~(err <= tol)  # NaN fails
    if bad.any():
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside the bound; first at {i}: "
                             f"got {got[tuple(i)].item():.6g} want {want[tuple(i)].item():.6g} tol {tol[tuple(i)].item():.3g}; "
                             f"max err {err.nan_to_num(float('inf')).max().item():.3g}")


def check_softmax(got, sc, v, dtype, what):
    """got [..., M, D] against softmax(sc) @ v in float64; sc [..., M, K] (masked entries -inf), v [..., K, D]."""
    p = torch.softmax(sc, -1)
    want = p @ v
    tol = softmax_bound(p, p @ v.abs(), want, dtype, sc.shape[-1], v.abs().amax(-2, keepdim=True))
    assert_within(got, want, tol, what)
    return p, want


# ---------------------------------------------------------------------------------------------------------- attention_qkv
def _heads(x, rows, heads, which):
    """[rows, 3 * heads * 64] -> float64 [heads, rows, 64] of q (0), k (1) or v (2)."""
    C = heads * 64
    return x[:rows, which * C: (which + 1) * C].double().view(rows, heads, 64).transpose(0, 1)


def attn_reference_check(got, qkv, num_seq, n_valid, heads, stride, causal, dtype, what, scale=0.125):
    for s in range(num_seq):
        x = qkv[s * stride: s * stride + n_valid]
        q, k, v = (_heads(x, n_valid, heads, i) for i in range(3))
        sc = q @ k.transpose(-1, -2) * scale
        if causal:
            sc = sc.masked_fill(torch.ones(n_valid, n_valid, dtype=torch.bool, device=DEV).triu(1), float("-inf"))
        o = got[s * stride: s * stride + n_valid].view(n_valid, heads, 64).transpose(0, 1)
        check_softmax(o, sc, v, dtype, f"{what} seq {s}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n_valid", [128, 129, 900, 4096])
@pytest.mark.parametrize("pattern", PATTERNS)
def test_attention_qkv_patterns(ops, pattern, n_valid, dtype):
    """n = 4096 rows (32 key blocks of 64), keys >= n_valid padded with +-6e4: within the bound of the float64 softmax, and
    bit-identical to the same call with zeros in the padding."""
    n, heads = 4096, 2
    qkv, _ = attn_qkv_case(pattern, dtype, 1, n, n_valid, heads, seed=n_valid, pad_fill=6e4)
    qkv = qkv.to(DEV)
    got = ops.attention_qkv(qkv, 1, n, heads, 64, 0.125, n_valid=n_valid)
    attn_reference_check(got, qkv, 1, n_valid, heads, n, False, dtype, pattern)
    if n_valid < n:
        zeroed = qkv.clone()
        zeroed[n_valid:] = 0
        assert torch.equal(ops.attention_qkv(zeroed, 1, n, heads, 64, 0.125, n_valid=n_valid)[:n_valid], got[:n_valid])
    if pattern == "ties" and n_valid & (n_valid - 1) == 0:  # P = 1, l = 2^k, values of a representable mean
        mean = _heads(qkv, n_valid, heads, 2).mean(1, keepdim=True).expand(heads, n_valid, 64)
        assert torch.equal(got[:n_valid].view(n_valid, heads, 64).transpose(0, 1).double(), mean)


@pytest.mark.parametrize("dtype", DTYPES)
def test_attention_qkv_single_key(ops, dtype):
    """n_valid = 1: every row returns value row 0 (to the output rounding), whatever the 4095 padded rows hold."""
    n, heads = 4096, 2
    qkv, _ = attn_qkv_case("dominant", dtype, 1, n, 1, heads, seed=1, pad_fill=6e4)
    qkv = qkv.to(DEV)
    got = ops.attention_qkv(qkv, 1, n, heads, 64, 0.125, n_valid=1)
    v0 = qkv[0, 2 * heads * 64:].double()
    torch.testing.assert_close(got[0].double(), v0, rtol=2 * U16[dtype], atol=0)
    zeroed = qkv.clone()
    zeroed[1:] = 0
    assert torch.equal(ops.attention_qkv(zeroed, 1, n, heads, 64, 0.125, n_valid=1)[:1], got[:1])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("pattern", PATTERNS)
def test_attention_qkv_causal_packed(ops, pattern, dtype):
    """Causal sequences of 200 rows packed at a stride of 208 in 256-row tiles (text tower): the 8 rows between two
    sequences hold +-6e4 and change nothing; row 0 of every sequence returns its value row 0."""
    num_seq, n, n_valid, stride, heads = 3, 256, 200, 208, 2
    qkv, _ = attn_qkv_case(pattern, dtype, num_seq, n, n_valid, heads, seed=7, stride=stride, pad_fill=6e4)
    qkv = qkv.to(DEV)
    run = lambda x: ops.attention_qkv(x, num_seq, n, heads, 64, 0.125, n_valid=n_valid, seq_stride=stride, causal=True)
    got = run(qkv)
    attn_reference_check(got, qkv, num_seq, n_valid, heads, stride, True, dtype, pattern)
    zeroed = qkv.clone()
    valid = torch.zeros(qkv.shape[0], dtype=torch.bool, device=DEV)
    for s in range(num_seq):
        valid[s * stride: s * stride + n_valid] = True
        torch.testing.assert_close(got[s * stride].double(), qkv[s * stride, 2 * heads * 64:].double(), rtol=2 * U16[dtype], atol=0)
    zeroed[~valid] = 0
    assert torch.equal(run(zeroed)[valid], got[valid])


SEG_STARTS = [[0, 1, 6, 63, 64, 65, 100, 127], [0, 1, 127]]  # segment starts inside each 128-row tile


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("pattern", PATTERNS)
def test_attention_qkv_segments(ops, pattern, dtype):
    """Length-packed causal tiles (seg_start): segments of length 1 at rows 0, 63, 64 and 127, segments that start inside
    the second key block; the contents of another segment (+-6e4) never reach a row."""
    heads, n = 2, 128
    num_seq = len(SEG_STARTS)
    qkv, _ = attn_qkv_case(pattern, dtype, num_seq, n, n, heads, seed=11)
    qkv = qkv.to(DEV)
    seg = torch.empty(num_seq * n, dtype=torch.int32)
    for t, starts in enumerate(SEG_STARTS):
        for a, b in zip(starts, starts[1:] + [n]):
            seg[t * n + a: t * n + b] = a
    seg = seg.to(DEV)
    run = lambda x: ops.attention_qkv(x, num_seq, n, heads, 64, 0.125, causal=True, seg_start=seg)
    got = run(qkv)
    pos = torch.arange(n, device=DEV)
    for t in range(num_seq):
        x = qkv[t * n: (t + 1) * n]
        q, k, v = (_heads(x, n, heads, i) for i in range(3))
        lo = seg[t * n: (t + 1) * n].long()
        masked = (pos[None, :] > pos[:, None]) | (pos[None, :] < lo[:, None])
        sc = (q @ k.transpose(-1, -2) * 0.125).masked_fill(masked, float("-inf"))
        check_softmax(got[t * n: (t + 1) * n].view(n, heads, 64).transpose(0, 1), sc, v, dtype, f"{pattern} tile {t}")
    for r in (0, 63, 64, 127):  # single-key segments
        torch.testing.assert_close(got[r].double(), qkv[r, 2 * heads * 64:].double(), rtol=2 * U16[dtype], atol=0)
    other = qkv.clone()
    other[6:63] = torch.where(torch.rand(57, qkv.shape[1], device=DEV) < 0.5, -6e4, 6e4).to(dtype)
    keep = torch.ones(num_seq * n, dtype=torch.bool, device=DEV)
    keep[6:63] = False
    assert torch.equal(run(other)[keep], got[keep])


# -------------------------------------------------------------------------------------------------------- attention_cross
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("hd,nkv,n_valid", [(256, 4096, 1), (256, 4096, 129), (256, 4096, 1537), (256, 4096, 4096),
                                            (64, 1024, 900)])
@pytest.mark.parametrize("pattern", PATTERNS)
def test_attention_cross_patterns(plain_ops, pattern, hd, nkv, n_valid, dtype):
    """attn_xfwd: 256-channel heads (and 64), keys >= n_valid padded with +-6e4 in K and V: within the bound, and
    bit-identical to the same call with zeros in the padding."""
    num_seq, nq, heads = 1, 128, 2
    C = heads * hd
    q, k, v, _ = cross_case(pattern, dtype, num_seq, nq, nkv, n_valid, heads, hd, seed=n_valid + hd, pad_fill=6e4)
    q, k, v = q.to(DEV), k.to(DEV), v.to(DEV)
    run = lambda k_, v_: plain_ops.attention_cross(q, k_, v_, num_seq, nq, nkv, n_valid, heads, hd, hd ** -0.5)
    got = run(k, v)
    qh, kh, vh = (x.double().view(-1, heads, hd).transpose(0, 1) for x in (q, k[:n_valid], v[:n_valid]))
    check_softmax(got.view(nq, heads, hd).transpose(0, 1), qh @ kh.transpose(-1, -2) * hd ** -0.5, vh, dtype, pattern)
    if n_valid < nkv:
        k0, v0 = k.clone(), v.clone()
        k0[n_valid:] = 0
        v0[n_valid:] = 0
        assert torch.equal(run(k0, v0), got)


# ------------------------------------------------------------------------------------------------------ vlf_fold_vision
def fold_vision_reference_check(got, v, qa, u, qc, gamma, bias, dtype, what):
    vd, qd, ud = v.double(), qa.double(), u.double()
    p = torch.softmax(torch.einsum("bsc,bhnc->bhsn", vd, qd) + qc.double()[:, :, None, :], -1)
    O = torch.einsum("bhsn,bhnc->bsc", p, ud)
    av = torch.einsum("bhsn,bhnc->bsc", p, ud.abs())
    g, bb = gamma.double(), bias.double()
    want = vd + g * (O + bb)
    N, NH = qa.shape[2], qa.shape[1]
    tol = softmax_bound(p, g * av, want, dtype, N * NH, g * ud.abs().amax((1, 2))[:, None, :])
    assert_within(got, want, tol, what)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("N", [1, 64, 65, 128, 1536])
@pytest.mark.parametrize("pattern", PATTERNS)
def test_fold_vision_patterns(plain_ops, pattern, N, dtype):
    """vlf_fold_vision: one pass (N <= 64) and statistics + P.U passes (N > 64); rows of the next image's keys past N (the
    last head of image 0 reads into image 1) hold +-6e4 in qa and U without changing image 0's output."""
    B, S, NH = 2, 100, 2
    v, qa, u, qc, gamma, bias, _ = fold_vision_case(pattern, dtype, B, S, N, NH, seed=N)
    v, qa, u, qc, gamma, bias = (x.to(DEV) for x in (v, qa, u, qc, gamma, bias))
    got = plain_ops.vlf_fold_vision(v, qa, u, qc, gamma, bias)
    fold_vision_reference_check(got, v, qa, u, qc, gamma, bias, dtype, pattern)
    if N % KB:
        qa2, u2 = qa.clone(), u.clone()
        qa2[1] = torch.where(torch.rand(qa2[1].shape, device=DEV) < 0.5, -6e4, 6e4).to(dtype)
        u2[1] = torch.where(torch.rand(u2[1].shape, device=DEV) < 0.5, -6e4, 6e4).to(dtype)
        assert torch.equal(plain_ops.vlf_fold_vision(v, qa2, u2, qc, gamma, bias)[0], got[0])


# -------------------------------------------------------------------------------------------------------- vlf_fold_pool
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,S,N", pool_shapes())
@pytest.mark.parametrize("pattern", PATTERNS)
def test_fold_pool_patterns(plain_ops, pattern, B, S, N, dtype):
    """vlf_fold_pool + combine: S split into nsplit >= 2 chunks whose last one holds 37 keys or a single key (pool_splits
    restated); with B = 2 the keys past image 0's last chunk are image 1's, which hold +-6e4 without changing image 0."""
    NH = 8
    v, qa, _ = fold_pool_case(pattern, dtype, B, S, N, NH, seed=S + B)
    v, qa = v.to(DEV), qa.to(DEV)
    got = plain_ops.vlf_fold_pool(v, qa)
    vd = v.double()
    sc = torch.einsum("bsc,brc->brs", vd, qa.double().view(B, NH * N, 256))
    o = got.view(B, N, NH, 256).transpose(1, 2).reshape(B, NH * N, 256)
    check_softmax(o, sc, vd, dtype, pattern)
    if B == 2:
        v2 = v.clone()
        v2[1] = torch.where(torch.rand(v2[1].shape, device=DEV) < 0.5, -6e4, 6e4).to(dtype)
        assert torch.equal(plain_ops.vlf_fold_pool(v2, qa)[:N], got[:N])


# ------------------------------------------------------------------------------------------------------------- vlf_pool
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,S", [(8, 1), (8, 5), (8, 8), (2, 87296)])
@pytest.mark.parametrize("pattern", PATTERNS)
def test_vlf_pool_patterns(plain_ops, pattern, B, S, dtype):
    """vlf_pool (three passes over strips, fuse_helper clamps): fp32 scores, accurate expf and fp32 sums over at most
    ~600 sequential terms, so the bound is 2^-14 of sum p |v| and of |out|; S < 8 runs one strip clamped to 8 tokens."""
    NH = 8
    v, qa, qc, _ = vlf_pool_case(pattern, dtype, B, S, NH, seed=S + B, score_block=vlf_pool_strip(S))
    v, qa, qc = v.to(DEV), qa.to(DEV), qc.to(DEV)
    got = plain_ops.vlf_pool(v, qa, qc, True)
    want, p = vlf_pool_reference(v, qa, qc)
    tol = 2.0 ** -14 * (torch.einsum("bhs,bsc->bhc", p, v.double().abs()) + want.abs()) + 1e-30
    assert_within(got, want, tol, pattern)


@pytest.mark.parametrize("S", [5, 87296])
def test_vlf_pool_ignores_the_next_image(plain_ops, S):
    """Without the global-max shift an image's pooling reads only its own S tokens: image 1 holding +-6e4 changes nothing
    in image 0, also when S < 8 and the strip is clamped to 8 tokens."""
    v, qa, qc, _ = vlf_pool_case("dominant", torch.float16, 2, S, 8, seed=3)
    v, qa, qc = v.to(DEV), qa.to(DEV), qc.to(DEV)
    got = plain_ops.vlf_pool(v, qa, qc, False)
    v2 = v.clone()
    v2[1] = torch.where(torch.rand(v2[1].shape, device=DEV) < 0.5, -6e4, 6e4).half()
    assert torch.equal(plain_ops.vlf_pool(v2, qa, qc, False)[0], got[0])
    torch.testing.assert_close(got[0].double(), vlf_pool_reference(v[:1], qa[:1], qc[:1], False)[0][0], rtol=2e-4, atol=1e-6)


# ---------------------------------------------------------------------------------------------------------------- MSDA
L5_1024 = [(256, 256), (128, 128), (64, 64), (32, 32), (16, 16)]  # APE-L_D encoder levels at 1024^2


@pytest.mark.parametrize("value_dtype,logit_dtype", [(torch.float32, torch.float32), (torch.float16, torch.float16),
                                                     (torch.bfloat16, torch.bfloat16), (torch.float16, torch.float32)])
@pytest.mark.parametrize("pattern", MSDA_PATTERNS)
def test_msda_fused_softmax(plain_ops, pattern, value_dtype, logit_dtype):
    """Fused MSDA softmax over the L * P = 20 logits of a (query, head), every sample exactly on a texel: the generic fused
    kernel (fp32 weights via __expf: 2^-16 of sum a |v| covers its error at these arguments) and, for 16-bit values, the
    pair kernel (weights rounded to 16 bit and the 4 points of a level summed in 16 bit: 5 u of sum a |v|)."""
    import ape_b200

    B, Q, H = 1, 600, 8
    value, ss, st, offs, logits, ref, texel, _ = msda_case(pattern, value_dtype, logit_dtype, B, Q, H, L5_1024, seed=5)
    value, ss, st, offs, logits, ref, texel = (x.to(DEV) for x in (value, ss, st, offs, logits, ref, texel))
    want, a, gathered = msda_reference(value, logits, texel, H)
    av = torch.einsum("bqhk,bqhkd->bqhd", a, gathered.abs()).reshape(B, Q, -1)
    u_out = U16.get(value_dtype, 2.0 ** -24)
    got = plain_ops.ms_deform_attn_fused_forward(value, ss, st, offs, logits, ref, 4)
    assert_within(got, want, 2.0 ** -16 * av + u_out * want.abs() + 1e-30, f"{pattern} fused")
    if value_dtype != torch.float32:
        assert ape_b200.ops.msda_pair_supported(L5_1024, H, 32, 4, value_dtype)
        v2 = plain_ops.msda_pair_values(value.view(B, value.shape[1], -1), H)
        got = plain_ops.ms_deform_attn_pair_fused_forward(v2, ss, st, L5_1024, offs, logits, ref, 4)
        assert_within(got, want, 5 * U16[value_dtype] * av + u_out * want.abs() + 1e-30, f"{pattern} pair")
