"""Score constructors for the softmax edge-case tests (tests/test_softmax_edges_gpu.py), and CPU checks that every
constructor produces its pattern exactly.

Each constructor builds 16-bit (or fp32) operands whose scores are designed exactly: the pattern sits in a few coordinates
of the queries and keys, with factors that 16-bit types represent, so that every product and every partial sum the
kernels form in fp32 is exact.  Query row r reads instance r % T of the pattern (coordinate triplet r % T), so one call
covers T independent draws.  A key score z in nats is stored as three 16-bit components (hi, lo, big):
    hi  = a multiple of 4 with |hi| <= 1020   (8 significant bits),
    lo  = a multiple of 1/64 in [0, 4)        (8 significant bits),
    big = a per-instance constant 0 or +-2^k  (the large-magnitude pattern),
and the query holds 1 / scale on the three coordinates, so that q . k * scale == hi + lo + big == z.  The checks below
recompute q k^T * scale in float64 on the rounded operands; a GPU failure then indicts the kernel, not the generator.

Patterns over the valid keys of one row (KB = keys per block of the flash-attention kernels):
    rising    the row maximum grows in every key block; the first block holds about 1e-6 of the mass
    last      the maximum is only the last valid key (the last, partial block)
    dominant  one key 38 or more nats above every other
    ties      every key equal (2 nats): the output is the mean of the valid values
    tie2      two equal maxima, 38 nats above the rest, in the first and in the last block
    large     scores of 1e3 to 1e4 nats (both signs) with a spread of a few nats
    cliff     the first half of the keys 120 nats below the second: their blocks / chunks weigh exp(-120), 0 in fp32
"""
import pytest
import torch

KB = 64  # keys per block of attn.cuh / vlf_fold.cu
T = 4    # pattern instances per call (coordinate triplets)
PATTERNS = ["rising", "last", "dominant", "ties", "tie2", "large", "cliff"]
BIGS = [8192.0, -4096.0, 2048.0, -1024.0]  # "large": one magnitude per instance, in nats
U16 = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}  # unit roundoff of the 16-bit types
DOMINANT_GAP = 38.0  # nats between a dominant key (or a pair of tied maxima) and the next key; >= 30 as required
RISING_FIRST_MASS = 1e-6


def _grid(x, q=64.0):
    """Round to multiples of 1/q."""
    return torch.round(x * q) / q


def _rising_slope(nk, block):
    """Slope s (nats per key) of z_j = s j such that the first block holds RISING_FIRST_MASS of the mass."""
    j = torch.arange(nk, dtype=torch.float64)

    def first_mass(s):
        w = torch.exp(s * (j - (nk - 1)))
        return (w[:block].sum() / w.sum()).item()

    lo, hi = 0.0, 60.0
    for _ in range(80):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if first_mass(mid) > RISING_FIRST_MASS else (lo, mid)
    return hi


def key_scores(pattern, nk, seed, block=KB, n_inst=T):
    """Designed scores z [n_inst, nk] (float64, nats) and the per-instance constant big [n_inst]: z = big + rel with rel a
    multiple of 1/64 in [-1020, 1024)."""
    g = torch.Generator().manual_seed(seed)
    rest = _grid(torch.rand(n_inst, nk, generator=g, dtype=torch.float64) * 4 - 2)  # background in [-2, 2]
    big = torch.zeros(n_inst, dtype=torch.float64)
    if pattern == "rising":
        s = _rising_slope(nk, block) if nk > block else 0.25
        rel = _grid(s * torch.arange(nk, dtype=torch.float64)).expand(n_inst, nk).clone()
        rel -= _grid(torch.full((n_inst, 1), s * (nk - 1) / 2))  # centred, so the scores stay small
    elif pattern == "last":
        rel = rest
        rel[:, nk - 1] = 8.0  # not dominant: the earlier keys keep a share, so their rescale by the last block matters
    elif pattern == "dominant":
        rel = rest
        pos = torch.randint(0, nk, (n_inst,), generator=g)
        rel[torch.arange(n_inst), pos] = 2.0 + DOMINANT_GAP
    elif pattern == "ties":
        rel = torch.full((n_inst, nk), 2.0, dtype=torch.float64)
    elif pattern == "tie2":
        rel = rest
        if nk <= block:  # one block: the first and the last key
            a, b = torch.zeros(n_inst, dtype=torch.long), torch.full((n_inst,), nk - 1)
        else:
            a = torch.randint(0, block, (n_inst,), generator=g)
            b = nk - 1 - torch.randint(0, nk - (nk - 1) // block * block, (n_inst,), generator=g)
        rel[torch.arange(n_inst), a] = 2.0 + DOMINANT_GAP
        rel[torch.arange(n_inst), b] = 2.0 + DOMINANT_GAP
    elif pattern == "large":
        rel = _grid(torch.rand(n_inst, nk, generator=g, dtype=torch.float64) * 8 - 4)
        big = torch.tensor(BIGS, dtype=torch.float64).repeat(n_inst // len(BIGS) + 1)[:n_inst]
    elif pattern == "cliff":
        rel = rest
        rel[:, : nk // 2] -= 120.0
    else:
        raise ValueError(pattern)
    return rel + big[:, None], big


def components(z, big):
    """[n_inst, nk] scores -> [nk, 3 n_inst] components (hi, lo, big per instance), each exact in fp16 and bf16."""
    rel = z - big[:, None]
    hi = torch.floor(rel / 4) * 4
    lo = rel - hi
    comp = torch.stack([hi, lo, big[:, None].expand_as(rel)], -1)  # [n_inst, nk, 3]
    return comp.permute(1, 0, 2).reshape(z.shape[1], -1)


def query_coeffs(rows, n_inst, coeff):
    """[rows, 3 n_inst]: row r holds `coeff` on the coordinates of triplet r % n_inst."""
    out = torch.zeros(rows, 3 * n_inst, dtype=torch.float64)
    r = torch.arange(rows)
    for c in range(3):
        out[r, 3 * (r % n_inst) + c] = coeff
    return out


def pad_values(shape, seed, fill):
    """Content of masked rows: +-fill (finite) in random signs, or zeros."""
    if fill == 0:
        return torch.zeros(shape)
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(0, 2, shape, generator=g) * 2 - 1).float() * fill


def tie_values(nk, width, seed):
    """Values whose mean over the nk keys is a multiple of 1/16 in [-1, 1] (exact in 16 bit), every entry a multiple of 1/16
    in [-3, 3]: the first half is random, the second half mirrors it around the mean.  nk must be even."""
    g = torch.Generator().manual_seed(seed)
    m = torch.randint(-16, 17, (width,), generator=g).double() / 16
    a = torch.randint(-32, 33, (nk // 2, width), generator=g).double() / 16
    return torch.cat([a, 2 * m - a], 0)


# ---------------------------------------------------------------------------------------------------------------- attention
def attn_qkv_case(pattern, dtype, num_seq, n, n_valid, heads, seed, stride=None, pad_fill=0.0, scale=0.125):
    """Fused qkv buffer for ops.attention_qkv (64-channel heads).  Every (sequence, head) gets its own draw of the pattern
    over its n_valid keys; rows of a sequence past n_valid (up to n, or to `stride` when packed) hold pad_fill.
    Returns (qkv [rows, 3 * heads * 64] in dtype, z [num_seq, heads, T, n_valid])."""
    stride = n if stride is None else stride
    rows = (num_seq - 1) * stride + (n if stride >= n else stride)
    C = heads * 64
    g = torch.Generator().manual_seed(seed)
    qkv = pad_values((rows, 3 * C), seed + 1, pad_fill)
    zs = torch.empty(num_seq, heads, T, n_valid, dtype=torch.float64)
    for s in range(num_seq):
        r0 = s * stride
        for h in range(heads):
            z, big = key_scores(pattern, n_valid, seed + 97 * s + 13 * h)
            zs[s, h] = z
            q = torch.randn(n_valid, 64, generator=g, dtype=torch.float64)
            q[:, : 3 * T] = query_coeffs(n_valid, T, 1.0 / scale)
            k = torch.zeros(n_valid, 64, dtype=torch.float64)
            k[:, : 3 * T] = components(z, big)
            if pattern == "ties" and n_valid % 2 == 0:
                v = tie_values(n_valid, 64, seed + 7 * s + h)
            else:
                v = torch.randn(n_valid, 64, generator=g, dtype=torch.float64)
            for i, x in enumerate((q, k, v)):
                qkv[r0: r0 + n_valid, i * C + h * 64: i * C + (h + 1) * 64] = x.float()
    return qkv.to(dtype), zs


def cross_case(pattern, dtype, num_seq, nq, nkv, n_valid, heads, hd, seed, pad_fill=0.0):
    """q [num_seq*nq, heads*hd], k / v [num_seq*nkv, heads*hd] for ops.attention_cross with scale hd^-0.5; keys >= n_valid
    hold pad_fill.  Returns (q, k, v, z [num_seq, heads, T, n_valid])."""
    scale = hd ** -0.5
    C = heads * hd
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(num_seq, nq, heads, hd, generator=g, dtype=torch.float64)
    k = pad_values((num_seq, nkv, heads, hd), seed + 1, pad_fill).double()
    v = pad_values((num_seq, nkv, heads, hd), seed + 2, pad_fill).double()
    zs = torch.empty(num_seq, heads, T, n_valid, dtype=torch.float64)
    for s in range(num_seq):
        for h in range(heads):
            z, big = key_scores(pattern, n_valid, seed + 97 * s + 13 * h)
            zs[s, h] = z
            q[s, :, h, : 3 * T] = query_coeffs(nq, T, 1.0 / scale)
            k[s, :n_valid, h] = 0
            k[s, :n_valid, h, : 3 * T] = components(z, big)
            v[s, :n_valid, h] = torch.randn(n_valid, hd, generator=g, dtype=torch.float64)
    return (q.reshape(-1, C).to(dtype), k.reshape(-1, C).to(dtype), v.reshape(-1, C).to(dtype), zs)


# -------------------------------------------------------------------------------------------------------- vision-language
def fold_vision_case(pattern, dtype, B, S, N, NH, seed):
    """Operands of ops.vlf_fold_vision: the rows of v are the queries (row s reads triplet s % T with coefficient 1), the N
    rows of qa[b, h] the keys.  qc = 0, so the score is v . qa.  Returns (v, qa, u, qc, gamma, bias, z [B, NH, T, N])."""
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(B, S, 256, generator=g, dtype=torch.float64)
    v[:, :, : 3 * T] = query_coeffs(S, T, 1.0)
    qa = torch.zeros(B, NH, N, 256, dtype=torch.float64)
    zs = torch.empty(B, NH, T, N, dtype=torch.float64)
    for b in range(B):
        for h in range(NH):
            z, big = key_scores(pattern, N, seed + 97 * b + 13 * h)
            zs[b, h] = z
            qa[b, h, :, : 3 * T] = components(z, big)
    u = torch.randn(B, NH, N, 256, generator=g, dtype=torch.float64)
    qc = torch.zeros(B, NH, N)
    gamma = _grid(torch.rand(256, generator=g, dtype=torch.float64), 256).float()
    bias = _grid(torch.randn(256, generator=g, dtype=torch.float64), 256).float()
    return v.to(dtype), qa.to(dtype), u.to(dtype), qc, gamma, bias, zs


def fold_pool_case(pattern, dtype, B, S, N, NH, seed, score_block=KB):
    """Operands of ops.vlf_fold_pool: the R = NH * N rows of qa[b] are the queries (row r reads triplet r % T with
    coefficient 1), the S rows of v[b] are the keys and the values.  Returns (v, qa, z [B, T, S])."""
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(B, S, 256, generator=g, dtype=torch.float64)
    zs = torch.empty(B, T, S, dtype=torch.float64)
    for b in range(B):
        z, big = key_scores(pattern, S, seed + 97 * b, block=score_block)
        zs[b] = z
        v[b, :, : 3 * T] = components(z, big)
    qa = torch.zeros(B, NH * N, 256, dtype=torch.float64)
    qa[:, :, : 3 * T] = query_coeffs(NH * N, T, 1.0)
    return v.to(dtype), qa.view(B, NH, N, 256).to(dtype), zs


def vlf_pool_case(pattern, dtype, B, S, NH, seed, score_block=KB):
    """Operands of ops.vlf_pool: head h reads triplet h % T (qa fp32 with coefficient 1, qc = 0), the S rows of v[b] are
    the keys and the values.  Returns (v, qa [B, NH, 256], qc [B, NH], z [B, T, S])."""
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(B, S, 256, generator=g, dtype=torch.float64)
    zs = torch.empty(B, T, S, dtype=torch.float64)
    for b in range(B):
        z, big = key_scores(pattern, S, seed + 97 * b, block=score_block)
        zs[b] = z
        v[b, :, : 3 * T] = components(z, big)
    qa = query_coeffs(NH, T, 1.0).float()
    qa = torch.cat([qa, torch.zeros(NH, 256 - 3 * T)], 1).expand(B, NH, 256).contiguous()
    return v.to(dtype), qa, torch.zeros(B, NH), zs


def vlf_pool_reference(v, qa, qc, stable_2d=True):
    """float64 restatement of the pooling with the fuse_helper clamps (stable_softmax_2d: global-max shift, +-5e4)."""
    vd = v.double()
    w = torch.einsum("bsc,bhc->bhs", vd, qa.double()) + qc.double()[..., None]
    if stable_2d:
        w = w - w.max()
    w = torch.clamp(w, -50000, 50000)
    wl = torch.clamp(w - w.max(-1, keepdim=True)[0], -50000, 50000)
    p = torch.softmax(wl, -1)
    return torch.einsum("bhs,bsc->bhc", p, vd), p


# ----------------------------------------------------------------------------------------------------------------- MSDA
MSDA_PATTERNS = ["dominant", "ties", "ties_large", "dominant_large"]


def msda_logits(pattern, rows, LP, seed):
    """[rows, LP] float64 logits, exact in fp16 and bf16: one logit 40 above the rest in [-2, 2] (at a random position), all
    equal, all equal at 30720, or a dominant one at 2^14 over a background at 2^14 - 128 or 2^14 - 256 (past exp's
    fp32 range: a maximum that misses the dominant logit overflows)."""
    g = torch.Generator().manual_seed(seed)
    pos = torch.randint(0, LP, (rows,), generator=g)
    r = torch.arange(rows)
    if pattern == "dominant":
        x = _grid(torch.rand(rows, LP, generator=g, dtype=torch.float64) * 4 - 2, 4)
        x[r, pos] = 42.0
    elif pattern == "ties":
        x = torch.full((rows, LP), 2.0, dtype=torch.float64)
    elif pattern == "ties_large":
        x = torch.full((rows, LP), 30720.0, dtype=torch.float64)
    elif pattern == "dominant_large":  # bf16 spacing just below 2^14 is 64
        x = 16384.0 - 128.0 * torch.randint(1, 3, (rows, LP), generator=g).double()
        x[r, pos] = 16384.0
    else:
        raise ValueError(pattern)
    return x


def msda_case(pattern, value_dtype, logit_dtype, B, Q, H, shapes, seed, P=4):
    """Operands of ops.ms_deform_attn_fused_forward with every sample landing exactly on a texel: reference points carry a
    box (ref_dim 4, box = 8 / size of the level, every level size a power of two), so point p of level l samples texel
    (y, x + p) of that level with bilinear weight 1.  Returns (value [B,S,H,32], shapes, starts, offsets, logits, ref,
    texel [B, Q, H, L * P] int64 rows of value, logits as float64)."""
    from oracle import msda as O

    L = len(shapes)
    LP = L * P
    g = torch.Generator().manual_seed(seed)
    ss = torch.tensor(shapes)
    st = O.level_start_index(ss)
    S = int((ss[:, 0] * ss[:, 1]).sum())
    value = torch.randn(B, S, H, 32, generator=g).to(value_dtype)
    logits = msda_logits(pattern, B * Q * H, LP, seed + 1).view(B, Q, H * LP)
    offs = torch.zeros(B, Q, H, L, P, 2)
    offs[..., 0] = torch.arange(P).float()
    ref = torch.empty(B, Q, L, 4)
    texel = torch.empty(B, Q, H, L, P, dtype=torch.int64)
    for l, (hl, wl) in enumerate(shapes):
        assert hl & (hl - 1) == 0 and wl & (wl - 1) == 0 and wl >= P
        y = torch.randint(0, hl, (B, Q), generator=g)
        x = torch.randint(0, wl - P + 1, (B, Q), generator=g)
        ref[:, :, l] = torch.stack([(x + 0.5) / wl, (y + 0.5) / hl, 8.0 / wl + 0 * x, 8.0 / hl + 0 * y], -1)
        texel[:, :, :, l] = (int(st[l]) + y * wl + x)[:, :, None, None] + torch.arange(P)
    return (value, ss, st, offs.view(B, Q, -1).to(logit_dtype), logits.to(logit_dtype), ref, texel.view(B, Q, H, LP), logits)


def msda_reference(value, logits, texel, H):
    """float64: out[b, q, h] = sum_k softmax(logits[b, q, h, :])_k value[b, texel[b, q, h, k], h]; also the weights."""
    B, Q = logits.shape[:2]
    a = torch.softmax(logits.double().view(B, Q, H, -1), -1)
    vd = value.double()
    bi = torch.arange(B, device=texel.device)[:, None, None, None]
    hi = torch.arange(H, device=texel.device)[None, None, :, None]
    gathered = vd[bi, texel, hi]  # [B, Q, H, LP, 32]
    return torch.einsum("bqhk,bqhkd->bqhd", a, gathered).reshape(B, Q, -1), a, gathered


# ======================================================================================================== CPU checks
def _check_pattern(pattern, z, nk, block=KB):
    """Pattern properties of one row of designed scores z [nk] (float64)."""
    nb = (nk + block - 1) // block
    bmax = torch.stack([z[i * block: (i + 1) * block].max() for i in range(nb)])
    top = z.max()
    if pattern == "rising":
        if nb > 1:
            assert (bmax[1:] > bmax[:-1]).all()
            w = torch.exp(z - top)
            assert 3e-7 < (w[:block].sum() / w.sum()).item() < 3e-6
    elif pattern == "last":
        assert (z[: nk - 1] < top).all() and z[nk - 1] == top
    elif pattern == "dominant":
        s = z.sort(descending=True)[0]
        assert nk == 1 or s[0] - s[1] >= 30
    elif pattern == "ties":
        assert (z == z[0]).all()
    elif pattern == "tie2":
        s, idx = z.sort(descending=True)
        if nk > 1:
            assert s[0] == s[1] and (nk == 2 or s[1] - s[2] >= 30)
            if nb > 1:
                assert {int(i) // block for i in idx[:2]} == {0, nb - 1}
    elif pattern == "large":
        assert (z.abs() >= 1e3).all() and (z.abs() <= 1e4).all() and z.max() - z.min() <= 10
    elif pattern == "cliff":
        assert (z[: nk // 2] <= z[nk // 2:].min() - 116).all()
    else:
        raise ValueError(pattern)


def _exact_in(x, dtype):
    return torch.equal(x.to(dtype).double(), x.double())


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("nk", [1, 2, 64, 65, 128, 129, 900, 1536, 4096])
def test_key_scores_have_their_pattern_and_exact_components(pattern, nk):
    z, big = key_scores(pattern, nk, seed=nk)
    comp = components(z, big)
    for dtype in (torch.float16, torch.bfloat16):
        assert _exact_in(comp, dtype)
    assert torch.equal(comp.view(nk, T, 3).sum(-1).T, z)
    for i in range(T):
        _check_pattern(pattern, z[i], nk)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("pattern", PATTERNS)
def test_attention_scores_are_designed_exactly(pattern, dtype):
    """float64 q k^T * scale on the rounded operands equals the designed scores, row r reading instance r % T; the pad rows
    hold the finite +-6e4."""
    num_seq, n, n_valid, heads, stride = 2, 256, 129, 2, 200
    qkv, z = attn_qkv_case(pattern, dtype, num_seq, n, n_valid, heads, seed=5, stride=stride, pad_fill=6e4)
    x = qkv.double()
    assert torch.isfinite(x).all() and x.abs().max() <= 65504
    for s in range(num_seq):
        rows = x[s * stride: s * stride + n_valid]
        assert (x[s * stride + n_valid: s * stride + stride].abs() == x.abs().max()).all()
        for h in range(heads):
            q, k = rows[:, h * 64: (h + 1) * 64], rows[:, 64 * heads + h * 64: 64 * heads + (h + 1) * 64]
            sc = q @ k.T * 0.125
            assert torch.equal(sc, z[s, h][torch.arange(n_valid) % T])
            assert torch.equal(sc.float().double(), sc)  # the kernel's fp32 scores are these numbers


@pytest.mark.parametrize("hd", [64, 256])
def test_cross_attention_scores_are_designed_exactly(hd):
    q, k, v, z = cross_case("large", torch.bfloat16, 1, 128, 192, 130, 2, hd, seed=3, pad_fill=6e4)
    for h in range(2):
        sc = q.double()[:, h * hd: (h + 1) * hd] @ k.double()[:130, h * hd: (h + 1) * hd].T * hd ** -0.5
        assert torch.equal(sc, z[0, h][torch.arange(128) % T])
    assert (k.double()[130:].abs() > 5e4).all() and (v.double()[130:].abs() > 5e4).all()


def test_tie_values_have_a_representable_mean():
    v = tie_values(128, 64, seed=1)
    m = v.mean(0)
    for dtype in (torch.float16, torch.bfloat16):
        assert _exact_in(v, dtype) and _exact_in(m, dtype)
    assert torch.equal(v.sum(0), m * 128)


@pytest.mark.parametrize("pattern", PATTERNS)
def test_fold_scores_are_designed_exactly(pattern):
    v, qa, u, qc, gamma, bias, z = fold_vision_case(pattern, torch.bfloat16, 2, 70, 65, 2, seed=4)
    sc = torch.einsum("bsc,bhnc->bhsn", v.double(), qa.double())
    assert torch.equal(sc, z[:, :, torch.arange(70) % T])
    for i in range(T):
        _check_pattern(pattern, z[0, 0, i], 65)
    v, qa, z = fold_pool_case(pattern, torch.float16, 2, 1100, 3, 2, seed=4)
    sc = torch.einsum("bsc,brc->brs", v.double(), qa.double().view(2, 6, 256))
    assert torch.equal(sc, z[:, torch.arange(6) % T])


@pytest.mark.parametrize("pattern", PATTERNS)
def test_vlf_pool_scores_are_designed_exactly(pattern):
    v, qa, qc, z = vlf_pool_case(pattern, torch.float16, 2, 300, 8, seed=2)
    sc = torch.einsum("bsc,bhc->bhs", v.double(), qa.double())
    assert torch.equal(sc, z[:, torch.arange(8) % T])
    assert torch.equal(sc.float().double(), sc)


def pool_splits(B, S, R):
    """Python restatement of vlf_fold.cu's pool_splits: (nsplit, chunk) of the language-side pooling."""
    tiles = (R + 63) // 64 * B
    nsplit = max(1, min((264 + tiles - 1) // tiles, (S + 1023) // 1024))
    chunk = ((S + nsplit - 1) // nsplit + KB - 1) // KB * KB
    return (S + chunk - 1) // chunk, chunk


def pool_shapes():
    """(B, S, N) of the fold pool whose last chunk is short or holds a single key, with nsplit >= 2."""
    out = []
    for B, N in ((1, 3), (2, 3)):
        for want_last, S in ((37, 2049), (1, 2049)):
            while True:
                nsplit, chunk = pool_splits(B, S, 8 * N)
                if nsplit >= 2 and S - (nsplit - 1) * chunk == want_last:
                    break
                S += 1
            out.append((B, S, N))
    return out


def test_pool_shapes_hit_the_chunk_boundaries():
    for B, S, N in pool_shapes():
        nsplit, chunk = pool_splits(B, S, 8 * N)
        assert nsplit >= 2 and S - (nsplit - 1) * chunk in (1, 37)


def vlf_pool_strip(S):
    """Python restatement of vlf_pool.cu's strips_for: tokens per CTA strip."""
    return max(8, min(512, (S + 263) // 264))


@pytest.mark.parametrize("pattern", MSDA_PATTERNS)
def test_msda_samples_land_on_texels_and_logits_are_exact(pattern):
    shapes = [(16, 16), (8, 8), (4, 4)]
    value, ss, st, offs, logits, ref, texel, zl = msda_case(pattern, torch.float16, torch.bfloat16, 1, 50, 2, shapes, seed=1)
    for dtype in (torch.float16, torch.bfloat16):
        assert _exact_in(zl, dtype)
    # restate the kernels' location arithmetic (ref_xy + off * box * 0.125, then * size - 0.5) in fp32: integer texels
    B, Q, L, P = 1, 50, 3, 4
    o = offs.float().view(B, Q, 2, L, P, 2)
    for l, (hl, wl) in enumerate(shapes):
        x = ref[:, :, None, l, None, 0] + o[..., l, :, 0] * (ref[:, :, None, l, None, 2] * 0.125)
        y = ref[:, :, None, l, None, 1] + o[..., l, :, 1] * (ref[:, :, None, l, None, 3] * 0.125)
        xi, yi = x * wl - 0.5, y * hl - 0.5
        assert torch.equal(xi, xi.round()) and torch.equal(yi, yi.round())
        assert (xi >= 0).all() and (xi <= wl - 1).all() and (yi >= 0).all() and (yi <= hl - 1).all()
        got = int(st[l]) + yi.long() * wl + xi.long()
        assert torch.equal(got, texel.view(B, Q, 2, L, P)[..., l, :])
    a = torch.softmax(zl.view(B, Q, 2, -1), -1)
    if pattern.startswith("ties"):
        assert torch.equal(a, torch.full_like(a, 1 / (L * P)))
    else:
        assert (a.max(-1)[0] > 1 - 1e-10).all()
