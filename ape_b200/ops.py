"""Operator surface of the reference's native library, backed by libape_b200.so.

Registers `torch.ops.ape.ms_deform_attn_forward` / `ms_deform_attn_backward` with the
reference's schemas (ape/layers/csrc/vision.cpp:76-79, ms_deform_attn.h:21-28,42-50) so
`MultiScaleDeformableAttnFunction` (ape/layers/multi_scale_deform_attn.py:32-81) works unchanged.
CUDA tensors only: like the reference (`AT_ERROR("Not implemented on the CPU")`,
ms_deform_attn.h:39) there is no CPU implementation."""
import ctypes

import torch

from . import _lib

_NS = "ape"

# bench.py sets this to a list to collect (tag, start_event, end_event) around every launch of the
# library's kernels on the current stream (None = off, zero overhead).
PROFILE_EVENTS = None


class _timed:
    def __init__(self, tag):
        self.tag = tag

    def __enter__(self):
        if PROFILE_EVENTS is not None:
            self.a = torch.cuda.Event(enable_timing=True)
            self.b = torch.cuda.Event(enable_timing=True)
            self.a.record()
        return self

    def __exit__(self, *exc):
        if PROFILE_EVENTS is not None:
            self.b.record()
            PROFILE_EVENTS.append((self.tag, self.a, self.b))
        return False
_FWD_SCHEMA = (
    "ms_deform_attn_forward(Tensor value, Tensor spatial_shapes, Tensor level_start_index, "
    "Tensor sampling_loc, Tensor attn_weight, int im2col_step) -> Tensor"
)
_BWD_SCHEMA = (
    "ms_deform_attn_backward(Tensor value, Tensor spatial_shapes, Tensor level_start_index, "
    "Tensor sampling_loc, Tensor attn_weight, Tensor grad_output, int im2col_step) -> Tensor[]"
)


def _require(cond: bool, msg: str) -> None:
    if not cond:
        raise RuntimeError(msg)


def _check_inputs(value, spatial_shapes, level_start_index, sampling_loc, attn_weight):
    # same asserts as ms_deform_attn_cuda.cu:29-39
    for name, t in (
        ("value", value),
        ("spatial_shapes", spatial_shapes),
        ("level_start_index", level_start_index),
        ("sampling_loc", sampling_loc),
        ("attn_weight", attn_weight),
    ):
        _require(t.is_contiguous(), f"{name} tensor has to be contiguous")
        _require(t.is_cuda, f"{name} must be a CUDA tensor")
    _require(value.dim() == 4, "value must be [B,S,H,D]")
    _require(sampling_loc.dim() == 6 and sampling_loc.size(-1) == 2, "sampling_loc must be [B,Q,H,L,P,2]")
    _require(spatial_shapes.dtype == torch.int64 and level_start_index.dtype == torch.int64,
             "spatial_shapes / level_start_index must be int64")
    _require(sampling_loc.dtype == value.dtype and attn_weight.dtype == value.dtype,
             "sampling_loc / attn_weight must have value's dtype")
    B, S, H, D = value.shape
    _, Q, H2, L, P, _ = sampling_loc.shape
    _require(H2 == H and sampling_loc.size(0) == B, "sampling_loc shape does not match value")
    _require(tuple(attn_weight.shape) == (B, Q, H, L, P), "attn_weight must be [B,Q,H,L,P]")
    _require(spatial_shapes.shape == (L, 2) and level_start_index.shape == (L,), "bad level tensors")
    return B, S, H, D, L, Q, P


def ms_deform_attn_forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight,
                           im2col_step=64, variant=-1):
    """out[B,Q,H*D]; `im2col_step` is accepted for signature parity and ignored (it only
    chunks the batch in the reference host code, ms_deform_attn_cuda.cu:51-62)."""
    if not value.is_cuda:
        raise RuntimeError("Not implemented on the CPU")  # ms_deform_attn.h:39
    B, S, H, D, L, Q, P = _check_inputs(value, spatial_shapes, level_start_index, sampling_loc, attn_weight)
    out = torch.empty((B, Q, H * D), dtype=value.dtype, device=value.device)
    with torch.cuda.device(value.device):
        rc = _lib.lib.ape_msda_fwd_variant(
            value.data_ptr(), spatial_shapes.data_ptr(), level_start_index.data_ptr(),
            sampling_loc.data_ptr(), attn_weight.data_ptr(), out.data_ptr(),
            B, S, H, D, L, Q, P, _lib.dtype_code(value.dtype), int(variant), _lib.current_stream_ptr())
    _lib.check(rc, "ape_msda_fwd")
    return out


def ms_deform_attn_fused_forward(value, spatial_shapes, level_start_index, sampling_offsets,
                                 attention_logits, reference_points, num_points):
    """Fused tail of MultiScaleDeformableAttention.forward (multi_scale_deform_attn.py:283-348).

    value [B,S,H,D]; sampling_offsets [B,Q,>=H*L*P*2] and attention_logits [B,Q,>=H*L*P] are the
    raw linear outputs (may be column slices of one wider GEMM output: only the last dim needs
    unit stride); reference_points [B,Q,L,2|4] fp32."""
    B, S, H, D = value.shape
    L = spatial_shapes.shape[0]
    Q = sampling_offsets.shape[1]
    P = int(num_points)
    _require(value.is_cuda and value.is_contiguous(), "value must be a contiguous CUDA tensor")
    ref = _check_fused(sampling_offsets, attention_logits, reference_points, B, Q, L)
    out = torch.empty((B, Q, H * D), dtype=value.dtype, device=value.device)
    with torch.cuda.device(value.device), _timed(("msda_fused", B, S, Q, L, P, value.element_size(),
                                                  sampling_offsets.element_size())):
        rc = _lib.lib.ape_msda_fused_fwd(
            value.data_ptr(), spatial_shapes.data_ptr(), level_start_index.data_ptr(),
            sampling_offsets.data_ptr(), sampling_offsets.stride(1),
            attention_logits.data_ptr(), attention_logits.stride(1),
            ref.data_ptr(), ref.shape[-1], out.data_ptr(),
            B, S, H, D, L, Q, P, _lib.dtype_code(value.dtype), _lib.dtype_code(sampling_offsets.dtype),
            _lib.current_stream_ptr())
    _lib.check(rc, "ape_msda_fused_fwd")
    return out


def _check_fused(sampling_offsets, attention_logits, reference_points, B, Q, L):
    _require(sampling_offsets.dtype == attention_logits.dtype, "offsets/logits dtype mismatch")
    _require(sampling_offsets.stride(-1) == 1 and attention_logits.stride(-1) == 1, "unit inner stride required")
    _require(sampling_offsets.stride(0) == Q * sampling_offsets.stride(1), "offsets batch stride")
    _require(attention_logits.stride(0) == Q * attention_logits.stride(1), "logits batch stride")
    ref = reference_points
    _require(ref.dtype == torch.float32 and ref.is_contiguous(), "reference_points must be contiguous fp32")
    _require(ref.shape[:3] == (B, Q, L), "reference_points must be [B,Q,L,2|4]")
    return ref


def msda_pair_supported(host_shapes, H, D, P, dtype):
    """True when the pair-layout kernel covers this geometry (16-bit value, D = 32, P = 4, L <= 8, levels >= 2 wide)."""
    if dtype not in (torch.float16, torch.bfloat16):
        return False
    L = len(host_shapes)
    hs = (ctypes.c_int * (2 * L))(*[int(v) for hw in host_shapes for v in hw])
    return bool(_lib.lib.ape_msda_pair_supported(hs, L, int(H), int(D), int(P), _lib.dtype_code(dtype)))


def msda_pair_values(value, num_heads, token_mask=None):
    """value [B,S,H*32] (16-bit, unit inner stride, uniform row pitch) -> pair layout [B,S,H,2,32] (ape_msda_pair_values):
    entry (s, h) = channels of token s then of token s+1.  token_mask [B,S] bool: masked tokens are written as zeros."""
    _require(value.is_cuda and value.dim() == 3 and value.stride(2) == 1 and value.stride(0) == value.shape[1] * value.stride(1),
             "msda_pair_values: CUDA [B,S,C] with uniform row pitch")
    B, S, C = value.shape
    H = int(num_heads)
    out = torch.empty((B, S, H, 2, C // H), dtype=value.dtype, device=value.device)
    mptr = None
    if token_mask is not None:  # a bool mask is read as its bytes (no conversion launch)
        token_mask = token_mask.contiguous()
        token_mask = token_mask.view(torch.uint8) if token_mask.dtype == torch.bool else token_mask.to(torch.uint8)
        _require(token_mask.numel() == B * S, "msda_pair_values: token_mask must be [B,S]")
        mptr = token_mask.data_ptr()
    with torch.cuda.device(value.device), _timed(("msda_pair_values", B, S, C)):
        rc = _lib.lib.ape_msda_pair_values(value.data_ptr(), value.stride(1), out.data_ptr(), mptr, B, S, H, C // H,
                                           _lib.dtype_code(value.dtype), _lib.current_stream_ptr())
    _lib.check(rc, "ape_msda_pair_values")
    return out


PAIR_TILE_W, PAIR_HEAD_MAJOR = -1, 0  # CTA tiling of the pair kernel for Q == S (tests / sweeps override)


def ms_deform_attn_pair_fused_forward(value2, spatial_shapes, level_start_index, host_shapes, sampling_offsets,
                                      attention_logits, reference_points, num_points, heads_per_cta=0, tile_w=None,
                                      head_major=None):
    """ms_deform_attn_fused_forward over the pair layout (ape_msda_pair_fused_fwd).  value2 [B,S,H,2,32]."""
    B, S, H, two, D = value2.shape
    L = spatial_shapes.shape[0]
    Q = sampling_offsets.shape[1]
    _require(value2.is_cuda and value2.is_contiguous() and two == 2, "value2 must be a contiguous CUDA [B,S,H,2,D] tensor")
    ref = _check_fused(sampling_offsets, attention_logits, reference_points, B, Q, L)
    hs = (ctypes.c_int * (2 * L))(*[int(v) for hw in host_shapes for v in hw])
    out = torch.empty((B, Q, H * D), dtype=value2.dtype, device=value2.device)
    with torch.cuda.device(value2.device), _timed(("msda_fused", B, S, Q, L, int(num_points), value2.element_size(),
                                                   sampling_offsets.element_size())):
        rc = _lib.lib.ape_msda_pair_fused_fwd(
            value2.data_ptr(), spatial_shapes.data_ptr(), level_start_index.data_ptr(), hs,
            sampling_offsets.data_ptr(), sampling_offsets.stride(1), attention_logits.data_ptr(),
            attention_logits.stride(1), ref.data_ptr(), ref.shape[-1], out.data_ptr(), B, S, H, D, L, Q, int(num_points),
            _lib.dtype_code(value2.dtype), _lib.dtype_code(sampling_offsets.dtype), int(heads_per_cta),
            int(PAIR_TILE_W if tile_w is None else tile_w) if Q == S else 0,
            int(PAIR_HEAD_MAJOR if head_major is None else head_major), _lib.current_stream_ptr())
    _lib.check(rc, "ape_msda_pair_fused_fwd")
    return out


ACT = {None: 0, "none": 0, "relu": 1, "gelu": 2, "swiglu": 3, "clamp": 4}


def linear_tc(x, weight, bias=None, act=None, out_dtype=None, residual=None, tile_n=0, out=None, ln_fold=None, stats_out=False):
    """act(x @ weight.T + bias) (+ residual) on the wgmma tensor cores (ape_gemm_tn).

    x [..., K] and weight [N, K] fp16/bf16 with unit inner stride; bias fp32 [N] (or None); residual
    [..., N] fp32 / fp16 / bf16 (any of them with any output dtype: fp32 sums over 16-bit operands).
    ln_fold = (part [M, nparts, 2] fp32, colsum [N] fp32, C, eps): a LayerNorm over x's C columns folded around the GEMM
    (ape_gemm_tn_fused): x is the RAW tensor, weight = gamma .* W, bias = beta W^T + b, fp32 output.
    stats_out=True (act "swiglu"): also returns fp32 [M, ceil(N/2/64), 2] row statistics of the output slabs.  act="swiglu": weight rows are interleaved (gate_j, up_j) pairs and the
    result has N/2 columns."""
    _require(x.is_cuda and weight.is_cuda, "linear_tc: CUDA tensors only")
    _require(x.dtype == weight.dtype and x.dtype in (torch.float16, torch.bfloat16), "linear_tc: fp16/bf16 operands")
    K = x.shape[-1]
    N = weight.shape[0]
    _require(weight.shape[1] == K and x.stride(-1) == 1 and weight.stride(-1) == 1, "linear_tc: bad operand layout")
    x2 = x.reshape(-1, K)
    if x2.stride(0) % 8 or x2.data_ptr() % 16:
        x2 = x2.contiguous()
    _require(weight.stride(0) % 8 == 0 and weight.data_ptr() % 16 == 0, "linear_tc: weight rows must be 16-byte aligned")
    M = x2.shape[0]
    n_out = N // 2 if act == "swiglu" else N
    if out is None:
        out_dtype = out_dtype or x.dtype
        out = torch.empty((M, n_out), dtype=out_dtype, device=x.device)
        ret_view = True
    else:
        _require(out.dim() == 2 and out.shape == (M, n_out) and out.stride(1) == 1 and out.is_cuda, "linear_tc: bad `out`")
        out_dtype = out.dtype
        ret_view = False
    res_ptr, ldr, res_dt = None, 0, 0
    if residual is not None:
        r2 = residual.reshape(-1, n_out)
        _require(r2.stride(1) == 1 and r2.is_cuda, "linear_tc: residual needs unit inner stride")
        res_ptr, ldr, res_dt = r2.data_ptr(), r2.stride(0), _lib.dtype_code(r2.dtype)
    if bias is not None:
        _require(bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == N, "linear_tc: bias must be fp32 [N]")
    stats = None
    if ln_fold is not None or stats_out:
        part, colsum, nparts, inv_c, eps = None, None, 0, 0.0, 0.0
        if ln_fold is not None:
            part, colsum, C, eps = ln_fold
            _require(part.dtype == torch.float32 and part.is_contiguous() and part.dim() == 3 and part.shape[0] == M and
                     part.shape[2] == 2, "linear_tc: ln_fold partials must be fp32 [M, nparts, 2]")
            _require(colsum.dtype == torch.float32 and colsum.is_contiguous() and colsum.numel() == N, "linear_tc: colsum fp32 [N]")
            nparts, inv_c = part.shape[1], 1.0 / float(C)
        nslab = 0
        if stats_out:
            nslab = (n_out + 63) // 64
            stats = torch.empty((M, nslab, 2), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device), _timed(("gemm_tn", M, N, K)):
            rc = _lib.lib.ape_gemm_tn_fused(
                x2.data_ptr(), x2.stride(0), weight.data_ptr(), weight.stride(0), out.data_ptr(), out.stride(0),
                bias.data_ptr() if bias is not None else None, res_ptr, ldr, res_dt, M, N, K, _lib.dtype_code(x.dtype),
                _lib.dtype_code(out_dtype), ACT[act], int(tile_n), part.data_ptr() if part is not None else None, int(nparts),
                colsum.data_ptr() if colsum is not None else None, float(inv_c), float(eps),
                stats.data_ptr() if stats is not None else None, int(nslab), _lib.current_stream_ptr())
        _lib.check(rc, "ape_gemm_tn_fused")
    else:
        with torch.cuda.device(x.device), _timed(("gemm_tn", M, N, K)):
            rc = _lib.lib.ape_gemm_tn_ex(x2.data_ptr(), x2.stride(0), weight.data_ptr(), weight.stride(0), out.data_ptr(),
                                         out.stride(0), bias.data_ptr() if bias is not None else None, res_ptr, ldr, res_dt,
                                         M, N, K, _lib.dtype_code(x.dtype), _lib.dtype_code(out_dtype), ACT[act], int(tile_n),
                                         _lib.current_stream_ptr())
        _lib.check(rc, "ape_gemm_tn")
    res = out.view(*x.shape[:-1], n_out) if ret_view else out
    return (res, stats) if stats_out else res


def quantize_rows_e4m3(w):
    """(q, scale): per-row e4m3 quantisation of a 2-D tensor, computed in fp32 on its device: scale = max|row| / 448 (1 for
    an all-zero row), q = e4m3(row / scale) rounded to nearest even.  Weight preparation for linear_fp8, done once."""
    w = w.detach().float()
    s = w.abs().amax(1) / 448.0
    s = torch.where(s > 0, s, torch.ones_like(s))
    return (w / s[:, None]).clamp(-448.0, 448.0).to(torch.float8_e4m3fn).contiguous(), s.contiguous()


def linear_fp8(xq, x_scale, wq, w_scale, bias=None, act=None, stats_out=False, out=None, out_dtype=torch.float16):
    """act((xq @ wq.T) * x_scale[:, None] * w_scale[None, :] + bias) on the FP8 tensor cores (ape_gemm_tn_e4m3).

    xq [M, K] and wq [N, K] torch.float8_e4m3fn with unit inner stride and 16-byte aligned rows, K a multiple of 16;
    x_scale fp32 [M], w_scale fp32 [N]; bias fp32 [N] or None.  act None or "swiglu" (interleaved weight rows, N/2 output
    columns; stats_out=True also returns the fp32 [M, ceil(N/2/64), 2] slab statistics, as linear_tc).  The output is fp16 or
    bf16: `out` [M, n_out] with unit inner stride, or a new tensor of out_dtype."""
    _require(xq.is_cuda and wq.is_cuda, "linear_fp8: CUDA tensors only")
    _require(xq.dtype == torch.float8_e4m3fn and wq.dtype == torch.float8_e4m3fn, "linear_fp8: e4m3 operands")
    _require(xq.dim() == 2 and wq.dim() == 2 and xq.shape[1] == wq.shape[1] and xq.stride(1) == 1 and wq.stride(1) == 1,
             "linear_fp8: xq [M, K] and wq [N, K] with unit inner stride")
    M, K = xq.shape
    N = wq.shape[0]
    for s, n, name in ((x_scale, M, "x_scale"), (w_scale, N, "w_scale")):
        _require(s.dtype == torch.float32 and s.is_contiguous() and s.numel() == n and s.is_cuda, f"linear_fp8: {name} fp32 [{n}]")
    if bias is not None:
        _require(bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == N, "linear_fp8: bias must be fp32 [N]")
    _require(act in (None, "swiglu"), "linear_fp8: act None or 'swiglu'")
    n_out = N // 2 if act == "swiglu" else N
    if out is None:
        out = torch.empty((M, n_out), dtype=out_dtype, device=xq.device)
    _require(out.dim() == 2 and out.shape == (M, n_out) and out.stride(1) == 1 and out.is_cuda, "linear_fp8: bad `out`")
    stats, nslab = None, 0
    if stats_out:
        nslab = (n_out + 63) // 64
        stats = torch.empty((M, nslab, 2), dtype=torch.float32, device=xq.device)
    with torch.cuda.device(xq.device), _timed(("gemm_tn_e4m3", M, N, K)):
        rc = _lib.lib.ape_gemm_tn_e4m3(xq.data_ptr(), xq.stride(0), wq.data_ptr(), wq.stride(0), x_scale.data_ptr(),
                                       w_scale.data_ptr(), out.data_ptr(), out.stride(0),
                                       bias.data_ptr() if bias is not None else None, M, N, K, _lib.dtype_code(out.dtype),
                                       ACT[act], stats.data_ptr() if stats is not None else None, int(nslab),
                                       _lib.current_stream_ptr())
    _lib.check(rc, "ape_gemm_tn_e4m3")
    return (out, stats) if stats_out else out


def ffn_fused(x, w1, b1, w2, b2, out=None, variant=0):
    """x + relu(x @ w1.T + b1) @ w2.T + b2 in one launch (ape_ffn_fused), fp32 [..., 256]; the hidden activation stays on chip.

    x [..., 256] and w1 [F, 256], w2 [256, F] (nn.Linear layouts) fp16/bf16 of one dtype, F a multiple of 64; b1 / b2 fp32 or
    None.  The result is bit-identical to linear_tc(x, w1, b1, act="relu") followed by linear_tc(h, w2, b2, residual=x,
    out_dtype=float32).  out: optional fp32 [M, 256] with unit inner stride (any even row pitch).  variant: 0 default,
    1 single CTA, 2 cluster of two (A/B runs)."""
    _require(x.is_cuda and w1.is_cuda and w2.is_cuda, "ffn_fused: CUDA tensors only")
    _require(x.dtype in (torch.float16, torch.bfloat16) and w1.dtype == x.dtype and w2.dtype == x.dtype,
             "ffn_fused: fp16/bf16 operands of one dtype")
    E = x.shape[-1]
    F = w1.shape[0]
    _require(w1.dim() == 2 and w2.dim() == 2 and tuple(w1.shape) == (F, E) and tuple(w2.shape) == (E, F) and
             w1.stride(1) == 1 and w2.stride(1) == 1, "ffn_fused: w1 must be [F, E] and w2 [E, F] with unit inner stride")
    for b, n in ((b1, F), (b2, E)):
        _require(b is None or (b.dtype == torch.float32 and b.is_contiguous() and b.numel() == n), "ffn_fused: biases fp32 [F] / [E]")
    x2 = x.reshape(-1, E)
    if x2.stride(1) != 1 or x2.stride(0) % 8 or x2.data_ptr() % 16:
        x2 = x2.contiguous()
    M = x2.shape[0]
    if out is None:
        out = torch.empty((M, E), dtype=torch.float32, device=x.device)
        res = out.view(*x.shape[:-1], E)
    else:
        _require(out.dtype == torch.float32 and out.dim() == 2 and tuple(out.shape) == (M, E) and out.stride(1) == 1 and out.is_cuda,
                 "ffn_fused: out must be fp32 [M, E] with unit inner stride")
        res = out
    with torch.cuda.device(x.device), _timed(("ffn_fused", M, E, F)):
        rc = _lib.lib.ape_ffn_fused(x2.data_ptr(), x2.stride(0), w1.data_ptr(), w1.stride(0),
                                    b1.data_ptr() if b1 is not None else None, w2.data_ptr(), w2.stride(0),
                                    b2.data_ptr() if b2 is not None else None, out.data_ptr(), out.stride(0), M, E, F,
                                    _lib.dtype_code(x.dtype), int(variant), _lib.current_stream_ptr())
    _lib.check(rc, "ape_ffn_fused")
    return res


def conv3x3_supported(H, W, Cin, Cout, dtype):
    if dtype not in (torch.float16, torch.bfloat16) or Cin % 64 or Cout % 8:
        return False
    tw = 128
    while tw > 8 and W % tw:
        tw >>= 1
    return W % tw == 0 and H % (128 // tw) == 0


def conv3x3_nhwc(x, weight_ohwi, bias=None, act=None):
    """3x3 / stride 1 / zero padding 1 convolution over token-major activations x [B,H,W,Cin] (ape_conv3x3_nhwc: implicit GEMM on
    the wgmma kernel, 4-D TMA boxes at shifted positions).  weight_ohwi [Cout,3,3,Cin] contiguous, same 16-bit dtype."""
    _require(x.is_cuda and x.dim() == 4 and x.is_contiguous() and weight_ohwi.is_contiguous() and x.dtype == weight_ohwi.dtype,
             "conv3x3: contiguous CUDA NHWC input and OHWI weight of one dtype")
    B, H, W, Cin = x.shape
    Cout = weight_ohwi.shape[0]
    _require(tuple(weight_ohwi.shape) == (Cout, 3, 3, Cin), "conv3x3: weight must be [Cout,3,3,Cin]")
    y = torch.empty((B, H, W, Cout), dtype=x.dtype, device=x.device)
    with torch.cuda.device(x.device), _timed(("conv3x3", B * H * W, Cout, 9 * Cin)):
        rc = _lib.lib.ape_conv3x3_nhwc(x.data_ptr(), weight_ohwi.data_ptr(), y.data_ptr(),
                                       bias.data_ptr() if bias is not None else None, B, H, W, Cin, Cout,
                                       _lib.dtype_code(x.dtype), ACT[act], _lib.current_stream_ptr())
    _lib.check(rc, "ape_conv3x3_nhwc")
    return y


def linear_rope_tc(x, weight, bias, cos, sin, num_channels, head_dim, pos_map=None):
    """Fused qkv projection + 2-D RoPE on the q and k thirds (ape_gemm_tn_rope): x [M, K] @ weight[3C, K]^T + bias with the
    rotary embedding applied in the GEMM epilogue (fp32, before the single rounding).  Returns [M, 3C]."""
    _require(x.is_cuda and x.dim() == 2 and x.dtype == weight.dtype and x.dtype in (torch.float16, torch.bfloat16),
             "linear_rope_tc: 2-D fp16/bf16 CUDA operands")
    M, K = x.shape
    N = weight.shape[0]
    _require(weight.shape[1] == K and x.stride(1) == 1 and weight.stride(1) == 1 and x.stride(0) % 8 == 0 and
             weight.stride(0) % 8 == 0, "linear_rope_tc: bad operand layout")
    _require(cos.dtype == torch.float32 and cos.is_contiguous() and sin.is_contiguous() and cos.shape[1] == head_dim,
             "linear_rope_tc: cos/sin must be contiguous fp32 [npos, head_dim]")
    out = torch.empty((M, N), dtype=x.dtype, device=x.device)
    with torch.cuda.device(x.device), _timed(("gemm_tn", M, N, K)):
        rc = _lib.lib.ape_gemm_tn_rope(x.data_ptr(), x.stride(0), weight.data_ptr(), weight.stride(0), out.data_ptr(), N,
                                       bias.data_ptr() if bias is not None else None, M, N, K, _lib.dtype_code(x.dtype),
                                       _lib.dtype_code(x.dtype), cos.data_ptr(), sin.data_ptr(),
                                       pos_map.data_ptr() if pos_map is not None else None, cos.shape[0], int(head_dim),
                                       2 * int(num_channels), 0, _lib.current_stream_ptr())
    _lib.check(rc, "ape_gemm_tn_rope")
    return out


def cached(obj, slot, dtype, key, build):
    """Per-object cache of re-laid-out weights with ONE ENTRY PER ENGINE DTYPE: `build()` runs when the entry of `dtype` is
    missing or its `key` (parameter versions / pointers) changed.  Entries of other dtypes are never evicted: a CUDA graph
    captured in fp16 keeps reading its fp16 copies after the model has also run in bf16 (capturing a new graph calls
    torch.cuda.empty_cache(), which would unmap an evicted copy under the old graph)."""
    d = obj.__dict__.setdefault(slot, {})
    e = d.get(dtype)
    if e is None or e[0] != key:
        with torch.no_grad():
            e = (key, build())
        d[dtype] = e
    return e[1]


def packed(module, dtype, extra=None):
    """(weight in `dtype`, fp32 bias) of an nn.Linear / nn.LayerNorm-like module, cached on the module and
    refreshed when its parameters change (load_state_dict, .to()).  LayerNorm weights stay fp32."""
    w, b = module.weight, getattr(module, "bias", None)
    key = (w._version, w.data_ptr(), None if b is None else (b._version, b.data_ptr()))
    return cached(module, "_ape_packed", dtype, key, lambda: (
        w.detach().to(dtype if w.dim() >= 2 else torch.float32).contiguous(),
        None if b is None else b.detach().to(torch.float32).contiguous()))


def linear_module_tc(module, x, act=None, residual=None, out_dtype=None, out=None):
    """nn.Linear forward on the tensor cores (weights packed once per dtype)."""
    w, b = packed(module, x.dtype)
    return linear_tc(x, w, b, act=act, residual=residual, out_dtype=out_dtype, out=out)


def layernorm_module(module, x, out_dtype=None):
    w, b = packed(module, torch.float32)
    return layernorm(x, w, b, eps=module.eps, out_dtype=out_dtype)


def layernorm(x, weight, bias, eps=1e-5, out_dtype=None, row_map=None, out=None, scale_out=None):
    """LayerNorm over the last dim (ape_layernorm).  x [..., C] with unit inner stride and uniform row
    pitch; weight / bias fp32.  row_map: int32 [rows] output row of each input row (or None).

    out_dtype=torch.float8_e4m3fn (or an e4m3 `out`): returns (q [rows, C] e4m3, scale [rows] fp32) with q * scale[:, None]
    the LayerNorm output, s = max|row| / 448 per row (ape_layernorm_e4m3; C <= 1024); `scale_out` is an optional fp32
    buffer for the scales, indexed like the output rows."""
    C = x.shape[-1]
    x2 = x.reshape(-1, C) if x.dim() != 2 else x
    _require(x2.is_cuda and x2.stride(1) == 1, "layernorm: CUDA tensor with unit inner stride")
    _require(weight.dtype == torch.float32 and bias.dtype == torch.float32, "layernorm: fp32 weight / bias")
    rows = x2.shape[0]
    out_dtype = out.dtype if out is not None else (out_dtype or x.dtype)
    if out_dtype == torch.float8_e4m3fn:
        if out is None:
            out = torch.empty((rows, (C + 15) // 16 * 16), dtype=out_dtype, device=x.device)[:, :C]
        _require(out.dim() == 2 and out.stride(1) == 1 and out.is_cuda, "layernorm: bad e4m3 `out`")
        if scale_out is None:
            scale_out = torch.empty((out.shape[0],), dtype=torch.float32, device=x.device)
        _require(scale_out.dtype == torch.float32 and scale_out.is_contiguous() and scale_out.numel() == out.shape[0],
                 "layernorm: scale_out must be fp32 [output rows]")
        with torch.cuda.device(x.device), _timed(("layernorm_e4m3", rows, C)):
            rc = _lib.lib.ape_layernorm_e4m3(x2.data_ptr(), x2.stride(0), out.data_ptr(), out.stride(0), scale_out.data_ptr(),
                                             weight.data_ptr(), bias.data_ptr(),
                                             row_map.data_ptr() if row_map is not None else None, rows, C, float(eps),
                                             _lib.dtype_code(x2.dtype), _lib.current_stream_ptr())
        _lib.check(rc, "ape_layernorm_e4m3")
        return out, scale_out
    if out is None:
        out = torch.empty((rows, C), dtype=out_dtype, device=x.device)
    with torch.cuda.device(x.device), _timed(("layernorm", rows, C)):
        rc = _lib.lib.ape_layernorm(x2.data_ptr(), x2.stride(0), out.data_ptr(), out.stride(0), weight.data_ptr(),
                                    bias.data_ptr(), row_map.data_ptr() if row_map is not None else None, rows, C,
                                    float(eps), _lib.dtype_code(x2.dtype), _lib.dtype_code(out.dtype),
                                    _lib.current_stream_ptr())
    _lib.check(rc, "ape_layernorm")
    return out if x.dim() == 2 or out.shape[1] != C else out.view(*x.shape[:-1], C)


def layernorm_ex(x, weight, bias, eps, weight2=None, bias2=None, eps2=0.0, col_add=None, row_add=None, out_dtype=None):
    """One pass over x [B, rows, C] (or [rows, C]) for LN -> optional second LN -> + col_add[image] -> (y, y + row_add)
    (ape_layernorm_ex; the previous encoder layer's last norm, the fusion layer's layer_norm_v, gamma_v * delta_v and
    `query + query_pos` in one kernel).  weights fp32 [C]; col_add fp32 [B, C]; row_add like x in the output dtype.
    Returns (y, y2) with y2 None when row_add is None.

    weight None: no normalisation.  With neither weight2 nor col_add, y is x itself (not copied) and the kernel only writes
    y2 = x + row_add: `query + query_pos` of an encoder's first layer when no fusion layer precedes it."""
    C = x.shape[-1]
    _require(x.is_cuda and x.is_contiguous(), "layernorm_ex: contiguous CUDA tensor")
    x2 = x.view(-1, C)
    rows = x2.shape[0]
    rpi = x.shape[-2] if x.dim() == 3 else rows
    out_dtype = out_dtype or x.dtype
    if weight is None:
        _require(bias is None and weight2 is None, "layernorm_ex: bias / weight2 without weight")
    add_only = weight is None and col_add is None and out_dtype == x.dtype
    _require(not add_only or row_add is not None, "layernorm_ex: nothing to compute")
    y = x if add_only else torch.empty(x.shape, dtype=out_dtype, device=x.device)
    y2 = None
    if row_add is not None:
        _require(row_add.dtype == out_dtype and row_add.is_contiguous() and row_add.numel() == x.numel(),
                 "layernorm_ex: row_add must match x in the output dtype")
        y2 = torch.empty(x.shape, dtype=out_dtype, device=x.device)
    if col_add is not None:
        col_add = col_add.reshape(-1, C)
        _require(col_add.dtype == torch.float32 and col_add.is_contiguous() and col_add.shape[0] * rpi == rows,
                 "layernorm_ex: col_add must be fp32 [images, C]")
    for t in (weight, bias, weight2, bias2):
        _require(t is None or (t.dtype == torch.float32 and t.is_contiguous()), "layernorm_ex: fp32 weights")
    with torch.cuda.device(x.device), _timed(("layernorm_ex", rows, C, weight2 is not None, row_add is not None)):
        rc = _lib.lib.ape_layernorm_ex(
            x2.data_ptr(), C, None if add_only else y.data_ptr(), C, weight.data_ptr() if weight is not None else None,
            bias.data_ptr() if bias is not None else None, float(eps),
            weight2.data_ptr() if weight2 is not None else None, bias2.data_ptr() if bias2 is not None else None, float(eps2),
            col_add.data_ptr() if col_add is not None else None, C, int(rpi),
            row_add.data_ptr() if row_add is not None else None, C, y2.data_ptr() if y2 is not None else None, C,
            rows, C, _lib.dtype_code(x.dtype), _lib.dtype_code(out_dtype), _lib.current_stream_ptr())
    _lib.check(rc, "ape_layernorm_ex")
    return y, y2


def groupnorm_nhwc(x, weight, bias, groups, eps=1e-5, out_dtype=None, out=None):
    """GroupNorm over token-major activations x [B, rows, C] (ape_groupnorm_nhwc); weight / bias fp32 [C].
    out: optional [B, rows, C] view (unit channel stride, any batch stride) the result is written into."""
    _require(x.is_cuda and x.dim() == 3 and x.is_contiguous(), "groupnorm_nhwc: contiguous CUDA [B, rows, C]")
    B, rows, C = x.shape
    if out is None:
        out = torch.empty((B, rows, C), dtype=out_dtype or x.dtype, device=x.device)
    _require(out.shape == x.shape and out.stride(2) == 1 and out.stride(1) == C, "groupnorm_nhwc: bad `out` view")
    ws = torch.empty((int(_lib.lib.ape_groupnorm_workspace_bytes(B, rows, C)),), dtype=torch.uint8, device=x.device)
    with torch.cuda.device(x.device), _timed(("groupnorm", B, rows, C)):
        rc = _lib.lib.ape_groupnorm_nhwc(x.data_ptr(), C, out.data_ptr(), C, out.stride(0) if B > 1 else 0, weight.data_ptr(),
                                         bias.data_ptr(), ws.data_ptr(), B, rows, C, int(groups), float(eps),
                                         _lib.dtype_code(x.dtype), _lib.dtype_code(out.dtype), _lib.current_stream_ptr())
    _lib.check(rc, "ape_groupnorm_nhwc")
    return out


def rope_qk_(qkv, cos, sin, num_channels, head_dim, pos_map=None):
    """In-place 2-D RoPE on the q and k thirds of qkv [M, 3*num_channels] (ape_rope_qk)."""
    _require(qkv.is_cuda and qkv.dim() == 2 and qkv.stride(1) == 1, "rope: qkv must be a 2-D CUDA tensor")
    _require(cos.dtype == torch.float32 and cos.is_contiguous() and sin.is_contiguous() and cos.shape[1] == head_dim,
             "rope: cos/sin must be contiguous fp32 [npos, head_dim]")
    with torch.cuda.device(qkv.device), _timed(("rope_qk", qkv.shape[0], num_channels)):
        rc = _lib.lib.ape_rope_qk(qkv.data_ptr(), qkv.stride(0), cos.data_ptr(), sin.data_ptr(),
                                  pos_map.data_ptr() if pos_map is not None else None, qkv.shape[0], num_channels,
                                  head_dim, cos.shape[0], _lib.dtype_code(qkv.dtype), _lib.current_stream_ptr())
    _lib.check(rc, "ape_rope_qk")
    return qkv


def attention_supported(n, head_dim, dtype):
    return head_dim == 64 and n % 128 == 0 and dtype in (torch.float16, torch.bfloat16)


def attention_qkv(qkv, num_seq, n, heads, head_dim, scale, n_valid=None, stats_out=False, seq_stride=None, causal=False,
                  out_row_map=None, out=None, seg_start=None):
    """softmax(q k^T * scale) v for every (sequence, head) straight from the fused qkv buffer [num_seq*n, 3*heads*64]
    (ape_attn_fwd: flash attention on the wgmma tensor cores).  Returns [num_seq*n, heads*64].
    n_valid: sequences are padded to n rows and only the first n_valid keys count (rows beyond must be finite).
    stats_out=True: also returns fp32 [rows, heads, 2] (sum, sum of squares of each row's stored values per head).
    seq_stride: rows between sequences when they are packed tighter than n (then n_valid <= seq_stride < n; rows of a tile
    past n_valid are not written); causal: key t attends to keys <= t.
    out_row_map: int32 [qkv rows] (ape_attn_fwd_mapped): query row r is stored at row out_row_map[r] of `out` (required
    then, [rows, heads*64] in qkv's dtype) and of the statistics ([out rows, heads, 2]); -1 stores nothing.  The mapped rows
    must be distinct rows of `out`; rows no query maps to keep what `out` held.
    seg_start: int32 [num_seq * 128] (ape_attn_fwd_seg): every 128-row tile holds several short sequences; query row r
    attends key k of its tile iff seg_start[r] <= k <= r, with seg_start[r] the position in the tile where r's sequence
    starts (a pad row: its own position).  Needs n = 128, causal=True and no n_valid / seq_stride / out_row_map."""
    _require(qkv.is_cuda and qkv.dim() == 2 and qkv.stride(1) == 1, "attention: qkv must be a 2-D CUDA tensor")
    stride = n if seq_stride is None else int(seq_stride)
    _require(qkv.shape[0] >= (num_seq - 1) * stride + (n_valid or n) and qkv.shape[1] == 3 * heads * head_dim, "attention: qkv shape")
    C = heads * head_dim
    if seg_start is not None:
        _require(seg_start.is_cuda and seg_start.dtype == torch.int32 and seg_start.dim() == 1 and seg_start.is_contiguous() and
                 seg_start.numel() == num_seq * n, "attention: seg_start must be a contiguous int32 CUDA vector with one entry per query row")
        _require(out_row_map is None and not stats_out, "attention: seg_start goes with neither out_row_map nor stats_out")
    if out_row_map is not None:
        _require(out_row_map.is_cuda and out_row_map.dtype == torch.int32 and out_row_map.dim() == 1 and
                 out_row_map.is_contiguous() and out_row_map.numel() >= (num_seq - 1) * stride + min(stride, n),
                 "attention: out_row_map must be a contiguous int32 CUDA vector with one entry per query row")
        _require(out is not None and out.is_cuda and out.dim() == 2 and out.dtype == qkv.dtype and out.shape[1] == C and
                 out.stride(1) == 1, "attention: out_row_map needs `out` [rows, heads*head_dim] in qkv's dtype")
    else:
        _require(out is None, "attention: `out` is only taken with out_row_map")
        # packed sequences leave the rows between n_valid and the stride unwritten; they come back as masked KEYS of the next
        # layer, and 0 * NaN in P V would poison it: those rows must stay finite
        alloc = torch.zeros if (stride < n or (n_valid is not None and n_valid < n)) else torch.empty
        out = alloc((qkv.shape[0], C), dtype=qkv.dtype, device=qkv.device)
    stats = torch.empty((out.shape[0], heads, 2), dtype=torch.float32, device=qkv.device) if stats_out else None
    args = (qkv.data_ptr(), qkv.stride(0), out.data_ptr(), out.stride(0), int(num_seq), int(n), int(n if n_valid is None else n_valid),
            int(heads), int(head_dim), float(scale), _lib.dtype_code(qkv.dtype), stats.data_ptr() if stats is not None else None,
            stride, 1 if causal else 0, int(qkv.shape[0]))
    with torch.cuda.device(qkv.device), _timed(("attention", num_seq, n, heads)):
        if seg_start is not None:
            rc = _lib.lib.ape_attn_fwd_seg(*args, seg_start.data_ptr(), _lib.current_stream_ptr())
        elif out_row_map is None:
            rc = _lib.lib.ape_attn_fwd_ex(*args, _lib.current_stream_ptr())
        else:
            rc = _lib.lib.ape_attn_fwd_mapped(*args, out_row_map.data_ptr(), _lib.current_stream_ptr())
    _lib.check(rc, "ape_attn_fwd")
    return (out, stats) if stats_out else out


def text_embed_packed(token_embedding, positional_embedding, tok, pos):
    """x[r] = token_embedding[tok[r]] + positional_embedding[pos[r]] as fp32 [rows, D] (ape_text_embed_packed): the text
    tower's first residual over length-packed prompts.  Tables fp32 [vocab, D] / [ctx, D]; tok / pos int32 [rows]; rows with
    pos < 0 (pad rows) are zeros."""
    for t in (token_embedding, positional_embedding):
        _require(t.is_cuda and t.dtype == torch.float32 and t.dim() == 2 and t.is_contiguous(), "text_embed_packed: contiguous fp32 CUDA tables")
    D = token_embedding.shape[1]
    _require(positional_embedding.shape[1] == D, "text_embed_packed: tables of one width")
    for t in (tok, pos):
        _require(t.is_cuda and t.dtype == torch.int32 and t.dim() == 1 and t.is_contiguous() and t.numel() == tok.numel(),
                 "text_embed_packed: tok / pos must be contiguous int32 CUDA vectors of one length")
    x = torch.empty((tok.numel(), D), dtype=torch.float32, device=tok.device)
    with torch.cuda.device(tok.device), _timed(("text_embed_packed", tok.numel(), D)):
        rc = _lib.lib.ape_text_embed_packed(token_embedding.data_ptr(), positional_embedding.data_ptr(), tok.data_ptr(), pos.data_ptr(),
                                            x.data_ptr(), tok.numel(), D, token_embedding.shape[0], positional_embedding.shape[0],
                                            _lib.current_stream_ptr())
    _lib.check(rc, "ape_text_embed_packed")
    return x


def rows_gather(x, rows):
    """x[rows] for fp32 x [M, D] (unit inner stride) and int64 rows [n], every entry in [0, M) (ape_rows_gather)."""
    _require(x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1, "rows_gather: fp32 2-D CUDA tensor")
    _require(rows.is_cuda and rows.dtype == torch.int64 and rows.dim() == 1 and rows.is_contiguous(), "rows_gather: contiguous int64 CUDA rows")
    out = torch.empty((rows.numel(), x.shape[1]), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device), _timed(("rows_gather", rows.numel(), x.shape[1])):
        rc = _lib.lib.ape_rows_gather(x.data_ptr(), x.stride(0), rows.data_ptr(), out.data_ptr(), out.stride(0), rows.numel(),
                                      x.shape[1], _lib.current_stream_ptr())
    _lib.check(rc, "ape_rows_gather")
    return out


def attention_cross(q, k, v, num_seq, nq, nkv, n_valid, heads, head_dim, scale):
    """softmax(q k^T * scale) v with separate tensors and 64- / 256-channel heads (ape_attn_cross_fwd).
    q [num_seq*nq, heads*head_dim], k / v [num_seq*nkv, heads*head_dim] (rows may be column slices of wider buffers);
    nq % 128 == 0, nkv % 64 == 0, keys >= n_valid masked.  Returns [num_seq*nq, heads*head_dim]."""
    for t in (q, k, v):
        _require(t.is_cuda and t.dim() == 2 and t.stride(1) == 1 and t.dtype == q.dtype, "attention_cross: 2-D CUDA tensors of one dtype")
    C = heads * head_dim
    _require(q.shape == (num_seq * nq, C) and k.shape == (num_seq * nkv, C) and v.shape == (num_seq * nkv, C), "attention_cross: shapes")
    out = torch.empty((num_seq * nq, C), dtype=q.dtype, device=q.device)
    with torch.cuda.device(q.device), _timed(("attention_cross", num_seq, nq, n_valid, heads, head_dim)):
        rc = _lib.lib.ape_attn_cross_fwd(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
                                         out.data_ptr(), out.stride(0), int(num_seq), int(nq), int(nkv), int(n_valid), int(heads),
                                         int(head_dim), float(scale), _lib.dtype_code(q.dtype), _lib.current_stream_ptr())
    _lib.check(rc, "ape_attn_cross_fwd")
    return out


def vlf_pool(v, qa, qc, stable_softmax_2d=True):
    """sum_s softmax_s(v_s . qa[h] + qc[h]) * v_s for every head -> fp32 [B, NH, C]  (ape_vlf_pool)."""
    _require(v.is_cuda and v.dim() == 3 and v.is_contiguous(), "vlf_pool: contiguous CUDA [B,S,C]")
    B, S, C = v.shape
    NH = qa.shape[1]
    qa = qa.float().contiguous()
    qc = qc.float().contiguous()
    nbytes = int(_lib.lib.ape_vlf_pool_workspace_bytes(B, S, C, NH))
    ws = torch.empty((nbytes // 4,), dtype=torch.float32, device=v.device)
    ptr, strips = ctypes.c_void_p(), ctypes.c_int()
    with torch.cuda.device(v.device), _timed(("vlf_pool", B, S, C, NH)):
        rc = _lib.lib.ape_vlf_pool(v.data_ptr(), qa.data_ptr(), qc.data_ptr(), ws.data_ptr(), ctypes.byref(ptr),
                                   ctypes.byref(strips), B, S, C, NH, 1 if stable_softmax_2d else 0,
                                   _lib.dtype_code(v.dtype), _lib.current_stream_ptr())
    _lib.check(rc, "ape_vlf_pool")
    off = (ptr.value - ws.data_ptr()) // 4
    part = ws[off: off + B * strips.value * NH * (C + 1)].view(B, strips.value, NH, C + 1).sum(1)  # fixed order
    return part[..., :C] / part[..., C:]


def nms_sorted_mask(sorted_boxes, iou_threshold, n_valid=None):
    """Greedy NMS over boxes ALREADY sorted by descending score: uint8 keep mask [n] (static shape, no host
    synchronisation: usable inside CUDA-graph capture) and the int32 [1] number of survivors.
    n_valid: optional int32 [1] device tensor; only the first n_valid boxes are real (keep = 0 for the rest)."""
    _require(sorted_boxes.is_cuda and sorted_boxes.dim() == 2 and sorted_boxes.shape[1] == 4 and
             sorted_boxes.dtype == torch.float32 and sorted_boxes.is_contiguous(), "nms: boxes must be contiguous CUDA fp32 [n,4]")
    n = sorted_boxes.shape[0]
    keep = torch.empty((n,), dtype=torch.uint8, device=sorted_boxes.device)
    count = torch.zeros((1,), dtype=torch.int32, device=sorted_boxes.device)
    if n == 0:
        return keep, count
    ws = torch.empty((int(_lib.lib.ape_nms_workspace_bytes(n)),), dtype=torch.uint8, device=sorted_boxes.device)
    with torch.cuda.device(sorted_boxes.device), _timed(("nms", n)):
        if n_valid is None:
            rc = _lib.lib.ape_nms_sorted(sorted_boxes.data_ptr(), n, float(iou_threshold), ws.data_ptr(), keep.data_ptr(),
                                         count.data_ptr(), _lib.current_stream_ptr())
        else:
            _require(n_valid.is_cuda and n_valid.dtype == torch.int32 and n_valid.numel() == 1, "nms: n_valid must be int32 [1]")
            rc = _lib.lib.ape_nms_sorted_dev(sorted_boxes.data_ptr(), n, n_valid.data_ptr(), float(iou_threshold), ws.data_ptr(),
                                             keep.data_ptr(), count.data_ptr(), _lib.current_stream_ptr())
    _lib.check(rc, "ape_nms_sorted")
    return keep, count


def nms_classwise(boxes, scores, score_thresh, iou_threshold, row_valid=None):
    """Class-aware NMS over ALL (query, class) pairs with score > score_thresh (ape_nms_classwise): boxes [Q,4] fp32 xyxy,
    scores [Q,N] fp32.  Returns fp32 [N,Q] (class-major): the score where the pair survives, -inf elsewhere.  Static
    shapes, no host synchronisation.  Bounded memory: Q*Q/8 bytes of workspace whatever N is (the dense n x n bit matrix of
    `nms_sorted_mask` would need terabytes for the 1.08 M pairs of a 1203-name vocabulary at threshold 0)."""
    _require(boxes.is_cuda and boxes.dtype == torch.float32 and boxes.is_contiguous() and boxes.dim() == 2 and boxes.shape[1] == 4,
             "nms_classwise: boxes must be contiguous CUDA fp32 [Q,4]")
    _require(scores.is_cuda and scores.dtype == torch.float32 and scores.dim() == 2 and scores.stride(1) == 1 and
             scores.shape[0] == boxes.shape[0], "nms_classwise: scores must be CUDA fp32 [Q,N]")
    Q, N = scores.shape
    _require(Q <= 1024, f"nms_classwise: at most 1024 queries (got {Q})")
    out = torch.empty((N, Q), dtype=torch.float32, device=scores.device)
    ws = torch.empty((max(1, int(_lib.lib.ape_nms_classwise_workspace_bytes(Q))),), dtype=torch.uint8, device=scores.device)
    if row_valid is not None:
        _require(row_valid.dtype == torch.uint8 and row_valid.is_contiguous() and row_valid.numel() == Q, "nms_classwise: row_valid uint8 [Q]")
    with torch.cuda.device(scores.device), _timed(("nms_classwise", Q, N)):
        rc = _lib.lib.ape_nms_classwise(boxes.data_ptr(), scores.data_ptr(), scores.stride(0),
                                        row_valid.data_ptr() if row_valid is not None else None, Q, N, float(score_thresh),
                                        float(iou_threshold), ws.data_ptr(), out.data_ptr(), _lib.current_stream_ptr())
    _lib.check(rc, "ape_nms_classwise")
    return out


def nms(boxes, scores, iou_threshold):
    """torchvision.ops.nms replacement: indices of kept boxes, sorted by descending score."""
    _require(boxes.is_cuda and boxes.dim() == 2 and boxes.shape[1] == 4, "nms: boxes must be CUDA [n,4]")
    n = boxes.shape[0]
    if n == 0:
        return torch.empty((0,), dtype=torch.int64, device=boxes.device)
    order = scores.sort(0, descending=True)[1]  # same ordering call as torchvision's nms kernel wrapper
    keep, _ = nms_sorted_mask(boxes.float().index_select(0, order).contiguous(), iou_threshold)
    return order[keep.bool()]


def batched_nms(boxes, scores, idxs, iou_threshold):
    """detectron2 / torchvision batched_nms (coordinate-offset trick, boxes.float()) on ape_nms_sorted."""
    if boxes.numel() == 0:
        return torch.empty((0,), dtype=torch.int64, device=boxes.device)
    if boxes.shape[0] > 32768:  # n x n/64 x 8 bytes of IoU bits: 134 MB at the limit
        raise RuntimeError(f"ape_b200.ops.batched_nms: {boxes.shape[0]} candidates need a dense IoU bit matrix of "
                           f"{boxes.shape[0] ** 2 // 8 / 2 ** 30:.1f} GiB; use ops.nms_classwise (per-class NMS over shared boxes)")
    boxes = boxes.float()
    max_coordinate = boxes.max()
    offsets = idxs.to(boxes) * (max_coordinate + torch.tensor(1).to(boxes))
    return nms(boxes + offsets[:, None], scores, iou_threshold)


def ref_update(delta, ref, valid_ratios, eps=1e-3):
    """(sigmoid(delta + inverse_sigmoid(ref)), new_ref[:, :, None] * cat(valid_ratios, valid_ratios)[:, None]) for 4-d reference
    points (ape_ref_update): delta / ref fp32 [B,Q,4], valid_ratios fp32 [B,L,2] -> fp32 [B,Q,4], [B,Q,L,4]."""
    _require(delta.is_cuda and delta.dtype == torch.float32 and ref.dtype == torch.float32 and delta.shape == ref.shape and
             delta.shape[-1] == 4 and delta.dim() == 3, "ref_update: CUDA fp32 [B,Q,4] tensors")
    B, Q, _ = delta.shape
    L = valid_ratios.shape[1]
    delta, ref = delta.contiguous(), ref.contiguous()
    vr = valid_ratios.float().contiguous()
    new_ref = torch.empty_like(delta)
    ref_in = torch.empty((B, Q, L, 4), dtype=torch.float32, device=delta.device)
    with torch.cuda.device(delta.device), _timed(("ref_update", B, Q, L)):
        rc = _lib.lib.ape_ref_update(delta.data_ptr(), ref.data_ptr(), vr.data_ptr(), new_ref.data_ptr(), ref_in.data_ptr(), B, Q, L,
                                     float(eps), _lib.current_stream_ptr())
    _lib.check(rc, "ape_ref_update")
    return new_ref, ref_in


def gemv_f32(x, weight, bias=None):
    """F.linear(x, weight, bias) in fp32 for 1..4 rows of x (ape_gemv_f32: one warp per output row); larger batches are split."""
    _require(x.is_cuda and weight.is_cuda and x.dtype == torch.float32 and weight.dtype == torch.float32, "gemv_f32: CUDA fp32 tensors")
    K = x.shape[-1]
    N = weight.shape[0]
    x2 = x.reshape(-1, K).contiguous()
    weight = weight.contiguous()
    _require(weight.shape[1] == K and K % 4 == 0, "gemv_f32: weight [N,K], K a multiple of 4")
    y = torch.empty((x2.shape[0], N), dtype=torch.float32, device=x.device)
    bptr = None
    if bias is not None:
        bias = bias.float().contiguous()
        bptr = bias.data_ptr()
    with torch.cuda.device(x.device), _timed(("gemv", x2.shape[0], N, K)):
        for b0 in range(0, x2.shape[0], 4):
            nb = min(4, x2.shape[0] - b0)
            rc = _lib.lib.ape_gemv_f32(weight.data_ptr(), x2[b0:].data_ptr(), bptr, y[b0:].data_ptr(), nb, N, K, _lib.current_stream_ptr())
            _lib.check(rc, "ape_gemv_f32")
    return y.view(*x.shape[:-1], N)


def mask_crop_and_resize(mask_logits, index, boxes, padded_hw, mask_size=128):
    """`BitMasks(F.interpolate(mask_logits[index], padded_hw, "bilinear").sigmoid() > 0.5).crop_and_resize(boxes, mask_size)`
    (deformable_detr_segm_vl.py:569-598) for the kept queries of one image: mask_logits [Q,h,w] (fp32 / fp16 / bf16, CUDA),
    index int64 [K], boxes fp32 [K,4] in padded-image pixels -> bool [K,mask_size,mask_size].  One bit per upsampled pixel of
    workspace; the fp32 full-resolution maps are never formed."""
    _require(mask_logits.is_cuda and mask_logits.dim() == 3 and mask_logits.is_contiguous(), "mask_crop: contiguous CUDA logits [Q,h,w]")
    K = int(index.numel())
    out = torch.empty((K, mask_size, mask_size), dtype=torch.uint8, device=mask_logits.device)
    if K == 0:
        return out.bool()
    index = index.to(device=mask_logits.device, dtype=torch.int64).contiguous()
    boxes = boxes.to(device=mask_logits.device, dtype=torch.float32).contiguous()
    _require(tuple(boxes.shape) == (K, 4), "mask_crop: boxes must be [K,4]")
    Hp, Wp = int(padded_hw[0]), int(padded_hw[1])
    ws = torch.empty((int(_lib.lib.ape_mask_crop_workspace_bytes(K, Hp, Wp)),), dtype=torch.uint8, device=mask_logits.device)
    with torch.cuda.device(mask_logits.device), _timed(("mask_crop", K, Hp, Wp)):
        rc = _lib.lib.ape_mask_crop(mask_logits.data_ptr(), index.data_ptr(), boxes.data_ptr(), ws.data_ptr(), out.data_ptr(), K,
                                    mask_logits.shape[1], mask_logits.shape[2], Hp, Wp, int(mask_size),
                                    _lib.dtype_code(mask_logits.dtype), _lib.current_stream_ptr())
    _lib.check(rc, "ape_mask_crop")
    return out.view(torch.bool)


def paste_masks_in_image(masks, boxes, image_shape, threshold=0.5):
    """detectron2.layers.mask_ops.paste_masks_in_image for 0 / 1 masks [N,S,S] (bool or float) and boxes [N,4] (output-image
    pixels) -> bool [N,H,W] (ape_mask_paste: no sampling grid, no float maps in memory)."""
    N, S = masks.shape[0], masks.shape[-1]
    img_h, img_w = int(image_shape[0]), int(image_shape[1])
    out = torch.empty((N, img_h, img_w), dtype=torch.uint8, device=masks.device)
    if N == 0:
        return out.view(torch.bool)
    _require(masks.is_cuda and masks.dim() == 3 and masks.shape[1] == S, "mask_paste: CUDA masks [N,S,S]")
    m8 = masks.view(torch.uint8) if masks.dtype == torch.bool else (masks >= 0.5).to(torch.uint8)
    m8 = m8.contiguous()
    boxes = boxes.to(device=masks.device, dtype=torch.float32).contiguous()
    with torch.cuda.device(masks.device), _timed(("mask_paste", N, img_h, img_w)):
        rc = _lib.lib.ape_mask_paste(m8.data_ptr(), boxes.data_ptr(), out.data_ptr(), N, S, img_h, img_w, float(threshold),
                                     _lib.current_stream_ptr())
    _lib.check(rc, "ape_mask_paste")
    return out.view(torch.bool)


def rle_counts_to_string(counts):
    """cocoapi rleToString (ape_rle_to_string, host): uint32 run lengths -> the compressed `counts` bytes of a COCO RLE."""
    import numpy as np

    c = np.ascontiguousarray(counts, dtype=np.uint32)
    out = np.empty((7 * max(len(c), 1),), dtype=np.uint8)
    n = int(_lib.lib.ape_rle_to_string(c.ctypes.data, len(c), out.ctypes.data))
    _lib.check(0 if n >= 0 else n, "ape_rle_to_string")
    return out[:n].tobytes()


def paste_masks_rle(masks, boxes, image_shape, threshold=0.5):
    """`[mask_util.encode(np.asfortranarray(m)) for m in paste_masks_in_image(masks, boxes, image_shape)]` without the dense
    masks (ape_mask_paste_rle): list of {"size": [H, W], "counts": bytes} — the run boundaries of every pasted mask are found on the
    device in column-major order (two passes over (mask, column) CTAs) and only they cross to the host."""
    import numpy as np

    N, S = masks.shape[0], masks.shape[-1]
    H, W = int(image_shape[0]), int(image_shape[1])
    if N == 0:
        return []
    _require(masks.is_cuda and masks.dim() == 3 and masks.shape[1] == S, "paste_masks_rle: CUDA masks [N,S,S]")
    m8 = (masks.view(torch.uint8) if masks.dtype == torch.bool else (masks >= 0.5).to(torch.uint8)).contiguous()
    boxes = boxes.to(device=masks.device, dtype=torch.float32).contiguous()
    stream = _lib.current_stream_ptr()
    col_count = torch.empty((N, W), dtype=torch.int32, device=masks.device)
    with torch.cuda.device(masks.device), _timed(("mask_rle", N, H, W)):
        rc = _lib.lib.ape_mask_paste_rle(m8.data_ptr(), boxes.data_ptr(), N, S, H, W, float(threshold), col_count.data_ptr(), None,
                                         None, stream)
        _lib.check(rc, "ape_mask_paste_rle")
        csum = col_count.view(-1).to(torch.int64).cumsum(0)
        col_offset = (csum - col_count.view(-1)).contiguous()
        per_mask = csum.view(N, W)[:, -1].cpu()           # boundaries up to the end of every mask (the one synchronisation)
        total = int(per_mask[-1])
        positions = torch.empty((max(total, 1),), dtype=torch.int32, device=masks.device)
        rc = _lib.lib.ape_mask_paste_rle(m8.data_ptr(), boxes.data_ptr(), N, S, H, W, float(threshold), None, col_offset.data_ptr(),
                                         positions.data_ptr(), stream)
        _lib.check(rc, "ape_mask_paste_rle")
    pos = positions[:total].cpu().numpy().astype(np.int64)
    ends = per_mask.numpy()
    out, lo = [], 0
    for n in range(N):
        p = pos[lo:int(ends[n])]
        lo = int(ends[n])
        counts = np.diff(np.concatenate(([0], p, [H * W])))  # leading run of zeros, ..., trailing run
        out.append({"size": [H, W], "counts": rle_counts_to_string(counts)})
    return out


MASK_PACK_HEAD = 60  # bytes before a mask slot: 13 fp32 selection columns, int32 kind, int32 length
MASK_SLOT_EMPTY, MASK_SLOT_CHARS, MASK_SLOT_BITS = 0, 1, 2


def mask_pack(mask_logits, rows, out_sizes, padded_hw, slot, mask_size=128):
    """The kept masks of the packed selection rows as COCO run-length codes in fixed-size slots (ape_mask_pack), with no host
    synchronisation: mask_logits [B,Q,h,w] (CUDA fp32 / fp16 / bf16), rows fp32 [B,topk,13] (`forward_packed`'s columns),
    out_sizes [(H, W)] per image (the rows' output sizes, as host ints) -> uint8 [B, topk, MASK_PACK_HEAD + slot]: each slot's
    13 columns as bytes, int32 kind (MASK_SLOT_*) and length, then the "counts" characters or, for a code longer than the slot,
    the mask_size^2 mask as bits (little-endian bit order).  Slots past the kept count and boxes that are empty after the
    rescale and clip hold no mask."""
    _require(mask_logits.is_cuda and mask_logits.dim() == 4 and mask_logits.is_contiguous(), "mask_pack: contiguous CUDA logits [B,Q,h,w]")
    B, Q, h, w = (int(v) for v in mask_logits.shape)
    _require(rows.dtype == torch.float32 and rows.is_contiguous() and rows.dim() == 3 and rows.shape[0] == B and rows.shape[2] == 13
             and rows.device == mask_logits.device, "mask_pack: rows must be contiguous fp32 [B,topk,13] on the logits' device")
    _require(len(out_sizes) == B, "mask_pack: one output size per image")
    topk, slot, S = int(rows.shape[1]), int(slot), int(mask_size)
    out = torch.empty((B, topk, MASK_PACK_HEAD + slot), dtype=torch.uint8, device=mask_logits.device)
    if B == 0 or topk == 0:
        return out
    Hp, Wp = int(padded_hw[0]), int(padded_hw[1])
    hw = (ctypes.c_int * (2 * B))(*[int(v) for s in out_sizes for v in s])
    max_w = max(int(s[1]) for s in out_sizes)
    ws = torch.empty((max(int(_lib.lib.ape_mask_pack_workspace_bytes(topk, Hp, Wp, max_w, S, slot)), 1),), dtype=torch.uint8,
                     device=mask_logits.device)
    with torch.cuda.device(mask_logits.device), _timed(("mask_pack", B, topk, Hp, Wp, slot)):
        rc = _lib.lib.ape_mask_pack(mask_logits.data_ptr(), rows.data_ptr(), hw, ws.data_ptr(), out.data_ptr(), B, topk, Q, h, w, Hp,
                                    Wp, S, slot, _lib.dtype_code(mask_logits.dtype), _lib.current_stream_ptr())
    _lib.check(rc, "ape_mask_pack")
    return out


SEMSEG_BAND_BYTES = 256 << 20  # bound of the resampled-operand workspace of semseg_label


def semseg_label(mask_logits, query_index, cls, padded_hw, img_hw, out_hw, class0_const=None, band_bytes=None):
    """Semantic label map of one image without the class-score maps: (label int64 [out_h, out_w], score fp32 [out_h, out_w]) =
    the argmax over classes, and its value, of

        sem_seg_postprocess(einsum("qc,qhw->chw", cls, F.interpolate(mask_logits[query_index][None], padded_hw,
                            "bilinear").sigmoid()[0]), img_hw, *out_hw)          (class 0 set to class0_const if given)

    (deformable_detr_segm_vl.py:875-918 + detectron2 sem_seg_postprocess + the evaluator's argmax).  Both resizes are linear,
    so the class contraction runs at the output resolution: bands of output rows are resampled once into a pixel-major 16-bit
    operand (ape_semseg_resample, at most `band_bytes`, default SEMSEG_BAND_BYTES) and contracted with cls^T by the wgmma GEMM
    whose epilogue keeps only the per-pixel argmax (ape_gemm_tn_argmax).  Nothing of size classes x pixels is ever written.

    mask_logits [Q, h, w] CUDA fp32 / fp16 / bf16; query_index int64 [K]; cls [K, N] fp16 / bf16 (the operand dtype: the
    class weights of the kept queries); class0_const: the constant of class 0 (stuff_prob_thing), which then stays out of the
    GEMM.  Ties resolve to the lowest class, as torch.argmax.  The band workspace comes from PyTorch's caching allocator, so a
    captured CUDA graph keeps it in the graph's own pool."""
    _require(mask_logits.is_cuda and mask_logits.dim() == 3 and mask_logits.is_contiguous(), "semseg_label: contiguous CUDA logits [Q,h,w]")
    _require(cls.dim() == 2 and cls.dtype in (torch.float16, torch.bfloat16), "semseg_label: cls must be fp16 / bf16 [K, N]")
    dev = mask_logits.device
    K, N = int(cls.shape[0]), int(cls.shape[1])
    _require(int(query_index.numel()) == K and N >= 1, "semseg_label: query_index [K] and cls [K, N >= 1] disagree")
    Hp, Wp = int(padded_hw[0]), int(padded_hw[1])
    ih, iw = int(img_hw[0]), int(img_hw[1])
    oh, ow = int(out_hw[0]), int(out_hw[1])
    _require(0 < ih <= Hp and 0 < iw <= Wp and oh > 0 and ow > 0, "semseg_label: bad image / output size")
    P = oh * ow
    keys = torch.empty((P,), dtype=torch.int64, device=dev)  # u64 keys (common.cuh argmax_key)
    label = torch.empty((oh, ow), dtype=torch.int64, device=dev)
    score = torch.empty((oh, ow), dtype=torch.float32, device=dev)
    col_base = 0 if class0_const is None else 1
    init = (float("-inf"), 0) if class0_const is None else (float(class0_const), 0)
    if K == 0 and N > col_base and (class0_const is None or float(class0_const) < 0.0):
        init = (0.0, col_base)  # no kept query: every class the GEMM would cover scores 0
    stream = _lib.current_stream_ptr()
    with torch.cuda.device(dev), _timed(("semseg_label", K, N, P)):
        _lib.check(_lib.lib.ape_semseg_keys_init(keys.data_ptr(), P, init[0], init[1], stream), "ape_semseg_keys_init")
        if K > 0:
            Kp = (K + 7) // 8 * 8
            dt = cls.dtype
            w = torch.zeros((N - col_base, Kp), dtype=dt, device=dev)
            w[:, :K] = cls[:, col_base:].t()
            index = query_index.to(device=dev, dtype=torch.int64).contiguous()
            budget = SEMSEG_BAND_BYTES if band_bytes is None else int(band_bytes)
            rows = max(1, min(oh, budget // (ow * Kp * 2)))
            ws = torch.empty((rows * ow, Kp), dtype=dt, device=dev)
            for r0 in range(0, oh, rows):
                nr = min(rows, oh - r0)
                rc = _lib.lib.ape_semseg_resample(mask_logits.data_ptr(), index.data_ptr(), ws.data_ptr(), Kp, K,
                                                  mask_logits.shape[1], mask_logits.shape[2], Hp, Wp, ih, iw, oh, ow, r0, nr,
                                                  _lib.dtype_code(mask_logits.dtype), _lib.dtype_code(dt), stream)
                _lib.check(rc, "ape_semseg_resample")
                if N > col_base:
                    rc = _lib.lib.ape_gemm_tn_argmax(ws.data_ptr(), Kp, w.data_ptr(), Kp, keys[r0 * ow:].data_ptr(), nr * ow,
                                                     N - col_base, Kp, col_base, _lib.dtype_code(dt), stream)
                    _lib.check(rc, "ape_gemm_tn_argmax")
        _lib.check(_lib.lib.ape_semseg_keys_decode(keys.data_ptr(), P, label.data_ptr(), score.data_ptr(), stream),
                   "ape_semseg_keys_decode")
    return label, score


def _label_rle_table(raw, P, H, W):
    """A codes body (P x (int32 label, character offset, length), then the characters) -> the list label_map_rle returns."""
    import numpy as np

    raw = np.asarray(raw, dtype=np.uint8)
    table = raw[:12 * P].view(np.int32).reshape(P, 3)
    chars = raw[12 * P:]
    return [{"label": int(c), "segmentation": {"size": [H, W], "counts": chars[o:o + n].tobytes()}} for c, o, n in table.tolist()]


def label_map_rle(label):
    """`[{"label": c, "segmentation": mask_util.encode(np.asfortranarray((label == c).astype(np.uint8)))} for c in np.unique(label)]`
    (detectron2's encode_json_sem_seg without the per-label masks, ape_label_rle): label int64 [H, W] on a CUDA device, values in
    [0, 65535] -> one cocoapi run-length code per label present, in ascending label order.  One synchronising read of the map's
    sizes (labels present, boundaries), then the codes are built on the device and copied to the host in one copy."""
    _require(label.is_cuda and label.dim() == 2 and label.dtype == torch.int64, "label_map_rle: CUDA int64 label map [H, W]")
    label = label.contiguous()
    H, W = int(label.shape[0]), int(label.shape[1])
    dev = label.device
    stream = _lib.current_stream_ptr()
    with torch.cuda.device(dev), _timed(("label_rle", H, W)):
        ws = torch.empty((int(_lib.lib.ape_label_rle_workspace_bytes(W, 0, 0)),), dtype=torch.uint8, device=dev)
        sizes = torch.empty((3,), dtype=torch.int32, device=dev)
        _lib.check(_lib.lib.ape_label_rle_sizes(label.data_ptr(), H, W, ws.data_ptr(), sizes.data_ptr(), stream), "ape_label_rle_sizes")
        host = sizes.cpu()  # P, m, labels out of range
        P, m = int(host[0]), int(host[1])
        hs = (ctypes.c_int * 3)(*[int(v) for v in host.tolist()])
        ws = torch.empty((int(_lib.lib.ape_label_rle_workspace_bytes(W, max(P, 0), 2 * max(m, 0) + 1)),), dtype=torch.uint8, device=dev)
        out = torch.empty((max(int(_lib.lib.ape_label_rle_out_bytes(max(P, 0), max(m, 0))), 4),), dtype=torch.uint8, device=dev)
        info = torch.empty((3,), dtype=torch.int32, device=dev)
        _lib.check(_lib.lib.ape_label_rle(label.data_ptr(), H, W, hs, ws.data_ptr(), out.data_ptr(), info.data_ptr(), stream),
                   "ape_label_rle")
        n = int(info[1])
        raw = out[:n].cpu().numpy()
    return _label_rle_table(raw, P, H, W)


def label_map_from_rle(sem_seg_rle):
    """The label map back from label_map_rle's list (host, numpy): int64 [H, W], each pixel the label whose code covers it."""
    import numpy as np

    H, W = sem_seg_rle[0]["segmentation"]["size"]
    flat = np.zeros((H * W,), dtype=np.int64)  # column-major pixel order, as the codes
    for entry in sem_seg_rle:
        s = entry["segmentation"]["counts"]
        counts, p = [], 0
        while p < len(s):  # cocoapi rleFrString
            x, k, more = 0, 0, True
            while more:
                c = s[p] - 48
                x |= (c & 0x1F) << (5 * k)
                more = bool(c & 0x20)
                p += 1
                k += 1
                if not more and (c & 0x10):
                    x |= -1 << (5 * k)
            if len(counts) > 2:
                x += counts[-2]
            counts.append(x)
        ends = np.cumsum(counts)
        for lo, hi in zip(ends[0::2], ends[1::2]):  # odd runs are the label's pixels
            flat[lo:hi] = entry["label"]
    return flat.reshape(W, H).T.copy()


SEM_PACK_HEAD = 32  # bytes before an image's detections in forward_packed's semantic form: 8 int32 header fields
SEM_SLOT_NONE, SEM_SLOT_CODES, SEM_SLOT_MAP, SEM_SLOT_OVER = 0, 1, 2, 3


def semseg_pack(labels, num_labels, slots, info):
    """One semantic slot per image with no host synchronisation (ape_label_rle_pack): labels [int64 [H_b, W_b] CUDA] with values
    in [0, num_labels); slots uint8 [B, slot] (rows 4-byte aligned, each row contiguous); info int32 [B, 3] <- kind
    (SEM_SLOT_*), bytes used, labels present.  A slot holds the codes of label_map_rle (a table of P x (int32 label, int32
    character offset, int32 length), then the characters) when they fit, else the map as uint16 [H, W] when that fits, else
    nothing."""
    B = len(labels)
    _require(slots.dim() == 2 and slots.shape[0] == B and slots.dtype == torch.uint8 and slots.stride(1) == 1,
             "semseg_pack: slots must be uint8 [B, slot] with contiguous rows")
    _require(info.dtype == torch.int32 and info.is_contiguous() and tuple(info.shape) == (B, 3), "semseg_pack: info int32 [B, 3]")
    if B == 0:
        return
    dev = slots.device
    slot = int(slots.shape[1])
    max_w = max(int(l.shape[1]) for l in labels)
    ws = torch.empty((max(int(_lib.lib.ape_label_rle_pack_workspace_bytes(max_w, int(num_labels), slot)), 1),), dtype=torch.uint8,
                     device=dev)
    stream = _lib.current_stream_ptr()
    with torch.cuda.device(dev), _timed(("semseg_pack", B, slot)):
        for b, l in enumerate(labels):
            _require(l.is_cuda and l.dim() == 2 and l.dtype == torch.int64 and l.is_contiguous() and l.device == dev,
                     "semseg_pack: contiguous CUDA int64 label maps on the slots' device")
            rc = _lib.lib.ape_label_rle_pack(l.data_ptr(), int(l.shape[0]), int(l.shape[1]), int(num_labels), slot, ws.data_ptr(),
                                             slots[b].data_ptr(), info[b].data_ptr(), stream)
            _lib.check(rc, "ape_label_rle_pack")


def panoptic_winners(mask_logits, query_index, scores, padded_hw, img_hw, out_hw, prob):
    """Per-pixel winners and segment areas of the panoptic merge of one image without the [K, H, W] mask stacks:
    (ids int32 [out_h, out_w], counts int32 [3, K]).  With

        p = sem_seg_postprocess(F.interpolate(mask_logits[query_index][None].float(), padded_hw, "bilinear")[0], img_hw,
                                *out_hw).sigmoid()                                   [K, out_h, out_w]
        win = (scores[:, None, None] * p).argmax(0)                                  first maximum, as torch.argmax

    ids = win where p[win] >= prob, else -1; counts = (bincount(win), bincount(win[p[win] >= prob]), (p >= prob).sum((1, 2))),
    each of length K (deformable_detr_segm_vl.py:919-998, the three areas of every kept query).  A query whose score is -inf
    takes no part: it never wins and its counts are 0, so a keep mask can be applied without compacting the queries.

    mask_logits [Q, h, w] CUDA fp32 / fp16 / bf16; query_index int64 [K]; scores fp32 [K].  One call to ape_panoptic_winners
    (two kernels, capturable in a CUDA graph); K <= APE_PANOPTIC_MAX_K (4096)."""
    _require(mask_logits.is_cuda and mask_logits.dim() == 3 and mask_logits.is_contiguous(),
             "panoptic_winners: contiguous CUDA logits [Q,h,w]")
    dev = mask_logits.device
    K = int(query_index.numel())
    _require(query_index.dim() == 1 and scores.dim() == 1 and int(scores.numel()) == K,
             "panoptic_winners: query_index [K] and scores [K] disagree")
    Hp, Wp = int(padded_hw[0]), int(padded_hw[1])
    ih, iw = int(img_hw[0]), int(img_hw[1])
    oh, ow = int(out_hw[0]), int(out_hw[1])
    _require(0 < ih <= Hp and 0 < iw <= Wp and oh > 0 and ow > 0, "panoptic_winners: bad image / output size")
    index = query_index.to(device=dev, dtype=torch.int64).contiguous()
    sc = scores.to(device=dev, dtype=torch.float32).contiguous()
    ids = torch.empty((oh, ow), dtype=torch.int32, device=dev)
    counts = torch.empty((3, K), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev), _timed(("panoptic_winners", K, oh * ow)):
        rc = _lib.lib.ape_panoptic_winners(mask_logits.data_ptr(), index.data_ptr(), sc.data_ptr(), ids.data_ptr(), counts.data_ptr(),
                                           K, mask_logits.shape[1], mask_logits.shape[2], Hp, Wp, ih, iw, oh, ow, float(prob),
                                           _lib.dtype_code(mask_logits.dtype), _lib.current_stream_ptr())
        _lib.check(rc, "ape_panoptic_winners")
    return ids, counts


APE_PANOPTIC_MAX_K = 4096  # = include/ape_b200.h: queries per panoptic merge
PAN_PACK_HEAD = 32  # bytes before a panoptic slot's segment table: 8 int32 header fields
PAN_ROW = 12        # bytes per segment table row: int32 id, isthing, category_id


def panoptic_slot_bytes_needed(K, out_hw):
    """Bytes a panoptic slot needs for K queries and an output of out_hw: header, K table rows, the uint16 map."""
    return PAN_PACK_HEAD + PAN_ROW * int(K) + 2 * int(out_hw[0]) * int(out_hw[1])


def panoptic_pack(ids, counts, classes, num_classes, num_things, stuff_first, overlap_threshold, slot):
    """One image's panoptic slot from `panoptic_winners`' (ids, counts) with no host synchronisation (ape_panoptic_pack):
    postprocess._segments' decisions over the K queries in order and the painting of the map, on the device.  classes int32 [K]
    (the label of each query, in [0, num_classes)); slot uint8 [slot_bytes] contiguous, 4-byte aligned, at least
    panoptic_slot_bytes_needed(K, ids.shape) bytes.  The slot gets a header of 8 int32 (1, segments S, out_h, out_w, K, bytes used,
    0, 0), K rows of (int32 id, isthing, category_id) of which the first S are the segments in id order, the map as uint16
    [out_h, out_w] (0 = no segment), and zeros to its end."""
    _require(ids.is_cuda and ids.dim() == 2 and ids.dtype == torch.int32 and ids.is_contiguous(), "panoptic_pack: CUDA int32 ids [H, W]")
    K = int(counts.shape[1]) if counts.dim() == 2 else -1
    _require(counts.dtype == torch.int32 and counts.is_contiguous() and tuple(counts.shape) == (3, K), "panoptic_pack: int32 counts [3, K]")
    _require(classes.dtype == torch.int32 and classes.is_contiguous() and tuple(classes.shape) == (K,), "panoptic_pack: int32 classes [K]")
    _require(slot.dtype == torch.uint8 and slot.dim() == 1 and slot.is_contiguous(), "panoptic_pack: contiguous uint8 slot")
    dev = ids.device
    _require(counts.device == dev and classes.device == dev and slot.device == dev, "panoptic_pack: all tensors on one device")
    oh, ow = int(ids.shape[0]), int(ids.shape[1])
    n = int(slot.numel())
    _require(n >= panoptic_slot_bytes_needed(K, (oh, ow)),
             f"panoptic_pack: {panoptic_slot_bytes_needed(K, (oh, ow))} bytes needed for K={K} and {oh} x {ow}, the slot has {n}")
    ws = torch.empty((max(int(_lib.lib.ape_panoptic_pack_workspace_bytes(K, int(num_classes))), 1),), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev), _timed(("panoptic_pack", K, oh * ow)):
        rc = _lib.lib.ape_panoptic_pack(ids.data_ptr(), counts.data_ptr(), classes.data_ptr(), K, int(num_classes), int(num_things),
                                        1 if stuff_first else 0, float(overlap_threshold), oh, ow, ws.data_ptr(), slot.data_ptr(), n,
                                        _lib.current_stream_ptr())
        _lib.check(rc, "ape_panoptic_pack")


_RESAMPLE_TABLES = {}


def resample_tables(in_size, out_size, device):
    """Pillow's bilinear taps for one axis (ape_resample_coeffs_u8, the arithmetic of libImaging/Resample.c:precompute_coeffs +
    normalize_coeffs_8bpc) as device tensors: (bounds int32 [out,2], taps int32 [out,ksize], ksize).  Cached per geometry."""
    key = (int(in_size), int(out_size), str(device))
    hit = _RESAMPLE_TABLES.get(key)
    if hit is None:
        ksize = int(_lib.lib.ape_resample_ksize(int(in_size), int(out_size)))
        _lib.check(0 if ksize > 0 else ksize, "ape_resample_ksize")
        bounds = torch.empty((out_size, 2), dtype=torch.int32)
        kk = torch.empty((out_size, ksize), dtype=torch.int32)
        _lib.check(_lib.lib.ape_resample_coeffs_u8(int(in_size), int(out_size), bounds.data_ptr(), kk.data_ptr()), "ape_resample_coeffs_u8")
        if len(_RESAMPLE_TABLES) > 64:
            _RESAMPLE_TABLES.clear()
        hit = _RESAMPLE_TABLES[key] = (bounds.to(device), kk.to(device), ksize)
    return hit


def resize_u8_bilinear(img, new_h, new_w, flip_channels=False, out=None):
    """PIL `Image.fromarray(img).resize((new_w, new_h), BILINEAR)` of a uint8 HWC (or HW) image on the device, bit for bit,
    returned as the float32 [C, new_h, new_w] tensor the predictor puts into the model's input dict
    (ape/engine/defaults.py:221-222: `torch.as_tensor(image.astype("float32").transpose(2, 0, 1))`).
    img: CUDA uint8 [H,W,C] / [H,W] with contiguous pixels (rows may be pitched); flip_channels folds the `[:, :, ::-1]` of
    defaults.py:218-220 into the write; out: optional float32 [C,>=new_h,>=new_w] view to write into (e.g. a padded batch)."""
    _require(img.is_cuda and img.dtype == torch.uint8 and img.dim() in (2, 3), "resize_u8_bilinear: CUDA uint8 [H,W,C] or [H,W] image")
    if img.dim() == 2:
        img = img.unsqueeze(-1)
    H, W, C = img.shape
    _require(1 <= C <= 4 and img.stride(2) == 1 and img.stride(1) == C, "resize_u8_bilinear: pixels must be contiguous (1-4 channels)")
    new_h, new_w = int(new_h), int(new_w)
    if out is None:
        out = torch.empty((C, new_h, new_w), dtype=torch.float32, device=img.device)
    _require(out.is_cuda and out.dtype == torch.float32 and out.dim() == 3 and out.shape[0] == C and out.shape[1] >= new_h and
             out.shape[2] >= new_w and out.stride(2) == 1, "resize_u8_bilinear: out must be float32 [C,>=new_h,>=new_w] with unit column stride")
    bh, kh, ksh = resample_tables(W, new_w, img.device)
    bv, kv, ksv = resample_tables(H, new_h, img.device)
    tmp = torch.empty((H, new_w, C), dtype=torch.uint8, device=img.device)
    with torch.cuda.device(img.device), _timed(("resample", H, W, new_h, new_w)):
        rc = _lib.lib.ape_resample_u8(img.data_ptr(), img.stride(0), tmp.data_ptr(), out.data_ptr(), out.stride(0), out.stride(1),
                                      bh.data_ptr(), kh.data_ptr(), ksh, bv.data_ptr(), kv.data_ptr(), ksv, H, W, C, new_h, new_w,
                                      1 if flip_channels else 0, _lib.current_stream_ptr())
    _lib.check(rc, "ape_resample_u8")
    return out[:, :new_h, :new_w]


def ms_deform_attn_backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output, im2col_step=64):
    """[grad_value, grad_sampling_loc, grad_attn_weight] (ape_msda_bwd; ms_deform_attn_cuda.cu:84-160).  grad_value is
    accumulated in fp32 by vector atomics and cast to value's dtype at the end."""
    if not value.is_cuda:
        raise RuntimeError("Not implemented on the CPU")  # ms_deform_attn.h:60
    B, S, H, D, L, Q, P = _check_inputs(value, spatial_shapes, level_start_index, sampling_loc, attn_weight)
    _require(grad_output.is_cuda and grad_output.is_contiguous(), "grad_output tensor has to be contiguous")
    _require(grad_output.dtype == value.dtype and grad_output.numel() == B * Q * H * D, "grad_output must be [B,Q,H*D] of value's dtype")
    gv = torch.zeros((B, S, H, D), dtype=torch.float32, device=value.device)
    gl = torch.empty_like(sampling_loc)
    ga = torch.empty_like(attn_weight)
    with torch.cuda.device(value.device), _timed(("msda_bwd", B, S, Q, L, P, value.element_size())):
        rc = _lib.lib.ape_msda_bwd(value.data_ptr(), spatial_shapes.data_ptr(), level_start_index.data_ptr(), sampling_loc.data_ptr(),
                                   attn_weight.data_ptr(), grad_output.data_ptr(), gv.data_ptr(), gl.data_ptr(), ga.data_ptr(),
                                   B, S, H, D, L, Q, P, _lib.dtype_code(value.dtype), _lib.current_stream_ptr())
    _lib.check(rc, "ape_msda_bwd")
    return [gv if value.dtype == torch.float32 else gv.to(value.dtype), gl, ga]


def _ms_deform_attn_backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight,
                             grad_output, im2col_step):
    return ms_deform_attn_backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output, im2col_step)


def _register():
    try:
        lib = torch.library.Library(_NS, "DEF")
    except Exception:  # namespace already defined in this process (e.g. the reference's ape._C)
        lib = torch.library.Library(_NS, "FRAGMENT")
    defined = []
    for schema in (_FWD_SCHEMA, _BWD_SCHEMA):
        try:
            lib.define(schema)
            defined.append(schema.split("(")[0])
        except RuntimeError:
            pass  # already defined by someone else: leave theirs in place

    def _fwd(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, im2col_step):
        return ms_deform_attn_forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, im2col_step)

    def _fwd_cpu(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, im2col_step):
        raise RuntimeError("Not implemented on the CPU")

    if "ms_deform_attn_forward" in defined:
        lib.impl("ms_deform_attn_forward", _fwd, "CUDA")
        lib.impl("ms_deform_attn_forward", _fwd_cpu, "CPU")
    if "ms_deform_attn_backward" in defined:
        lib.impl("ms_deform_attn_backward", _ms_deform_attn_backward, "CUDA")
        lib.impl("ms_deform_attn_backward", lambda *a: _fwd_cpu(*a[:6]), "CPU")
    return lib


_LIBRARY = _register()


def pad_geometry(sizes, padded_hw, shapes, dim_t, level_embeds, engine_dtype, offset=0.0, eps=1e-6, scale=6.283185307179586,
                 normalize=True, want_pos=False):
    """The per-image-size geometry of a padded batch in one launch (ape_pad_geometry), what
    DeformableDetrTransformerVL.geometry returns for the padding masks F.interpolate'd from the image sizes, plus
    PositionEmbeddingSine's embedding: sizes int32 [B, 2] (h, w) on the device; padded_hw and the level shapes [L, 2] host ints;
    dim_t fp32 [E/2] (PositionEmbeddingSine.dim_t); level_embeds [L, E].  Returns a dict of mask_flatten bool [B, S],
    pos_lvl engine_dtype [B, S, E] (pos + level embedding), pos_flatten fp32 [B, S, E] (only with want_pos, else None),
    valid_ratios fp32 [B, L, 2], reference_points fp32 [B, S, L, 2], output_proposals fp32 [B, S, 4] and proposal_invalid
    bool [B, S, 1].  The outputs are allocated here, so inside a capture they belong to the graph's pool."""
    _require(sizes.is_cuda and sizes.dtype == torch.int32 and sizes.dim() == 2 and sizes.shape[1] == 2 and sizes.is_contiguous(),
             "pad_geometry: sizes must be a contiguous CUDA int32 [B, 2] tensor")
    dev = sizes.device
    B = int(sizes.shape[0])
    L = len(shapes)
    E = int(level_embeds.shape[-1]) if level_embeds.dim() == 2 else -1
    _require(level_embeds.dim() == 2 and int(level_embeds.shape[0]) >= L, "pad_geometry: level_embeds must be [L, E]")
    _require(dim_t.dim() == 1 and 2 * int(dim_t.numel()) == E, f"pad_geometry: dim_t must have E/2 = {E // 2} entries")
    hw = (ctypes.c_int * max(2 * L, 1))(*[int(v) for sh in shapes for v in sh])
    S = sum(int(h) * int(w) for h, w in shapes)
    dt = dim_t.to(device=dev, dtype=torch.float32).contiguous()
    lv = level_embeds.detach()[:L].to(device=dev, dtype=torch.float32).contiguous()
    out = dict(mask_flatten=torch.empty((B, S), dtype=torch.bool, device=dev),
               pos_lvl=torch.empty((B, S, E), dtype=engine_dtype, device=dev),
               pos_flatten=torch.empty((B, S, E), dtype=torch.float32, device=dev) if want_pos else None,
               valid_ratios=torch.empty((B, L, 2), dtype=torch.float32, device=dev),
               reference_points=torch.empty((B, S, L, 2), dtype=torch.float32, device=dev),
               output_proposals=torch.empty((B, S, 4), dtype=torch.float32, device=dev),
               proposal_invalid=torch.empty((B, S, 1), dtype=torch.bool, device=dev))
    code = _lib.dtype_code(engine_dtype) if engine_dtype in (torch.float32, torch.float16, torch.bfloat16) else -1
    pf = out["pos_flatten"]
    with torch.cuda.device(dev), _timed(("pad_geometry", B, S, E)):
        rc = _lib.lib.ape_pad_geometry(sizes.data_ptr(), B, int(padded_hw[0]), int(padded_hw[1]), hw, L, dt.data_ptr(), lv.data_ptr(),
                                       E, float(offset), float(eps), float(scale), 1 if normalize else 0,
                                       out["mask_flatten"].data_ptr(), out["pos_lvl"].data_ptr(), code,
                                       pf.data_ptr() if pf is not None else None, out["valid_ratios"].data_ptr(),
                                       out["reference_points"].data_ptr(), out["output_proposals"].data_ptr(),
                                       out["proposal_invalid"].data_ptr(), _lib.current_stream_ptr())
        _lib.check(rc, "ape_pad_geometry")
    return out


def zero_masked_rows_(x, mask):
    """In place: the rows of x [B, S, C] (CUDA, unit inner stride, uniform row pitch) whose mask [B, S] entry is true become +0.0,
    as `x.masked_fill(mask[..., None], 0)` would give them (ape_zero_masked_rows); the other rows are not written, so an all-false
    mask costs its read alone.  Returns x."""
    _require(x.is_cuda and x.dim() == 3 and x.stride(2) == 1 and x.stride(0) == x.shape[1] * x.stride(1),
             "zero_masked_rows_: CUDA [B,S,C] with uniform row pitch")
    _require(tuple(mask.shape) == tuple(x.shape[:2]) and mask.device == x.device, "zero_masked_rows_: mask must be [B,S] on x's device")
    m = mask.contiguous()
    m = m.view(torch.uint8) if m.dtype == torch.bool else m.to(torch.uint8)
    with torch.cuda.device(x.device), _timed(("zero_masked_rows", x.shape[0], x.shape[1], x.shape[2])):
        rc = _lib.lib.ape_zero_masked_rows(x.data_ptr(), x.stride(1), m.data_ptr(), x.shape[0] * x.shape[1], x.shape[2],
                                           _lib.dtype_code(x.dtype), _lib.current_stream_ptr())
    _lib.check(rc, "ape_zero_masked_rows")
    return x
