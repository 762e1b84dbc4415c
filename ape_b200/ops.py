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
    if token_mask is not None:
        token_mask = token_mask.to(torch.uint8).contiguous()
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


def layernorm(x, weight, bias, eps=1e-5, out_dtype=None, row_map=None, out=None):
    """LayerNorm over the last dim (ape_layernorm).  x [..., C] with unit inner stride and uniform row
    pitch; weight / bias fp32.  row_map: int32 [rows] output row of each input row (or None)."""
    C = x.shape[-1]
    x2 = x.reshape(-1, C) if x.dim() != 2 else x
    _require(x2.is_cuda and x2.stride(1) == 1, "layernorm: CUDA tensor with unit inner stride")
    _require(weight.dtype == torch.float32 and bias.dtype == torch.float32, "layernorm: fp32 weight / bias")
    rows = x2.shape[0]
    out_dtype = out_dtype or x.dtype
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
    Returns (y, y2) with y2 None when row_add is None."""
    C = x.shape[-1]
    _require(x.is_cuda and x.is_contiguous(), "layernorm_ex: contiguous CUDA tensor")
    x2 = x.view(-1, C)
    rows = x2.shape[0]
    rpi = x.shape[-2] if x.dim() == 3 else rows
    out_dtype = out_dtype or x.dtype
    y = torch.empty(x.shape, dtype=out_dtype, device=x.device)
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
            x2.data_ptr(), C, y.data_ptr(), C, weight.data_ptr(), bias.data_ptr(), float(eps),
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


def attention_qkv(qkv, num_seq, n, heads, head_dim, scale, n_valid=None, stats_out=False, seq_stride=None, causal=False):
    """softmax(q k^T * scale) v for every (sequence, head) straight from the fused qkv buffer [num_seq*n, 3*heads*64]
    (ape_attn_fwd: flash attention on the wgmma tensor cores).  Returns [num_seq*n, heads*64].
    n_valid: sequences are padded to n rows and only the first n_valid keys count (rows beyond must be finite).
    stats_out=True: also returns fp32 [rows, heads, 2] (sum, sum of squares of each row's stored values per head).
    seq_stride: rows between sequences when they are packed tighter than n (then n_valid <= seq_stride < n; rows of a tile
    past n_valid are not written); causal: key t attends to keys <= t."""
    _require(qkv.is_cuda and qkv.dim() == 2 and qkv.stride(1) == 1, "attention: qkv must be a 2-D CUDA tensor")
    stride = n if seq_stride is None else int(seq_stride)
    _require(qkv.shape[0] >= (num_seq - 1) * stride + (n_valid or n) and qkv.shape[1] == 3 * heads * head_dim, "attention: qkv shape")
    # packed sequences leave the rows between n_valid and the stride unwritten; they come back as masked KEYS of the next
    # layer, and 0 * NaN in P V would poison it: those rows must stay finite
    alloc = torch.zeros if (stride < n or (n_valid is not None and n_valid < n)) else torch.empty
    out = alloc((qkv.shape[0], heads * head_dim), dtype=qkv.dtype, device=qkv.device)
    stats = torch.empty((qkv.shape[0], heads, 2), dtype=torch.float32, device=qkv.device) if stats_out else None
    with torch.cuda.device(qkv.device), _timed(("attention", num_seq, n, heads)):
        rc = _lib.lib.ape_attn_fwd_ex(qkv.data_ptr(), qkv.stride(0), out.data_ptr(), out.stride(0), int(num_seq), int(n),
                                      int(n if n_valid is None else n_valid), int(heads), int(head_dim), float(scale),
                                      _lib.dtype_code(qkv.dtype), stats.data_ptr() if stats is not None else None,
                                      stride, 1 if causal else 0, int(qkv.shape[0]), _lib.current_stream_ptr())
    _lib.check(rc, "ape_attn_fwd")
    return (out, stats) if stats_out else out


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
