"""Host-side mirror of the reference's MultiScaleDeformableAttention module
(ape/layers/multi_scale_deform_attn.py:127-358): same constructor arguments, same parameter
names (`sampling_offsets`, `attention_weights`, `value_proj`, `output_proj`) so reference
checkpoints load, same forward signature and semantics — but the tail (softmax, sampling-location
arithmetic, bilinear gather) is ONE launch of libape_b200's fused kernel, and the two
query-side linears run as one GEMM.  CUDA only; no CPU / PyTorch fallback."""
import math
import os
import warnings
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops


def _is_power_of_2(n):
    if (not isinstance(n, int)) or (n < 0):
        raise ValueError("invalid input for _is_power_of_2: {} (type: {})".format(n, type(n)))
    return (n & (n - 1) == 0) and n != 0


class MultiScaleDeformableAttention(nn.Module):
    def __init__(
        self,
        embed_dim: int = 256,
        num_heads: int = 8,
        num_levels: int = 4,
        num_points: int = 4,
        img2col_step: int = 64,
        dropout: float = 0.1,
        batch_first: bool = False,
        pytorch_attn: bool = False,
    ):
        super().__init__()
        if embed_dim % num_heads != 0:
            raise ValueError(
                "embed_dim must be divisible by num_heads, but got {} and {}".format(embed_dim, num_heads))
        if not _is_power_of_2(embed_dim // num_heads):
            warnings.warn("head dim should be a power of 2 for the vectorised sm_90a path")
        self.dropout = nn.Dropout(dropout)
        self.batch_first = batch_first
        self.im2col_step = img2col_step
        self.embed_dim = embed_dim
        self.num_heads = num_heads
        self.num_levels = num_levels
        self.num_points = num_points
        self.sampling_offsets = nn.Linear(embed_dim, num_heads * num_levels * num_points * 2)
        self.attention_weights = nn.Linear(embed_dim, num_heads * num_levels * num_points)
        self.value_proj = nn.Linear(embed_dim, embed_dim)
        self.output_proj = nn.Linear(embed_dim, embed_dim)
        # accepted for config compatibility; this engine has exactly one (CUDA) path
        self.pytorch_attn = pytorch_attn
        # engine: calls with at least this many queries gather from the pair layout (csrc/msda_pair.cu).  Off by default
        # (None): the gather itself is faster than the generic fused kernel on the encoder call, but the pairing pass
        # costs more than it saves in the model; APE_MSDA_PAIR=<min queries> (e.g. 2048) switches it on for A/B runs.
        env = os.environ.get("APE_MSDA_PAIR", "")
        self.pair_layout_min_queries = int(env) if env.isdigit() and int(env) > 0 else None
        self._qcat = None
        self.init_weights()

    def init_weights(self):
        """Same initialisation as multi_scale_deform_attn.py:190-213."""
        nn.init.constant_(self.sampling_offsets.weight.data, 0.0)
        thetas = torch.arange(self.num_heads, dtype=torch.float32) * (2.0 * math.pi / self.num_heads)
        grid = torch.stack([thetas.cos(), thetas.sin()], -1)
        grid = (grid / grid.abs().max(-1, keepdim=True)[0]).view(self.num_heads, 1, 1, 2)
        grid = grid.repeat(1, self.num_levels, self.num_points, 1)
        for i in range(self.num_points):
            grid[:, :, i, :] *= i + 1
        with torch.no_grad():
            self.sampling_offsets.bias = nn.Parameter(grid.view(-1))
        nn.init.constant_(self.attention_weights.weight.data, 0.0)
        nn.init.constant_(self.attention_weights.bias.data, 0.0)
        nn.init.xavier_uniform_(self.value_proj.weight.data)
        nn.init.constant_(self.value_proj.bias.data, 0.0)
        nn.init.xavier_uniform_(self.output_proj.weight.data)
        nn.init.constant_(self.output_proj.bias.data, 0.0)

    def _query_side_weights(self):
        """[sampling_offsets ; attention_weights] stacked so both come out of one GEMM."""
        ws, wa = self.sampling_offsets.weight, self.attention_weights.weight
        bs, ba = self.sampling_offsets.bias, self.attention_weights.bias
        key = (ws._version, wa._version, bs._version, ba._version, ws.data_ptr(), wa.data_ptr(), ws.dtype)
        if self._qcat is None or self._qcat[0] != key:
            with torch.no_grad():
                self._qcat = (key, torch.cat([ws, wa], 0).contiguous(), torch.cat([bs, ba], 0).contiguous())
        return self._qcat[1], self._qcat[2]

    def forward(
        self,
        query: torch.Tensor,
        key: Optional[torch.Tensor] = None,
        value: Optional[torch.Tensor] = None,
        identity: Optional[torch.Tensor] = None,
        query_pos: Optional[torch.Tensor] = None,
        key_padding_mask: Optional[torch.Tensor] = None,
        reference_points: Optional[torch.Tensor] = None,
        spatial_shapes: Optional[torch.Tensor] = None,
        level_start_index: Optional[torch.Tensor] = None,
        **kwargs,
    ) -> torch.Tensor:
        if not query.is_cuda:
            raise RuntimeError("ape_b200.MultiScaleDeformableAttention: CUDA tensors only (no CPU fallback)")
        if value is None:
            value = query
        if identity is None:
            identity = query
        if kwargs.get("query_with_pos") is not None:
            query = kwargs["query_with_pos"]  # engine: `query + query_pos` already formed by the producing kernel
        elif query_pos is not None:
            query = query + query_pos
        if not self.batch_first:
            query = query.permute(1, 0, 2)
            value = value.permute(1, 0, 2)
        bs, num_query, _ = query.shape
        bs, num_value, _ = value.shape
        if reference_points.shape[-1] not in (2, 4):
            raise ValueError("Last dim of reference_points must be 2 or 4, but get {} instead.".format(
                reference_points.shape[-1]))

        engine = query.dtype in (torch.float16, torch.bfloat16) and value.dtype == query.dtype
        wq, bq = self._query_side_weights()
        if engine:
            # tensor-core path: wgmma GEMMs (fp32 accumulate), fused gather kernel, residual in the epilogue
            value = ops.linear_module_tc(self.value_proj, value)
            w16, b32 = ops.cached(self, "_q16", query.dtype, (wq._version, wq.data_ptr()),
                                  lambda: (wq.to(query.dtype).contiguous(), bq.float().contiguous()))
            qo = ops.linear_tc(query, w16, b32)
        else:
            value = self.value_proj(value)
            qo = F.linear(query, wq, bq)  # [B,Q, H*L*P*2 + H*L*P]
        n_off = self.num_heads * self.num_levels * self.num_points * 2
        ref32 = reference_points.to(torch.float32).contiguous()
        host_shapes = kwargs.get("host_shapes")
        head_dim = self.embed_dim // self.num_heads
        if engine and host_shapes is not None and self.pair_layout_min_queries is not None and \
                num_query >= self.pair_layout_min_queries and \
                ops.msda_pair_supported(host_shapes, self.num_heads, head_dim, self.num_points, value.dtype):
            # many queries: pair layout (token s | token s+1 in one 128-byte line) + 16-bit corner blend
            value2 = ops.msda_pair_values(value, self.num_heads, token_mask=key_padding_mask)
            output = ops.ms_deform_attn_pair_fused_forward(value2, spatial_shapes, level_start_index, host_shapes,
                                                           qo[..., :n_off], qo[..., n_off:], ref32, self.num_points)
        else:
            if key_padding_mask is not None:
                value = value.masked_fill(key_padding_mask[..., None], float(0))
            value = value.view(bs, num_value, self.num_heads, -1).contiguous()
            output = ops.ms_deform_attn_fused_forward(value, spatial_shapes, level_start_index, qo[..., :n_off], qo[..., n_off:],
                                                      ref32, self.num_points)
        if engine and self.batch_first and identity.dtype in (output.dtype, torch.float32):
            # `sum_dtype=torch.float32` (engine layers): identity + output_proj(...) leaves the epilogue as fp32
            return ops.linear_module_tc(self.output_proj, output, residual=identity.contiguous(),
                                        out_dtype=kwargs.get("sum_dtype"))
        output = self.output_proj(output)
        if not self.batch_first:
            output = output.permute(1, 0, 2)
        return self.dropout(output) + identity
