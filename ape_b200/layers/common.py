"""Small building blocks whose parameter names match the third-party modules the reference
instantiates (detrex MLP / FFN, detectron2 Conv2d+norm, channels-first LayerNorm), so reference
checkpoints load by name.  Semantics restated from detrex@776058e / detectron2@017abbf
(SURVEY.md Appendix B)."""
import torch
import torch.nn as nn
import torch.nn.functional as F


class LayerNorm2d(nn.Module):
    """detectron2 `LayerNorm` (get_norm("LN")): normalise over C of an NCHW tensor, eps 1e-6."""

    def __init__(self, channels, eps=1e-6):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(channels))
        self.bias = nn.Parameter(torch.zeros(channels))
        self.eps = eps

    def forward(self, x):
        # as F.layer_norm over the channel dim (same statistics as the d2 formula)
        return F.layer_norm(x.permute(0, 2, 3, 1), (x.shape[1],), self.weight, self.bias, self.eps).permute(0, 3, 1, 2)


class ConvNorm(nn.Conv2d):
    """detectron2 `Conv2d(..., norm=, activation=)`: parameters `weight`, `bias`, `norm.*`."""

    def __init__(self, cin, cout, kernel_size, padding=0, bias=True, norm=None, activation=None):
        super().__init__(cin, cout, kernel_size, padding=padding, bias=bias)
        self.norm = norm
        self.activation = activation

    def forward(self, x):
        x = F.conv2d(x, self.weight, self.bias, self.stride, self.padding)
        if self.norm is not None:
            x = self.norm(x)
        if self.activation is not None:
            x = self.activation(x)
        return x


class MLP(nn.Module):
    """detrex MLP: `layers.{i}` Linear, ReLU between."""

    def __init__(self, input_dim, hidden_dim, output_dim, num_layers):
        super().__init__()
        self.num_layers = num_layers
        h = [hidden_dim] * (num_layers - 1)
        self.layers = nn.ModuleList(nn.Linear(n, k) for n, k in zip([input_dim] + h, h + [output_dim]))

    def forward(self, x, out_dtype=None):
        if x.is_cuda and x.dtype in (torch.float16, torch.bfloat16):
            from .. import ops  # tensor-core path: bias + ReLU in the GEMM epilogue, weights packed once

            for i, layer in enumerate(self.layers):
                last = i == self.num_layers - 1
                x = ops.linear_module_tc(layer, x, act=None if last else "relu", out_dtype=out_dtype if last else None)
            return x
        for i, layer in enumerate(self.layers):
            x = F.relu(layer(x)) if i < self.num_layers - 1 else layer(x)
        return x


class FFN(nn.Module):
    """detrex FFN(num_fcs=2): `layers.0.0` Linear -> ReLU -> `layers.1` Linear, + identity."""

    def __init__(self, embed_dim, feedforward_dim):
        super().__init__()
        self.layers = nn.Sequential(
            nn.Sequential(nn.Linear(embed_dim, feedforward_dim), nn.ReLU(inplace=True), nn.Dropout(0.0)),
            nn.Linear(feedforward_dim, embed_dim),
            nn.Dropout(0.0),
        )

    def forward(self, x, out_dtype=None):
        if x.is_cuda and x.dtype in (torch.float16, torch.bfloat16):
            from .. import ops  # tensor-core path: ReLU and the residual add live in the GEMM epilogues

            fc1, fc2 = self.layers[0][0], self.layers[1]
            if out_dtype == torch.float32 and x.shape[-1] == 256 and fc1.out_features % 64 == 0:
                # one kernel, the [tokens, feedforward_dim] hidden activation never reaches memory; same bits as below
                w1, b1 = ops.packed(fc1, x.dtype)
                w2, b2 = ops.packed(fc2, x.dtype)
                return ops.ffn_fused(x, w1, b1, w2, b2)
            h = ops.linear_module_tc(fc1, x, act="relu")
            # out_dtype float32: the sum x + ffn(x) leaves the epilogue unrounded (it feeds a LayerNorm)
            return ops.linear_module_tc(fc2, h, residual=x.contiguous(), out_dtype=out_dtype)
        return x + self.layers[1](F.relu(self.layers[0][0](x)))


def inverse_sigmoid(x, eps=1e-3):
    """detrex.utils.inverse_sigmoid (eps 1e-3, not the 1e-5 of ape/utils/misc.py:543)."""
    x = x.clamp(min=0, max=1)
    return torch.log(x.clamp(min=eps) / (1 - x).clamp(min=eps))


def box_cxcywh_to_xyxy(b):
    cx, cy, w, h = b.unbind(-1)
    return torch.stack([cx - 0.5 * w, cy - 0.5 * h, cx + 0.5 * w, cy + 0.5 * h], dim=-1)
