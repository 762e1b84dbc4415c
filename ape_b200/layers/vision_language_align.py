"""VisionLanguageAlign: the query x text-embedding open-vocabulary classifier.
Mirror of ape/layers/vision_language_align.py:8-52 (same constructor, same parameter names
`dot_product_projection_text`, `log_scale`, `bias_lang`, `bias0`)."""
import math

import torch
import torch.nn.functional as F
from torch import nn


class VisionLanguageAlign(nn.Module):
    def __init__(self, embed_dim, embed_dim_language, prior_prob=0.01, log_scale=0.0, clamp_dot_product=True):
        super().__init__()
        bias_value = -math.log((1 - prior_prob) / prior_prob)
        self.dot_product_projection_image = nn.Identity()
        self.dot_product_projection_text = nn.Linear(embed_dim_language, embed_dim, bias=True)
        self.log_scale = nn.Parameter(torch.Tensor([log_scale]))
        self.bias_lang = nn.Parameter(torch.zeros(embed_dim_language))
        self.bias0 = nn.Parameter(torch.Tensor([bias_value]))
        self.clamp_dot_product = clamp_dot_product

    def project_text(self, embedding, dtype):
        """Text-side half (vision_language_align.py:32-41); depends only on the vocabulary, so the
        engine computes it once per vocabulary instead of once per decoder level and image."""
        embedding = F.normalize(embedding.to(dtype), p=2, dim=-1)
        tokens = self.dot_product_projection_text(embedding / 2.0)
        bias = torch.matmul(embedding, self.bias_lang) + self.bias0
        return tokens, bias

    def _engine_weights(self, dtype):
        """Text projection with 1 / (2 * exp(log_scale)) folded in (16-bit operand) and `bias_lang` as an 8-row weight."""
        lin = self.dot_product_projection_text
        ps = (lin.weight, lin.bias, self.log_scale, self.bias_lang, self.bias0)
        from .. import ops

        def build():
            inv = torch.exp(-self.log_scale.detach().float())
            wt = (lin.weight.detach().float() * (0.5 * inv)).to(dtype).contiguous()
            bt = (lin.bias.detach().float() * inv).contiguous()
            wl = torch.zeros(8, lin.weight.shape[1], dtype=dtype, device=lin.weight.device)
            wl[0] = self.bias_lang.detach().to(dtype)
            bl = torch.zeros(8, dtype=torch.float32, device=lin.weight.device)
            bl[0] = self.bias0.detach().float()[0]
            return wt, bt, wl, bl

        return ops.cached(self, "_pk", dtype, (tuple(p._version for p in ps), lin.weight.data_ptr()), build)

    def forward_engine(self, x, embedding, n_cols=None):
        """Engine path (x [B,Q,C] fp16 / bf16 CUDA): the text projection, the language bias and the query x text contraction
        are wgmma GEMMs (ape_gemm_tn); fp32 accumulation, fp32 logits, bias + clamp in the epilogue.  The reference's own
        eval recipe runs this module in fp16 end to end (tools/train_net.py:641-642); here only the operands are 16-bit.
        n_cols (int32 [1] on the device, or None): the text is padded to embedding.shape[1] rows and only the first n_cols are
        classes; the contraction (ape_gemm_tn_cols_dev) writes -inf into the other columns."""
        from .. import ops

        wt, bt, wl, bl = self._engine_weights(x.dtype)
        e = F.normalize(embedding.float(), p=2, dim=-1).to(x.dtype)                      # (:35)
        tokens = ops.linear_tc(e, wt, bt)                                                # [B,N,C]: Linear(e / 2) / exp(log_scale)
        bias = ops.linear_tc(e, wl, bl, out_dtype=torch.float32)[..., 0].contiguous()    # [B,N]:   e . bias_lang + bias0
        act = "clamp" if self.clamp_dot_product else None
        if n_cols is not None:
            if act != "clamp":
                raise NotImplementedError("ape_b200: a padded prompt needs clamp_dot_product (the kernel clamps)")
            out = [ops.linear_cols_dev(x[b].contiguous(), tokens[b], bias[b], n_cols) for b in range(x.shape[0])]
            return torch.stack(out) if len(out) > 1 else out[0][None]
        out = [ops.linear_tc(x[b].contiguous(), tokens[b], bias[b], act=act, out_dtype=torch.float32) for b in range(x.shape[0])]
        return torch.stack(out) if len(out) > 1 else out[0][None]

    def forward(self, x, embedding, n_cols=None):
        if x.is_cuda and x.dtype in (torch.float16, torch.bfloat16) and x.dim() == 3 and x.shape[-1] % 8 == 0 \
                and embedding.shape[-1] % 8 == 0:
            return self.forward_engine(x, embedding, n_cols)
        if n_cols is not None:
            raise NotImplementedError("ape_b200: padded prompts run on the engine path only (16-bit CUDA operands)")
        tokens, bias = self.project_text(embedding, x.dtype)
        logit = torch.matmul(x, tokens.transpose(-1, -2)) / self.log_scale.exp() + bias.unsqueeze(1)
        if self.clamp_dot_product:
            logit = torch.clamp(logit, max=50000)
            logit = torch.clamp(logit, min=-50000)
        return logit
