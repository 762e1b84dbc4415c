"""Deformable VL transformer (encoder with VisionLanguageFusion, two-stage proposal selection,
decoder with iterative box refinement).

Mirror of ape/modeling/ape_deta/deformable_transformer_vl.py (`DeformableDetrTransformerEncoderVL`
:20-121, `DeformableDetrTransformerDecoderVL` :124-255, `DeformableDetrTransformerVL` :258-699) and
of the detrex containers it is built from (BaseTransformerLayer / TransformerLayerSequence / FFN /
MultiheadAttention, SURVEY.md Appendix B): same constructor arguments, same forward signatures,
same parameter names (`layers.{i}.attentions.{j}`, `layers.{i}.ffns.0.layers.{0.0,1}`,
`layers.{i}.norms.{k}`, `vl_layers.{i}.b_attn…`, `level_embeds`, `enc_output`, `pos_trans`, …)."""
import copy
import math

import torch
import torch.nn as nn
import torch.nn.functional as F
import torchvision

from .. import ops
from ..layers import MultiScaleDeformableAttention
from ..layers.common import FFN, box_cxcywh_to_xyxy, inverse_sigmoid


class _SelfAttention(nn.Module):
    """detrex MultiheadAttention wrapper (parameters under `.attn`): q = k = x + pos, v = x."""

    def __init__(self, embed_dim, num_heads):
        super().__init__()
        self.embed_dim, self.num_heads = embed_dim, num_heads
        self.attn = nn.MultiheadAttention(embed_dim, num_heads, dropout=0.0, batch_first=True)

    def _packed(self, dtype):
        """In / out projections re-laid out for ape_attn_fwd: every head padded from E/nh to 64 channels with zero rows
        (zero columns in the output projection), q | k | v thirds as the kernel's fused-qkv column layout."""
        w, b = self.attn.in_proj_weight, self.attn.in_proj_bias
        wo, bo = self.attn.out_proj.weight, self.attn.out_proj.bias
        E, nh = self.embed_dim, self.num_heads
        hd = E // nh

        def build():
            def pad_rows(wpart, bpart):  # [E, E] / [E] -> [nh*64, E] / [nh*64]
                wp = wpart.new_zeros(nh, 64, E)
                wp[:, :hd] = wpart.view(nh, hd, E)
                bp = bpart.new_zeros(nh, 64)
                bp[:, :hd] = bpart.view(nh, hd)
                return wp.view(nh * 64, E), bp.view(nh * 64)
            wq, bq = pad_rows(w[:E], b[:E])
            wk, bk = pad_rows(w[E:2 * E], b[E:2 * E])
            wv, bv = pad_rows(w[2 * E:], b[2 * E:])
            wop = wo.new_zeros(E, nh, 64)
            wop[:, :, :hd] = wo.view(E, nh, hd)
            return (torch.cat([wq, wk], 0).detach().to(dtype).contiguous(), torch.cat([bq, bk]).detach().float().contiguous(),
                    wv.detach().to(dtype).contiguous(), bv.detach().float().contiguous(),
                    wop.view(E, nh * 64).detach().to(dtype).contiguous(), bo.detach().float().contiguous())

        return ops.cached(self, "_pk", dtype, (w._version, b._version, wo._version, bo._version, w.data_ptr()), build)

    def forward(self, x, pos):
        E, nh = self.embed_dim, self.num_heads
        if x.is_cuda and x.dtype in (torch.float16, torch.bfloat16) and E // nh <= 64:
            # engine path: wgmma GEMMs for the in / out projections (residual in the epilogue) and the repo's wgmma
            # flash-attention kernel over the queries (rows padded to a multiple of 128, padded keys masked)
            wqk, bqk, wv, bv, wo, bo = self._packed(x.dtype)
            B, N, _ = x.shape
            NP = (N + 127) // 128 * 128
            C = nh * 64
            # padded rows must be finite (zeros): they are never written, so one zero-filled buffer per geometry serves every call
            # (a fresh torch.zeros here was a fill kernel per layer inside the captured graph)
            bk = (B, NP, C, x.dtype, str(x.device))
            if getattr(self, "_qkv_buf", (None,))[0] != bk:
                self._qkv_buf = (bk, torch.zeros((B, NP, 3 * C), dtype=x.dtype, device=x.device))
            buf = self._qkv_buf[1]
            xp = x + pos.to(x.dtype)
            for b in range(B):
                ops.linear_tc(xp[b], wqk, bqk, out=buf[b, :N, : 2 * C])
                ops.linear_tc(x[b], wv, bv, out=buf[b, :N, 2 * C:])
            o = ops.attention_qkv(buf.view(B * NP, 3 * C), B, NP, nh, 64, (E // nh) ** -0.5, n_valid=N).view(B, NP, C)
            outs = [ops.linear_tc(o[b, :N], wo, bo, residual=x[b].contiguous(), out_dtype=torch.float32) for b in range(B)]
            return outs[0].unsqueeze(0) if B == 1 else torch.stack(outs)
        w, b = self.attn.in_proj_weight, self.attn.in_proj_bias
        qk = F.linear(x + pos, w[: 2 * E], b[: 2 * E])
        v = F.linear(x, w[2 * E:], b[2 * E:])
        B, N, _ = x.shape
        q, k = qk[..., :E], qk[..., E:]
        q, k, v = (t.reshape(B, N, nh, E // nh).transpose(1, 2) for t in (q, k, v))
        o = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, N, E)
        return x + self.attn.out_proj(o)


class _EncoderLayer(nn.Module):
    """BaseTransformerLayer(("self_attn","norm","ffn","norm")) with an MSDA self-attention."""

    def __init__(self, embed_dim, num_heads, ffn_dim, num_levels):
        super().__init__()
        self.embed_dim = embed_dim
        self.pre_norm = False
        self.attentions = nn.ModuleList([MultiScaleDeformableAttention(
            embed_dim=embed_dim, num_heads=num_heads, dropout=0.0, batch_first=True, num_levels=num_levels)])
        self.ffns = nn.ModuleList([FFN(embed_dim, ffn_dim)])
        self.norms = nn.ModuleList([nn.LayerNorm(embed_dim), nn.LayerNorm(embed_dim)])

    def forward(self, query, query_pos, key_padding_mask, reference_points, spatial_shapes, level_start_index,
                host_shapes=None, query_with_pos=None, defer_last_norm=False):
        x = self.attentions[0](query, None, query, None, query_pos=query_pos, key_padding_mask=key_padding_mask,
                               reference_points=reference_points, spatial_shapes=spatial_shapes,
                               level_start_index=level_start_index, host_shapes=host_shapes,
                               query_with_pos=query_with_pos,
                               sum_dtype=torch.float32 if query.dtype != torch.float32 else None)
        if query.dtype in (torch.float16, torch.bfloat16):
            # engine path: the two residual sums (query + attention, x + ffn) are fp32 tensors written by the GEMM epilogues;
            # the LayerNorm kernels read them and emit the 16-bit operands of the next GEMMs
            x = ops.layernorm_module(self.norms[0], x, out_dtype=query.dtype)
            x = self.ffns[0](x, out_dtype=torch.float32)
            if defer_last_norm:  # the caller folds norms[1] into the kernel that consumes this layer's output
                return x
            return ops.layernorm_module(self.norms[1], x, out_dtype=query.dtype)
        x = self.norms[0](x)
        x = self.ffns[0](x)
        return self.norms[1](x)


class _DecoderLayer(nn.Module):
    """BaseTransformerLayer(("self_attn","norm","cross_attn","norm","ffn","norm"))."""

    def __init__(self, embed_dim, num_heads, ffn_dim, num_levels):
        super().__init__()
        self.embed_dim = embed_dim
        self.pre_norm = False
        self.attentions = nn.ModuleList([
            _SelfAttention(embed_dim, num_heads),
            MultiScaleDeformableAttention(embed_dim=embed_dim, num_heads=num_heads, dropout=0.0, batch_first=True,
                                          num_levels=num_levels)])
        self.ffns = nn.ModuleList([FFN(embed_dim, ffn_dim)])
        self.norms = nn.ModuleList([nn.LayerNorm(embed_dim) for _ in range(3)])

    def forward(self, query, value, query_pos, key_padding_mask, reference_points, spatial_shapes, level_start_index):
        if query.is_cuda and query.dtype in (torch.float16, torch.bfloat16) and value.dtype == query.dtype:
            # engine path: every linear is a wgmma GEMM, norms are libape_b200 row kernels
            dt = query.dtype  # residual sums in fp32 (GEMM epilogues), LayerNorm outputs / GEMM operands in dt
            x = self.attentions[0](query, query_pos)
            x = ops.layernorm_module(self.norms[0], x, out_dtype=dt)
            x = self.attentions[1](x, None, value, None, query_pos=query_pos.to(dt), key_padding_mask=key_padding_mask,
                                   reference_points=reference_points, spatial_shapes=spatial_shapes,
                                   level_start_index=level_start_index, sum_dtype=torch.float32)
            x = ops.layernorm_module(self.norms[1], x, out_dtype=dt)
            x = self.ffns[0](x, out_dtype=torch.float32)
            return ops.layernorm_module(self.norms[2], x, out_dtype=dt)
        x = self.attentions[0](query, query_pos)
        x = self.norms[0](x)
        x = self.attentions[1](x, None, value, None, query_pos=query_pos, key_padding_mask=key_padding_mask,
                               reference_points=reference_points, spatial_shapes=spatial_shapes,
                               level_start_index=level_start_index)
        x = self.norms[1](x)
        x = self.ffns[0](x)
        return self.norms[2](x)


class DeformableDetrTransformerEncoderVL(nn.Module):
    def __init__(self, embed_dim=256, num_heads=8, feedforward_dim=1024, attn_dropout=0.1, ffn_dropout=0.1,
                 num_layers=6, post_norm=False, num_feature_levels=4, vl_layer=None, use_act_checkpoint=False,
                 pytorch_attn=False):
        super().__init__()
        self.num_layers = num_layers
        self.layers = nn.ModuleList([_EncoderLayer(embed_dim, num_heads, feedforward_dim, num_feature_levels)
                                     for _ in range(num_layers)])
        self.embed_dim = embed_dim
        self.pre_norm = False
        self.post_norm_layer = nn.LayerNorm(embed_dim) if post_norm else None
        self.vl_layers = nn.ModuleList([copy.deepcopy(vl_layer) for _ in range(num_layers)])
        self.record_taps = False  # tests: keep per-layer outputs ("vlf{i}.v" after the fusion, "enc{i}" after the layer) in self.taps

    def forward(self, query, key, value, query_l, attention_mask_l, query_pos=None, key_pos=None, attn_masks=None,
                query_key_padding_mask=None, key_padding_mask=None, **kwargs):
        engine_dtype = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else None
        if engine_dtype is not None:
            query, query_pos = query.to(engine_dtype), query_pos.to(engine_dtype)
            if query_l is not None and query_l.shape[1] == 1 and attention_mask_l is None and query.shape[-1] % 8 == 0 \
                    and all(v is not None and not v.b_attn.attn.use_attention_mask_v for v in self.vl_layers):
                return self._engine_single_token(query.contiguous(), query_pos.contiguous(), query_l,
                                                 query_key_padding_mask, kwargs)
        if self.record_taps:
            self.taps = {}
        for i, (vl_layer, layer) in enumerate(zip(self.vl_layers, self.layers)):
            if vl_layer is not None and query_l is not None:
                query, query_l = vl_layer(query, query_l, attention_mask_v=query_key_padding_mask,
                                          attention_mask_l=attention_mask_l)
                if engine_dtype is not None:
                    query = query.to(engine_dtype)
                if self.record_taps:
                    self.taps[f"vlf{i}.v"] = query
            query = layer(query, query_pos, query_key_padding_mask, kwargs["reference_points"],
                          kwargs["spatial_shapes"], kwargs["level_start_index"], kwargs.get("host_shapes"))
            if self.record_taps:
                self.taps[f"enc{i}"] = query
        if self.post_norm_layer is not None:
            query = self.post_norm_layer(query)
        return query, query_l

    def _engine_single_token(self, x, query_pos, query_l, key_padding_mask, kwargs):
        """Engine schedule of the encoder for "name" prompts (one language token).  Per layer:
          tiny fp32 ops on the language token (delta_v, folded score operands)
          -> ONE row kernel: [last norm of the previous layer] -> layer_norm_v -> + gamma_v*delta_v -> (query, query+pos)
          -> pooling kernels over `query` (language-side update; fuse_helper.py:67-166 restructured)
          -> deformable self-attention + FFN (wgmma GEMMs, fused gather), last norm deferred to the next layer.
        Same functions as `vl_layer(...)` followed by `layer(...)`; the activations cross HBM once per row kernel."""
        pending = None
        dt = x.dtype
        if self.record_taps:
            self.taps = {}
        for i, (vl_layer, layer) in enumerate(zip(self.vl_layers, self.layers)):
            b = vl_layer.b_attn
            with torch.autocast("cuda", enabled=False):
                ln_l = ops.layernorm(query_l.float().contiguous(), b.layer_norm_l.weight.float(), b.layer_norm_l.bias.float(),
                                     eps=b.layer_norm_l.eps, out_dtype=torch.float32)  # own row kernel (fp32 in / out)
                dv, qa, qc = b.single_token_language_side(ln_l)
                shift = (b.gamma_v.float() * dv.float()).reshape(x.shape[0], -1).contiguous()  # [B, C]
            vw, vb = ops.packed(b.layer_norm_v, dt)
            if pending is None:
                query, qpos = ops.layernorm_ex(x, vw, vb, b.layer_norm_v.eps, col_add=shift, row_add=query_pos, out_dtype=dt)
            else:  # x is the previous layer's fp32 sum (x + ffn(x))
                query, qpos = ops.layernorm_ex(x, pending[0], pending[1], pending[2], weight2=vw, bias2=vb,
                                               eps2=b.layer_norm_v.eps, col_add=shift, row_add=query_pos, out_dtype=dt)
            if self.record_taps:
                self.taps[f"vlf{i}.v"] = query
            with torch.autocast("cuda", enabled=False):
                dl = b.single_token_pool(query, qa, qc, shift=shift)
                query_l = ln_l + b.gamma_l.float() * dl
            x = layer(query, query_pos, key_padding_mask, kwargs["reference_points"], kwargs["spatial_shapes"],
                      kwargs["level_start_index"], kwargs.get("host_shapes"), query_with_pos=qpos, defer_last_norm=True)
            nw, nb = ops.packed(layer.norms[1], dt)
            pending = (nw, nb, layer.norms[1].eps)
        x = ops.layernorm(x, pending[0], pending[1], eps=pending[2], out_dtype=dt)
        if self.post_norm_layer is not None:
            x = self.post_norm_layer(x)
        return x, query_l


class DeformableDetrTransformerDecoderVL(nn.Module):
    def __init__(self, embed_dim=256, num_heads=8, feedforward_dim=1024, attn_dropout=0.1, ffn_dropout=0.1,
                 num_layers=6, return_intermediate=True, num_feature_levels=4, use_act_checkpoint=False,
                 look_forward_twice=False, pytorch_attn=False):
        super().__init__()
        self.num_layers = num_layers
        self.layers = nn.ModuleList([_DecoderLayer(embed_dim, num_heads, feedforward_dim, num_feature_levels)
                                     for _ in range(num_layers)])
        self.return_intermediate = return_intermediate
        self.bbox_embed = None
        self.class_embed = None
        self.look_forward_twice = look_forward_twice

    def forward(self, query, key, value, query_pos=None, key_pos=None, attn_masks=None, query_key_padding_mask=None,
                key_padding_mask=None, reference_points=None, valid_ratios=None, **kwargs):
        output = query
        engine_dtype = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else None
        if engine_dtype is not None and value.dtype == engine_dtype:
            output, query_pos = output.to(engine_dtype), query_pos.to(engine_dtype)
        intermediate, intermediate_ref = [], []
        # engine: the reference-point arithmetic between two layers (inverse_sigmoid, add, sigmoid, scaling by the valid ratios:
        # nine elementwise launches) is one kernel with the same fp32 operations in the same order (ape_ref_update)
        fused_ref = engine_dtype is not None and self.bbox_embed is not None and reference_points.is_cuda and \
            reference_points.shape[-1] == 4 and reference_points.dtype == torch.float32
        next_ref_in = None
        for i, layer in enumerate(self.layers):
            if next_ref_in is not None:
                ref_in = next_ref_in
            elif reference_points.shape[-1] == 4:
                ref_in = reference_points[:, :, None] * torch.cat([valid_ratios, valid_ratios], -1)[:, None]
            else:
                ref_in = reference_points[:, :, None] * valid_ratios[:, None]
            output = layer(output, value, query_pos, key_padding_mask, ref_in, kwargs["spatial_shapes"],
                           kwargs["level_start_index"])
            if self.bbox_embed is not None:
                tmp = self.bbox_embed[i](output, out_dtype=torch.float32).float()
                if fused_ref:
                    new_ref, next_ref_in = ops.ref_update(tmp, reference_points, valid_ratios)
                elif reference_points.shape[-1] == 4:
                    new_ref = (tmp + inverse_sigmoid(reference_points)).sigmoid()
                else:
                    new_ref = tmp
                    new_ref[..., :2] = tmp[..., :2] + inverse_sigmoid(reference_points)
                    new_ref = new_ref.sigmoid()
                reference_points = new_ref.detach()
            if self.return_intermediate:
                intermediate.append(output)
                intermediate_ref.append(new_ref if self.look_forward_twice else reference_points)
        if self.return_intermediate:
            return torch.stack(intermediate), torch.stack(intermediate_ref)
        return output, reference_points


class DeformableDetrTransformerVL(nn.Module):
    def __init__(self, encoder=None, decoder=None, num_feature_levels=4, as_two_stage=False,
                 two_stage_num_proposals=300, assign_first_stage=False, pre_nms_topk=1000, nms_thresh_enc=0.9,
                 proposal_ambiguous=0):
        super().__init__()
        if not (as_two_stage and assign_first_stage):
            raise NotImplementedError("ape_b200: only the two-stage / assign_first_stage configuration APE uses")
        self.encoder, self.decoder = encoder, decoder
        self.num_feature_levels = num_feature_levels
        self.as_two_stage = as_two_stage
        self.two_stage_num_proposals = two_stage_num_proposals
        self.assign_first_stage = assign_first_stage
        self.pre_nms_topk = pre_nms_topk
        self.nms_thresh_enc = nms_thresh_enc
        self.proposal_ambiguous = proposal_ambiguous
        self.embed_dim = encoder.embed_dim
        E = self.embed_dim
        self.level_embeds = nn.Parameter(torch.Tensor(num_feature_levels, E))
        self.enc_output = nn.Linear(E, E)
        self.enc_output_norm = nn.LayerNorm(E)
        self.pos_trans = nn.Linear(E * 2, E * 2)
        self.pos_trans_norm = nn.LayerNorm(E * 2)
        self.pix_trans = nn.Linear(E, E)
        self.pix_trans_norm = nn.LayerNorm(E)
        self.init_weights()

    def init_weights(self):
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)
        for m in self.modules():
            if isinstance(m, MultiScaleDeformableAttention):
                m.init_weights()
        nn.init.normal_(self.level_embeds)

    # -- deformable_transformer_vl.py:321-369 ----------------------------------------------------
    def gen_encoder_output_proposals(self, memory, memory_padding_mask, spatial_shapes, mask_prompt_flatten=None):
        N, S, C = memory.shape
        dev = memory.device
        proposals, level_ids = [], []
        cur = 0
        for lvl, (H, W) in enumerate(spatial_shapes):
            m = memory_padding_mask[:, cur:cur + H * W].view(N, H, W, 1)
            valid_H = torch.sum(~m[:, :, 0, 0], 1)
            valid_W = torch.sum(~m[:, 0, :, 0], 1)
            gy, gx = torch.meshgrid(torch.linspace(0, H - 1, H, dtype=torch.float32, device=dev),
                                    torch.linspace(0, W - 1, W, dtype=torch.float32, device=dev), indexing="ij")
            grid = torch.cat([gx.unsqueeze(-1), gy.unsqueeze(-1)], -1)
            scale = torch.cat([valid_W.unsqueeze(-1), valid_H.unsqueeze(-1)], 1).view(N, 1, 1, 2)
            grid = (grid.unsqueeze(0).expand(N, -1, -1, -1) + 0.5) / scale
            wh = torch.ones_like(grid) * 0.05 * (2.0 ** lvl)
            proposals.append(torch.cat((grid, wh), -1).view(N, -1, 4))
            cur += H * W
            level_ids.append(grid.new_ones(H * W, dtype=torch.long) * lvl)
        out = torch.cat(proposals, 1)
        valid = ((out > 0.01) & (out < 0.99)).all(-1, keepdim=True)
        out = torch.log(out / (1 - out))
        out = out.masked_fill(memory_padding_mask.unsqueeze(-1), float("inf"))
        out = out.masked_fill(~valid, float("inf"))
        mem = memory.masked_fill(memory_padding_mask.unsqueeze(-1), float(0)).masked_fill(~valid, float(0))
        if mask_prompt_flatten is not None:
            out = out.masked_fill(~mask_prompt_flatten.unsqueeze(-1), float("inf"))
            mem = mem.masked_fill(~mask_prompt_flatten.unsqueeze(-1), float(0))
        mem = self.enc_output_norm(self.enc_output(mem))
        return mem, out.to(mem.dtype), torch.cat(level_ids)

    @staticmethod
    def get_reference_points(spatial_shapes, valid_ratios, device):
        pts = []
        for lvl, (H, W) in enumerate(spatial_shapes):
            ry, rx = torch.meshgrid(torch.linspace(0.5, H - 0.5, H, dtype=torch.float32, device=device),
                                    torch.linspace(0.5, W - 0.5, W, dtype=torch.float32, device=device), indexing="ij")
            ry = ry.reshape(-1)[None] / (valid_ratios[:, None, lvl, 1] * H)
            rx = rx.reshape(-1)[None] / (valid_ratios[:, None, lvl, 0] * W)
            pts.append(torch.stack((rx, ry), -1))
        ref = torch.cat(pts, 1)
        return ref[:, :, None] * valid_ratios[:, None]

    @staticmethod
    def get_valid_ratio(mask):
        _, H, W = mask.shape
        vh = torch.sum(~mask[:, :, 0], 1).float() / H
        vw = torch.sum(~mask[:, 0, :], 1).float() / W
        return torch.stack([vw, vh], -1)

    @staticmethod
    def get_proposal_pos_embed(proposals, num_pos_feats=128, temperature=10000):
        dim_t = torch.arange(num_pos_feats, dtype=torch.float32, device=proposals.device)
        dim_t = temperature ** (2 * torch.div(dim_t, 2, rounding_mode="floor") / num_pos_feats)
        proposals = proposals.sigmoid() * (2 * math.pi)
        pos = proposals[:, :, :, None] / dim_t
        return torch.stack((pos[:, :, :, 0::2].sin(), pos[:, :, :, 1::2].cos()), dim=4).flatten(2)

    def select_proposals(self, logit, coord_unact, level_ids, n_levels):
        """deformable_transformer_vl.py:569-625 for one image -> LongTensor[min(two_stage_num_proposals, S)].

        Same decisions as the reference's loop (per-level top-k -> class-aware NMS by level -> per-level quota ->
        pad in score order), written with static shapes and no host synchronisation (masks + cumulative sums +
        nonzero_static instead of boolean indexing), so the whole selection is CUDA-graph capturable."""
        topk = self.two_stage_num_proposals
        S = logit.size(0)
        fallback = torch.sort(logit, descending=True, stable=True)[1][: min(topk, S)]  # (:598-599)
        if S < topk:
            return fallback  # fewer tokens than queries: NMS can never keep `topk`, the reference takes this branch
        dev = logit.device
        boxes = box_cxcywh_to_xyxy(coord_unact.sigmoid()).clamp(0, 1)
        lvls = torch.arange(n_levels, device=dev)
        lvl_mask = level_ids[None] == lvls[:, None]                                           # [L,S]
        # The reference calls torch.topk per level; for a level with fewer tokens than pre_nms_topk (the 16x16 level
        # at 1024^2) the result is padded with zero-score tokens of OTHER levels in an implementation-defined order
        # (CPU and CUDA top-k differ).  The engine fixes the rule: stable descending sort = lowest index first.
        k = min(self.pre_nms_topk, S)
        pre = torch.sort(logit.sigmoid()[None] * lvl_mask, dim=1, descending=True, stable=True)[1][:, :k].reshape(-1)
        # detectron2 / torchvision batched_nms: coordinate-offset trick on boxes.float(), scores sorted descending
        b = boxes[pre].float()
        sc = logit[pre].float()
        ids = level_ids[pre]
        b = b + (ids.to(b) * (b.max() + 1))[:, None]  # offsets = idxs * (max_coordinate + 1)
        order = sc.sort(0, descending=True)[1]
        keep_mask, count = ops.nms_sorted_mask(b.index_select(0, order).contiguous(), self.nms_thresh_enc)
        cand = pre[order]                       # candidates in NMS (descending score) order
        kept = keep_mask.bool()                 # `keep = pre[post]` is cand[kept]
        q_per_l = topk // n_levels
        per_lvl = (level_ids[cand][None] == lvls[:, None]) & kept[None]                       # [L,n]
        km = (per_lvl & (per_lvl.cumsum(1) <= q_per_l)).any(0)
        num_to_add = topk - km.sum()
        extra = kept & ~km
        km = km | (extra & (extra.cumsum(0) <= num_to_add))
        sel = torch.nonzero_static(km, size=topk, fill_value=0)[:, 0]
        picked = cand[sel]
        return torch.where(count.to(torch.int64) < topk, fallback, picked)

    # -- staged forward ------------------------------------------------------------------------------
    # forward() = geometry() [pure function of the padded-image geometry, cacheable] -> stage_encode()
    # [static shapes, no host sync: CUDA-graph capturable] -> stage_select() [top-k / NMS, data dependent]
    # -> stage_decode() [static shapes again].
    def geometry(self, shapes, multi_level_masks, multi_level_pos_embeds):
        """Everything that depends only on the feature-map shapes and the padding masks
        (deformable_transformer_vl.py:435-477 and the anchor part of :321-353)."""
        dev = multi_level_masks[0].device
        mask_flatten = torch.cat([m.flatten(1) for m in multi_level_masks], 1)
        pos_flatten = torch.cat([p.flatten(2).transpose(1, 2) for p in multi_level_pos_embeds], 1)
        spatial_shapes = torch.as_tensor(shapes, dtype=torch.long, device=dev)
        level_start_index = torch.cat((spatial_shapes.new_zeros((1,)), spatial_shapes.prod(1).cumsum(0)[:-1]))
        valid_ratios = torch.stack([self.get_valid_ratio(m) for m in multi_level_masks], 1).to(torch.float32)
        reference_points = self.get_reference_points(shapes, valid_ratios, dev).to(torch.float32)
        N = mask_flatten.shape[0]
        proposals, level_ids = [], []
        cur = 0
        for lvl, (H, W) in enumerate(shapes):
            m = mask_flatten[:, cur:cur + H * W].view(N, H, W, 1)
            valid_H = torch.sum(~m[:, :, 0, 0], 1)
            valid_W = torch.sum(~m[:, 0, :, 0], 1)
            gy, gx = torch.meshgrid(torch.linspace(0, H - 1, H, dtype=torch.float32, device=dev),
                                    torch.linspace(0, W - 1, W, dtype=torch.float32, device=dev), indexing="ij")
            grid = torch.cat([gx.unsqueeze(-1), gy.unsqueeze(-1)], -1)
            scale = torch.cat([valid_W.unsqueeze(-1), valid_H.unsqueeze(-1)], 1).view(N, 1, 1, 2)
            grid = (grid.unsqueeze(0).expand(N, -1, -1, -1) + 0.5) / scale
            wh = torch.ones_like(grid) * 0.05 * (2.0 ** lvl)
            proposals.append(torch.cat((grid, wh), -1).view(N, -1, 4))
            cur += H * W
            level_ids.append(grid.new_ones(H * W, dtype=torch.long) * lvl)
        out = torch.cat(proposals, 1)
        valid = ((out > 0.01) & (out < 0.99)).all(-1, keepdim=True)
        out = torch.log(out / (1 - out))
        out = out.masked_fill(mask_flatten.unsqueeze(-1), float("inf")).masked_fill(~valid, float("inf"))
        return dict(shapes=list(shapes), mask_flatten=mask_flatten, pos_flatten=pos_flatten, spatial_shapes=spatial_shapes,
                    level_start_index=level_start_index, valid_ratios=valid_ratios, reference_points=reference_points,
                    output_proposals=out, proposal_invalid=mask_flatten.unsqueeze(-1) | ~valid,
                    level_ids=torch.cat(level_ids), has_padding=bool(mask_flatten.any()))

    def stage_encode(self, multi_level_feats, geo, query_l, attention_mask_l=None, mask_prompt_flatten=None,
                     feat_flatten=None):
        """feat_flatten: optional [B,S,C] tensor that already holds the flattened levels (the engine neck writes its
        outputs straight into it; `multi_level_feats` are then views of its slices)."""
        if feat_flatten is None:
            feat_flatten = torch.cat([f.flatten(2).transpose(1, 2) for f in multi_level_feats], 1)
        engine_dtype = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else torch.float32
        ck = (self.level_embeds._version, self.level_embeds.data_ptr())
        cache = geo.setdefault("_pos_lvl", {})  # position + level embedding: constant per geometry and weights, one entry per dtype
        if engine_dtype not in cache or cache[engine_dtype][0] != ck:
            with torch.no_grad():
                lvl_embed = torch.cat([self.level_embeds[i].view(1, 1, -1).expand(1, h * w, -1)
                                       for i, (h, w) in enumerate(geo["shapes"])], 1)
                cache[engine_dtype] = (ck, (geo["pos_flatten"] + lvl_embed.float()).to(engine_dtype).contiguous())
        pos_flatten = cache[engine_dtype][1]
        memory, query_l = self.encoder(
            query=feat_flatten, key=None, value=None, query_l=query_l, attention_mask_l=attention_mask_l,
            query_pos=pos_flatten, query_key_padding_mask=geo["mask_flatten"] if geo["has_padding"] else None,
            spatial_shapes=geo["spatial_shapes"], reference_points=geo["reference_points"],
            level_start_index=geo["level_start_index"], valid_ratios=geo["valid_ratios"],
            host_shapes=geo["shapes"])
        # gen_encoder_output_proposals (:354-369): zero the memory of invalid anchors, project, normalise
        output_proposals = geo["output_proposals"]
        invalid = geo["proposal_invalid"]
        if mask_prompt_flatten is not None:
            output_proposals = output_proposals.masked_fill(~mask_prompt_flatten.unsqueeze(-1), float("inf"))
            invalid = invalid | ~mask_prompt_flatten.unsqueeze(-1)
        nd = self.decoder.num_layers
        if memory.is_cuda and memory.dtype in (torch.float16, torch.bfloat16):
            output_memory, enc_cls, enc_coord = self._engine_proposal_heads(memory, invalid, output_proposals, nd)
            return memory, query_l, output_memory, enc_cls, enc_coord
        output_memory = self.enc_output_norm(self.enc_output(memory.masked_fill(invalid, float(0))))
        output_proposals = output_proposals.to(output_memory.dtype)
        enc_cls = self.decoder.class_embed[nd](output_memory)
        enc_coord = self.decoder.bbox_embed[nd](output_memory) + output_proposals
        if self.proposal_ambiguous:
            cls_all = torch.stack([enc_cls] + [m(output_memory) for m in self.decoder.class_embed_ambiguous], dim=1)
            coord_all = torch.stack([enc_coord] + [m(output_memory) + output_proposals
                                                   for m in self.decoder.bbox_embed_ambiguous], dim=1)
            idx = torch.argmax(cls_all, dim=1, keepdim=True)
            enc_cls = torch.gather(cls_all, 1, idx).squeeze(1)
            enc_coord = torch.gather(coord_all, 1, idx.repeat(1, 1, 1, 4)).squeeze(1)
        return memory, query_l, output_memory, enc_cls, enc_coord

    def _engine_proposal_heads(self, memory, invalid, output_proposals, nd):
        """deformable_transformer_vl.py:354-369 + :503-533 on the tensor cores: enc_output -> LayerNorm, then the
        class heads (Linear 256->1, main + ambiguous, stacked into one 8-row GEMM) and the box MLPs (first layers
        of all heads stacked into one GEMM with a ReLU epilogue).  Logits and box deltas leave the last GEMMs in
        fp32 (they feed top-k / NMS); the ambiguous-head argmax follows the reference."""
        dt = memory.dtype
        cls_mods = [self.decoder.class_embed[nd]] + (list(self.decoder.class_embed_ambiguous) if self.proposal_ambiguous else [])
        box_mods = [self.decoder.bbox_embed[nd]] + (list(self.decoder.bbox_embed_ambiguous) if self.proposal_ambiguous else [])
        params = [p for m in cls_mods + box_mods for p in m.parameters()]
        def build():
            E = self.embed_dim
            wc = torch.zeros(8, E, device=memory.device, dtype=dt)
            bc = torch.zeros(8, device=memory.device, dtype=torch.float32)
            for j, m in enumerate(cls_mods):
                wc[j] = m.weight[0].to(dt)
                bc[j] = m.bias[0].float()
            w0 = torch.cat([m.layers[0].weight for m in box_mods], 0).to(dt).contiguous()
            b0 = torch.cat([m.layers[0].bias for m in box_mods], 0).float().contiguous()
            rest = []
            for m in box_mods:
                mids = [(l.weight.detach().to(dt).contiguous(), l.bias.detach().float().contiguous()) for l in m.layers[1:-1]]
                wl = torch.zeros(8, m.layers[-1].weight.shape[1], device=memory.device, dtype=dt)
                bl = torch.zeros(8, device=memory.device, dtype=torch.float32)
                wl[:4] = m.layers[-1].weight.to(dt)
                bl[:4] = m.layers[-1].bias.float()
                rest.append((mids, wl, bl))
            return wc, bc, w0, b0, rest, len(cls_mods)

        wc, bc, w0, b0, rest, n = ops.cached(self, "_heads_pk", dt, (tuple(p._version for p in params), params[0].data_ptr()), build)
        om = ops.linear_module_tc(self.enc_output, memory.masked_fill(invalid, float(0)))
        output_memory = ops.layernorm_module(self.enc_output_norm, om)
        B, S, E = output_memory.shape
        cls_all = ops.linear_tc(output_memory, wc, bc, out_dtype=torch.float32)[..., :n]      # [B,S,n] fp32
        h0 = ops.linear_tc(output_memory, w0, b0, act="relu")                                  # [B,S,n*E]
        props = output_proposals.float()
        coords = []
        for j, (mids, wl, bl) in enumerate(rest):
            h = h0[..., j * E:(j + 1) * E]
            for (w, b) in mids:
                h = ops.linear_tc(h, w, b, act="relu")
            coords.append(ops.linear_tc(h, wl, bl, out_dtype=torch.float32)[..., :4] + props)
        if n == 1:
            return output_memory, cls_all, coords[0]
        idx = torch.argmax(cls_all, dim=-1, keepdim=True)                                      # [B,S,1]
        enc_cls = torch.gather(cls_all, 2, idx)
        coord_all = torch.stack(coords, dim=2)                                                 # [B,S,n,4]
        enc_coord = torch.gather(coord_all, 2, idx.unsqueeze(-1).expand(-1, -1, 1, 4)).squeeze(2)
        return output_memory, enc_cls, enc_coord

    def stage_select(self, enc_cls, enc_coord, geo):
        logit = enc_cls[..., 0].float()
        coord = enc_coord.float()
        return torch.stack([self.select_proposals(logit[b], coord[b], geo["level_ids"], len(geo["shapes"]))
                            for b in range(logit.shape[0])])

    def stage_decode(self, memory, output_memory, enc_coord, topk_proposals, geo):
        c = memory.shape[-1]
        topk_unact = torch.gather(enc_coord.float(), 1, topk_proposals.unsqueeze(-1).repeat(1, 1, 4)).detach()
        reference = topk_unact.sigmoid()
        topk_feats = torch.gather(output_memory, 1, topk_proposals.unsqueeze(-1).expand(-1, -1, c)).detach()
        if memory.is_cuda and memory.dtype in (torch.float16, torch.bfloat16):
            emb = self.get_proposal_pos_embed(topk_unact).to(memory.dtype)
            pos_trans_out = ops.layernorm_module(self.pos_trans_norm, ops.linear_module_tc(self.pos_trans, emb))
            query_pos, query = torch.split(pos_trans_out, c, dim=2)
            query = query + ops.layernorm_module(self.pix_trans_norm, ops.linear_module_tc(self.pix_trans, topk_feats.to(memory.dtype)))
        else:
            pos_trans_out = self.pos_trans_norm(self.pos_trans(self.get_proposal_pos_embed(topk_unact).to(topk_unact.dtype)))
            query_pos, query = torch.split(pos_trans_out, c, dim=2)
            query = query + self.pix_trans_norm(self.pix_trans(topk_feats))
        inter_states, inter_references = self.decoder(
            query=query, key=None, value=memory, query_pos=query_pos,
            key_padding_mask=geo["mask_flatten"] if geo["has_padding"] else None,
            reference_points=reference, spatial_shapes=geo["spatial_shapes"],
            level_start_index=geo["level_start_index"], valid_ratios=geo["valid_ratios"])
        return inter_states, reference, inter_references

    def forward(self, multi_level_feats, multi_level_masks, multi_level_pos_embeds, query_embed, query_l,
                attention_mask_l, multi_level_masks_prompt, **kwargs):
        shapes = [(int(f.shape[2]), int(f.shape[3])) for f in multi_level_feats]
        geo = kwargs.get("geometry") or self.geometry(shapes, multi_level_masks, multi_level_pos_embeds)
        mask_prompt_flatten = None
        if multi_level_masks_prompt is not None:
            mask_prompt_flatten = torch.cat([m.flatten(1) for m in multi_level_masks_prompt], 1)
        memory, query_l, output_memory, enc_cls, enc_coord = self.stage_encode(
            multi_level_feats, geo, query_l, attention_mask_l, mask_prompt_flatten)
        topk_proposals = self.stage_select(enc_cls, enc_coord, geo)
        inter_states, init_reference_out, inter_references = self.stage_decode(
            memory, output_memory, enc_coord, topk_proposals, geo)
        self.last_topk_proposals = topk_proposals  # kept for parity tests (bit-exact index requirement)
        return (inter_states, init_reference_out, inter_references, enc_cls, enc_coord,
                geo["output_proposals"].sigmoid(), memory, query_l)
