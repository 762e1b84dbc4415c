"""VisionLanguageFusion: bi-directional vision<->language cross attention of the VL encoder.
Mirror of ape/layers/vision_language_fusion.py:7-53 and ape/layers/fuse_helper.py:8-232 (same
constructor arguments, same parameter names: `b_attn.{layer_norm_v,layer_norm_l,gamma_v,gamma_l}`,
`b_attn.attn.{v_proj,l_proj,values_v_proj,values_l_proj,out_v_proj,out_l_proj}`).

Inference engine: dropout / drop-path / checkpointing arguments are accepted and ignored."""
import torch
import torch.nn as nn
import torch.nn.functional as F


class BiMultiHeadAttention(nn.Module):
    def __init__(self, v_dim, l_dim, embed_dim, num_heads, dropout=0.1, stable_softmax_2d=False,
                 clamp_min_for_underflow=True, clamp_max_for_overflow=True, use_attention_mask_v=False):
        super().__init__()
        self.embed_dim, self.num_heads, self.head_dim = embed_dim, num_heads, embed_dim // num_heads
        self.v_dim, self.l_dim = v_dim, l_dim
        assert self.head_dim * num_heads == embed_dim
        self.scale = self.head_dim ** (-0.5)
        self.v_proj = nn.Linear(v_dim, embed_dim)
        self.l_proj = nn.Linear(l_dim, embed_dim)
        self.values_v_proj = nn.Linear(v_dim, embed_dim)
        self.values_l_proj = nn.Linear(l_dim, embed_dim)
        self.out_v_proj = nn.Linear(embed_dim, v_dim)
        self.out_l_proj = nn.Linear(embed_dim, l_dim)
        self.stable_softmax_2d = stable_softmax_2d
        self.clamp_min_for_underflow = clamp_min_for_underflow
        self.clamp_max_for_overflow = clamp_max_for_overflow
        self.use_attention_mask_v = use_attention_mask_v
        # Phrase prompts at scale (BASELINE.json configs[3]: S = 196 416 vision tokens x 5 000 phrases x 8 heads) would
        # materialise 31 GB of fp32 scores several times over.  Above this many score bytes the two softmaxes are
        # evaluated as two streaming attention calls (no S x N_t tensor) — identical mathematics as long as the +-5e4
        # clamps cannot bind, which is checked from the operand norms first.
        self.stream_threshold_bytes = 1 << 30
        for m in (self.v_proj, self.l_proj, self.values_v_proj, self.values_l_proj, self.out_v_proj, self.out_l_proj):
            nn.init.xavier_uniform_(m.weight)
            m.bias.data.fill_(0)

    def forward_engine(self, v, l):
        """Engine path for several language tokens (phrase / text prompts): the six projections are wgmma GEMMs and
        each softmax direction is ONE flash-attention pass of ape_attn_cross_fwd over 256-channel heads — the S x N_t
        score matrix of fuse_helper.py:86 (31 GB per head set at 1536^2 / 5 000 phrases) is never materialised, there is
        no host synchronisation and no data-dependent choice of algorithm.  v [B,S,v_dim] 16-bit and l [B,N,l_dim] are the
        layer-normed inputs.  Returns (delta_v [B,S,v_dim] 16-bit, delta_l [B,N,l_dim] fp32)."""
        from .. import ops

        dt = v.dtype
        B, S, _ = v.shape
        N = l.shape[1]
        nh, hd, E = self.num_heads, self.head_dim, self.embed_dim
        Sp, Np = (S + 127) // 128 * 128, (N + 127) // 128 * 128  # padded rows (zeros): queries in tiles of 128, keys of 64
        l16 = l.to(dt)
        qv = torch.zeros((B, Sp, E), dtype=dt, device=v.device)   # v_proj(v): queries of direction 1, keys of direction 2
        vv = torch.zeros((B, Sp, E), dtype=dt, device=v.device)   # values_v_proj(v)
        kl = torch.zeros((B, Np, E), dtype=dt, device=v.device)   # l_proj(l)
        vl = torch.zeros((B, Np, E), dtype=dt, device=v.device)   # values_l_proj(l)
        for b in range(B):
            ops.linear_module_tc(self.v_proj, v[b], out=qv[b, :S])
            ops.linear_module_tc(self.values_v_proj, v[b], out=vv[b, :S])
            ops.linear_module_tc(self.l_proj, l16[b], out=kl[b, :N])
            ops.linear_module_tc(self.values_l_proj, l16[b], out=vl[b, :N])
        # vision <- language: softmax over the N phrases (fuse_helper.py:127-141);  language <- vision: over the S tokens (:94-125)
        out_v = ops.attention_cross(qv.view(B * Sp, E), kl.view(B * Np, E), vl.view(B * Np, E), B, Sp, Np, N, nh, hd, self.scale)
        out_l = ops.attention_cross(kl.view(B * Np, E), qv.view(B * Sp, E), vv.view(B * Sp, E), B, Np, Sp, S, nh, hd, self.scale)
        dv = torch.stack([ops.linear_module_tc(self.out_v_proj, out_v.view(B, Sp, E)[b, :S]) for b in range(B)])
        dl = torch.stack([ops.linear_module_tc(self.out_l_proj, out_l.view(B, Np, E)[b, :N], out_dtype=torch.float32) for b in range(B)])
        return dv, dl

    def _clamp(self, w):
        if self.clamp_min_for_underflow:
            w = torch.clamp(w, min=-50000)
        if self.clamp_max_for_overflow:
            w = torch.clamp(w, max=50000)
        return w

    def forward(self, v, l, attention_mask_v=None, attention_mask_l=None):
        """fuse_helper.py:67-166 (v, l already layer-normed by the block)."""
        bsz, tgt_len, _ = v.shape
        nh, hd = self.num_heads, self.head_dim

        def heads(t):
            return t.view(bsz, -1, nh, hd).transpose(1, 2).reshape(bsz * nh, -1, hd)

        q = heads(self.v_proj(v) * self.scale)
        k = heads(self.l_proj(l))
        val_v = heads(self.values_v_proj(v))
        val_l = heads(self.values_l_proj(l))
        src_len = k.shape[1]
        masked = attention_mask_l is not None or (attention_mask_v is not None and self.use_attention_mask_v)
        if not masked and bsz * nh * tgt_len * src_len * 4 > self.stream_threshold_bytes:
            # |score| <= |q_s| |k_t|: if that bound stays inside the clamps, every shift in fuse_helper.py:88-108
            # (global max, row max) is a softmax-invariant translation and both clamps are identities
            bound = q.float().norm(dim=-1).max() * k.float().norm(dim=-1).max()
            if float(bound) < 25000.0:
                q4, k4 = q.view(bsz, nh, tgt_len, hd), k.view(bsz, nh, src_len, hd)
                out_v = F.scaled_dot_product_attention(q4, k4, val_l.view(bsz, nh, src_len, hd), scale=1.0)   # softmax over phrases
                out_l = F.scaled_dot_product_attention(k4, q4, val_v.view(bsz, nh, tgt_len, hd), scale=1.0)   # softmax over pixels
                out_v = out_v.transpose(1, 2).reshape(bsz, tgt_len, self.embed_dim)
                out_l = out_l.transpose(1, 2).reshape(bsz, src_len, self.embed_dim)
                return self.out_v_proj(out_v), self.out_l_proj(out_l)
        w = torch.bmm(q, k.transpose(1, 2))
        if self.stable_softmax_2d:
            w = w - w.max()
        w = self._clamp(w)
        wT = w.transpose(1, 2)
        wl = self._clamp(wT - torch.max(wT, dim=-1, keepdim=True)[0])
        if attention_mask_v is not None and self.use_attention_mask_v:
            mv = attention_mask_v[:, None, None, :].repeat(1, nh, 1, 1).flatten(0, 1)
            wl = wl.masked_fill(mv, float("-inf"))
        wl = wl.softmax(dim=-1)
        if attention_mask_l is not None:
            ml = attention_mask_l[:, None, None, :].repeat(1, nh, 1, 1).flatten(0, 1)
            w = w.masked_fill(ml, float("-inf"))
        wv = w.softmax(dim=-1)
        out_v = torch.bmm(wv, val_l).view(bsz, nh, tgt_len, hd).transpose(1, 2).reshape(bsz, tgt_len, self.embed_dim)
        out_l = torch.bmm(wl, val_v).view(bsz, nh, -1, hd).transpose(1, 2).reshape(bsz, -1, self.embed_dim)
        return self.out_v_proj(out_v), self.out_l_proj(out_l)


class BiAttentionBlock(nn.Module):
    def __init__(self, v_dim, l_dim, embed_dim, num_heads, dropout=0.1, drop_path=0.0, init_values=1e-4,
                 stable_softmax_2d=False, clamp_min_for_underflow=True, clamp_max_for_overflow=True,
                 use_attention_mask_v=False):
        super().__init__()
        self.layer_norm_v = nn.LayerNorm(v_dim)
        self.layer_norm_l = nn.LayerNorm(l_dim)
        self.attn = BiMultiHeadAttention(v_dim, l_dim, embed_dim, num_heads, dropout, stable_softmax_2d,
                                         clamp_min_for_underflow, clamp_max_for_overflow, use_attention_mask_v)
        self.gamma_v = nn.Parameter(init_values * torch.ones(v_dim))
        self.gamma_l = nn.Parameter(init_values * torch.ones(l_dim))
        self.fold_language_side = True  # one-token case: fold the small projection chains into two GEMVs (CUDA)

    def forward(self, v, l, attention_mask_v=None, attention_mask_l=None):
        # fuse_helper.py:221-232 — note the residual is added to the *normalised* v / l
        a = self.attn
        if v.is_cuda and v.dtype in (torch.float16, torch.bfloat16) and l.shape[1] > 1 and attention_mask_l is None and \
                not (a.use_attention_mask_v and attention_mask_v is not None) and a.head_dim in (64, 256) and \
                v.shape[-1] % 8 == 0 and l.shape[-1] % 8 == 0:
            from .. import ops  # engine: LayerNorm kernel, wgmma GEMMs, two flash-attention passes (forward_engine)

            vn = ops.layernorm_module(self.layer_norm_v, v.contiguous())
            with torch.autocast("cuda", enabled=False):
                ln = self.layer_norm_l(l.float())
            dv, dl = a.forward_engine(vn, ln)
            return vn + self.gamma_v.to(vn.dtype) * dv, ln + self.gamma_l.float() * dl
        v = self.layer_norm_v(v)
        l = self.layer_norm_l(l)
        if l.shape[1] == 1 and attention_mask_l is None and not (self.attn.use_attention_mask_v and attention_mask_v is not None):
            dv, dl = self.single_token(v, l)
        else:
            dv, dl = self.attn(v, l, attention_mask_v=attention_mask_v, attention_mask_l=attention_mask_l)
        return v + self.gamma_v * dv, l + self.gamma_l * dl

    def single_token(self, v, l):
        """BiMultiHeadAttention.forward (fuse_helper.py:67-166) for ONE language token — the "name" prompt
        case, where the fusion feature is the single `name_prompt_fusion_feature` row
        (deformable_detr_segm_vl.py:342-360).  Same function, restructured (SURVEY.md §0):
          * vision side: softmax over one key is exactly 1, so delta_v = out_v_proj(values_l_proj(l)) for
            every token — no S x 2048 projections of v at all;
          * language side: scores[s,h] = scale*(W_q,h v_s + b_q,h).k_h = v_s.(scale W_q,h^T k_h) + const and
            sum_s p[s,h] (W_vv,h v_s + b_vv,h) = W_vv,h (sum_s p[s,h] v_s) + b_vv,h — O(S*256*8) instead of
            three S x 256 x 2048 GEMMs (1.65 TFLOP per image over the six encoder layers).
        fp32 regardless of the engine dtype (tiny); differs from the literal op order by fp32 reassociation."""
        dv, qa, qc = self.single_token_language_side(l)
        dl = self.single_token_pool(v, qa, qc)
        return dv.to(v.dtype), dl.to(l.dtype)

    def _folded_language_maps(self):
        """The one-token case is affine in the language token on both sides, so the chains of small projections are
        folded once per set of weights (fp64, stored fp32):
          [qa | qc | delta_v] = ln_l @ G^T + g0     (l_proj -> per-head v_proj^T; l_proj -> v_proj bias; values_l_proj -> out_v_proj)
          delta_l             = pooled @ E^T + e0   (values_v_proj per head -> out_l_proj)
        One GEMV each per layer instead of ~25 small kernels; results differ from the op-by-op order by fp32 rounding."""
        a = self.attn
        params = [a.l_proj.weight, a.l_proj.bias, a.v_proj.weight, a.v_proj.bias, a.values_l_proj.weight, a.values_l_proj.bias,
                  a.out_v_proj.weight, a.out_v_proj.bias, a.values_v_proj.weight, a.values_v_proj.bias, a.out_l_proj.weight,
                  a.out_l_proj.bias]
        key = tuple((t._version, t.data_ptr()) for t in params)
        if getattr(self, "_folded", (None,))[0] != key:
            nh, hd = a.num_heads, a.head_dim
            with torch.no_grad():
                d = lambda t: t.detach().double()
                wl, bl = d(a.l_proj.weight).view(nh, hd, -1), d(a.l_proj.bias).view(nh, hd)           # [nh,hd,L]
                wq, bq = d(a.v_proj.weight).view(nh, hd, -1), d(a.v_proj.bias).view(nh, hd)           # [nh,hd,C]
                A = torch.einsum("hdc,hdj->hcj", wq, wl) * a.scale                                    # [nh,C,L]
                a0 = torch.einsum("hdc,hd->hc", wq, bl) * a.scale
                Cm = torch.einsum("hd,hdj->hj", bq, wl) * a.scale                                     # [nh,L]
                c0 = torch.einsum("hd,hd->h", bq, bl) * a.scale
                D = d(a.out_v_proj.weight) @ d(a.values_l_proj.weight)                                # [C,L]
                d0 = d(a.out_v_proj.weight) @ d(a.values_l_proj.bias) + d(a.out_v_proj.bias)
                G = torch.cat([A.reshape(-1, A.shape[-1]), Cm, D], 0).float().contiguous()
                g0 = torch.cat([a0.reshape(-1), c0, d0], 0).float().contiguous()
                wvv, bvv = d(a.values_v_proj.weight).view(nh, hd, -1), d(a.values_v_proj.bias)        # [nh,hd,C]
                wol = d(a.out_l_proj.weight).view(-1, nh, hd)                                         # [L,nh,hd]
                E = torch.einsum("jhd,hdc->jhc", wol, wvv).reshape(wol.shape[0], -1).float().contiguous()
                e0 = (d(a.out_l_proj.weight) @ bvv + d(a.out_l_proj.bias)).float().contiguous()
            self._folded = (key, G, g0, E, e0)
        return self._folded[1:]

    def single_token_language_side(self, l):
        """Everything of the one-token case that depends on the language token only: delta_v [B,1,v_dim] and the
        folded score operands qa [B,nh,v_dim], qc [B,nh] (scores[s,h] = v_s . qa[h] + qc[h])."""
        a = self.attn
        nh, hd = a.num_heads, a.head_dim
        if l.is_cuda and self.fold_language_side:
            with torch.autocast("cuda", enabled=False):
                G, g0, _, _ = self._folded_language_maps()
                B = l.shape[0]
                from .. import ops

                y = ops.gemv_f32(l.float().reshape(B, -1), G, g0)  # own fp32 GEMV (PyTorch would run cuBLAS gemv kernels here)
                C = a.v_proj.weight.shape[1]
                return y[:, nh * C + nh:].reshape(B, 1, C), y[:, : nh * C].reshape(B, nh, C), y[:, nh * C: nh * C + nh]
        with torch.autocast("cuda", enabled=False):
            lf = l.float()
            B = lf.shape[0]
            k = F.linear(lf, a.l_proj.weight.float(), a.l_proj.bias.float()).view(B, nh, hd)
            val_l = F.linear(lf, a.values_l_proj.weight.float(), a.values_l_proj.bias.float())       # [B,1,E]
            dv = F.linear(val_l, a.out_v_proj.weight.float(), a.out_v_proj.bias.float())             # [B,1,v_dim]
            wq = a.v_proj.weight.float().view(nh, hd, -1)                                            # [nh,hd,v_dim]
            qa = torch.einsum("bhd,hdc->bhc", k, wq) * a.scale                                       # [B,nh,v_dim]
            qc = torch.einsum("bhd,hd->bh", k, a.v_proj.bias.float().view(nh, hd)) * a.scale         # [B,nh]
        return dv, qa, qc

    def single_token_pool(self, v, qa, qc, shift=None):
        """delta_l [B,1,l_dim] from the vision tokens.  `shift` [B,1,v_dim] (fp32): the tensor passed as `v` is
        v_true + shift (the engine hands over the already updated query = LN_v(x) + gamma_v * delta_v and avoids
        materialising LN_v(x)); scores and the pooled vector are corrected exactly:
        v_true.qa + qc = v.qa + (qc - shift.qa),  sum_s p_s v_true_s = sum_s p_s v_s - shift."""
        a = self.attn
        nh, hd = a.num_heads, a.head_dim
        with torch.autocast("cuda", enabled=False):
            B, S, _ = v.shape
            if shift is not None:
                qc = qc - torch.einsum("bc,bhc->bh", shift.reshape(B, -1).float(), qa)
            if v.is_cuda and nh <= 8 and a.clamp_min_for_underflow and a.clamp_max_for_overflow and \
                    v.shape[-1] == 256 and B * nh <= 64:
                from .. import ops  # fused pooling kernels: v is read twice in its own dtype, nothing else of size S

                pooled = ops.vlf_pool(v.contiguous(), qa, qc, a.stable_softmax_2d)
            else:
                vf = v.float()
                w = torch.einsum("bsc,bhc->bhs", vf, qa) + qc[..., None]                             # [B,nh,S]
                if a.stable_softmax_2d:
                    w = w - w.max()
                w = a._clamp(w)
                wl = a._clamp(w - w.max(dim=-1, keepdim=True)[0]).softmax(dim=-1)
                pooled = torch.einsum("bhs,bsc->bhc", wl, vf)                                        # [B,nh,v_dim]
            if shift is not None:
                pooled = pooled - shift.reshape(B, 1, -1).float()
            if v.is_cuda and self.fold_language_side:
                _, _, E, e0 = self._folded_language_maps()
                from .. import ops

                return ops.gemv_f32(pooled.reshape(B, 1, -1).contiguous(), E, e0)
            wvv = a.values_v_proj.weight.float().view(nh, hd, -1)
            out_l = torch.einsum("bhc,hdc->bhd", pooled, wvv) + a.values_v_proj.bias.float().view(nh, hd)
            dl = F.linear(out_l.reshape(B, 1, nh * hd), a.out_l_proj.weight.float(), a.out_l_proj.bias.float())
        return dl


class VisionLanguageFusion(nn.Module):
    def __init__(self, v_dim, l_dim, embed_dim, num_heads, dropout=0.1, drop_path=0.0, init_values=1e-4,
                 stable_softmax_2d=False, clamp_min_for_underflow=True, clamp_max_for_overflow=True,
                 use_checkpoint=False, use_attention_mask_v=False):
        super().__init__()
        self.use_checkpoint = use_checkpoint
        self.b_attn = BiAttentionBlock(v_dim, l_dim, embed_dim, num_heads, dropout, drop_path, init_values,
                                       stable_softmax_2d, clamp_min_for_underflow, clamp_max_for_overflow,
                                       use_attention_mask_v)

    def forward(self, v, l, attention_mask_v=None, attention_mask_l=None):
        return self.b_attn(v, l, attention_mask_v, attention_mask_l)
