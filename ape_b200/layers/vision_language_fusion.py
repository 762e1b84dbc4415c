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

    def forward(self, v, l, attention_mask_v=None, attention_mask_l=None, n_tokens=None):
        """n_tokens (int32 [1] on the device, or None): l is padded and only its first n_tokens tokens are real (a prompt padded
        to a capacity); the folded path reads the count on the device, and no other path takes padded text."""
        # fuse_helper.py:221-232 — note the residual is added to the *normalised* v / l
        a = self.attn
        if v.is_cuda and v.dtype in (torch.float16, torch.bfloat16) and l.shape[1] > 1 and attention_mask_l is None and \
                not (a.use_attention_mask_v and attention_mask_v is not None) and a.head_dim in (64, 256) and \
                v.shape[-1] % 8 == 0 and l.shape[-1] % 8 == 0:
            from .. import ops  # engine: LayerNorm kernel, then the folded fusion (256-channel vision tokens) or forward_engine

            vn = ops.layernorm_module(self.layer_norm_v, v.contiguous())
            with torch.autocast("cuda", enabled=False):
                ln = self.layer_norm_l(l.float())
            if self.folds(vn.shape[-1], ln.shape[-1], ln.shape[1]):
                return self.folded(vn, ln, n_tokens)
            if n_tokens is not None:
                raise NotImplementedError("ape_b200: a padded prompt needs the folded fusion path")
            dv, dl = a.forward_engine(vn, ln)
            return vn + self.gamma_v.to(vn.dtype) * dv, ln + self.gamma_l.float() * dl
        if n_tokens is not None:
            raise NotImplementedError("ape_b200: a padded prompt needs the folded fusion path (16-bit CUDA)")
        v = self.layer_norm_v(v)
        l = self.layer_norm_l(l)
        if l.shape[1] == 1 and attention_mask_l is None and not (self.attn.use_attention_mask_v and attention_mask_v is not None):
            dv, dl = self.single_token(v, l)
        else:
            dv, dl = self.attn(v, l, attention_mask_v=attention_mask_v, attention_mask_l=attention_mask_l)
        return v + self.gamma_v * dv, l + self.gamma_l * dl

    # The folded path removes three S x v_dim x embed_dim projections but evaluates each head's vision-side softmax in two
    # passes over the keys once they exceed one block, so its cost grows faster with N than forward_engine's.  On an H100 SXM
    # (700 W) it is faster up to at least N = 1203 (one fusion layer at 1024^2: 6.1 ms against 7.1 ms) and slower at N = 5000
    # (bench.py --workload ape_l_d_1536_phrase); forward_engine takes the longer prompts.
    fold_max_tokens = 1536

    def folds(self, v_dim, l_dim, n_tokens, masked_v=True):
        """True when a 16-bit CUDA call with n_tokens > 1 unmasked language tokens takes the folded path (`folded`): the
        engine gate of `forward` with 256-channel vision tokens and at most fold_max_tokens tokens.  masked_v: a vision
        padding mask is passed (as inside a CUDA graph)."""
        a = self.attn
        return a.head_dim in (64, 256) and v_dim == 256 and l_dim % 8 == 0 and n_tokens <= self.fold_max_tokens and \
            not (a.use_attention_mask_v and masked_v)

    def folded(self, vn, ln, n_tokens=None):
        """BiMultiHeadAttention.forward (fuse_helper.py:67-166) for N >= 1 unmasked language tokens, with the language side
        folded into the 256-dimensional vision space (fold_maps): per layer ONE GEMM maps the LayerNormed tokens to the
        per-head keys qa, biases qc and values U, and
          vision side:   out_s = vn_s + gamma_v (sum_h sum_n softmax_n(vn_s . qa[h,n] + qc[h,n]) U[h,n] + b_out_v)
          language side: pooled[h,n] = sum_s softmax_s(vn_s . qa[h,n]) vn_s  (qc is constant in s and cancels),
                         delta_l = E pooled + e0.
        Nothing of width embed_dim is formed over the S vision tokens: no v_proj / values_v_proj / out_v_proj GEMMs.  The
        +-5e4 clamps and the global-max shift are treated as softmax-invariant translations, as in forward_engine.
        vn [B,S,256] 16-bit (layer-normed), ln [B,N,l_dim] fp32.  Returns (query [B,S,256] in vn's dtype, l [B,N,l_dim] fp32).
        n_tokens: see forward; the padding tokens are no keys of the vision side and their pooled rows are zeros."""
        from .. import ops

        a = self.attn
        nh, dt = a.num_heads, vn.dtype
        B, N, L = ln.shape
        C = vn.shape[-1]
        Gm, gm0, E, e0 = self._folded_multi_maps(dt)
        with torch.autocast("cuda", enabled=False):
            y = ops.linear_tc(ln.to(dt).reshape(B * N, L), Gm, gm0, out_dtype=torch.float32).view(B, N, -1)  # [qa | U | qc]
            qa = torch.empty((B, nh, N, C), dtype=dt, device=vn.device)
            qa.copy_(y[..., : nh * C].view(B, N, nh, C).transpose(1, 2))
            u = torch.empty_like(qa)
            u.copy_(y[..., nh * C: 2 * nh * C].view(B, N, nh, C).transpose(1, 2))
            qc = y[..., 2 * nh * C:].transpose(1, 2).contiguous()
            vn = vn.contiguous()
            _, bo = ops.packed(a.out_v_proj, dt)
            out = ops.vlf_fold_vision(vn, qa, u, qc, self.gamma_v.detach().float().contiguous(), bo, n_dev=n_tokens)
            pooled = ops.vlf_fold_pool(vn, qa, n_dev=n_tokens)
            dl = ops.linear_tc(pooled, E, e0, out_dtype=torch.float32).view(B, N, L)
        return out, ln + self.gamma_l.float() * dl

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

    def _fold_params(self):
        a = self.attn
        return [a.l_proj.weight, a.l_proj.bias, a.v_proj.weight, a.v_proj.bias, a.values_l_proj.weight, a.values_l_proj.bias,
                a.out_v_proj.weight, a.out_v_proj.bias, a.values_v_proj.weight, a.values_v_proj.bias, a.out_l_proj.weight,
                a.out_l_proj.bias]

    def fold_maps(self, dtype=torch.float64):
        """The fusion is affine in each language token on both sides, so the chains of small projections fold (computed in
        fp64, returned in `dtype`):
          one token:  [qa | qc | delta_v] = ln_l @ G^T + g0     (l_proj -> per-head v_proj^T; l_proj -> v_proj bias;
                                                                 values_l_proj -> out_v_proj summed over heads)
          N tokens:   [qa | U | qc]       = ln_l @ Gm^T + gm0   (the same qa / qc; U[h] = out_v_proj restricted to head h
                                                                 after values_l_proj: the per-head values in the vision space)
          both:       delta_l             = pooled @ E^T + e0   (values_v_proj per head -> out_l_proj)
        qa [nh, v_dim], qc [nh] per token: scores[s, h] = v_s . qa[h] + qc[h]; pooled [nh * v_dim] per token."""
        a = self.attn
        nh, hd = a.num_heads, a.head_dim
        with torch.no_grad():
            d = lambda t: t.detach().double()
            wl, bl = d(a.l_proj.weight).view(nh, hd, -1), d(a.l_proj.bias).view(nh, hd)           # [nh,hd,L]
            wq, bq = d(a.v_proj.weight).view(nh, hd, -1), d(a.v_proj.bias).view(nh, hd)           # [nh,hd,C]
            A = torch.einsum("hdc,hdj->hcj", wq, wl) * a.scale                                    # [nh,C,L]
            a0 = torch.einsum("hdc,hd->hc", wq, bl) * a.scale
            Cm = torch.einsum("hd,hdj->hj", bq, wl) * a.scale                                     # [nh,L]
            c0 = torch.einsum("hd,hd->h", bq, bl) * a.scale
            wvl, bvl = d(a.values_l_proj.weight).view(nh, hd, -1), d(a.values_l_proj.bias).view(nh, hd)
            wov = d(a.out_v_proj.weight).view(-1, nh, hd)                                         # [C,nh,hd]
            U = torch.einsum("chd,hdj->hcj", wov, wvl)                                            # [nh,C,L]
            u0 = torch.einsum("chd,hd->hc", wov, bvl)                                             # [nh,C]
            D = d(a.out_v_proj.weight) @ d(a.values_l_proj.weight)                                # [C,L]
            d0 = d(a.out_v_proj.weight) @ d(a.values_l_proj.bias) + d(a.out_v_proj.bias)
            G = torch.cat([A.reshape(-1, A.shape[-1]), Cm, D], 0)
            g0 = torch.cat([a0.reshape(-1), c0, d0], 0)
            Gm = torch.cat([A.reshape(-1, A.shape[-1]), U.reshape(-1, U.shape[-1]), Cm], 0)
            gm0 = torch.cat([a0.reshape(-1), u0.reshape(-1), c0], 0)
            wvv, bvv = d(a.values_v_proj.weight).view(nh, hd, -1), d(a.values_v_proj.bias)        # [nh,hd,C]
            wol = d(a.out_l_proj.weight).view(-1, nh, hd)                                         # [L,nh,hd]
            E = torch.einsum("jhd,hdc->jhc", wol, wvv).reshape(wol.shape[0], -1)
            e0 = d(a.out_l_proj.weight) @ bvv + d(a.out_l_proj.bias)
        return tuple(t.to(dtype).contiguous() for t in (G, g0, E, e0, Gm, gm0))

    def _folded_language_maps(self):
        """fold_maps in fp32, cached per set of weights: (G, g0, E, e0, Gm, gm0).  One GEMV / GEMM each per layer instead of
        ~25 small kernels; results differ from the op-by-op order by rounding."""
        key = tuple((t._version, t.data_ptr()) for t in self._fold_params())
        if getattr(self, "_folded", (None,))[0] != key:
            self._folded = (key,) + self.fold_maps(torch.float32)
        return self._folded[1:]

    def _folded_multi_maps(self, dtype):
        """(Gm, gm0, E, e0) for the N-token GEMMs: weights in the engine dtype, biases fp32; one copy per dtype (ops.cached)."""
        from .. import ops

        key = tuple((t._version, t.data_ptr()) for t in self._fold_params())

        def build():
            _, _, E, e0, Gm, gm0 = self._folded_language_maps()
            return Gm.to(dtype).contiguous(), gm0, E.to(dtype).contiguous(), e0

        return ops.cached(self, "_ape_fold_multi", dtype, key, build)

    def single_token_language_side(self, l):
        """Everything of the one-token case that depends on the language token only: delta_v [B,1,v_dim] and the
        folded score operands qa [B,nh,v_dim], qc [B,nh] (scores[s,h] = v_s . qa[h] + qc[h])."""
        a = self.attn
        nh, hd = a.num_heads, a.head_dim
        if l.is_cuda and self.fold_language_side:
            with torch.autocast("cuda", enabled=False):
                G, g0 = self._folded_language_maps()[:2]
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
                E, e0 = self._folded_language_maps()[2:4]
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

    def forward(self, v, l, attention_mask_v=None, attention_mask_l=None, n_tokens=None):
        return self.b_attn(v, l, attention_mask_v, attention_mask_l, n_tokens)
