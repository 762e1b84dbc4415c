"""EVA-02 ViT backbone + SimpleFeaturePyramid of APE-L_D.

Mirror of ape/modeling/backbone/vit_eva_clip.py (`ViT` :570-754, `Block` :383-567, `Attention`
:135-319, `SwiGLU` :101-132, `SimpleFeaturePyramid` :757-922) and utils_eva02.py (`PatchEmbed`
:190-216, `get_abs_pos` :158-187, `VisionRotaryEmbeddingFast` :307-346, window partition :19-63):
same constructor arguments, same parameter / buffer names, so `DetectionCheckpointer.load` fills
them.  Only the configuration APE uses is implemented (sub-LN, naive SwiGLU, 2-D RoPE, q/v bias,
window + global blocks, no rel-pos bias, pre-norm, no layer scale); other switches raise."""
import math
import os
from functools import partial

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from ..layers.common import ConvNorm, LayerNorm2d


class ShapeSpec:
    def __init__(self, channels=None, height=None, width=None, stride=None):
        self.channels, self.height, self.width, self.stride = channels, height, width, stride


class VisionRotaryEmbeddingFast(nn.Module):
    """utils_eva02.py:307-346: cos/sin tables (ft_seq_len^2, 2*dim) for 2-D rotary embedding."""

    def __init__(self, dim, pt_seq_len=16, ft_seq_len=None, theta=10000):
        super().__init__()
        freqs = 1.0 / (theta ** (torch.arange(0, dim, 2)[: (dim // 2)].float() / dim))
        if ft_seq_len is None:
            ft_seq_len = pt_seq_len
        t = torch.arange(ft_seq_len) / ft_seq_len * pt_seq_len
        freqs = torch.einsum("i,f->if", t, freqs).repeat_interleave(2, dim=-1)
        fh = freqs[:, None, :].expand(ft_seq_len, ft_seq_len, -1)
        fw = freqs[None, :, :].expand(ft_seq_len, ft_seq_len, -1)
        freqs = torch.cat([fh, fw], dim=-1)
        self.register_buffer("freqs_cos", freqs.cos().reshape(-1, freqs.shape[-1]))
        self.register_buffer("freqs_sin", freqs.sin().reshape(-1, freqs.shape[-1]))

    def forward(self, t):
        x = t.reshape(*t.shape[:-1], -1, 2)
        x1, x2 = x.unbind(dim=-1)
        rot = torch.stack((-x2, x1), dim=-1).flatten(-2)
        return t * self.freqs_cos + rot * self.freqs_sin


class PatchEmbed(nn.Module):
    def __init__(self, kernel_size=(16, 16), stride=(16, 16), padding=(0, 0), in_chans=3, embed_dim=768):
        super().__init__()
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=kernel_size, stride=stride, padding=padding)

    def forward(self, x):
        return self.proj(x).permute(0, 2, 3, 1)


def get_abs_pos(abs_pos, has_cls_token, hw):
    h, w = hw
    if has_cls_token:
        abs_pos = abs_pos[:, 1:]
    size = int(math.sqrt(abs_pos.shape[1]))
    assert size * size == abs_pos.shape[1]
    if size != h or size != w:
        new = F.interpolate(abs_pos.reshape(1, size, size, -1).permute(0, 3, 1, 2), size=(h, w), mode="bicubic",
                            align_corners=False)
        return new.permute(0, 2, 3, 1)
    return abs_pos.reshape(1, h, w, -1)


def window_partition(x, ws):
    B, H, W, C = x.shape
    pad_h, pad_w = (ws - H % ws) % ws, (ws - W % ws) % ws
    if pad_h > 0 or pad_w > 0:
        x = F.pad(x, (0, 0, 0, pad_w, 0, pad_h))
    Hp, Wp = H + pad_h, W + pad_w
    x = x.view(B, Hp // ws, ws, Wp // ws, ws, C)
    return x.permute(0, 1, 3, 2, 4, 5).contiguous().view(-1, ws, ws, C), (Hp, Wp)


def window_unpartition(win, ws, pad_hw, hw):
    Hp, Wp = pad_hw
    H, W = hw
    B = win.shape[0] // (Hp * Wp // ws // ws)
    x = win.view(B, Hp // ws, Wp // ws, ws, ws, -1).permute(0, 1, 3, 2, 4, 5).contiguous().view(B, Hp, Wp, -1)
    if Hp > H or Wp > W:
        x = x[:, :H, :W, :].contiguous()
    return x


class SwiGLU(nn.Module):
    def __init__(self, in_features, hidden_features, norm_layer):
        super().__init__()
        self.w1 = nn.Linear(in_features, hidden_features)
        self.w2 = nn.Linear(in_features, hidden_features)
        self.ffn_ln = norm_layer(hidden_features)
        self.w3 = nn.Linear(hidden_features, in_features)

    def forward(self, x):
        return self.w3(self.ffn_ln(F.silu(self.w1(x)) * self.w2(x)))


class PackedSwiGLU(nn.Module):
    """vit_eva02.py `xops_SwiGLU` (:41-160): w1 and w2 stacked in one `w12` Linear, no inner LayerNorm."""

    def __init__(self, in_features, hidden_features):
        super().__init__()
        self.w12 = nn.Linear(in_features, 2 * hidden_features)
        self.w3 = nn.Linear(hidden_features, in_features)

    def forward(self, x):
        w1, w2 = torch.unbind(self.w12.weight.view(2, self.w12.weight.shape[0] // 2, -1), dim=0)
        b1, b2 = torch.unbind(self.w12.bias.view(2, -1), dim=0)
        return self.w3(F.silu(F.linear(x, w1, b1)) * F.linear(x, w2, b2))


class Attention(nn.Module):
    """subln=True: vit_eva_clip.py:135-319 (separate q/k/v projections + inner_attn_ln, APE-L);
    subln=False: vit_eva02.py `Attention` (fused `qkv` projection, no inner norm, APE-Ti)."""

    def __init__(self, dim, num_heads, rope, norm_layer, subln=True):
        super().__init__()
        self.num_heads = num_heads
        head_dim = dim // num_heads
        self.scale = head_dim ** -0.5
        self.subln = subln
        if subln:
            self.q_proj = nn.Linear(dim, dim, bias=False)
            self.k_proj = nn.Linear(dim, dim, bias=False)
            self.v_proj = nn.Linear(dim, dim, bias=False)
        else:
            self.qkv = nn.Linear(dim, dim * 3, bias=False)
        self.q_bias = nn.Parameter(torch.zeros(dim))
        self.v_bias = nn.Parameter(torch.zeros(dim))
        if subln:
            self.inner_attn_ln = norm_layer(dim)
        self.proj = nn.Linear(dim, dim)
        self.rope = rope

    def forward(self, x):
        B, H, W, C = x.shape
        N = H * W
        x = x.reshape(B, N, C)
        if self.subln:
            q = F.linear(x, self.q_proj.weight, self.q_bias)
            k = F.linear(x, self.k_proj.weight, None)
            v = F.linear(x, self.v_proj.weight, self.v_bias)
            q = q.reshape(B, N, self.num_heads, -1).permute(0, 2, 1, 3)
            k = k.reshape(B, N, self.num_heads, -1).permute(0, 2, 1, 3)
            v = v.reshape(B, N, self.num_heads, -1).permute(0, 2, 1, 3)
        else:
            bias = torch.cat((self.q_bias, torch.zeros_like(self.v_bias), self.v_bias))
            qkv = F.linear(x, self.qkv.weight, bias).reshape(B, N, 3, self.num_heads, -1).permute(2, 0, 3, 1, 4)
            q, k, v = qkv[0], qkv[1], qkv[2]
        q = self.rope(q).type_as(v)
        k = self.rope(k).type_as(v)
        o = F.scaled_dot_product_attention(q, k, v, dropout_p=0.0, scale=self.scale)
        o = o.permute(0, 2, 1, 3).reshape(B, N, -1)
        if self.subln:
            o = self.inner_attn_ln(o)
        return self.proj(o).view(B, H, W, C)


class Block(nn.Module):
    def __init__(self, dim, num_heads, mlp_ratio, norm_layer, window_size, rope, subln=True, packed_swiglu=False):
        super().__init__()
        self.norm1 = norm_layer(dim)
        self.attn = Attention(dim, num_heads, rope, norm_layer, subln=subln)
        self.norm2 = norm_layer(dim)
        self.mlp = PackedSwiGLU(dim, int(dim * mlp_ratio)) if packed_swiglu else SwiGLU(dim, int(dim * mlp_ratio), norm_layer)
        self.window_size = window_size

    def forward(self, x):
        shortcut = x
        x = self.norm1(x)
        if self.window_size > 0:
            H, W = x.shape[1], x.shape[2]
            x, pad_hw = window_partition(x, self.window_size)
        x = self.attn(x)
        if self.window_size > 0:
            x = window_unpartition(x, self.window_size, pad_hw, (H, W))
        x = shortcut + x
        return x + self.mlp(self.norm2(x))


class ViT(nn.Module):
    def __init__(self, img_size=1024, patch_size=16, in_chans=3, embed_dim=768, depth=12, num_heads=12,
                 mlp_ratio=4.0, qkv_bias=False, qk_scale=None, drop_rate=0.0, attn_drop_rate=0.0, drop_path_rate=0.0,
                 norm_layer=partial(nn.LayerNorm, eps=1e-6), init_values=None, use_abs_pos=True, use_rel_pos=False,
                 rope=False, postnorm=False, pt_hw_seq_len=16, intp_freq=False, naiveswiglu=False, subln=False,
                 window_size=0, window_block_indexes=(), residual_block_indexes=(), use_act_checkpoint=False,
                 pretrain_img_size=224, pretrain_use_cls_token=True, out_feature="last_feat", xattn=False,
                 frozen_stages=-1, swiglu=False):
        super().__init__()
        variant_l = naiveswiglu and subln and not swiglu        # vit_eva_clip.py (APE-L_*: sub-LN, naive SwiGLU)
        variant_ti = swiglu and not naiveswiglu and not subln   # vit_eva02.py   (APE-Ti: packed SwiGLU, fused qkv)
        if not (rope and (variant_l or variant_ti) and qkv_bias and use_abs_pos and intp_freq) or postnorm or init_values \
                or len(residual_block_indexes) or qk_scale is not None:
            raise NotImplementedError("ape_b200.ViT implements the two EVA-02 configurations APE uses "
                                      "(rope, qkv_bias, abs pos, intp_freq, pre-norm; naiveswiglu + subln, or packed swiglu)")
        self._variant_l = variant_l
        self.pretrain_use_cls_token = pretrain_use_cls_token
        self.patch_embed = PatchEmbed((patch_size, patch_size), (patch_size, patch_size), in_chans=in_chans,
                                      embed_dim=embed_dim)
        num_patches = (pretrain_img_size // patch_size) ** 2
        self.pos_embed = nn.Parameter(torch.zeros(1, num_patches + (1 if pretrain_use_cls_token else 0), embed_dim))
        half = embed_dim // num_heads // 2
        self.rope_win = VisionRotaryEmbeddingFast(half, pt_hw_seq_len, window_size)
        self.rope_glb = VisionRotaryEmbeddingFast(half, pt_hw_seq_len, img_size // patch_size)
        self.blocks = nn.ModuleList([
            Block(embed_dim, num_heads, mlp_ratio, norm_layer, window_size if i in window_block_indexes else 0,
                  self.rope_win if i in window_block_indexes else self.rope_glb, subln=variant_l, packed_swiglu=variant_ti)
            for i in range(depth)])
        # RoPE in the qkv GEMM's epilogue (ape_gemm_tn_rope) instead of the in-place ape_rope_qk pass: measured slower twice
        # (+26 us per GEMM with the general epilogue, +27 us with a lean one: per-thread cos / sin rows are 32 different lines per
        # warp load) against 8.7 us for the pass; APE_FUSED_ROPE=1 switches it on for A/B runs
        self.fused_rope = os.environ.get("APE_FUSED_ROPE", "0") == "1"
        self.engine_attention = True  # ape_attn_fwd (own wgmma kernel) for head_dim 64 / n % 128 == 0, else library SDPA
        # inner_attn_ln / ffn_ln folded around proj / w3 (ape_gemm_tn_fused): two LayerNorm launches and two trips of the
        # activations through HBM fewer per block
        self.fold_sub_layernorms = True
        self._out_feature_channels = {out_feature: embed_dim}
        self._out_feature_strides = {out_feature: patch_size}
        self._out_features = [out_feature]
        nn.init.trunc_normal_(self.pos_embed, std=0.02)
        self.apply(self._init_weights)

    @staticmethod
    def _init_weights(m):
        if isinstance(m, nn.Linear):
            nn.init.trunc_normal_(m.weight, std=0.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def output_shape(self):
        return {n: ShapeSpec(channels=self._out_feature_channels[n], stride=self._out_feature_strides[n])
                for n in self._out_features}

    def forward(self, x):
        if x.is_cuda and x.dtype in (torch.float16, torch.bfloat16) and self._engine_ok(x):
            return {self._out_features[0]: self._engine_forward(x)}
        # fp32 (strict-parity) path on PyTorch library kernels
        x = self.patch_embed(x)
        x = x + get_abs_pos(self.pos_embed, self.pretrain_use_cls_token, (x.shape[1], x.shape[2])).to(x.dtype)
        for blk in self.blocks:
            x = blk(x)
        return {self._out_features[0]: x.permute(0, 3, 1, 2)}

    # ---------------------------------------------------------------------------------------------
    # Engine path (fp16 / bf16): libape_b200 kernels — wgmma GEMMs with fused bias / SwiGLU /
    # residual epilogues, LayerNorm and RoPE kernels; tokens stay in WINDOW-MAJOR order for the
    # whole network (attention is permutation-equivariant once the RoPE table follows the tokens), so
    # window_partition / window_unpartition (utils_eva02.py:19-63) cost one permutation at the
    # patch embedding and one at the end instead of two copies per block.
    # ---------------------------------------------------------------------------------------------
    def _engine_ok(self, x):
        if not self._variant_l:  # the tensor-core token path is written for the APE-L block layout
            return False
        ws = next((b.window_size for b in self.blocks if b.window_size > 0), 0)
        g = x.shape[-1] // self.patch_embed.proj.kernel_size[0]
        return x.shape[-1] == x.shape[-2] and (ws == 0 or g % ws == 0)

    def _pack(self, dtype, device):
        """Weights re-laid out once for the kernels (fused qkv, interleaved SwiGLU pairs, K padded to 8)."""
        key = (str(device), tuple(p._version for p in self.parameters()))
        packs = self.__dict__.setdefault("_packs", {})  # one entry per engine dtype, never evicted (ops.cached)
        if dtype in packs and packs[dtype][0] == key:
            return packs[dtype][1]
        f32 = dict(dtype=torch.float32, device=device)
        packed = {"blocks": []}
        with torch.no_grad():
            pw = self.patch_embed.proj.weight
            packed["patch_w"] = pw.reshape(pw.shape[0], -1).to(device, dtype).contiguous()
            packed["patch_b"] = self.patch_embed.proj.bias.to(**f32).contiguous()
            for blk in self.blocks:
                a, m = blk.attn, blk.mlp
                hid = m.w1.weight.shape[0]
                hid_p = (hid + 7) // 8 * 8
                w12 = torch.stack([m.w1.weight, m.w2.weight], 1).reshape(2 * hid, -1)  # rows (w1_j, w2_j)
                b12 = torch.stack([m.w1.bias, m.w2.bias], 1).reshape(2 * hid)
                w3 = torch.zeros(m.w3.weight.shape[0], hid_p, dtype=dtype, device=device)
                w3[:, :hid] = m.w3.weight
                packed["blocks"].append(dict(
                    n1w=blk.norm1.weight.to(**f32), n1b=blk.norm1.bias.to(**f32),
                    wqkv=torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], 0).to(device, dtype).contiguous(),
                    bqkv=torch.cat([a.q_bias, torch.zeros_like(a.v_bias), a.v_bias]).to(**f32).contiguous(),
                    lnw=a.inner_attn_ln.weight.to(**f32), lnb=a.inner_attn_ln.bias.to(**f32),
                    wproj=a.proj.weight.to(device, dtype).contiguous(), bproj=a.proj.bias.to(**f32).contiguous(),
                    n2w=blk.norm2.weight.to(**f32), n2b=blk.norm2.bias.to(**f32),
                    w12=w12.to(device, dtype).contiguous(), b12=b12.to(**f32).contiguous(),
                    fw=m.ffn_ln.weight.to(**f32).contiguous(), fb=m.ffn_ln.bias.to(**f32).contiguous(),
                    w3=w3, b3=m.w3.bias.to(**f32).contiguous(), hid=hid, hid_p=hid_p))
                # sub-LayerNorms folded around the GEMM that follows them (ape_gemm_tn_fused): gamma .* W as the 16-bit
                # operand, its row sums, and beta W^T + b as the bias
                d = packed["blocks"][-1]
                wp = (a.proj.weight.float() * a.inner_attn_ln.weight.float()[None, :]).to(device, dtype).contiguous()
                d.update(wproj_ln=wp, sproj=wp.float().sum(1).contiguous(),
                         bproj_ln=(a.proj.weight.float() @ a.inner_attn_ln.bias.float() + a.proj.bias.float()).to(**f32).contiguous())
                w3l = torch.zeros(m.w3.weight.shape[0], hid_p, dtype=dtype, device=device)
                w3l[:, :hid] = (m.w3.weight.float() * m.ffn_ln.weight.float()[None, :]).to(dtype)
                d.update(w3_ln=w3l, s3=w3l.float().sum(1).contiguous(),
                         b3_ln=(m.w3.weight.float() @ m.ffn_ln.bias.float() + m.w3.bias.float()).to(**f32).contiguous())
        packs[dtype] = (key, packed)
        return packed

    def _geometry(self, B, g, ws, dtype, device):
        """Per input geometry: window-major token permutation, abs-pos table, RoPE position maps."""
        k = (B, g, ws, dtype, str(device), self.pos_embed._version)
        geom = self.__dict__.setdefault("_geom", {})
        if k in geom:
            return geom[k]
        nw = g // ws if ws else 1
        w = ws if ws else g
        ids = torch.arange(g * g, device=device).view(nw, w, nw, w).permute(0, 2, 1, 3).reshape(-1)  # window-major -> raster
        pos = get_abs_pos(self.pos_embed.detach().float(), self.pretrain_use_cls_token, (g, g)).reshape(g * g, -1)
        geo = dict(ids=ids, pos=pos[ids].float().repeat(B, 1).contiguous(),  # fp32: first value of the residual stream
                   glb_map=ids.to(torch.int32).repeat(B).contiguous(), inv=torch.argsort(ids))
        geom[k] = geo
        return geo

    def _engine_forward(self, img):
        return self._engine_tokens(img).permute(0, 3, 1, 2)  # NCHW view over NHWC memory (channels_last)

    def _engine_tokens(self, img):
        B, _, Hh, Ww = img.shape
        ps = self.patch_embed.proj.kernel_size[0]
        g = Hh // ps
        ws = next((b.window_size for b in self.blocks if b.window_size > 0), 0)
        dtype, dev = img.dtype, img.device
        pk = self._pack(dtype, dev)
        geo = self._geometry(B, g, ws, dtype, dev)
        C = self.pos_embed.shape[-1]
        heads = self.blocks[0].attn.num_heads
        hd = C // heads
        nw = g // ws if ws else 1
        w = ws if ws else g
        # patch embedding as a GEMM over window-major im2col rows; abs-pos added as the epilogue residual
        cols = img.view(B, 3, nw, w, ps, nw, w, ps).permute(0, 2, 5, 3, 6, 1, 4, 7).reshape(B * g * g, 3 * ps * ps)
        # The residual stream `x` stays fp32 for all 24 blocks (only GEMM / attention operands and LayerNorm outputs are
        # 16-bit): every branch output is added in the GEMM epilogue to the fp32 stream and written back as fp32.
        x = ops.linear_tc(cols, pk["patch_w"], pk["patch_b"], residual=geo["pos"], out_dtype=torch.float32)
        M = x.shape[0]
        rope_win = (self.rope_win.freqs_cos.float().contiguous(), self.rope_win.freqs_sin.float().contiguous())
        rope_glb = (self.rope_glb.freqs_cos.float().contiguous(), self.rope_glb.freqs_sin.float().contiguous())
        hid_p = pk["blocks"][0]["hid_p"]
        hbuf = torch.empty((M, hid_p), dtype=dtype, device=dev)
        hbuf2 = torch.empty((M, hid_p), dtype=dtype, device=dev)
        for blk, p in zip(self.blocks, pk["blocks"]):
            h = ops.layernorm(x, p["n1w"], p["n1b"], eps=1e-6, out_dtype=dtype)
            # RoPE in the qkv GEMM epilogue (ape_gemm_tn_rope) is available but OFF: measured +26 us per qkv GEMM (the 8
            # epilogue warps wait on the cos/sin rows) against 8.7 us for the separate ape_rope_qk pass
            fused_rope = self.fused_rope and hd == 64 and C % 8 == 0
            if blk.window_size > 0:
                if fused_rope:
                    qkv = ops.linear_rope_tc(h, p["wqkv"], p["bqkv"], rope_win[0], rope_win[1], C, hd)
                else:
                    qkv = ops.linear_tc(h, p["wqkv"], p["bqkv"])
                    ops.rope_qk_(qkv, rope_win[0], rope_win[1], C, hd)  # position = index inside the window
                nb, n = B * nw * nw, w * w
            else:
                if fused_rope:
                    qkv = ops.linear_rope_tc(h, p["wqkv"], p["bqkv"], rope_glb[0], rope_glb[1], C, hd, pos_map=geo["glb_map"])
                else:
                    qkv = ops.linear_tc(h, p["wqkv"], p["bqkv"])
                    ops.rope_qk_(qkv, rope_glb[0], rope_glb[1], C, hd, pos_map=geo["glb_map"])
                nb, n = B, g * g
            fold = self.fold_sub_layernorms
            if self.engine_attention and ops.attention_supported(n, hd, qkv.dtype):
                # wgmma flash attention, no head-split copies; with `fold` it also leaves per-(row, head) statistics
                o = ops.attention_qkv(qkv, nb, n, heads, hd, blk.attn.scale, stats_out=fold)
                o, st = o if fold else (o, None)
            else:
                q5 = qkv.view(nb, n, 3, heads, hd)
                o = F.scaled_dot_product_attention(q5[:, :, 0].transpose(1, 2), q5[:, :, 1].transpose(1, 2),
                                                   q5[:, :, 2].transpose(1, 2), scale=blk.attn.scale)
                o, st = o.transpose(1, 2).reshape(M, C), None
            if st is not None:  # inner_attn_ln folded into proj: the raw attention output is the GEMM operand
                x = ops.linear_tc(o, p["wproj_ln"], p["bproj_ln"], residual=x, out_dtype=torch.float32,
                                  ln_fold=(st, p["sproj"], C, 1e-6))
            else:
                a = ops.layernorm(o, p["lnw"], p["lnb"], eps=1e-6)
                x = ops.linear_tc(a, p["wproj"], p["bproj"], residual=x, out_dtype=torch.float32)
            h = ops.layernorm(x, p["n2w"], p["n2b"], eps=1e-6, out_dtype=dtype)
            if fold:  # ffn_ln folded into w3: the SwiGLU epilogue leaves the row statistics of the hidden it writes
                _, st2 = ops.linear_tc(h, p["w12"], p["b12"], act="swiglu", out=hbuf[:, :p["hid"]], stats_out=True)
                x = ops.linear_tc(hbuf[:, :p["hid"]], p["w3_ln"][:, :p["hid"]], p["b3_ln"], residual=x, out_dtype=torch.float32,
                                  ln_fold=(st2, p["s3"], p["hid"], 1e-6))
            else:
                ops.linear_tc(h, p["w12"], p["b12"], act="swiglu", out=hbuf[:, :p["hid"]])
                ops.layernorm(hbuf[:, :p["hid"]], p["fw"], p["fb"], eps=1e-6, out=hbuf2[:, :p["hid"]])
                x = ops.linear_tc(hbuf2[:, :p["hid"]], p["w3"][:, :p["hid"]], p["b3"], residual=x, out_dtype=torch.float32)
        # back to raster order: [B, g, g, C] tokens (NHWC memory), 16-bit operand of the pyramid GEMMs
        return x.to(dtype).view(B, g * g, C)[:, geo["inv"]].view(B, g, g, C)


def _convT_as_gemm(ct, dtype):
    """ConvTranspose2d(k=2, s=2) as a GEMM over tokens: weight [(dy,dx,co), ci], bias tiled 4x (cached)."""
    return ops.cached(ct, "_ape_packed_ct", dtype, (ct.weight._version, ct.weight.data_ptr()), lambda: (
        ct.weight.detach().permute(2, 3, 1, 0).reshape(-1, ct.weight.shape[0]).to(dtype).contiguous(),
        ct.bias.detach().float().repeat(4).contiguous()))


def _conv_weights_ohwi(conv, dtype):
    """3x3 Conv2d weight as [Cout, 3, 3, Cin] (the K-major operand of ape_conv3x3_nhwc)."""
    return ops.cached(conv, "_ape_packed_ohwi", dtype, (conv.weight._version, conv.weight.data_ptr()),
                      lambda: conv.weight.detach().permute(0, 2, 3, 1).to(dtype).contiguous())


def conv3x3_tokens(conv, y, B, H, W, engine):
    """3x3 convolution (no bias) over token-major activations y [B*H*W, C] -> [B, H, W, Cout] contiguous: the repo's implicit-GEMM
    kernel when `engine` and the geometry is covered, else cuDNN on the channels_last view (no copies)."""
    ch = y.shape[-1]
    if engine and conv.bias is None and ops.conv3x3_supported(H, W, ch, conv.weight.shape[0], y.dtype):
        return ops.conv3x3_nhwc(y.view(B, H, W, ch), _conv_weights_ohwi(conv, y.dtype))
    z = F.conv2d(y.view(B, H, W, ch).permute(0, 3, 1, 2), _conv_weights(conv, y.dtype), padding=1).permute(0, 2, 3, 1)
    return z if z.is_contiguous() else z.contiguous()


def _conv_weights(conv, dtype):
    def build():
        w = conv.weight.detach().to(dtype)
        return w.reshape(w.shape[0], -1).contiguous() if w.shape[-1] == 1 else w.contiguous(memory_format=torch.channels_last)

    return ops.cached(conv, "_ape_packed_cv", dtype, (conv.weight._version, conv.weight.data_ptr()), build)


class LastLevelMaxPool(nn.Module):
    def __init__(self):
        super().__init__()
        self.num_levels = 1
        self.in_feature = "p5"

    def forward(self, x):
        return [F.max_pool2d(x, kernel_size=1, stride=2, padding=0)]


class SimpleFeaturePyramid(nn.Module):
    def __init__(self, net, in_feature, out_channels, scale_factors, top_block=None, norm="LN", square_pad=0):
        super().__init__()
        assert norm == "LN"
        self.scale_factors = scale_factors
        shapes = net.output_shape()
        strides = [int(shapes[in_feature].stride / s) for s in scale_factors]
        dim = shapes[in_feature].channels
        self.stages = []
        for idx, scale in enumerate(scale_factors):
            out_dim = dim
            if scale == 4.0:
                layers = [nn.ConvTranspose2d(dim, dim // 2, kernel_size=2, stride=2), LayerNorm2d(dim // 2), nn.GELU(),
                          nn.ConvTranspose2d(dim // 2, dim // 4, kernel_size=2, stride=2)]
                out_dim = dim // 4
            elif scale == 2.0:
                layers = [nn.ConvTranspose2d(dim, dim // 2, kernel_size=2, stride=2)]
                out_dim = dim // 2
            elif scale == 1.0:
                layers = []
            elif scale == 0.5:
                layers = [nn.MaxPool2d(kernel_size=2, stride=2)]
            else:
                raise NotImplementedError(f"scale_factor={scale} is not supported yet.")
            layers.extend([ConvNorm(out_dim, out_channels, 1, bias=False, norm=LayerNorm2d(out_channels)),
                           ConvNorm(out_channels, out_channels, 3, padding=1, bias=False, norm=LayerNorm2d(out_channels))])
            seq = nn.Sequential(*layers)
            stage = int(math.log2(strides[idx]))
            self.add_module(f"simfp_{stage}", seq)
            self.stages.append(seq)
        self.net = net
        self.in_feature = in_feature
        self.top_block = top_block
        self._out_feature_strides = {"p{}".format(int(math.log2(s))): s for s in strides}
        if top_block is not None:
            for s in range(stage, stage + top_block.num_levels):
                self._out_feature_strides["p{}".format(s + 1)] = 2 ** (s + 1)
        self._out_features = list(self._out_feature_strides.keys())
        self._out_feature_channels = {k: out_channels for k in self._out_features}
        self._size_divisibility = strides[-1]
        self._square_pad = square_pad
        # 3x3 convolutions on the repo's implicit-GEMM kernel (ape_conv3x3_nhwc) instead of cuDNN
        self.conv3x3_engine = os.environ.get("APE_CONV3X3", "1") == "1"

    @property
    def size_divisibility(self):
        return 0  # detectron2 Backbone default; the reference's SFP does not override it

    @property
    def padding_constraints(self):
        return {"size_divisiblity": self._size_divisibility, "square_size": self._square_pad}

    def output_shape(self):
        return {n: ShapeSpec(channels=self._out_feature_channels[n], stride=self._out_feature_strides[n])
                for n in self._out_features}

    # Engine path: activations stay token-major (NHWC) from the ViT to the encoder.  2x2/stride-2 transposed
    # convolutions and 1x1 convolutions are wgmma GEMMs over tokens; the pixel shuffle of a transposed conv is
    # folded into the row map of the LayerNorm kernel that follows it; channels-first LayerNorm (detectron2 "LN")
    # is a row LayerNorm in this layout; only the 3x3 convolutions still go to cuDNN (channels_last, no copies).
    def _shuffle_map(self, B, g, device):
        key = (B, g, str(device))
        cache = self.__dict__.setdefault("_maps", {})
        if key not in cache:
            b, y, x, dy, dx = torch.meshgrid(torch.arange(B), torch.arange(g), torch.arange(g), torch.arange(2),
                                             torch.arange(2), indexing="ij")
            cache[key] = (b * (4 * g * g) + (2 * y + dy) * (2 * g) + 2 * x + dx).reshape(-1).to(device, torch.int32)
        return cache[key]

    def _engine_forward(self, img):
        tok = self.net._engine_tokens(img)  # [B, g, g, C]
        B, g, _, C = tok.shape
        dt, dev = tok.dtype, tok.device
        results = {}
        for scale, seq, name in zip(self.scale_factors, self.stages, self._out_features):
            mods = list(seq)
            if scale == 4.0:
                ct1, ln, _, ct2, c1, c3 = mods
                w, b = _convT_as_gemm(ct1, dt)
                y = ops.linear_tc(tok.view(-1, C), w, b).view(-1, C // 2)            # rows (t, dy, dx)
                lw, lb = ops.packed(ln, dt)
                y = ops.layernorm(y, lw, lb, eps=ln.eps, row_map=self._shuffle_map(B, g, dev))  # -> raster 2g x 2g
                y = F.gelu(y)
                w, b = _convT_as_gemm(ct2, dt)
                y = ops.linear_tc(y, w, b).view(-1, C // 4)                          # rows (t2, dy, dx), t2 raster 2g
                y = ops.linear_tc(y, _conv_weights(c1, dt))                          # 1x1 conv commutes with the shuffle
                nw, nb = ops.packed(c1.norm, dt)
                y = ops.layernorm(y, nw, nb, eps=c1.norm.eps, row_map=self._shuffle_map(B, 2 * g, dev))
                hw = 4 * g
            elif scale == 2.0:
                ct1, c1, c3 = mods
                w, b = _convT_as_gemm(ct1, dt)
                y = ops.linear_tc(tok.view(-1, C), w, b).view(-1, C // 2)
                y = ops.linear_tc(y, _conv_weights(c1, dt))
                nw, nb = ops.packed(c1.norm, dt)
                y = ops.layernorm(y, nw, nb, eps=c1.norm.eps, row_map=self._shuffle_map(B, g, dev))
                hw = 2 * g
            else:
                if scale == 1.0:
                    c1, c3 = mods
                    src, hw = tok.view(-1, C), g
                elif scale == 0.5:
                    _, c1, c3 = mods
                    src = F.max_pool2d(tok.permute(0, 3, 1, 2), kernel_size=2, stride=2).permute(0, 2, 3, 1).reshape(-1, C)
                    hw = g // 2
                else:
                    raise NotImplementedError(f"scale_factor={scale} is not supported yet.")
                y = ops.linear_tc(src, _conv_weights(c1, dt))
                nw, nb = ops.packed(c1.norm, dt)
                y = ops.layernorm(y, nw, nb, eps=c1.norm.eps)
            ch = y.shape[-1]
            z = conv3x3_tokens(c3, y, B, hw, hw, self.conv3x3_engine)
            nw, nb = ops.packed(c3.norm, dt)
            z = ops.layernorm(z.view(-1, ch), nw, nb, eps=c3.norm.eps)
            results[name] = z.view(B, hw, hw, ch).permute(0, 3, 1, 2)
        top = self.top_block(results[self.top_block.in_feature])
        for n, t in zip(self._out_features[len(self.stages):], top):
            results[n] = t
        return {n: results[n] for n in self._out_features}

    def forward(self, x):
        if x.is_cuda and x.dtype in (torch.float16, torch.bfloat16) and hasattr(self.net, "_engine_ok") \
                and self.net._engine_ok(x) and isinstance(self.top_block, LastLevelMaxPool):
            return self._engine_forward(x)
        feats = self.net(x)
        f = feats[self.in_feature]
        results = [stage(f) for stage in self.stages]
        if self.top_block is not None:
            src = feats[self.top_block.in_feature] if self.top_block.in_feature in feats else \
                results[self._out_features.index(self.top_block.in_feature)]
            results.extend(self.top_block(src))
        return dict(zip(self._out_features, results))
