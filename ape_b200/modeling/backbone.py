"""EVA-02 ViT backbone + SimpleFeaturePyramid of APE-L_D, APE-L_B / L_C (ape_b200.modeling.vit_eva02.ViT) and APE-Ti.

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
    """subln=True: separate q/k/v projections; inner_ln=True adds vit_eva_clip.py's inner_attn_ln (:135-319, APE-L_D), which
    vit_eva02.py's sub-LN Attention does not have (:206-291, APE-L_B / L_C); subln=False: vit_eva02.py's fused `qkv`
    projection, no inner norm (APE-Ti).  inner_ln defaults to subln (the vit_eva_clip.py reading)."""

    def __init__(self, dim, num_heads, rope, norm_layer, subln=True, inner_ln=None):
        super().__init__()
        self.num_heads = num_heads
        head_dim = dim // num_heads
        self.scale = head_dim ** -0.5
        self.subln = subln
        self.inner_ln = subln if inner_ln is None else inner_ln
        if subln:
            self.q_proj = nn.Linear(dim, dim, bias=False)
            self.k_proj = nn.Linear(dim, dim, bias=False)
            self.v_proj = nn.Linear(dim, dim, bias=False)
        else:
            self.qkv = nn.Linear(dim, dim * 3, bias=False)
        self.q_bias = nn.Parameter(torch.zeros(dim))
        self.v_bias = nn.Parameter(torch.zeros(dim))
        if self.inner_ln:
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
        if self.inner_ln:
            o = self.inner_attn_ln(o)
        return self.proj(o).view(B, H, W, C)


class Block(nn.Module):
    def __init__(self, dim, num_heads, mlp_ratio, norm_layer, window_size, rope, subln=True, packed_swiglu=False,
                 inner_ln=None):
        super().__init__()
        self.norm1 = norm_layer(dim)
        self.attn = Attention(dim, num_heads, rope, norm_layer, subln=subln, inner_ln=inner_ln)
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
    """EVA-02 ViT of APE.  `fp8_linears=True` (off by default, not a reference keyword) runs the qkv and w12 GEMMs of every
    block in FP8 on the window-major engine path (APE-L_D, APE-L_B / L_C); the APE-Ti raster path and the fp32 path ignore
    it and run as without it."""
    # reference file whose meaning of `subln` this class follows: vit_eva_clip.py (inner_attn_ln) here, vit_eva02.py (none)
    # in ape_b200.modeling.vit_eva02.ViT
    _reference_file = "vit_eva_clip"

    def __init__(self, img_size=1024, patch_size=16, in_chans=3, embed_dim=768, depth=12, num_heads=12,
                 mlp_ratio=4.0, qkv_bias=False, qk_scale=None, drop_rate=0.0, attn_drop_rate=0.0, drop_path_rate=0.0,
                 norm_layer=partial(nn.LayerNorm, eps=1e-6), init_values=None, use_abs_pos=True, use_rel_pos=False,
                 rope=False, postnorm=False, pt_hw_seq_len=16, intp_freq=False, naiveswiglu=False, subln=False,
                 window_size=0, window_block_indexes=(), residual_block_indexes=(), use_act_checkpoint=False,
                 pretrain_img_size=224, pretrain_use_cls_token=True, out_feature="last_feat", xattn=False,
                 frozen_stages=-1, swiglu=False, fp8_linears=False):
        super().__init__()
        naive_subln = naiveswiglu and subln and not swiglu
        variant_l = naive_subln and self._reference_file == "vit_eva_clip"  # APE-L_D: sub-LN with inner_attn_ln, naive SwiGLU
        variant_lb = naive_subln and self._reference_file == "vit_eva02"    # APE-L_B / L_C: q/k/v projections, ffn_ln only
        variant_ti = swiglu and not naiveswiglu and not subln                # APE-Ti: packed SwiGLU, fused qkv
        if not (rope and (variant_l or variant_lb or variant_ti) and qkv_bias and use_abs_pos and intp_freq) or postnorm \
                or init_values or len(residual_block_indexes) or qk_scale is not None:
            raise NotImplementedError("ape_b200.ViT implements the three EVA-02 configurations APE uses "
                                      "(rope, qkv_bias, abs pos, intp_freq, pre-norm; naiveswiglu + subln, or packed swiglu)")
        self._variant_l = variant_l
        self._flavour = "eva_clip" if variant_l else "eva02_subln" if variant_lb else "eva02_swiglu"
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
                  self.rope_win if i in window_block_indexes else self.rope_glb, subln=not variant_ti, packed_swiglu=variant_ti,
                  inner_ln=variant_l)
            for i in range(depth)])
        # RoPE in the qkv GEMM's epilogue (ape_gemm_tn_rope) instead of the in-place ape_rope_qk pass: measured slower twice
        # (+26 us per GEMM with the general epilogue, +27 us with a lean one: per-thread cos / sin rows are 32 different lines per
        # warp load) against 8.7 us for the pass; APE_FUSED_ROPE=1 switches it on for A/B runs
        self.fused_rope = os.environ.get("APE_FUSED_ROPE", "0") == "1"
        # APE-L path: ape_attn_fwd (own wgmma kernel) for head_dim 64 / n % 128 == 0, else library SDPA (the APE-Ti path
        # always runs ape_attn_fwd*: _engine_ok requires 64-channel heads)
        self.engine_attention = True
        # inner_attn_ln / ffn_ln folded around proj / w3 (ape_gemm_tn_fused): two LayerNorm launches and two trips of the
        # activations through HBM fewer per block
        self.fold_sub_layernorms = True
        # Opt-in FP8 (e4m3) for the two GEMMs that follow a LayerNorm in every block, qkv (after norm1) and w12 (after
        # norm2): the LayerNorm writes e4m3 values with a scale per row (ape_layernorm_e4m3) and the GEMM runs on the FP8
        # tensor cores (ape_gemm_tn_e4m3) against weights quantised once per output row.  RoPE, attention, proj, w3, the
        # folds and the fp32 residual stream are unchanged.  Only the window-major engine path (APE-L_D, APE-L_B / L_C)
        # honours it; the APE-Ti raster path and the fp32 path ignore it.  Off by default: its accuracy on the released
        # checkpoints has not been measured.
        self.fp8_linears = bool(fp8_linears)
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
    # residual epilogues, LayerNorm and RoPE kernels.  APE-L_*: tokens stay in WINDOW-MAJOR order for
    # the whole network (attention is permutation-equivariant once the RoPE table follows the tokens),
    # so window_partition / window_unpartition (utils_eva02.py:19-63) cost one permutation at the
    # patch embedding and one at the end instead of two copies per block.  APE-Ti (windows that need
    # not tile the grid): tokens stay in RASTER order and each window block scatters / gathers them
    # through row maps (_engine_tokens_raster).
    # ---------------------------------------------------------------------------------------------
    def _engine_ok(self, x):
        ws = next((b.window_size for b in self.blocks if b.window_size > 0), 0)
        ps = self.patch_embed.proj.kernel_size[0]
        g = x.shape[-1] // ps
        if self._variant_l:
            return x.shape[-1] == x.shape[-2] and (ws == 0 or g % ws == 0)
        if self._flavour == "eva02_subln":  # window-major path of APE-L_D, RoPE tables of this grid
            return x.shape[-1] == x.shape[-2] and x.shape[-1] % ps == 0 and (ws == 0 or g % ws == 0) and \
                self.rope_glb.freqs_cos.shape[0] == g * g
        # APE-Ti raster path: any window size (windows are padded), 64-channel heads for the attention kernel, and the global
        # RoPE table of this grid
        C, heads = self.pos_embed.shape[-1], self.blocks[0].attn.num_heads
        return x.shape[-1] == x.shape[-2] and x.shape[-1] % ps == 0 and C == 64 * heads and \
            self.rope_glb.freqs_cos.shape[0] == g * g

    def _pack(self, dtype, device):
        """Weights re-laid out once for the kernels (fused qkv, interleaved SwiGLU pairs, K padded to 8)."""
        key = (str(device), self.fold_sub_layernorms, tuple(p._version for p in self.parameters()))
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
                if self._flavour == "eva02_subln":
                    packed["blocks"].append(self._pack_block_eva02_subln(blk, dtype, device))
                    continue
                if self._variant_l:
                    wqkv = torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], 0)
                    w1, w2, b1, b2 = m.w1.weight, m.w2.weight, m.w1.bias, m.w2.bias
                else:  # vit_eva02.py: fused qkv projection, w12 = [w1; w2] stacked halves
                    wqkv = a.qkv.weight
                    w1, w2 = m.w12.weight.chunk(2, 0)
                    b1, b2 = m.w12.bias.chunk(2, 0)
                hid = w1.shape[0]
                hid_p = (hid + 7) // 8 * 8
                w12 = torch.stack([w1, w2], 1).reshape(2 * hid, -1)  # rows (w1_j, w2_j)
                b12 = torch.stack([b1, b2], 1).reshape(2 * hid)
                w3 = torch.zeros(m.w3.weight.shape[0], hid_p, dtype=dtype, device=device)
                w3[:, :hid] = m.w3.weight
                d = dict(
                    n1w=blk.norm1.weight.to(**f32), n1b=blk.norm1.bias.to(**f32),
                    wqkv=wqkv.to(device, dtype).contiguous(),
                    bqkv=torch.cat([a.q_bias, torch.zeros_like(a.v_bias), a.v_bias]).to(**f32).contiguous(),
                    wproj=a.proj.weight.to(device, dtype).contiguous(), bproj=a.proj.bias.to(**f32).contiguous(),
                    n2w=blk.norm2.weight.to(**f32), n2b=blk.norm2.bias.to(**f32),
                    w12=w12.to(device, dtype).contiguous(), b12=b12.to(**f32).contiguous(),
                    w3=w3, b3=m.w3.bias.to(**f32).contiguous(), hid=hid, hid_p=hid_p)
                packed["blocks"].append(d)
                if not self._variant_l:
                    continue
                d.update(lnw=a.inner_attn_ln.weight.to(**f32), lnb=a.inner_attn_ln.bias.to(**f32),
                         fw=m.ffn_ln.weight.to(**f32).contiguous(), fb=m.ffn_ln.bias.to(**f32).contiguous())
                # sub-LayerNorms folded around the GEMM that follows them (ape_gemm_tn_fused): gamma .* W as the 16-bit
                # operand, its row sums, and beta W^T + b as the bias
                wp = (a.proj.weight.float() * a.inner_attn_ln.weight.float()[None, :]).to(device, dtype).contiguous()
                d.update(wproj_ln=wp, sproj=wp.float().sum(1).contiguous(),
                         bproj_ln=(a.proj.weight.float() @ a.inner_attn_ln.bias.float() + a.proj.bias.float()).to(**f32).contiguous())
                w3l = torch.zeros(m.w3.weight.shape[0], hid_p, dtype=dtype, device=device)
                w3l[:, :hid] = (m.w3.weight.float() * m.ffn_ln.weight.float()[None, :]).to(dtype)
                d.update(w3_ln=w3l, s3=w3l.float().sum(1).contiguous(),
                         b3_ln=(m.w3.weight.float() @ m.ffn_ln.bias.float() + m.w3.bias.float()).to(**f32).contiguous())
        packs[dtype] = (key, packed)
        return packed

    def _pack_block_eva02_subln(self, blk, dtype, device):
        """vit_eva02.py sub-LN block (APE-L_B / L_C): fused [q; k; v] weight, plain proj (no inner_attn_ln), interleaved
        SwiGLU pairs, and w3 with ffn_ln folded in (or ffn_ln and w3 apart when fold_sub_layernorms is off)."""
        f32 = dict(dtype=torch.float32, device=device)
        a, m = blk.attn, blk.mlp
        hid = m.w1.weight.shape[0]
        hid_p = (hid + 7) // 8 * 8
        w12 = torch.stack([m.w1.weight, m.w2.weight], 1).reshape(2 * hid, -1)  # rows (w1_j, w2_j)
        b12 = torch.stack([m.w1.bias, m.w2.bias], 1).reshape(2 * hid)
        d = dict(
            n1w=blk.norm1.weight.to(**f32), n1b=blk.norm1.bias.to(**f32),
            wqkv=torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], 0).to(device, dtype).contiguous(),
            bqkv=torch.cat([a.q_bias, torch.zeros_like(a.v_bias), a.v_bias]).to(**f32).contiguous(),
            wproj=a.proj.weight.to(device, dtype).contiguous(), bproj=a.proj.bias.to(**f32).contiguous(),
            n2w=blk.norm2.weight.to(**f32), n2b=blk.norm2.bias.to(**f32),
            w12=w12.to(device, dtype).contiguous(), b12=b12.to(**f32).contiguous(), hid=hid, hid_p=hid_p)
        w3 = torch.zeros(m.w3.weight.shape[0], hid_p, dtype=dtype, device=device)
        if self.fold_sub_layernorms:  # gamma .* W3 as the operand, its row sums, beta W3^T + b3 as the bias
            w3[:, :hid] = (m.w3.weight.float() * m.ffn_ln.weight.float()[None, :]).to(dtype)
            d.update(w3_ln=w3, s3=w3.float().sum(1).contiguous(),
                     b3_ln=(m.w3.weight.float() @ m.ffn_ln.bias.float() + m.w3.bias.float()).to(**f32).contiguous())
        else:
            w3[:, :hid] = m.w3.weight
            d.update(w3=w3, b3=m.w3.bias.to(**f32).contiguous(),
                     fw=m.ffn_ln.weight.to(**f32).contiguous(), fb=m.ffn_ln.bias.to(**f32).contiguous())
        return d

    def _pack_fp8(self, packed, device):
        """e4m3 copies of the fused qkv and interleaved w12 weights with one scale per output row (ops.quantize_rows_e4m3),
        quantised from the fp32 parameters and added to the blocks of the 16-bit pack `packed` on first use, so the 16-bit
        weights of a graph captured without FP8 stay where they are."""
        for blk, d in zip(self.blocks, packed["blocks"]):
            if "wqkv_q" in d:
                continue
            a, m = blk.attn, blk.mlp
            wqkv = torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], 0).to(device)
            w12 = torch.stack([m.w1.weight, m.w2.weight], 1).reshape(2 * m.w1.weight.shape[0], -1).to(device)
            d["wqkv_q"], d["sqkv"] = ops.quantize_rows_e4m3(wqkv)
            d["w12_q"], d["s12"] = ops.quantize_rows_e4m3(w12)

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

    def _raster_geometry(self, B, g, ws, device):
        """APE-Ti, per input geometry: abs-pos table in raster order, and the maps between raster rows and the padded
        window-major rows of window_partition (windows of ws x ws over the grid padded to a multiple of ws)."""
        k = ("raster", B, g, ws, str(device), self.pos_embed._version)
        geom = self.__dict__.setdefault("_geom", {})
        if k in geom:
            return geom[k]
        pos = get_abs_pos(self.pos_embed.detach().float(), self.pretrain_use_cls_token, (g, g)).reshape(g * g, -1)
        geo = dict(pos=pos.float().repeat(B, 1).contiguous())  # fp32: first value of the residual stream
        if ws:
            nw = -(-g // ws)
            b, y, x = torch.meshgrid(torch.arange(B), torch.arange(g), torch.arange(g), indexing="ij")
            row = ((b * nw + y // ws) * nw + x // ws) * (ws * ws) + (y % ws) * ws + x % ws  # raster -> padded window-major
            inv = torch.full((B * nw * nw * ws * ws,), -1, dtype=torch.int32)
            inv[row.reshape(-1)] = torch.arange(B * g * g, dtype=torch.int32)  # pad rows stay -1
            geo.update(win_map=row.reshape(-1).to(device, torch.int32), win_out_map=inv.to(device), windows=B * nw * nw)
        geom[k] = geo
        return geo

    def _engine_forward(self, img):
        return self._engine_tokens(img).permute(0, 3, 1, 2)  # NCHW view over NHWC memory (channels_last)

    def _engine_tokens(self, img):
        if self._flavour == "eva02_swiglu":
            return self._engine_tokens_raster(img)
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
        fp8 = self.fp8_linears
        if fp8:
            self._pack_fp8(pk, dev)
        for blk, p in zip(self.blocks, pk["blocks"]):
            # RoPE in the qkv GEMM epilogue (ape_gemm_tn_rope) is available but OFF: measured +26 us per qkv GEMM (the 8
            # epilogue warps wait on the cos/sin rows) against 8.7 us for the separate ape_rope_qk pass; the FP8 qkv GEMM
            # always leaves RoPE to that pass
            fused_rope = self.fused_rope and hd == 64 and C % 8 == 0 and not fp8
            if fp8:  # e4m3 LayerNorm output with a scale per row -> FP8 qkv GEMM
                hq, hs = ops.layernorm(x, p["n1w"], p["n1b"], eps=1e-6, out_dtype=torch.float8_e4m3fn)
                qkv = ops.linear_fp8(hq, hs, p["wqkv_q"], p["sqkv"], p["bqkv"], out_dtype=dtype)
            else:
                h = ops.layernorm(x, p["n1w"], p["n1b"], eps=1e-6, out_dtype=dtype)
            if blk.window_size > 0:
                if fused_rope:
                    qkv = ops.linear_rope_tc(h, p["wqkv"], p["bqkv"], rope_win[0], rope_win[1], C, hd)
                else:
                    if not fp8:
                        qkv = ops.linear_tc(h, p["wqkv"], p["bqkv"])
                    ops.rope_qk_(qkv, rope_win[0], rope_win[1], C, hd)  # position = index inside the window
                nb, n = B * nw * nw, w * w
            else:
                if fused_rope:
                    qkv = ops.linear_rope_tc(h, p["wqkv"], p["bqkv"], rope_glb[0], rope_glb[1], C, hd, pos_map=geo["glb_map"])
                else:
                    if not fp8:
                        qkv = ops.linear_tc(h, p["wqkv"], p["bqkv"])
                    ops.rope_qk_(qkv, rope_glb[0], rope_glb[1], C, hd, pos_map=geo["glb_map"])
                nb, n = B, g * g
            fold = self.fold_sub_layernorms
            stats = fold and self._variant_l  # statistics only feed the inner_attn_ln fold
            if self.engine_attention and ops.attention_supported(n, hd, qkv.dtype):
                # wgmma flash attention, no head-split copies; with `stats` it also leaves per-(row, head) statistics
                o = ops.attention_qkv(qkv, nb, n, heads, hd, blk.attn.scale, stats_out=stats)
                o, st = o if stats else (o, None)
            else:
                q5 = qkv.view(nb, n, 3, heads, hd)
                o = F.scaled_dot_product_attention(q5[:, :, 0].transpose(1, 2), q5[:, :, 1].transpose(1, 2),
                                                   q5[:, :, 2].transpose(1, 2), scale=blk.attn.scale)
                o, st = o.transpose(1, 2).reshape(M, C), None
            if st is not None:  # inner_attn_ln folded into proj: the raw attention output is the GEMM operand
                x = ops.linear_tc(o, p["wproj_ln"], p["bproj_ln"], residual=x, out_dtype=torch.float32,
                                  ln_fold=(st, p["sproj"], C, 1e-6))
            elif not self._variant_l:  # vit_eva02.py sub-LN block: no inner_attn_ln
                x = ops.linear_tc(o, p["wproj"], p["bproj"], residual=x, out_dtype=torch.float32)
            else:
                a = ops.layernorm(o, p["lnw"], p["lnb"], eps=1e-6)
                x = ops.linear_tc(a, p["wproj"], p["bproj"], residual=x, out_dtype=torch.float32)
            if fp8:
                hq, hs = ops.layernorm(x, p["n2w"], p["n2b"], eps=1e-6, out_dtype=torch.float8_e4m3fn)
                w12 = lambda **kw: ops.linear_fp8(hq, hs, p["w12_q"], p["s12"], p["b12"], act="swiglu", **kw)
            else:
                h = ops.layernorm(x, p["n2w"], p["n2b"], eps=1e-6, out_dtype=dtype)
                w12 = lambda **kw: ops.linear_tc(h, p["w12"], p["b12"], act="swiglu", **kw)
            if fold:  # ffn_ln folded into w3: the SwiGLU epilogue leaves the row statistics of the hidden it writes
                _, st2 = w12(out=hbuf[:, :p["hid"]], stats_out=True)
                x = ops.linear_tc(hbuf[:, :p["hid"]], p["w3_ln"][:, :p["hid"]], p["b3_ln"], residual=x, out_dtype=torch.float32,
                                  ln_fold=(st2, p["s3"], p["hid"], 1e-6))
            else:
                w12(out=hbuf[:, :p["hid"]])
                ops.layernorm(hbuf[:, :p["hid"]], p["fw"], p["fb"], eps=1e-6, out=hbuf2[:, :p["hid"]])
                x = ops.linear_tc(hbuf2[:, :p["hid"]], p["w3"][:, :p["hid"]], p["b3"], residual=x, out_dtype=torch.float32)
        # back to raster order: [B, g, g, C] tokens (NHWC memory), 16-bit operand of the pyramid GEMMs
        return x.to(dtype).view(B, g * g, C)[:, geo["inv"]].view(B, g, g, C)

    def _engine_tokens_raster(self, img):
        """APE-Ti blocks (vit_eva02.py: fused qkv, packed SwiGLU, no sub-LayerNorms) with the fp32 residual stream in raster
        order.  A window block's norm1 scatters the tokens into a zero-initialised buffer of padded ws x ws windows (pad rows
        are never written, so they stay the zeros window_partition pads with and attend as keys k = 0, v = v_bias), and its
        attention writes each real query row straight back to its raster row; global blocks attend over the raster rows."""
        B, _, Hh, _ = img.shape
        ps = self.patch_embed.proj.kernel_size[0]
        g = Hh // ps
        ws = next((b.window_size for b in self.blocks if b.window_size > 0), 0)
        dtype, dev = img.dtype, img.device
        pk = self._pack(dtype, dev)
        geo = self._raster_geometry(B, g, ws, dev)
        C = self.pos_embed.shape[-1]
        heads = self.blocks[0].attn.num_heads
        hd = C // heads
        M = B * g * g
        cols = img.view(B, 3, g, ps, g, ps).permute(0, 2, 4, 1, 3, 5).reshape(M, 3 * ps * ps)  # raster im2col rows
        x = ops.linear_tc(cols, pk["patch_w"], pk["patch_b"], residual=geo["pos"], out_dtype=torch.float32)
        rope_win = (self.rope_win.freqs_cos.float().contiguous(), self.rope_win.freqs_sin.float().contiguous())
        rope_glb = (self.rope_glb.freqs_cos.float().contiguous(), self.rope_glb.freqs_sin.float().contiguous())
        hid, hid_p = pk["blocks"][0]["hid"], pk["blocks"][0]["hid_p"]
        hbuf = torch.empty((M, hid_p), dtype=dtype, device=dev)[:, :hid]
        hwin = torch.zeros((geo["windows"] * ws * ws, C), dtype=dtype, device=dev) if ws else None
        pad128 = lambda n: -(-n // 128) * 128  # the attention kernel's sequence length: 128-row query tiles
        for blk, p in zip(self.blocks, pk["blocks"]):
            if blk.window_size > 0:
                ops.layernorm(x, p["n1w"], p["n1b"], eps=1e-6, row_map=geo["win_map"], out=hwin)
                qkv = ops.linear_tc(hwin, p["wqkv"], p["bqkv"])  # pad rows: q_bias, 0, v_bias
                ops.rope_qk_(qkv, rope_win[0], rope_win[1], C, hd)  # position = row % (ws * ws) = index inside the window
                o = torch.empty((M, C), dtype=dtype, device=dev)
                ops.attention_qkv(qkv, geo["windows"], pad128(ws * ws), heads, hd, blk.attn.scale, n_valid=ws * ws,
                                  seq_stride=ws * ws, out_row_map=geo["win_out_map"], out=o)
            else:
                h = ops.layernorm(x, p["n1w"], p["n1b"], eps=1e-6, out_dtype=dtype)
                qkv = ops.linear_tc(h, p["wqkv"], p["bqkv"])
                ops.rope_qk_(qkv, rope_glb[0], rope_glb[1], C, hd)  # position = row % (g * g)
                o = ops.attention_qkv(qkv, B, pad128(g * g), heads, hd, blk.attn.scale, n_valid=g * g, seq_stride=g * g)
            x = ops.linear_tc(o, p["wproj"], p["bproj"], residual=x, out_dtype=torch.float32)
            h = ops.layernorm(x, p["n2w"], p["n2b"], eps=1e-6, out_dtype=dtype)
            ops.linear_tc(h, p["w12"], p["b12"], act="swiglu", out=hbuf)
            x = ops.linear_tc(hbuf, p["w3"][:, :hid], p["b3"], residual=x, out_dtype=torch.float32)
        return x.to(dtype).view(B, g, g, C)  # [B, g, g, C] tokens (NHWC memory), 16-bit operand of the pyramid GEMMs


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
        # Engine path for a model without a neck (DeformableDETRSegmVL(neck=None) sets it): every level's final LayerNorm, and
        # the p6 subsample, write into their slice of one [B, S, C] buffer (`last_flat`), the flattened levels the encoder
        # consumes (deformable_transformer_vl.py:435-452); the returned levels are views of it
        self.flat_output = False
        self.last_flat = None

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

    def _flat_map(self, B, S, start, n, device):
        """LayerNorm output rows of one level in the flat [B*S, C] buffer: row (b, r) -> b * S + start + r."""
        key = ("flat", B, S, start, n, str(device))
        cache = self.__dict__.setdefault("_maps", {})
        if key not in cache:
            b, r = torch.meshgrid(torch.arange(B), torch.arange(n), indexing="ij")
            cache[key] = (b * S + start + r).reshape(-1).to(device, torch.int32)
        return cache[key]

    def _engine_forward(self, img):
        tok = self.net._engine_tokens(img)  # [B, g, g, C]
        B, g, _, C = tok.shape
        dt, dev = tok.dtype, tok.device
        results = {}
        flat = None
        if self.flat_output:
            sides = [int(g * s) for s in self.scale_factors]
            sides.append((sides[-1] + 1) // 2)  # LastLevelMaxPool: kernel 1, stride 2
            starts = [sum(h * h for h in sides[:i]) for i in range(len(sides) + 1)]
            flat = torch.empty((B, starts[-1], self._out_feature_channels[self._out_features[0]]), dtype=dt, device=dev)
        self.last_flat = flat
        for li, (scale, seq, name) in enumerate(zip(self.scale_factors, self.stages, self._out_features)):
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
            if flat is not None:
                s0, n = starts[li], hw * hw
                ops.layernorm(z.view(-1, ch), nw, nb, eps=c3.norm.eps, row_map=self._flat_map(B, starts[-1], s0, n, dev),
                              out=flat.view(-1, ch))
                results[name] = flat[:, s0:s0 + n].view(B, hw, hw, ch).permute(0, 3, 1, 2)
                continue
            z = ops.layernorm(z.view(-1, ch), nw, nb, eps=c3.norm.eps)
            results[name] = z.view(B, hw, hw, ch).permute(0, 3, 1, 2)
        if flat is not None:  # p6 = p5[::2, ::2] into the last slice
            h5, h6 = sides[-2], sides[-1]
            p6 = flat[:, starts[-2]:starts[-1]].view(B, h6, h6, -1)
            p6.copy_(flat[:, starts[-3]:starts[-2]].view(B, h5, h5, -1)[:, ::2, ::2])
            results[self._out_features[len(self.stages)]] = p6.permute(0, 3, 1, 2)
            return {n: results[n] for n in self._out_features}
        top = self.top_block(results[self.top_block.in_feature])
        for n, t in zip(self._out_features[len(self.stages):], top):
            results[n] = t
        return {n: results[n] for n in self._out_features}

    def forward(self, x):
        if x.is_cuda and x.dtype in (torch.float16, torch.bfloat16) and hasattr(self.net, "_engine_ok") \
                and self.net._engine_ok(x) and isinstance(self.top_block, LastLevelMaxPool):
            return self._engine_forward(x)
        self.last_flat = None
        feats = self.net(x)
        f = feats[self.in_feature]
        results = [stage(f) for stage in self.stages]
        if self.top_block is not None:
            src = feats[self.top_block.in_feature] if self.top_block.in_feature in feats else \
                results[self._out_features.index(self.top_block.in_feature)]
            results.extend(self.top_block(src))
        return dict(zip(self._out_features, results))
