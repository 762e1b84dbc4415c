"""Drop-in classes for configs that build ape/modeling/backbone/vit_eva02.py (`configs/common/backbone/vitl_eva02.py`: APE-L_A,
APE-L_B, APE-L_C; `vitt_eva02.py`: APE-Ti).

`ViT` takes vit_eva02.ViT's signature and defaults (:468-498) and reads its switches the way that file does:
  swiglu=True                    packed `w12` SwiGLU, fused `qkv`, no sub-LayerNorms (APE-Ti)
  naiveswiglu=True, subln=True   separate q/k/v projections with q/v biases, NO inner_attn_ln, SwiGLU w1, w2, ffn_ln, w3
                                 (:179-291; APE-L_B / L_C)
It is ape_b200.modeling.ViT with that reading; ape_b200.modeling.ViT keeps vit_eva_clip.py's (subln = inner_attn_ln too).
`fp8_linears` (not in the reference, off by default) is ape_b200.modeling.ViT's opt-in FP8 qkv / w12 mode; the APE-Ti path
ignores it."""
from functools import partial

import torch.nn as nn

from . import backbone as _backbone
from .backbone import SimpleFeaturePyramid  # noqa: F401  (vit_eva02.py defines the same pyramid)


class ViT(_backbone.ViT):
    _reference_file = "vit_eva02"

    def __init__(self, img_size=1024, patch_size=16, in_chans=3, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4 * 2 / 3,
                 qkv_bias=True, drop_path_rate=0.0, norm_layer=partial(nn.LayerNorm, eps=1e-6), act_layer=nn.GELU,
                 use_abs_pos=True, use_rel_pos=False, rope=True, pt_hw_seq_len=16, intp_freq=True, window_size=0,
                 window_block_indexes=(), residual_block_indexes=(), use_act_checkpoint=False, pretrain_img_size=224,
                 pretrain_use_cls_token=True, out_feature="last_feat", xattn=True, subln=False, swiglu=False,
                 naiveswiglu=False, frozen_stages=-1, fp8_linears=False):
        # act_layer is accepted and unused, as in the reference (its blocks use SiLU gates only)
        super().__init__(img_size=img_size, patch_size=patch_size, in_chans=in_chans, embed_dim=embed_dim, depth=depth,
                         num_heads=num_heads, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias, drop_path_rate=drop_path_rate,
                         norm_layer=norm_layer, use_abs_pos=use_abs_pos, use_rel_pos=use_rel_pos, rope=rope,
                         pt_hw_seq_len=pt_hw_seq_len, intp_freq=intp_freq, naiveswiglu=naiveswiglu, subln=subln,
                         window_size=window_size, window_block_indexes=window_block_indexes,
                         residual_block_indexes=residual_block_indexes, use_act_checkpoint=use_act_checkpoint,
                         pretrain_img_size=pretrain_img_size, pretrain_use_cls_token=pretrain_use_cls_token,
                         out_feature=out_feature, xattn=xattn, frozen_stages=frozen_stages, swiglu=swiglu,
                         fp8_linears=fp8_linears)
