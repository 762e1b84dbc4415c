"""Engine-side model classes (reference-compatible constructors and parameter names)."""
from functools import partial

import torch
import torch.nn as nn

from ..layers import VisionLanguageFusion
from .backbone import LastLevelMaxPool, ShapeSpec, SimpleFeaturePyramid, ViT
from .detr import ChannelMapper, DeformableDETRSegm, DeformableDETRSegmVL, PositionEmbeddingSine, SomeThing, _Criterion
from .text import EVA01CLIP, EVA02CLIP, TextTransformer  # noqa: F401
from .transformer import (DeformableDetrTransformer, DeformableDetrTransformerDecoder, DeformableDetrTransformerDecoderVL,
                          DeformableDetrTransformerEncoder, DeformableDetrTransformerEncoderVL, DeformableDetrTransformerVL)
from . import vit_eva02  # noqa: F401  (ape_b200.modeling.vit_eva02.ViT: drop-in for vit_eva02.py configs)
from .vit_eva02 import ViT as VitEva02


class SyntheticTextModel:
    """`model_language` stand-in for synthetic benchmarks: seeded features instead of the EVA02-CLIP
    text tower (SURVEY.md §8f row 1; text features are a cached input of the hot path)."""

    def __init__(self, lang_dim, n_max=8192, seed=2, dtype=torch.float32):
        g = torch.Generator().manual_seed(seed)
        self.bank = torch.randn(n_max, lang_dim, generator=g).to(dtype)

    def forward_text(self, text_list, cache=False):
        return {"last_hidden_state_eot": self.bank[: len(text_list)].clone()}


def build_model(spec, num_text=None):
    """Instantiate the engine's DeformableDETRSegmVL (DeformableDETRSegm for specs without fusion fields) from a plain-dict
    spec (ape_b200/configs.py) — what detectron2's `instantiate(cfg.model.model_vision)` does from the LazyConfig tree, with
    `_target_`s pointing at this package (INTEGRATION.md)."""
    b = spec["backbone"]
    variant = b.get("variant", "eva_clip")
    # "eva_clip": vit_eva_clip.py (APE-L_D); "eva02": vit_eva02.py packed SwiGLU (APE-Ti); "eva02_subln": vit_eva02.py sub-LN
    # blocks (APE-L_B / L_C), whose `subln` means no inner_attn_ln: the vit_eva02 class reads it so
    vit_cls = VitEva02 if variant == "eva02_subln" else ViT
    net = vit_cls(img_size=b["img_size"], patch_size=b["patch_size"], embed_dim=b["embed_dim"], depth=b["depth"],
                  num_heads=b["num_heads"], drop_path_rate=0.0, window_size=b["window_size"], mlp_ratio=b["mlp_ratio"],
                  qkv_bias=True, norm_layer=partial(nn.LayerNorm, eps=1e-6), window_block_indexes=b["window_block_indexes"],
                  residual_block_indexes=[], use_rel_pos=True, out_feature="last_feat", use_act_checkpoint=False,
                  xattn=False, rope=True, pt_hw_seq_len=b["pt_hw_seq_len"], intp_freq=True,
                  naiveswiglu=variant != "eva02", subln=variant != "eva02", swiglu=variant == "eva02",
                  pretrain_img_size=b["pretrain_img_size"], pretrain_use_cls_token=True)
    backbone = SimpleFeaturePyramid(net=net, in_feature="last_feat", out_channels=b["out_channels"],
                                    scale_factors=b["scale_factors"], top_block=LastLevelMaxPool(), norm="LN",
                                    square_pad=b["square_pad"])
    E = spec["embed_dim"]
    feats = ["p2", "p3", "p4", "p5", "p6"]
    shapes = {f: ShapeSpec(channels=b["out_channels"]) for f in feats}
    neck = None
    if spec.get("neck", "ChannelMapper") is not None:
        neck = ChannelMapper(input_shapes=shapes, in_features=feats, out_channels=E, num_outs=5, kernel_size=1,
                             norm_layer=nn.GroupNorm(num_groups=spec["gn_groups"], num_channels=E))
    fusion = spec.get("vlf_embed") is not None  # APE-L_A (configs.APE_L_A): the non-VL classes of deformable_detr_segm.py
    enc_kw = dict(embed_dim=E, num_heads=spec["num_heads"], feedforward_dim=spec["ffn_dim"], attn_dropout=0.0, ffn_dropout=0.0,
                  num_layers=spec["enc_layers"], post_norm=False, num_feature_levels=spec["num_levels"])
    dec_kw = dict(embed_dim=E, num_heads=spec["num_heads"], feedforward_dim=spec["ffn_dim"], attn_dropout=0.0, ffn_dropout=0.0,
                  num_layers=spec["dec_layers"], return_intermediate=True, num_feature_levels=spec["num_levels"])
    tr_kw = dict(as_two_stage=True, num_feature_levels=spec["num_levels"], two_stage_num_proposals=spec["num_queries"],
                 assign_first_stage=True, pre_nms_topk=spec["pre_nms_topk"], nms_thresh_enc=spec["nms_thresh_enc"],
                 proposal_ambiguous=spec["proposal_ambiguous"])
    if fusion:
        vl_layer = VisionLanguageFusion(v_dim=E, l_dim=spec["lang_dim"], embed_dim=spec["vlf_embed"],
                                        num_heads=spec["vlf_heads"], dropout=0.1, drop_path=0.0,
                                        init_values=spec["vlf_init"], stable_softmax_2d=True,
                                        clamp_min_for_underflow=True, clamp_max_for_overflow=True, use_checkpoint=False)
        transformer = DeformableDetrTransformerVL(encoder=DeformableDetrTransformerEncoderVL(vl_layer=vl_layer, **enc_kw),
                                                  decoder=DeformableDetrTransformerDecoderVL(**dec_kw), **tr_kw)
    else:
        transformer = DeformableDetrTransformer(encoder=DeformableDetrTransformerEncoder(**enc_kw),
                                                decoder=DeformableDetrTransformerDecoder(**dec_kw), **tr_kw)
    n_text = num_text if num_text is not None else spec["num_classes"]
    name = f"synthetic_{spec['name']}"
    # the _vlf_ configs set name_prompt_fusion_type = "zero" and text_feature_bank = True; APE-L_A keeps ape_deta_r50.py's defaults
    model = (DeformableDETRSegmVL if fusion else DeformableDETRSegm)(
        instance_on=True, semantic_on=False, panoptic_on=False, input_shapes=shapes, mask_in_features=["p2"],
        mask_encode_level=0, stuff_dataset_learn_thing=False, stuff_prob_thing=0.9,
        name_prompt_fusion_type="zero" if fusion else "none",
        test_mask_on=False, backbone=backbone,
        position_embedding=PositionEmbeddingSine(num_pos_feats=E // 2, temperature=10000, normalize=True, offset=-0.5),
        neck=neck, transformer=transformer, embed_dim=E, num_classes=spec["num_classes"],
        num_queries=spec["num_queries"], criterion=[_Criterion(spec["num_classes"])],
        pixel_mean=spec["pixel_mean"], pixel_std=spec["pixel_std"], aux_loss=True, with_box_refine=True,
        as_two_stage=True, select_box_nums_for_evaluation=spec["test_topk"], input_format="RGB",
        dataset_names=[name], dataset_metas=[name], dataset_prompts=["name"], embed_dim_language=spec["lang_dim"],
        text_feature_bank=fusion, text_feature_reduce_before_fusion=True, text_feature_batch_repeat=True,
        test_nms_thresh=spec["test_nms_thresh"], test_score_thresh=spec["test_score_thresh"],
        vocabulary={name: [f"c{i}" for i in range(n_text)]})
    model.set_model_language(SyntheticTextModel(spec["lang_dim"]))
    model.eval()
    return model
