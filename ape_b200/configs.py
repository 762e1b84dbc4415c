"""Model specifications as plain dicts (the reference expresses the same values as detectron2
LazyConfig trees; file:line cited per entry).  Shared by the engine, the tests and bench.py.

APE_L_D   configs/LVISCOCOCOCOSTUFF_O365_OID_VGR_SA1B_REFCOCO_GQA_PhraseCut_Flickr30k/ape_deta/
          ape_deta_vitl_eva02_clip_vlf_lsj1024_cp_16x4_1080k.py:19-227 on top of
          configs/COCO_InstanceSegmentation/ape_deta/models/ape_deta_r50.py:24-155 and
          configs/common/backbone/vitl_eva02_clip.py:9-48
MINI      same architecture, toy sizes: used for golden fixtures small enough to commit.
APE_L_B   APE-L_B and APE-L_C (vit_eva02.py ViT-L, no neck); MINI_EVA02L is its toy-size twin.
APE_L_A   APE-L_B without vision-language fusion; MINI_L_A is its toy-size twin.
"""
import copy


def _window_blocks(depth, every=3):
    # global attention on every 3rd block (2,5,8,...), window attention elsewhere
    return [i for i in range(depth) if i % every != every - 1]


APE_L_D = dict(
    name="APE-L_D",
    backbone=dict(
        img_size=1024, patch_size=16, embed_dim=1024, depth=24, num_heads=16,
        window_size=32, mlp_ratio=4 * 2 / 3, window_block_indexes=_window_blocks(24),
        pretrain_img_size=336, pt_hw_seq_len=16,                      # vitl_eva02_clip.py:10-41
        out_channels=256, scale_factors=(4.0, 2.0, 1.0, 0.5), square_pad=1024,  # :42-48
    ),
    embed_dim=256, num_heads=8, num_points=4, ffn_dim=2048,            # ape_deta_r50.py:55-75
    enc_layers=6, dec_layers=6, num_levels=5, num_queries=900,         # ape_deta_r50.py:75-82
    gn_groups=32,                                                      # …1080k.py:42-55
    vlf_embed=2048, vlf_heads=8, vlf_init=1.0 / 6, lang_dim=1024,      # …1080k.py:86-98,40
    num_classes=1256, proposal_ambiguous=1,                            # …1080k.py:106,174
    pre_nms_topk=1000, nms_thresh_enc=0.9,                             # deformable_transformer_vl.py:277-279
    test_topk=300, test_nms_thresh=0.7, test_score_thresh=0.0,         # …1080k.py:107; deformable_detr.py:81-82
    pixel_mean=(123.675, 116.280, 103.530), pixel_std=(58.395, 57.120, 57.375),  # ape_deta_r50.py:124-125
)

APE_L_D_1536 = copy.deepcopy(APE_L_D)
APE_L_D_1536["name"] = "APE-L_D-1536"
APE_L_D_1536["backbone"].update(img_size=1536, square_pad=1536)         # configs/common/backbone/vitl_eva02_clip_1536.py

# APE-Ti (BASELINE.json configs[0]): configs/common/backbone/vitt_eva02.py:10-41 (ape/modeling/backbone/vit_eva02.py:
# packed-SwiGLU "w12", fused qkv, no sub-LN, 14x14 windows over a 64x64 token grid padded to 70x70) under the same
# deformable transformer as APE-L_D (…/ape_deta_vitt_eva02_vlf_lsj1024_cp_16x4_1080k.py:19-176).
APE_TI = copy.deepcopy(APE_L_D)
APE_TI["name"] = "APE-Ti"
APE_TI["backbone"] = dict(
    variant="eva02",                                                   # vit_eva02.py: swiglu=True, naiveswiglu=False, subln=False
    img_size=1024, patch_size=16, embed_dim=192, depth=12, num_heads=3,
    window_size=14, mlp_ratio=4 * 2 / 3, window_block_indexes=[0, 1, 3, 4, 6, 7, 9, 10],
    pretrain_img_size=224, pt_hw_seq_len=16,
    out_channels=256, scale_factors=(4.0, 2.0, 1.0, 0.5), square_pad=1024,
)

# APE-L_B: configs/LVISCOCOCOCOSTUFF_O365_OID_VGR_REFCOCO/ape_deta/ape_deta_vitl_eva02_vlf_lsj1024_cp_1080k.py on top of
# …_vlf_lsj1024_cp_720k.py:12-47 (VL classes, fusion layer), …_lsj1024_cp_720k.py:16-53 (1256 classes, top-300, no neck),
# LVIS_InstanceSegmentation/ape_deta/ape_deta_vitl_eva02_lsj1024_cp_24ep.py and
# COCO_InstanceSegmentation/ape_deta/ape_deta_vitl_eva02_lsj1024_cp_12ep.py:9-29,83-86 (backbone, neck = None, EVA01-CLIP
# text features of width 1024) over models/ape_deta_r50.py.  APE-L_C (LVISCOCOCOCOSTUFF_O365_OID_VGR_SA1B_REFCOCO/…_1080k.py)
# imports that model unchanged; only its criterion list (7 entries) differs, which shapes nothing but the non-persistent
# features_phrase_bank.  Both configs also set semantic_on=True and stuff_prob_thing=0.9 (…_lsj1024_cp_720k.py:47-51):
# the semantic branch is switched per run with `model.semantic_on`.
APE_L_B = copy.deepcopy(APE_L_D)
APE_L_B["name"] = "APE-L_B"
APE_L_B["backbone"] = dict(
    variant="eva02_subln",              # vit_eva02.py: subln=True, naiveswiglu=True (q/k/v projections, ffn_ln, no inner_attn_ln)
    img_size=1024, patch_size=16, embed_dim=1024, depth=24, num_heads=16,
    window_size=16, mlp_ratio=4 * 2 / 3, window_block_indexes=_window_blocks(24, every=6),  # vitl_eva02.py:10-27
    pretrain_img_size=224, pt_hw_seq_len=16,  # vit_eva02.ViT defaults (:468-498): not set by the config
    out_channels=256, scale_factors=(4.0, 2.0, 1.0, 0.5), square_pad=1024,  # vitl_eva02.py:35-40
)
APE_L_B.update(neck=None, num_classes=1256, proposal_ambiguous=0)  # …_lsj1024_cp_720k.py:16,53; deformable_transformer_vl.py:280

MINI = dict(
    name="MINI",
    backbone=dict(
        img_size=64, patch_size=16, embed_dim=64, depth=3, num_heads=2,
        window_size=2, mlp_ratio=4 * 2 / 3, window_block_indexes=_window_blocks(3),
        pretrain_img_size=48, pt_hw_seq_len=16,
        out_channels=64, scale_factors=(4.0, 2.0, 1.0, 0.5), square_pad=64,
    ),
    embed_dim=256, num_heads=8, num_points=4, ffn_dim=128,   # 256: get_proposal_pos_embed hard-codes 4x128 (deformable_transformer_vl.py:412)
    enc_layers=2, dec_layers=2, num_levels=5, num_queries=20,
    gn_groups=32,
    vlf_embed=128, vlf_heads=4, vlf_init=1.0 / 6, lang_dim=32,
    num_classes=12, proposal_ambiguous=1,
    pre_nms_topk=1000, nms_thresh_enc=0.9,
    test_topk=10, test_nms_thresh=0.7, test_score_thresh=0.0,
    pixel_mean=(123.675, 116.280, 103.530), pixel_std=(58.395, 57.120, 57.375),
)

# APE-L_B's structure at MINI sizes (no neck, proposal_ambiguous = 0, the vit_eva02.py sub-LN blocks): golden fixtures.
# The pyramid's 64 channels are the encoder's width here, so embed_dim follows out_channels = 256 as in APE-L_B.
MINI_EVA02L = copy.deepcopy(MINI)
MINI_EVA02L["name"] = "MINI-EVA02L"
MINI_EVA02L["backbone"].update(variant="eva02_subln", out_channels=256)
MINI_EVA02L.update(neck=None, proposal_ambiguous=0)


# APE-L_A: configs/LVISCOCOCOCOSTUFF_O365_OID_VG/ape_deta/ape_deta_vitl_eva02_lsj1024_cp_720k.py:11-53 (1256 classes, top-300,
# no neck) on the same LVIS / COCO chain as APE-L_B, without the _vlf_ step: DeformableDETRSegm over DeformableDetrTransformer
# (deformable_detr_segm.py, deformable_transformer.py), i.e. APE-L_B without the fusion fields.  The model builds no fusion
# layer and no name-prompt fusion feature (ape_deta_r50.py leaves name_prompt_fusion_type at "none").
_FUSION_FIELDS = ("vlf_embed", "vlf_heads", "vlf_init")
APE_L_A = {k: copy.deepcopy(v) for k, v in APE_L_B.items() if k not in _FUSION_FIELDS}
APE_L_A["name"] = "APE-L_A"

# APE-L_A's structure at MINI sizes: golden fixtures.
MINI_L_A = {k: copy.deepcopy(v) for k, v in MINI_EVA02L.items() if k not in _FUSION_FIELDS}
MINI_L_A["name"] = "MINI-L_A"


def level_shapes(spec):
    """Feature-map sizes p2..p6 for the padded square input (strides 4..64)."""
    s = spec["backbone"]["square_pad"]
    return [(s // st, s // st) for st in (4, 8, 16, 32, 64)]
