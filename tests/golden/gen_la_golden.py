"""Generates the golden data of APE-L_A (the vit_eva02.py ViT-L sub-LN backbone of APE-L_B, no neck, proposal_ambiguous = 0,
WITHOUT vision-language fusion: deformable_detr_segm.py over deformable_transformer.py) and of its EVA01-CLIP text tower, by
running the REFERENCE's own model files on the CPU (unmodified, under oracle/refshim.py's import shims), with name-derived
synthetic weights (oracle/synth.py).  Build container only; run from the repository root:

  python tests/golden/gen_la_golden.py [cpu|mini|la|text]

  model_mini_la.npz          MINI_L_A, one 48 x 64 image, test_mask_on + semantic_on        (tests/test_ape_l_a_gpu.py)
  model_la_1024.npz          APE-L_A, one 1024 x 768 image padded to 1024^2, 1203 names    (tests/test_ape_l_a_gpu.py)
  state_dict_shapes_la.json.gz   parameter names and shapes for MINI_L_A and APE_L_A       (tests/test_ape_l_a_cpu.py)
  ref_config_tree_la.json    the LazyConfig model tree of APE-L_A                          (tests/test_ape_l_a_cpu.py)
  text_eva01.npz             eva01_clip/eva_model.py TextTransformer at EVA_CLIP_g_14 size  (tests/test_ape_l_a_{cpu,gpu}.py)"""
import gzip
import importlib
import json
import os
import sys
import time
import types
from functools import partial

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
from ape_b200 import configs  # noqa: E402
from oracle import ref_model, refshim, synth  # noqa: E402

REF = "/root/reference"
LA_CONFIGS = ("configs/common/backbone/vitl_eva02.py",
              "configs/COCO_InstanceSegmentation/ape_deta/models/ape_deta_r50.py",
              "configs/COCO_InstanceSegmentation/ape_deta/ape_deta_vitl_eva02_lsj1024_cp_12ep.py",
              "configs/LVIS_InstanceSegmentation/ape_deta/ape_deta_vitl_eva02_lsj1024_cp_24ep.py",
              "configs/LVISCOCOCOCOSTUFF_O365_OID_VG/ape_deta/ape_deta_vitl_eva02_lsj1024_cp_720k.py")
# EVA_CLIP_g_14 / EVA_CLIP_g_14_X text_cfg (eva01_clip/model_configs/*.json) and embed_dim
TEXT_CFG = dict(vocab_size=49408, width=768, layers=12, heads=12, context_length=77, embed_dim=1024)


def build_reference_la(spec, num_text=None, test_mask_on=False, semantic_on=False):
    """The reference APE-L_A model of a fusion-free spec: DeformableDETRSegm over DeformableDetrTransformer{,Encoder,Decoder}
    (deformable_detr_segm.py, deformable_transformer.py), with the constructor values of oracle/ref_model.py's model except
    what the L_A config leaves at ape_deta_r50.py's defaults (name_prompt_fusion_type "none", no text feature bank), the
    vit_eva02.ViT(subln=True, naiveswiglu=True) backbone under vit_eva02.SimpleFeaturePyramid and no neck."""
    assert spec["backbone"]["variant"] == "eva02_subln" and spec["neck"] is None and "vlf_embed" not in spec
    refshim.install()
    vit_mod = refshim.load("ape.modeling.backbone.vit_eva02")
    tr = refshim.load("ape.modeling.ape_deta.deformable_transformer")
    segm = refshim.load("ape.modeling.ape_deta.deformable_detr_segm")
    torch.manual_seed(0)
    b = spec["backbone"]
    net = vit_mod.ViT(
        img_size=b["img_size"], patch_size=b["patch_size"], embed_dim=b["embed_dim"], depth=b["depth"],
        num_heads=b["num_heads"], drop_path_rate=0.0, window_size=b["window_size"], mlp_ratio=b["mlp_ratio"],
        qkv_bias=True, norm_layer=partial(nn.LayerNorm, eps=1e-6), window_block_indexes=b["window_block_indexes"],
        residual_block_indexes=[], use_rel_pos=True, out_feature="last_feat", use_act_checkpoint=False, xattn=False,
        subln=True, swiglu=False, naiveswiglu=True, pt_hw_seq_len=b["pt_hw_seq_len"], pretrain_img_size=b["pretrain_img_size"])
    backbone = vit_mod.SimpleFeaturePyramid(
        net=net, in_feature="last_feat", out_channels=b["out_channels"], scale_factors=b["scale_factors"],
        top_block=refshim.LastLevelMaxPool(), norm="LN", square_pad=b["square_pad"])
    E = spec["embed_dim"]
    shapes = {f: refshim.ShapeSpec(channels=b["out_channels"]) for f in ("p2", "p3", "p4", "p5", "p6")}
    transformer = tr.DeformableDetrTransformer(
        encoder=tr.DeformableDetrTransformerEncoder(
            embed_dim=E, num_heads=spec["num_heads"], feedforward_dim=spec["ffn_dim"], attn_dropout=0.0,
            ffn_dropout=0.0, num_layers=spec["enc_layers"], post_norm=False, num_feature_levels=spec["num_levels"],
            use_act_checkpoint=False, pytorch_attn=True),
        decoder=tr.DeformableDetrTransformerDecoder(
            embed_dim=E, num_heads=spec["num_heads"], feedforward_dim=spec["ffn_dim"], attn_dropout=0.0,
            ffn_dropout=0.0, num_layers=spec["dec_layers"], return_intermediate=True,
            num_feature_levels=spec["num_levels"], pytorch_attn=True),
        as_two_stage=True, num_feature_levels=spec["num_levels"], two_stage_num_proposals=spec["num_queries"],
        assign_first_stage=True, pre_nms_topk=spec["pre_nms_topk"], nms_thresh_enc=spec["nms_thresh_enc"],
        proposal_ambiguous=spec["proposal_ambiguous"])
    n_text = num_text if num_text is not None else spec["num_classes"]
    names = [f"c{i}" for i in range(n_text)]
    meta = refshim.MetadataCatalog.get(f"fake_{spec['name']}_{n_text}")
    meta.thing_classes = names
    model = segm.DeformableDETRSegm(
        instance_on=True, semantic_on=semantic_on, panoptic_on=False, input_shapes=shapes, mask_in_features=["p2"],
        mask_encode_level=0, stuff_dataset_learn_thing=False, stuff_prob_thing=0.9, test_mask_on=test_mask_on,
        backbone=backbone, position_embedding=refshim.PositionEmbeddingSine(num_pos_feats=E // 2, temperature=10000,
                                                                           normalize=True, offset=-0.5),
        neck=None, transformer=transformer, embed_dim=E, num_classes=spec["num_classes"],
        num_queries=spec["num_queries"], criterion=[ref_model.FakeCriterion(spec["num_classes"])],
        pixel_mean=list(spec["pixel_mean"]), pixel_std=list(spec["pixel_std"]), aux_loss=True, with_box_refine=True,
        as_two_stage=True, select_box_nums_for_evaluation=spec["test_topk"], input_format="RGB",
        dataset_names=[meta.name], dataset_metas=[meta.name], dataset_prompts=["name"],
        embed_dim_language=spec["lang_dim"], text_feature_reduce_before_fusion=True, text_feature_batch_repeat=True,
        expression_cumulative_gt_class=True, test_nms_thresh=spec["test_nms_thresh"],
        test_score_thresh=spec["test_score_thresh"])
    model.set_model_language(ref_model.FakeLanguageModel(spec["lang_dim"]))
    ref_model.randomize_degenerate_parameters(model)
    model.eval()
    return model, names


def _spy_topk(spec):
    gathered, orig = [], torch.gather

    def spy(inp, dim, index, *a, **k):
        if index.dim() == 3 and index.shape[-1] == 4 and index.shape[1] == spec["num_queries"]:
            gathered.append(index[..., 0].clone())
        return orig(inp, dim, index, *a, **k)

    return gathered, orig, spy


def main_mini():
    """model_mini_la.npz: MINI_L_A with test_mask_on and semantic_on, one 48 x 64 image shown at 96 x 128."""
    spec = configs.MINI_L_A
    model, names = build_reference_la(spec, test_mask_on=True, semantic_on=True)
    synth.fill_state_dict(model)
    cap = {}
    model.backbone.register_forward_hook(lambda m, i, o: cap.__setitem__("backbone", o))
    model.transformer.register_forward_hook(lambda m, i, o: cap.__setitem__("transformer", o))
    orig_mf = model.maskdino_mask_features

    def mf_spy(*a, **k):
        cap["mask_features"] = orig_mf(*a, **k)
        return cap["mask_features"]

    model.maskdino_mask_features = mf_spy
    import ape.modeling.ape_deta.deformable_detr_segm as segm  # the module object refshim loaded

    orig_interp = torch.nn.functional.interpolate

    def interp_spy(x, *a, **k):  # first 4-D call with num_queries channels is `mask_pred`
        if x.dim() == 4 and x.shape[1] == spec["num_queries"] and "pred_masks" not in cap:
            cap["pred_masks"] = x.clone()
        return orig_interp(x, *a, **k)

    gathered, orig_gather, spy = _spy_topk(spec)
    segm.F.interpolate = interp_spy
    torch.gather = spy
    try:
        with torch.no_grad():
            out = model([{"image": synth.image(48, 64, seed=0), "height": 96, "width": 128}])
    finally:
        segm.F.interpolate = orig_interp
        torch.gather = orig_gather
    (inter_states, init_reference, inter_references, enc_cls, enc_coord_unact, anchors, memory) = cap["transformer"]
    assert len(gathered) == 1
    inst = out[0]["instances"]
    rec = {f"backbone.{k}": v[:, ::4] for k, v in cap["backbone"].items()}
    rec.update(memory=memory[:, ::4], inter_states=inter_states, init_reference=init_reference,
               inter_references=inter_references, enc_outputs_class=enc_cls, topk_proposals=gathered[0],
               mask_features=cap["mask_features"][:, ::8], pred_masks=cap["pred_masks"], sem_seg=out[0]["sem_seg"],
               **{"det0.boxes": inst.pred_boxes.tensor, "det0.scores": inst.scores, "det0.classes": inst.pred_classes,
                  "det0.masks_packed": torch.from_numpy(np.packbits(inst.pred_masks.numpy().astype(np.uint8), axis=-1)),
                  "det0.masks_shape": torch.tensor(inst.pred_masks.shape)})
    np.savez_compressed(os.path.join(HERE, "model_mini_la.npz"), **{k: v.detach().cpu().numpy() for k, v in rec.items()})
    print("mini_la", {k: tuple(v.shape) for k, v in rec.items()})


def main_la():
    """model_la_1024.npz: APE-L_A, one 1024 x 768 image padded to 1024^2, 1203-name vocabulary, "name" prompt, boxes only,
    fp32 on the CPU (pytorch_attn=True / SDPA-math).  Per-token tensors are stored sub-sampled; indices, boxes and detections
    in full (the layout of model_lb_1024.npz)."""
    spec = configs.APE_L_A
    n_text = 1203
    model, names = build_reference_la(spec, num_text=n_text)
    synth.fill_state_dict(model)
    synth.suppress_invalid_anchor_logits(model)
    cap = {}
    model.backbone.register_forward_hook(lambda m, i, o: cap.__setitem__("backbone", o))
    model.transformer.register_forward_hook(lambda m, i, o: cap.__setitem__("transformer", o))
    for i, layer in enumerate(model.transformer.encoder.layers):
        layer.register_forward_hook(lambda m, inp, o, i=i: cap.__setitem__(f"enc{i}", o))
    orig_inf = model.inference

    def inf_spy(box_cls, box_pred, image_sizes, *a, **k):
        cap["box_cls"], cap["box_pred"] = box_cls.clone(), box_pred.clone()
        return orig_inf(box_cls, box_pred, image_sizes, *a, **k)

    model.inference = inf_spy
    gathered, orig_gather, spy = _spy_topk(spec)
    torch.gather = spy
    t0 = time.time()
    try:
        with torch.no_grad():
            out = model([{"image": synth.image(1024, 768, seed=0), "height": 1024, "width": 768}])
    finally:
        torch.gather = orig_gather
    print(f"reference APE-L_A forward on CPU: {time.time() - t0:.1f} s")
    (inter_states, init_reference, inter_references, enc_cls, enc_coord_unact, anchors, memory) = cap["transformer"]
    inst = out[0]["instances"]
    rec = {f"backbone.{k}": v[:, ::16, ::8, ::8] for k, v in cap["backbone"].items()}
    for i in range(spec["enc_layers"]):
        rec[f"enc{i}"] = cap[f"enc{i}"][:, ::2048, ::4]
    box_cls, box_pred = cap["box_cls"], cap["box_pred"]
    rec.update(memory=memory[:, ::512, ::4], enc_outputs_class=enc_cls[:, ::16], topk_proposals=gathered[0],
               init_reference=init_reference, inter_references=inter_references, pred_logits=box_cls[:, :, ::32],
               pred_boxes=box_pred, **{"det0.boxes": inst.pred_boxes.tensor, "det0.scores": inst.scores,
                                       "det0.classes": inst.pred_classes})
    np.savez_compressed(os.path.join(HERE, "model_la_1024.npz"), **{k: v.detach().cpu().numpy() for k, v in rec.items()})
    print("la", {k: tuple(v.shape) for k, v in rec.items()})


def main_cpu():
    from test_integration_cpu import _run_config

    out = {}
    for name in ("MINI_L_A", "APE_L_A"):
        ref, _ = build_reference_la(getattr(configs, name), num_text=16)
        out[name] = {k: list(v.shape) for k, v in ref.state_dict().items()}
    json.dump(out, gzip.open(os.path.join(HERE, "state_dict_shapes_la.json.gz"), "wt"), indent=0, sort_keys=True)
    env = {}
    for rel in LA_CONFIGS:
        _run_config(open(os.path.join(REF, rel)).read(), env)
    la = env["model"]
    assert la["_target_"] == "SomeThing" and la["model_vision"]["_target_"] == "DeformableDETRSegm"
    json.dump({"APE_L_A": la}, open(os.path.join(HERE, "ref_config_tree_la.json"), "w"), indent=0, sort_keys=True)


def reference_eva01_text():
    """eva01_clip/eva_model.py, executed unmodified.  The eva01_clip package __init__ is bypassed (it builds the whole
    EVA-CLIP with its vision tower); the timm helpers vit_model.py imports are shimmed, `clip` (OpenAI's tokenizer, which
    only the wrapper imports) is not needed: the prompts are pre-tokenised."""
    refshim.install()
    tl = sys.modules["timm.models.layers"]
    tl.trunc_normal_ = getattr(tl, "trunc_normal_", torch.nn.init.trunc_normal_)
    tl.to_2tuple = getattr(tl, "to_2tuple", lambda x: tuple(x) if isinstance(x, (tuple, list)) else (x, x))
    tl.drop_path = getattr(tl, "drop_path", lambda x, drop_prob=0.0, training=False: x)
    m = types.ModuleType("ape.modeling.text.eva01_clip")
    m.__path__ = [os.path.join(REF, "ape/modeling/text/eva01_clip")]
    sys.modules["ape.modeling.text.eva01_clip"] = m
    return importlib.import_module("ape.modeling.text.eva01_clip.eva_model")


def text_tokens():
    """Prompts of 2 to 77 tokens: random ids below the end-of-text id 49407 (the highest, which argmax picks), zero padding."""
    g = torch.Generator().manual_seed(4)
    lens = [2, 5, 9, 17, 40, 76, 77]
    t = torch.zeros(len(lens), TEXT_CFG["context_length"], dtype=torch.long)
    for i, n in enumerate(lens):
        t[i, : n - 1] = torch.randint(1, TEXT_CFG["vocab_size"] - 1, (n - 1,), generator=g)
        t[i, n - 1] = TEXT_CFG["vocab_size"] - 1
    return t


def main_text():
    mod = reference_eva01_text()
    torch.manual_seed(0)
    ref = mod.TextTransformer(**TEXT_CFG).eval()
    synth.fill_state_dict(ref)
    t = text_tokens()
    with torch.no_grad():
        eot = ref(t)
        x = ref.token_embedding(t) + ref.positional_embedding
        x = ref.transformer(x.permute(1, 0, 2), attn_mask=ref.attn_mask).permute(1, 0, 2)
        xx = ref.ln_final(x) @ ref.text_projection
    keys = "\n".join(sorted("net.text." + k for k in ref.state_dict()))  # the wrapper's names: self.net = EVA_CLIP, visual deleted
    np.savez_compressed(os.path.join(HERE, "text_eva01.npz"), tokens=t.numpy(), eot=eot.numpy(), all=xx[:, ::7].numpy(),
                        keys=np.frombuffer(keys.encode(), dtype=np.uint8))
    print("eva01 text golden", tuple(eot.shape), tuple(xx.shape), float(eot.abs().mean()))


if __name__ == "__main__":
    what = sys.argv[1] if len(sys.argv) > 1 else "all"
    if what in ("cpu", "all"):
        main_cpu()
    if what in ("text", "all"):
        main_text()
    if what in ("mini", "all"):
        main_mini()
    if what in ("la", "all"):
        main_la()
