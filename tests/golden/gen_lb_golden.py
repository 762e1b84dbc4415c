"""Generates the golden data of APE-L_B / APE-L_C (vit_eva02.py ViT-L sub-LN backbone, no neck, proposal_ambiguous = 0) by
running the REFERENCE's own model files on the CPU (unmodified, under oracle/refshim.py's import shims), with name-derived
synthetic weights (oracle/synth.py).  Build container only; run from the repository root:

  python tests/golden/gen_lb_golden.py [mini|lb|cpu]

  model_mini_lb.npz          MINI_EVA02L, one 48 x 64 image, test_mask_on + semantic_on    (tests/test_ape_l_b_gpu.py)
  model_lb_1024.npz          APE-L_B, one 1024 x 768 image padded to 1024^2, 1203 names   (tests/test_ape_l_b_gpu.py)
  state_dict_shapes_lb.json.gz   parameter names and shapes for MINI_EVA02L and APE_L_B    (tests/test_ape_l_b_cpu.py)
  ref_config_tree_lb.json    the LazyConfig model tree of APE-L_B and the APE-Ti backbone node (tests/test_ape_l_b_cpu.py)"""
import gzip
import json
import os
import sys
import time
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
LB_CONFIGS = ("configs/common/backbone/vitl_eva02.py",
              "configs/COCO_InstanceSegmentation/ape_deta/models/ape_deta_r50.py",
              "configs/COCO_InstanceSegmentation/ape_deta/ape_deta_vitl_eva02_lsj1024_cp_12ep.py",
              "configs/LVIS_InstanceSegmentation/ape_deta/ape_deta_vitl_eva02_lsj1024_cp_24ep.py",
              "configs/LVISCOCOCOCOSTUFF_O365_OID_VGR_REFCOCO/ape_deta/ape_deta_vitl_eva02_lsj1024_cp_720k.py",
              "configs/LVISCOCOCOCOSTUFF_O365_OID_VGR_REFCOCO/ape_deta/ape_deta_vitl_eva02_vlf_lsj1024_cp_720k.py",
              "configs/LVISCOCOCOCOSTUFF_O365_OID_VGR_REFCOCO/ape_deta/ape_deta_vitl_eva02_vlf_lsj1024_cp_1080k.py")


def build_reference_lb(spec, num_text=None, test_mask_on=False, semantic_on=False):
    """The reference model of an APE-L_B-structured spec: oracle/ref_model.py's model (same transformer, heads and
    proposal_ambiguous from the spec) with vit_eva02.ViT(subln=True, naiveswiglu=True) under vit_eva02.SimpleFeaturePyramid
    as its backbone and no neck (…_lsj1024_cp_720k.py:53)."""
    assert spec["backbone"]["variant"] == "eva02_subln" and spec["neck"] is None
    model, names = ref_model.build_reference_model(spec, num_text=num_text, test_mask_on=test_mask_on, semantic_on=semantic_on)
    vit_mod = refshim.load("ape.modeling.backbone.vit_eva02")
    b = spec["backbone"]
    net = vit_mod.ViT(
        img_size=b["img_size"], patch_size=b["patch_size"], embed_dim=b["embed_dim"], depth=b["depth"],
        num_heads=b["num_heads"], drop_path_rate=0.0, window_size=b["window_size"], mlp_ratio=b["mlp_ratio"],
        qkv_bias=True, norm_layer=partial(nn.LayerNorm, eps=1e-6), window_block_indexes=b["window_block_indexes"],
        residual_block_indexes=[], use_rel_pos=True, out_feature="last_feat", use_act_checkpoint=False, xattn=False,
        subln=True, swiglu=False, naiveswiglu=True, pt_hw_seq_len=b["pt_hw_seq_len"], pretrain_img_size=b["pretrain_img_size"])
    model.backbone = vit_mod.SimpleFeaturePyramid(
        net=net, in_feature="last_feat", out_channels=b["out_channels"], scale_factors=b["scale_factors"],
        top_block=refshim.LastLevelMaxPool(), norm="LN", square_pad=b["square_pad"])
    model.neck = None
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
    """model_mini_lb.npz: MINI_EVA02L with test_mask_on and semantic_on, one 48 x 64 image shown at 96 x 128."""
    spec = configs.MINI_EVA02L
    model, names = build_reference_lb(spec, test_mask_on=True, semantic_on=True)
    synth.fill_state_dict(model)
    cap = {}
    model.backbone.register_forward_hook(lambda m, i, o: cap.__setitem__("backbone", o))
    model.transformer.register_forward_hook(lambda m, i, o: cap.__setitem__("transformer", o))
    orig_mf = model.maskdino_mask_features

    def mf_spy(*a, **k):
        cap["mask_features"] = orig_mf(*a, **k)
        return cap["mask_features"]

    model.maskdino_mask_features = mf_spy
    import ape.modeling.ape_deta.deformable_detr_segm_vl as segm  # the module object refshim loaded

    orig_interp = torch.nn.functional.interpolate

    def interp_spy(x, *a, **k):  # first 4-D call with num_queries channels is `mask_pred` (:563-566)
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
    (inter_states, init_reference, inter_references, enc_cls, enc_coord_unact, anchors, memory, feats_l) = cap["transformer"]
    assert len(gathered) == 1
    inst = out[0]["instances"]
    rec = {f"backbone.{k}": v[:, ::4] for k, v in cap["backbone"].items()}
    rec.update(memory=memory[:, ::4], inter_states=inter_states, init_reference=init_reference,
               inter_references=inter_references, enc_outputs_class=enc_cls, topk_proposals=gathered[0],
               mask_features=cap["mask_features"][:, ::8], pred_masks=cap["pred_masks"], sem_seg=out[0]["sem_seg"],
               **{"det0.boxes": inst.pred_boxes.tensor, "det0.scores": inst.scores, "det0.classes": inst.pred_classes,
                  "det0.masks_packed": torch.from_numpy(np.packbits(inst.pred_masks.numpy().astype(np.uint8), axis=-1)),
                  "det0.masks_shape": torch.tensor(inst.pred_masks.shape)})
    np.savez_compressed(os.path.join(HERE, "model_mini_lb.npz"), **{k: v.detach().cpu().numpy() for k, v in rec.items()})
    print("mini_lb", {k: tuple(v.shape) for k, v in rec.items()})


def main_lb():
    """model_lb_1024.npz: APE-L_B, one 1024 x 768 image padded to 1024^2, 1203-name vocabulary, "name" prompt, boxes only,
    fp32 on the CPU (pytorch_attn=True / SDPA-math).  Per-token tensors are stored sub-sampled; indices, boxes and detections
    in full (the layout of model_ld_1024.npz)."""
    spec = configs.APE_L_B
    n_text = 1203
    model, names = build_reference_lb(spec, num_text=n_text)
    synth.fill_state_dict(model)
    synth.suppress_invalid_anchor_logits(model)
    cap = {}
    model.backbone.register_forward_hook(lambda m, i, o: cap.__setitem__("backbone", o))
    model.transformer.register_forward_hook(lambda m, i, o: cap.__setitem__("transformer", o))
    for i, layer in enumerate(model.transformer.encoder.vl_layers):
        layer.register_forward_hook(lambda m, inp, o, i=i: cap.__setitem__(f"vlf{i}", o))
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
    print(f"reference APE-L_B forward on CPU: {time.time() - t0:.1f} s")
    (inter_states, init_reference, inter_references, enc_cls, enc_coord_unact, anchors, memory, feats_l) = cap["transformer"]
    inst = out[0]["instances"]
    rec = {f"backbone.{k}": v[:, ::16, ::8, ::8] for k, v in cap["backbone"].items()}
    for i in range(spec["enc_layers"]):
        rec[f"vlf{i}.v"] = cap[f"vlf{i}"][0][:, ::2048, ::4]
        rec[f"vlf{i}.l"] = cap[f"vlf{i}"][1][:, ::2048, ::4]
        rec[f"enc{i}"] = cap[f"enc{i}"][:, ::2048, ::4]
    box_cls, box_pred = cap["box_cls"], cap["box_pred"]
    rec.update(memory=memory[:, ::512, ::4], enc_outputs_class=enc_cls[:, ::16], topk_proposals=gathered[0],
               init_reference=init_reference, inter_references=inter_references, pred_logits=box_cls[:, :, ::32],
               pred_boxes=box_pred, **{"det0.boxes": inst.pred_boxes.tensor, "det0.scores": inst.scores,
                                       "det0.classes": inst.pred_classes})
    np.savez_compressed(os.path.join(HERE, "model_lb_1024.npz"), **{k: v.detach().cpu().numpy() for k, v in rec.items()})
    print("lb", {k: tuple(v.shape) for k, v in rec.items()})


def main_cpu():
    from test_integration_cpu import _run_config

    out = {}
    for name in ("MINI_EVA02L", "APE_L_B"):
        ref, _ = build_reference_lb(getattr(configs, name), num_text=16)
        out[name] = {k: list(v.shape) for k, v in ref.state_dict().items()}
    json.dump(out, gzip.open(os.path.join(HERE, "state_dict_shapes_lb.json.gz"), "wt"), indent=0, sort_keys=True)
    env = {}
    for rel in LB_CONFIGS:
        _run_config(open(os.path.join(REF, rel)).read(), env)
    lb = env["model"]
    assert lb["_target_"] == "SomeThing" and lb["model_vision"]["_target_"] == "DeformableDETRSegmVL"
    env = {}
    _run_config(open(os.path.join(REF, "configs/common/backbone/vitt_eva02.py")).read(), env)
    json.dump({"APE_L_B": lb, "APE_Ti_backbone": env["backbone"]}, open(os.path.join(HERE, "ref_config_tree_lb.json"), "w"),
              indent=0, sort_keys=True)


if __name__ == "__main__":
    what = sys.argv[1] if len(sys.argv) > 1 else "all"
    if what in ("cpu", "all"):
        main_cpu()
    if what in ("mini", "all"):
        main_mini()
    if what in ("lb", "all"):
        main_lb()
