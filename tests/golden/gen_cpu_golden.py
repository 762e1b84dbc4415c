"""Regenerates the golden data of the CPU tests that compare with the reference's own code (needs the reference checkout
and oracle/refshim.py's import shims; run from the repository root):
  state_dict_shapes.json.gz  parameter names and shapes of the reference model per spec   (tests/test_state_dict_cpu.py)
  panoptic_ref.npz         DeformableDETRSegmVL._postprocess_panoptic on seeded inputs   (tests/test_panoptic_cpu.py)
  vlf_block_ref.npz        the reference BiAttentionBlock on seeded weights / inputs     (tests/test_vlf_cpu.py)
  ref_model_config_tree.json  the LazyConfig model tree of the reference's configs       (tests/test_integration_cpu.py)"""
import gzip
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))


def state_dicts():
    from ape_b200 import configs
    from oracle import ref_model

    out = {}
    for name in ("MINI", "APE_TI", "APE_L_D"):
        ref, _ = ref_model.build_reference_model(getattr(configs, name), num_text=16)
        out[name] = {k: list(v.shape) for k, v in ref.state_dict().items()}
    json.dump(out, gzip.open(os.path.join(HERE, "state_dict_shapes.json.gz"), "wt"), indent=0, sort_keys=True)


def panoptic():
    from oracle import refshim
    from test_panoptic_cpu import CASES, make_case

    refshim.install()
    segm = refshim.load("ape.modeling.ape_deta.deformable_detr_segm_vl")
    rec = {}
    for i, case in enumerate(CASES):
        mask_cls, mask_pred, image_size, out_hw, meta, cfg, images = make_case(*case)
        seg, info = segm.DeformableDETRSegmVL._postprocess_panoptic([mask_cls], [mask_pred], [{"height": out_hw[0], "width": out_hw[1]}],
                                                                   images, meta, cfg)[0]["panoptic_seg"]
        rec[f"case{i}.seg"] = seg.numpy()
        rec[f"case{i}.info"] = np.array(json.dumps(info))
    np.savez_compressed(os.path.join(HERE, "panoptic_ref.npz"), **rec)


def vlf():
    from oracle import refshim
    from test_vlf_cpu import make_block_and_inputs

    refshim.install()
    fh = refshim.load("ape.layers.fuse_helper")
    mine, v, l = make_block_and_inputs()
    ref = fh.BiAttentionBlock(v_dim=256, l_dim=128, embed_dim=512, num_heads=8, dropout=0.0, drop_path=0.0, init_values=1 / 6,
                              stable_softmax_2d=True, clamp_min_for_underflow=True, clamp_max_for_overflow=True).eval()
    ref.load_state_dict(mine.state_dict())
    with torch.no_grad():
        rv, rl = ref(v, l, attention_mask_v=None, attention_mask_l=None)
    np.savez_compressed(os.path.join(HERE, "vlf_block_ref.npz"), v=rv.numpy(), l=rl.numpy())


def config_tree():
    from test_integration_cpu import _reference_model_tree

    json.dump(_reference_model_tree(), open(os.path.join(HERE, "ref_model_config_tree.json"), "w"), indent=0, sort_keys=True)


if __name__ == "__main__":
    config_tree()
    state_dicts()
    panoptic()
    vlf()
