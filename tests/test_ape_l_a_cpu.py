"""CPU: APE-L_A drop-in surface and the EVA01-CLIP text tower.

* The engine's `state_dict` for APE_L_A and MINI_L_A equals the reference non-VL model's (deformable_detr_segm.py over
  deformable_transformer.py) name for name and shape: no `vl_layers`, no name-prompt fusion feature
  (tests/golden/state_dict_shapes_la.json.gz, tests/golden/gen_la_golden.py cpu).
* Every `_target_` override INTEGRATION.md gives for APE-L_A names a LazyCall node of the L_A config tree
  (tests/golden/ref_config_tree_la.json) and the engine class accepts every keyword the node passes; the EVA01CLIP override
  names the config's `model_language` node.
* The non-VL classes keep the reference's forward signatures; the VL classes are unchanged.
* EVA01CLIP: parameter names of the reference's text half, `cache_dir` loading of an EVA-CLIP checkpoint, and the fp32
  literal path against tests/golden/text_eva01.npz (the reference's eva01_clip TextTransformer at EVA_CLIP_g_14 size)."""
import gzip
import inspect
import json
import os
import re

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT, load_golden
from oracle import synth
from ape_b200 import configs
from test_ape_l_b_cpu import _blocks, _check


@pytest.mark.parametrize("spec_name", ["MINI_L_A", "APE_L_A"])
def test_la_state_dict_keys_and_shapes_equal_reference(spec_name):
    from ape_b200.modeling import DeformableDETRSegm, DeformableDetrTransformer, build_model

    a = {k: tuple(v) for k, v in json.load(gzip.open(os.path.join(GOLDEN, "state_dict_shapes_la.json.gz"), "rt"))[spec_name].items()}
    eng = build_model(getattr(configs, spec_name), num_text=16)
    b = {k: tuple(v.shape) for k, v in eng.state_dict().items()}
    assert sorted(a) == sorted(b), (sorted(set(a) - set(b))[:5], sorted(set(b) - set(a))[:5])
    assert a == b
    assert type(eng) is DeformableDETRSegm and type(eng.transformer) is DeformableDetrTransformer
    assert not any("vl_layers" in k or "name_prompt_fusion" in k for k in b)
    assert not hasattr(eng.transformer.encoder, "vl_layers")


def test_vl_specs_still_build_the_vl_classes():
    from ape_b200.modeling import DeformableDETRSegmVL, DeformableDetrTransformerEncoderVL, build_model

    eng = build_model(configs.MINI_EVA02L, num_text=4)
    assert type(eng) is DeformableDETRSegmVL and type(eng.transformer.encoder) is DeformableDetrTransformerEncoderVL
    assert any(k.startswith("transformer.encoder.vl_layers.") for k in eng.state_dict())


def test_non_vl_forward_signatures_follow_the_reference():
    from ape_b200.modeling import transformer as t

    enc = inspect.signature(t.DeformableDetrTransformerEncoder.forward).parameters
    assert "query_l" not in enc and list(enc)[1:4] == ["query", "key", "value"]
    assert "look_forward_twice" not in inspect.signature(t.DeformableDetrTransformerDecoder.__init__).parameters
    tr = inspect.signature(t.DeformableDetrTransformer.forward).parameters
    assert list(tr)[1:5] == ["multi_level_feats", "multi_level_masks", "multi_level_pos_embeds", "query_embed"]
    assert "query_l" not in tr and "multi_level_masks_prompt" not in tr
    g = inspect.signature(t.DeformableDetrTransformer.gen_encoder_output_proposals).parameters
    assert list(g) == ["self", "memory", "memory_padding_mask", "spatial_shapes"]
    vl = inspect.signature(t.DeformableDetrTransformerEncoderVL.forward).parameters
    assert "query_l" in vl  # the VL classes keep theirs


def test_la_overrides_name_real_config_nodes():
    import ape_b200  # noqa: F401

    tree = json.load(open(os.path.join(GOLDEN, "ref_config_tree_la.json")))["APE_L_A"]
    text = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    pat = r"(model(?:\.\w+)+)\._target_=(ape_b200(?:\.\w+)+)"
    la = [b.replace("$E.", "ape_b200.modeling.") for b in _blocks(text) if "LVISCOCOCOCOSTUFF_O365_OID_VG/ape_deta/ape_deta_vitl_eva02_lsj1024_cp_720k.py" in b]
    assert len(la) == 1
    overrides = re.findall(pat, la[0])
    paths = {p for p, _ in overrides}
    for p in ("model.model_vision", "model.model_vision.backbone", "model.model_vision.transformer",
              "model.model_vision.transformer.encoder", "model.model_vision.transformer.decoder", "model.model_language"):
        assert p in paths, f"INTEGRATION.md's APE-L_A command does not override {p}"
    assert not any(".neck" in p for p in paths) and tree["model_vision"]["neck"] == "<value>"
    for path, target in overrides:
        _check(tree, path.split(".")[1:], target)
    # the language model line applies to L_B / L_C too: their config tree has the same node
    lb = json.load(open(os.path.join(GOLDEN, "ref_config_tree_lb.json")))["APE_L_B"]
    assert lb["model_language"]["_target_"] == tree["model_language"]["_target_"] == "EVA01CLIP"
    assert "E=ape_b200.modeling" in text


# -- EVA01-CLIP ----------------------------------------------------------------------------------------------------------
def test_eva01_parameter_names_equal_the_reference():
    from ape_b200.modeling import EVA01CLIP

    want = set(bytes(load_golden("text_eva01.npz")["keys"].numpy()).decode().split("\n"))
    for name in ("EVA_CLIP_g_14", "EVA_CLIP_g_14_X"):
        with torch.device("meta"):
            clip = EVA01CLIP(name, cache_dir=None)
        sd = clip.state_dict()
        assert set(sd) == want
        assert "net.text.logit_scale" in sd and "net.logit_scale" not in sd
        assert sd["net.text.text_projection"].shape == (768, 1024)
        assert sd["net.text.transformer.resblocks.11.attn.in_proj_weight"].shape == (3 * 768, 768)
    sig = inspect.signature(EVA01CLIP.__init__).parameters
    assert list(sig)[1:5] == ["clip_model", "cache_dir", "dtype", "max_batch_size"] and sig["dtype"].default == "float32"
    assert "tokenizer" in sig


def _small_eva01(**kw):
    from ape_b200.modeling import EVA01CLIP

    return EVA01CLIP("EVA_CLIP_g_14", text_cfg=dict(context_length=77, vocab_size=1000, width=128, heads=2, layers=2),
                     embed_dim=64, **kw)


def test_eva01_cache_dir_loading(tmp_path):
    src = _small_eva01(cache_dir=None)
    synth.fill_state_dict(src)
    text_sd = {"text." + k: v.clone() for k, v in src.net.text.state_dict().items()}
    visual = {"visual.blocks.0.attn.qkv.weight": torch.randn(12, 4), "visual.cls_token": torch.randn(1, 1, 4)}
    # EVA-CLIP layout: {"module": ...} with DataParallel's "module." prefix, vision tower included
    path = tmp_path / "eva_clip_psz14.pt"
    torch.save({"module": {"module." + k: v for k, v in {**visual, **text_sd}.items()}, "epoch": 3}, path)
    clip = _small_eva01(cache_dir=str(path))
    for k, v in src.net.text.state_dict().items():
        assert torch.equal(clip.net.text.state_dict()[k], v), k
    assert not any(k.startswith("net.visual") for k in clip.state_dict())
    # a bare dict without prefix and a "state_dict"-wrapped one load the same
    for i, obj in enumerate(({**visual, **text_sd}, {"state_dict": text_sd})):
        p = tmp_path / f"ckpt{i}.pt"
        torch.save(obj, p)
        assert torch.equal(_small_eva01(cache_dir=str(p)).net.text.positional_embedding, src.net.text.positional_embedding)
    # a missing text entry is an error
    bad = dict(text_sd)
    del bad["text.transformer.resblocks.1.mlp.c_fc.weight"]
    p = tmp_path / "missing.pt"
    torch.save({"model": bad}, p)
    with pytest.raises(RuntimeError, match="c_fc"):
        _small_eva01(cache_dir=str(p))
    with pytest.raises(FileNotFoundError):
        _small_eva01(cache_dir=str(tmp_path / "absent.pt"))


def test_eva01_fp32_literal_path_matches_reference_golden():
    from ape_b200.modeling import EVA01CLIP

    g = load_golden("text_eva01.npz")
    clip = EVA01CLIP("EVA_CLIP_g_14_X", cache_dir=None)
    synth.fill_state_dict(clip.net.text)
    assert clip.net.text.engine_dtype is None  # dtype "float32": the literal path, as the reference runs it
    out = clip.forward_text(g["tokens"])
    assert set(out) == {"end_token_idx", "attention_mask", "last_hidden_state", "last_hidden_state_eot"}
    torch.testing.assert_close(out["last_hidden_state_eot"], g["eot"], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(out["last_hidden_state"][:, ::7], g["all"], rtol=1e-4, atol=1e-5)
    ends = out["end_token_idx"].tolist()
    assert ends == [1, 4, 8, 16, 39, 75, 76] and out["attention_mask"].sum(1).tolist() == [e + 1 for e in ends]


def test_eva01_dtype_selects_the_path():
    for dt, want in (("float32", None), ("float16", torch.float16), ("bfloat16", torch.bfloat16)):
        assert _small_eva01(cache_dir=None, dtype=dt).net.text.engine_dtype == want
    clip = _small_eva01(cache_dir=None, tokenizer=lambda texts: torch.stack(
        [torch.cat([torch.arange(1, 1 + len(t.split())), torch.tensor([999]), torch.zeros(76 - len(t.split()), dtype=torch.long)])
         for t in texts]))
    out = clip.forward_text(["a dog", "the red apple"], cache=True)
    assert out["last_hidden_state_eot"].shape == (2, 64) and out["end_token_idx"].tolist() == [2, 3]
    assert clip.forward_text(["a dog", "the red apple"], cache=True) is out
