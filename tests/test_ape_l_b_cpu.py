"""CPU: APE-L_B / APE-L_C drop-in surface.

* The engine's `state_dict` for APE_L_B and MINI_EVA02L equals the reference's name for name and shape (vit_eva02.py sub-LN
  blocks without inner_attn_ln, RoPE buffers under every attention block, no neck), recorded from the reference model in
  tests/golden/state_dict_shapes_lb.json.gz (tests/golden/gen_lb_golden.py cpu).
* Every `_target_` override INTEGRATION.md gives for the APE-L_B / L_C configs names a LazyCall node of APE-L_B's config tree,
  and every backbone override of the APE-Ti command names a node of `vitt_eva02.py`'s tree (tests/golden/ref_config_tree_lb.json);
  the engine class accepts every keyword the node passes.
* `ape_b200.modeling.vit_eva02.ViT` reads the switches as vit_eva02.py does; `ape_b200.modeling.ViT` keeps vit_eva_clip.py's."""
import gzip
import importlib
import inspect
import json
import os
import re

import pytest
import torch

from ape_b200 import configs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.mark.parametrize("spec_name", ["MINI_EVA02L", "APE_L_B"])
def test_lb_state_dict_keys_and_shapes_equal_reference(spec_name):
    from ape_b200.modeling import build_model

    a = {k: tuple(v) for k, v in json.load(gzip.open(os.path.join(GOLDEN, "state_dict_shapes_lb.json.gz"), "rt"))[spec_name].items()}
    eng = build_model(getattr(configs, spec_name), num_text=16)
    b = {k: tuple(v.shape) for k, v in eng.state_dict().items()}
    assert sorted(a) == sorted(b), (sorted(set(a) - set(b))[:5], sorted(set(b) - set(a))[:5])
    assert a == b
    assert eng.neck is None and eng.transformer.proposal_ambiguous == 0
    assert not any("inner_attn_ln" in k or k.startswith("neck.") for k in b)
    assert all(f"backbone.net.blocks.{i}.attn.rope.freqs_cos" in b for i in range(len(eng.backbone.net.blocks)))


def _blocks(text):
    """Contents of the fenced code blocks of a markdown text."""
    blocks, cur = [], None
    for line in text.splitlines():
        if line.startswith("```"):
            if cur is None:
                cur = []
            else:
                blocks.append("\n".join(cur))
                cur = None
        elif cur is not None:
            cur.append(line)
    return blocks


def _check(tree, path, target):
    node = tree
    for k in path:
        assert isinstance(node, dict) and k in node, f"override {'.'.join(path)}: `{k}` is not a key of the reference config"
        node = node[k]
    assert isinstance(node, dict) and "_target_" in node, f"{'.'.join(path)} is not a LazyCall node in the reference config"
    mod, cls = target.rsplit(".", 1)
    engine_cls = getattr(importlib.import_module(mod), cls)
    assert engine_cls.__name__ == node["_target_"], f"{'.'.join(path)}: reference builds {node['_target_']}, override names {cls}"
    params = inspect.signature(engine_cls.__init__).parameters
    accepts_kwargs = any(p.kind == p.VAR_KEYWORD for p in params.values())
    for kw in node:
        if kw != "_target_":
            assert accepts_kwargs or kw in params, f"{target} does not accept the config keyword `{kw}` of {'.'.join(path)}"


def test_lb_and_ti_overrides_name_real_config_nodes():
    import ape_b200  # noqa: F401

    trees = json.load(open(os.path.join(GOLDEN, "ref_config_tree_lb.json")))
    text = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    pat = r"(model(?:\.\w+)+)\._target_=(ape_b200(?:\.\w+)+)"
    lb = [b for b in _blocks(text) if "ape_deta_vitl_eva02_vlf_lsj1024_cp_1080k.py" in b]
    ti = [b for b in _blocks(text) if "ape_deta_vitt_eva02" in b]
    assert len(lb) == 1 and len(ti) == 1
    lb_overrides = re.findall(pat, lb[0])
    assert len(lb_overrides) >= 8 and not any(".neck" in p for p, _ in lb_overrides)  # the configs set neck = None
    assert trees["APE_L_B"]["model_vision"]["neck"] == "<value>"
    for path, target in lb_overrides:
        _check(trees["APE_L_B"], path.split(".")[1:], target)
    ti_overrides = re.findall(pat, ti[0])
    assert any(t.endswith("vit_eva02.ViT") for _, t in ti_overrides)
    for path, target in ti_overrides:
        assert path.startswith("model.model_vision.backbone")
        _check({"backbone": trees["APE_Ti_backbone"]}, path.split(".")[2:], target)


def test_vit_eva02_class_reads_switches_like_vit_eva02():
    from ape_b200.modeling import ViT
    from ape_b200.modeling import vit_eva02

    sig = inspect.signature(vit_eva02.ViT.__init__).parameters
    for k, v in dict(rope=True, intp_freq=True, xattn=True, qkv_bias=True, pretrain_img_size=224, mlp_ratio=4 * 2 / 3,
                     subln=False, swiglu=False, naiveswiglu=False).items():
        assert sig[k].default == v, k
    assert "act_layer" in sig
    assert inspect.signature(ViT.__init__).parameters["rope"].default is False  # the vit_eva_clip.py defaults stay
    kw = dict(img_size=64, patch_size=16, embed_dim=64, depth=2, num_heads=2, window_size=2, window_block_indexes=[0])
    lb = vit_eva02.ViT(subln=True, naiveswiglu=True, **kw)
    ld = ViT(subln=True, naiveswiglu=True, rope=True, intp_freq=True, qkv_bias=True, **kw)
    ti = vit_eva02.ViT(swiglu=True, **kw)
    assert lb._flavour == "eva02_subln" and ld._flavour == "eva_clip" and ti._flavour == "eva02_swiglu"
    names = set(lb.state_dict())
    assert "blocks.0.attn.q_proj.weight" in names and "blocks.0.mlp.ffn_ln.weight" in names
    assert not any("inner_attn_ln" in k for k in names) and any("inner_attn_ln" in k for k in ld.state_dict())
    assert "blocks.0.attn.qkv.weight" in ti.state_dict() and "blocks.0.mlp.w12.weight" in ti.state_dict()
    with pytest.raises(NotImplementedError):  # vit_eva02.py's default (neither MLP switch) is not an APE configuration
        vit_eva02.ViT(**kw)


def test_lb_fp32_forward_is_the_module_forward():
    """The fp32 path of the new flavour is the literal block forward: one block against its hand-written composition."""
    from ape_b200.modeling import vit_eva02
    from ape_b200.synthetic import fill_state_dict
    import torch.nn.functional as F

    vit = vit_eva02.ViT(img_size=64, patch_size=16, embed_dim=64, depth=1, num_heads=2, window_size=0, subln=True,
                        naiveswiglu=True).eval()
    fill_state_dict(vit)
    blk = vit.blocks[0]
    x = torch.randn(1, 4, 4, 64, generator=torch.Generator().manual_seed(0))
    with torch.no_grad():
        got = blk(x)
        a, m = blk.attn, blk.mlp
        h = blk.norm1(x).reshape(1, 16, 64)
        q = F.linear(h, a.q_proj.weight, a.q_bias).view(1, 16, 2, 32).transpose(1, 2)
        k = F.linear(h, a.k_proj.weight).view(1, 16, 2, 32).transpose(1, 2)
        v = F.linear(h, a.v_proj.weight, a.v_bias).view(1, 16, 2, 32).transpose(1, 2)
        o = F.scaled_dot_product_attention(a.rope(q), a.rope(k), v).transpose(1, 2).reshape(1, 16, 64)
        y = x + a.proj(o).view(1, 4, 4, 64)
        z = blk.norm2(y)
        want = y + m.w3(m.ffn_ln(F.silu(m.w1(z)) * m.w2(z)))
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5)
