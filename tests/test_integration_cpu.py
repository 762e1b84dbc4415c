"""CPU: the drop-in boundary artefacts (SURVEY.md 8(b)).

* `integration/ape/_C.py` satisfies the reference's import contract (`from ape import _C`,
  ape/layers/multi_scale_deform_attn.py:415-423): with it in place the reference module file defines the real
  MultiScaleDeformableAttention class and finds `torch.ops.ape.ms_deform_attn_forward`.
* every `_target_` override INTEGRATION.md tells a user to pass names a node of the reference's own LazyConfig tree
  (configs/…/ape_deta_vitl_eva02_clip_vlf_lsj1024_cp_16x4_1080k.py and the files it builds on), parsed with `ast` (detectron2
  is not installed here), and the engine class behind it accepts every keyword the config passes to the reference class.
* `Instances.to_detectron2()` maps the fields onto detectron2's types.
* entity gates and thing-class slicing of the instance branch (deformable_detr_segm_vl.py:575-593)."""
import ast
import importlib.util
import inspect
import json
import os
import re
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
needs_ref = pytest.mark.skipif(not os.path.isdir(REF), reason="the reference checkout only exists in the build container")


def _load(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@needs_ref
def test_shipped_C_shim_satisfies_the_reference_import_contract(built):
    saved = {k: sys.modules.get(k) for k in ("ape", "ape._C", "ape.layers", "ape.layers.multi_scale_deform_attn")}
    try:
        pkg = types.ModuleType("ape")
        pkg.__path__ = [os.path.join(REF, "ape")]
        sys.modules["ape"] = pkg
        shim = _load(os.path.join(ROOT, "integration", "ape", "_C.py"), "ape._C")
        sys.modules["ape._C"] = shim
        pkg._C = shim
        ref = _load(os.path.join(REF, "ape", "layers", "multi_scale_deform_attn.py"), "ape.layers.multi_scale_deform_attn")
        assert inspect.isclass(ref.MultiScaleDeformableAttention) and issubclass(ref.MultiScaleDeformableAttention, torch.nn.Module)
        m = ref.MultiScaleDeformableAttention(embed_dim=64, num_heads=4, num_levels=2, num_points=4)  # dummy class would raise ImportError
        assert hasattr(m, "sampling_offsets")
        schema = str(torch.ops.ape.ms_deform_attn_forward.default._schema)
        assert "Tensor value, Tensor spatial_shapes, Tensor level_start_index, Tensor sampling_loc, Tensor attn_weight, int im2col_step" in schema
        with pytest.raises(RuntimeError, match="Not implemented on the CPU"):  # ms_deform_attn.h:39
            z = torch.zeros
            torch.ops.ape.ms_deform_attn_forward(z(1, 4, 4, 16), z(1, 2, dtype=torch.long), z(1, dtype=torch.long),
                                                 z(1, 3, 4, 1, 4, 2), z(1, 3, 4, 1, 4), 64)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


# ---- LazyConfig tree from the config sources -----------------------------------------------------------------------
LEAF = "<value>"


def _lazy_tree(node, env):
    """`L(Target)(kw=...)` -> {"_target_": "Target", kw: subtree | LEAF}; a bare name bound to a tree -> that tree."""
    if isinstance(node, ast.Call) and isinstance(node.func, ast.Call) and getattr(node.func.func, "id", "") == "L":
        tgt = node.func.args[0]
        name = tgt.id if isinstance(tgt, ast.Name) else ast.unparse(tgt)
        return {"_target_": name, **{kw.arg: _lazy_tree(kw.value, env) for kw in node.keywords if kw.arg}}
    if isinstance(node, ast.Name) and isinstance(env.get(node.id), dict):
        return env[node.id]
    return LEAF


def _attr_path(t):
    path = []
    while isinstance(t, ast.Attribute):
        path.append(t.attr)
        t = t.value
    return (t.id if isinstance(t, ast.Name) else None), path[::-1]


def _run_config(src, env):
    """The three statement forms the configs use to build the model tree: `name = L(..)(..)`,
    `name.a.b = <L-call | value>` and `name.a.b.update(_target_=X, ...)`."""
    for stmt in ast.parse(src).body:
        if isinstance(stmt, ast.Assign) and len(stmt.targets) == 1:
            tgt = stmt.targets[0]
            if isinstance(tgt, ast.Name):
                tree = _lazy_tree(stmt.value, env)
                if isinstance(tree, dict):
                    env[tgt.id] = tree
                continue
            root, path = _attr_path(tgt)
            node = env.get(root)
            for k in path[:-1]:
                node = node.get(k) if isinstance(node, dict) else None
            if isinstance(node, dict) and path:
                node[path[-1]] = _lazy_tree(stmt.value, env)
        elif isinstance(stmt, ast.Expr) and isinstance(stmt.value, ast.Call) and isinstance(stmt.value.func, ast.Attribute) \
                and stmt.value.func.attr == "update":
            root, path = _attr_path(stmt.value.func.value)
            node = env.get(root)
            for k in path:
                node = node.get(k) if isinstance(node, dict) else None
            if isinstance(node, dict):
                for kw in stmt.value.keywords:
                    if kw.arg == "_target_":
                        node["_target_"] = kw.value.id if isinstance(kw.value, ast.Name) else ast.unparse(kw.value)
                    elif kw.arg:
                        node[kw.arg] = _lazy_tree(kw.value, env)


def _reference_model_tree():
    env = {}
    for rel in ("configs/common/backbone/vitl_eva02_clip.py",
                "configs/COCO_InstanceSegmentation/ape_deta/models/ape_deta_r50.py",
                "configs/LVISCOCOCOCOSTUFF_O365_OID_VGR_SA1B_REFCOCO_GQA_PhraseCut_Flickr30k/ape_deta/"
                "ape_deta_vitl_eva02_clip_vlf_lsj1024_cp_16x4_1080k.py"):
        _run_config(open(os.path.join(REF, rel)).read(), env)
    tree = env["model"]
    assert tree["_target_"] == "SomeThing" and tree["model_vision"]["_target_"] == "DeformableDETRSegmVL"
    return tree


def test_integration_target_overrides_name_real_config_nodes(built):
    """The overrides name real nodes of the reference's model config tree (_reference_model_tree over the reference's own
    config files), recorded in tests/golden/ref_model_config_tree.json by tests/golden/gen_cpu_golden.py."""
    tree = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_model_config_tree.json")))
    text = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    overrides = re.findall(r"(model(?:\.\w+)+)\._target_=(ape_b200(?:\.\w+)+)", text)
    assert len(overrides) >= 9
    import ape_b200  # noqa: F401
    for path, target in overrides:
        node = tree
        for k in path.split(".")[1:]:
            assert isinstance(node, dict) and k in node, f"INTEGRATION.md overrides {path}: `{k}` is not a key of the reference config"
            node = node[k]
        assert isinstance(node, dict) and "_target_" in node, f"{path} is not a LazyCall node in the reference config"
        mod, cls = target.rsplit(".", 1)
        engine_cls = getattr(importlib.import_module(mod), cls)
        assert engine_cls.__name__ == node["_target_"], f"{path}: reference builds {node['_target_']}, override names {cls}"
        params = inspect.signature(engine_cls.__init__).parameters
        accepts_kwargs = any(p.kind == p.VAR_KEYWORD for p in params.values())
        for kw in node:
            if kw != "_target_":
                assert accepts_kwargs or kw in params, f"{target} does not accept the config keyword `{kw}` of {path}"


def test_instances_to_detectron2_maps_fields(monkeypatch):
    from ape_b200.structures import Boxes, Instances

    class D2Boxes:
        def __init__(self, tensor):
            self.tensor = tensor

    class D2Instances:
        def __init__(self, image_size, **kw):
            self.image_size = image_size
            self.fields = {}
            for k, v in kw.items():
                self.set(k, v)

        def set(self, k, v):
            self.fields[k] = v

        def __setattr__(self, k, v):
            if k in ("image_size", "fields"):
                object.__setattr__(self, k, v)
            else:
                self.fields[k] = v

    d2 = types.ModuleType("detectron2")
    d2s = types.ModuleType("detectron2.structures")
    d2s.Boxes, d2s.Instances = D2Boxes, D2Instances
    monkeypatch.setitem(sys.modules, "detectron2", d2)
    monkeypatch.setitem(sys.modules, "detectron2.structures", d2s)
    inst = Instances((48, 64), pred_boxes=Boxes(torch.rand(3, 4)), scores=torch.rand(3), pred_classes=torch.arange(3))
    out = inst.to_detectron2()
    assert isinstance(out, D2Instances) and out.image_size == (48, 64)
    assert isinstance(out.fields["pred_boxes"], D2Boxes) and torch.equal(out.fields["pred_boxes"].tensor, inst.pred_boxes.tensor)
    assert torch.equal(out.fields["scores"], inst.scores) and torch.equal(out.fields["pred_classes"], inst.pred_classes)


def test_entity_gates_and_thing_class_slicing(built):
    """deformable_detr_segm_vl.py:575-593 / :628-630 / :671-673 and deformable_detr.py:246-262, 524-532."""
    from ape_b200 import configs
    from ape_b200.modeling import build_model

    m = build_model(configs.MINI)
    name = m.dataset_names[0]
    box_cls = torch.randn(1, 5, 12)
    assert m._detector_box_cls(box_cls) is box_cls          # no dataset selected (eval_dataset_id = -1): all classes
    things, stuff = [f"t{i}" for i in range(8)], [f"s{i}" for i in range(4)]
    m.dataset_stuff = {name: (things, stuff)}
    m.set_eval_dataset(name)
    assert m.eval_dataset_entity == "thing+stuff"
    assert torch.equal(m._detector_box_cls(box_cls), box_cls[..., :8])   # disjoint lists: the first len(things) columns
    m.dataset_stuff = {name: (things[:4], things, None, [0, 2, 5, 7])}   # thing classes are a subset of the stuff classes
    m.set_eval_dataset(name)
    out = m._detector_box_cls(box_cls)
    assert torch.equal(out[..., [0, 2, 5, 7]], box_cls[..., [0, 2, 5, 7]]) and torch.isinf(out[..., [1, 3, 4, 6, 8]]).all()
    m.dataset_stuff = {name: ([], stuff)}
    m.set_eval_dataset(name)
    assert m.eval_dataset_entity == "stuff"                  # instance branch is skipped for stuff-only datasets
    m.set_eval_dataset("some_other_dataset")
    assert m.eval_dataset_id == -1 and m.eval_dataset_entity == ""
