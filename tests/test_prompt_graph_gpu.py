"""GPU: prompts that put several language tokens into the vision-language fusion replay a CUDA graph.  A MINI model with APE's
fusion geometry (8 heads of 256 channels, 1024-wide text features) in fp16 under `use_cuda_graphs`: a phrase prompt, a
two-image expression batch and a fused-vocabulary name prompt (`name_prompt_fusion_text`) give logits, boxes and detections
(and `forward_packed` bytes with masks, semantic and panoptic maps) bit-identical to the eager 16-bit call; a new token count
is captured on its second call, not its first; another text with the same count replays the same graph with its own inputs;
the text-feature bank is still updated before the step."""
import copy
import zlib

import pytest
import torch

from ape_b200 import configs, parallel
from ape_b200.modeling import build_model
from oracle import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SPEC = copy.deepcopy(configs.MINI)
SPEC.update(name="MINI-VLF2048", vlf_embed=2048, vlf_heads=8, lang_dim=1024)


class _TextByContent:
    """Text features seeded by each string's content, so that two texts with the same count differ."""

    def forward_text(self, text_list, cache=False, **kw):
        rows = [torch.randn(SPEC["lang_dim"], generator=torch.Generator().manual_seed(zlib.crc32(t.encode()))) for t in text_list]
        return {"last_hidden_state_eot": torch.stack(rows)}


@pytest.fixture(scope="module")
def model(built):
    m = build_model(SPEC)
    synth.fill_state_dict(m)
    m = m.to(DEV).eval()
    m.engine_dtype = torch.float16
    m.set_model_language(_TextByContent())
    return m


def _images(n, seed):
    sizes = [(56, 64), (48, 40)][:n]
    return [{"image": synth.image(h, w, seed=seed + i), "height": 2 * h, "width": 2 * w} for i, (h, w) in enumerate(sizes)]


def _phrases(seed, n=1):
    return [dict(x, prompt="text", text_prompt=f"red car {seed},person,traffic light {seed}") for x in _images(n, seed)]


def _expressions(seed):
    return [dict(x, prompt="expression", expressions=[f"the dog on the left {seed}", f"a man in a hat {seed}"][i])
            for i, x in enumerate(_images(2, seed))]


def _run(model, inputs, graphs, packed=False):
    model.use_cuda_graphs = graphs
    out = model.forward_packed(inputs).clone() if packed else model(inputs)
    lo = model.last_outputs
    return out, lo["pred_logits"].clone(), lo["pred_boxes"].clone()


def _same(got, want, packed):
    if packed:
        assert torch.equal(got, want)
        return
    assert len(got) == len(want)
    for x, y in zip(got, want):
        i, j = x["instances"], y["instances"]
        assert torch.equal(i.pred_boxes.tensor, j.pred_boxes.tensor) and torch.equal(i.scores, j.scores)
        assert torch.equal(i.pred_classes, j.pred_classes)


def _graphs(model):
    return [k for k in model._graph_cache if k[0][0] == "forward"]


def _check(model, make, packed=False):
    """First call of a token count: eager, nothing captured.  Second: captured, replay == eager.  Another text with the same
    count: the same graph replays and matches that text's eager call."""
    model._graph_cache.clear()
    model.__dict__.pop("_graph_seen_keys", None)
    inputs = make(0)
    first = _run(model, inputs, True, packed)
    assert len(_graphs(model)) == 0
    want = _run(model, inputs, False, packed)
    got = _run(model, inputs, True, packed)
    assert len(_graphs(model)) == 1
    for g, w in ((first, want), (got, want)):
        assert torch.equal(g[1], w[1]) and torch.equal(g[2], w[2])
        _same(g[0], w[0], packed)
    other = make(1)
    got = _run(model, other, True, packed)
    want2 = _run(model, other, False, packed)
    assert len(_graphs(model)) == 1
    assert not torch.equal(want2[1], want[1])
    assert torch.equal(got[1], want2[1]) and torch.equal(got[2], want2[2])
    _same(got[0], want2[0], packed)
    return want


def test_phrase_prompt_replays_a_graph(model):
    _check(model, _phrases)
    _check(model, _phrases, packed=True)


def test_expression_batch_replays_a_graph(model):
    _check(model, _expressions)


def test_new_token_count_is_captured_on_its_second_call(model):
    model._graph_cache.clear()
    model.__dict__.pop("_graph_seen_keys", None)
    model.use_cuda_graphs = True
    four = lambda s: [dict(x, text_prompt=x["text_prompt"] + f",a blue kite {s}") for x in _phrases(s)]
    model(_phrases(0))
    model(four(0))
    assert len(_graphs(model)) == 0
    model(_phrases(1))
    assert len(_graphs(model)) == 1
    model(four(1))
    assert len(_graphs(model)) == 2
    model(four(2))
    assert len(_graphs(model)) == 2


def test_fused_vocabulary_with_masks_semantic_and_panoptic(model):
    name = model.dataset_names[0]
    saved = (model.name_prompt_fusion_text, dict(model.dataset_stuff), model.test_mask_on, model.semantic_on, model.panoptic_on,
             model.mask_format)
    model.name_prompt_fusion_text = [True]
    model.dataset_stuff[name] = ([f"c{i}" for i in range(6)], [f"c{i}" for i in range(6, 12)], "thing+stuff")
    model.set_eval_dataset(name)
    model.test_mask_on, model.semantic_on, model.panoptic_on, model.mask_format = True, True, True, "rle"
    try:
        inputs = _images(1, 3)
        model._graph_cache.clear()
        model.__dict__.pop("_graph_seen_keys", None)
        model.use_cuda_graphs = True
        model.forward_packed(inputs)
        assert len(_graphs(model)) == 0
        got = model.forward_packed(inputs).clone()
        assert len(_graphs(model)) == 1
        model.use_cuda_graphs = False
        want = model.forward_packed(inputs).clone()
        assert torch.equal(got, want)
        assert len(parallel.unpack_packed(got)) == 1
        _check(model, lambda s: _images(1, s))
    finally:
        (model.name_prompt_fusion_text, model.dataset_stuff, model.test_mask_on, model.semantic_on, model.panoptic_on,
         model.mask_format) = saved
        model.set_eval_dataset("")


def test_text_feature_bank_is_updated_under_graphs(model):
    name = model.dataset_names[0]
    prompts = list(model.dataset_prompts)
    model.dataset_prompts[0] = "expression"
    model.set_eval_dataset(name)
    try:
        model._graph_cache.clear()
        model.__dict__.pop("_graph_seen_keys", None)
        model.use_cuda_graphs = True
        for seed in (0, 0, 1):
            inputs = _expressions(seed)
            model(inputs)
            texts = [x["expressions"][0] for x in inputs]
            feats = model.model_language.forward_text(texts)["last_hidden_state_eot"].to(DEV)
            assert torch.equal(model.features_phrase_bank[0, : len(texts)], feats.to(model.features_phrase_bank.dtype))
        assert len(_graphs(model)) == 1
    finally:
        model.dataset_prompts[:] = prompts
        model.set_eval_dataset("")
