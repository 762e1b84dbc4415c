"""GPU: region prompts (`mask_prompt`) on the device and on the captured step.

Kernel: `ops.region_prompt` gives the region flags, folded anchors and invalid flags of the torch path (prompts padded, an
all-zero batch set to 255, F.interpolate(mode="bilinear") on the device, `.to(bool)`, masked_fill) bit for bit, +inf included, over
the sweep of tests/test_region_prompt_cpu.py, whose prompts on the rows and columns where a fused and an unfused source index
differ pin the fused one against torch's CUDA kernel; one empty prompt beside a set one keeps no token, an all-empty batch keeps
all.

Model: MINI in fp16 under `use_cuda_graphs` over a stream of (image size, region) pairs inside the 64^2 pad that revisits one
pair captures exactly one "forward" graph with a region, and each call's logits, boxes and detections equal the eager 16-bit
call bit for bit: for name prompts, for a 3-phrase prompt (captured on its second call), for `forward_packed` (boxes only, then
masks with `packed_output_capacity`), and for instance masks + semantic maps through `model(inputs)`.  After capture, a
boxes-only `forward_packed` with a region prompt runs under set_sync_debug_mode("error"); `DefaultPredictor` with two masks
replays one graph and equals the eager result."""
import numpy as np
import pytest
import torch

from ape_b200 import configs, parallel
from ape_b200.modeling import build_model
from oracle import synth
from test_prompt_graph_gpu import SPEC as VLF_SPEC, _TextByContent
from test_region_prompt_cpu import GEOMETRIES, cases, padded_nonzero, region_np, region_torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _anchors(B, S, seed):
    """Geometry-like anchors: finite logits with some +inf rows, and invalid flags on some of the finite ones too."""
    g = torch.Generator().manual_seed(seed)
    p = torch.randn((B, S, 4), generator=g) * 3
    inv = torch.rand((B, S, 1), generator=g) < 0.2
    p[inv.expand(-1, -1, 4)] = float("inf")
    inv |= torch.rand((B, S, 1), generator=g) < 0.05
    return p.to(DEV), inv.to(DEV)


@pytest.mark.parametrize("geometry", sorted(GEOMETRIES))
def test_kernel_matches_torch_path(built, geometry):
    from ape_b200 import ops

    padded, shapes, _ = GEOMETRIES[geometry]
    S = sum(h * w for h, w in shapes)
    kept = 0
    for k, (name, prompts) in enumerate(cases(geometry)):
        B = len(prompts)
        props, inv = _anchors(B, S, k)
        region = region_torch(prompts, padded, shapes, device=DEV)
        want_p = props.masked_fill(~region.unsqueeze(-1), float("inf"))
        want_i = inv | ~region.unsqueeze(-1)
        rmap = padded_nonzero(prompts, padded, device=DEV).to(torch.uint8)
        got_p, got_i, got_r = ops.region_prompt(rmap, shapes, props, inv, want_region=True)
        assert torch.equal(got_r, region), f"{geometry} {name}: region flags"
        assert torch.equal(got_p, want_p), f"{geometry} {name}: folded anchors"
        assert torch.equal(got_i, want_i), f"{geometry} {name}: invalid flags"
        if name == "one-empty":
            assert region[0].any() and not region[1].any()
        if name == "all-empty":
            assert region.all()
        kept += int(region.sum())
    assert kept > 0


@pytest.mark.parametrize("axis", ["row", "column"])
def test_kernel_follows_the_fused_source_index(built, axis):
    """33 -> 13, token row 6: the fused source index 15.999999 reads rows 15 and 16, the unfused 16.0 row 16 alone; 65 -> 25,
    token column 12, likewise columns 31 and 32.  A prompt on row 15 (column 31) alone puts that token row (column) inside the
    region for torch's CUDA F.interpolate and for the kernel, and outside it for the unfused rule."""
    from ape_b200 import ops

    padded, shapes = (33, 65), [(13, 25)]
    m = torch.zeros(padded)
    if axis == "row":
        m[15, :] = 1
    else:
        m[:, 31] = 1
    want = region_torch([m], padded, shapes, device=DEV)
    rmap = padded_nonzero([m], padded, device=DEV).to(torch.uint8)
    props, inv = _anchors(1, 13 * 25, 0)
    got = ops.region_prompt(rmap, shapes, props, inv, want_region=True)[2]
    assert torch.equal(got, want)
    line = got.view(13, 25)[6] if axis == "row" else got.view(13, 25)[:, 12]
    assert line.all()
    unfused = region_np(rmap.bool().cpu().numpy(), shapes, fused=False).reshape(13, 25)
    assert not (unfused[6] if axis == "row" else unfused[:, 12]).any()


def test_kernel_is_capturable_and_reads_the_flag(built):
    from ape_b200 import ops

    padded, shapes, _ = GEOMETRIES["mini"]
    S = sum(h * w for h, w in shapes)
    props, inv = _anchors(1, S, 0)
    rmap = torch.zeros((1,) + padded, dtype=torch.uint8, device=DEV)
    g = torch.cuda.CUDAGraph()
    ops.region_prompt(rmap, shapes, props, inv)  # warm-up
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        out = ops.region_prompt(rmap, shapes, props, inv, want_region=True)
    for y0, y1 in ((0, 0), (5, 9), (0, 64), (0, 0)):
        rmap.zero_()
        rmap[0, y0:y1, 3:40] = 1
        g.replay()
        m = torch.zeros((1,) + padded)
        m[0, y0:y1, 3:40] = 1
        assert torch.equal(out[2], region_torch([m[0]], padded, shapes, device=DEV))
    # a caller's flag replaces the reduction: "empty" means everywhere whatever the map holds
    flag = torch.ones((1,), dtype=torch.uint8, device=DEV)
    assert ops.region_prompt(rmap, shapes, props, inv, empty=flag, want_region=True)[2].all()
    with pytest.raises(RuntimeError, match="region_prompt"):
        ops.region_prompt(rmap.float(), shapes, props, inv)
    with pytest.raises(RuntimeError, match="output_proposals"):
        ops.region_prompt(rmap, shapes, props[:, :-1], inv)


# -- the model --------------------------------------------------------------------------------------------------------------
STREAM = [((56, 64), (8, 40, 16, 56)), ((64, 64), (0, 64, 0, 64)), ((33, 17), (30, 33, 0, 17)), ((64, 1), (10, 11, 0, 1)),
          ((40, 48), (0, 0, 0, 0)), ((56, 64), (20, 21, 5, 60)), ((56, 64), (8, 40, 16, 56))]  # the first pair revisited


@pytest.fixture(scope="module")
def model(built):
    m = build_model(configs.MINI)
    synth.fill_state_dict(m)
    m = m.to(DEV).eval()
    m.engine_dtype = torch.float16
    return m


def _inputs(step, seed, **extra):
    (h, w), (y0, y1, x0, x1) = STREAM[step]
    mp = torch.zeros((h, w))
    mp[y0:y1, x0:x1] = 1.0
    return [dict({"image": synth.image(h, w, seed=seed), "height": 2 * h, "width": 2 * w, "mask_prompt": mp}, **extra)]


def _region_graphs(model):
    return [k for k in model._graph_cache if k[0][0] == "forward" and k[0][-1] is True]


def _run(model, inputs, graphs, packed=False):
    model.use_cuda_graphs = graphs
    out = model.forward_packed(inputs).clone() if packed else model(inputs)
    lo = model.last_outputs
    return out, lo["pred_logits"].clone(), lo["pred_boxes"].clone()


def _same_instances(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert set(x) == set(y)
        for k in x:
            if k == "instances":
                i, j = x[k], y[k]
                assert i.image_size == j.image_size and len(i) == len(j)
                assert torch.equal(i.pred_boxes.tensor, j.pred_boxes.tensor) and torch.equal(i.scores, j.scores)
                assert torch.equal(i.pred_classes, j.pred_classes)
                if i.has("pred_masks") or j.has("pred_masks"):
                    assert torch.equal(i.pred_masks, j.pred_masks)
                if i.has("pred_masks_rle") or j.has("pred_masks_rle"):
                    assert [r["counts"] for r in i.pred_masks_rle] == [r["counts"] for r in j.pred_masks_rle]
            elif torch.is_tensor(x[k]):
                assert torch.equal(x[k], y[k]), k
            else:
                assert x[k] == y[k], k


def _check_stream(model, packed=False, first_graph_call=0, **extra):
    model._graph_cache.clear()
    n = 0
    for step in range(len(STREAM)):
        inputs = _inputs(step, step, **extra)
        got, logits, boxes = _run(model, inputs, True, packed)
        assert len(_region_graphs(model)) == (step >= first_graph_call), f"step {step}"
        want, elogits, eboxes = _run(model, inputs, False, packed)
        assert torch.equal(logits, elogits) and torch.equal(boxes, eboxes), f"graph differs from eager at step {step}"
        got, want = (parallel.unpack_packed(got), parallel.unpack_packed(want)) if packed else (got, want)
        _same_instances(got, want)
        n += sum(len(o["instances"]) for o in want)
    assert n > 0
    return [k for k in model._graph_cache if k[0][0] == "forward"]


def test_one_region_graph_for_a_stream_of_sizes_and_regions(model):
    model.test_mask_on = False
    assert len(_check_stream(model)) == 1


def test_region_changes_the_result(model):
    """The region reaches the step: a prompt on one corner keeps other proposals than the whole image."""
    model.test_mask_on, model.use_cuda_graphs = False, True
    model._graph_cache.clear()
    a = _inputs(0, 0)
    b = [dict(a[0], mask_prompt=torch.ones(a[0]["mask_prompt"].shape))]
    model(a)
    ta = model.transformer.last_topk_proposals.clone()
    model(b)
    assert not torch.equal(ta, model.transformer.last_topk_proposals)
    assert len(_region_graphs(model)) == 1


def test_profile_stages_split_with_region(model):
    """With profile_stages the step runs as an "encode" graph keyed with the region flag and a "decode" graph: one encode graph
    with a region for the whole stream, equal to the eager call bit for bit."""
    model.test_mask_on, model.profile_stages = False, True
    try:
        model._graph_cache.clear()
        for step in range(len(STREAM)):
            inputs = _inputs(step, step)
            got, logits, boxes = _run(model, inputs, True)
            want, elogits, eboxes = _run(model, inputs, False)
            assert torch.equal(logits, elogits) and torch.equal(boxes, eboxes), f"graph differs from eager at step {step}"
            _same_instances(got, want)
        enc = [k for k in model._graph_cache if k[0][0] == "encode"]
        assert len(enc) == 1 and enc[0][0][-1] is True
        assert not [k for k in model._graph_cache if k[0][0] == "forward"]
    finally:
        model.profile_stages = False


def test_packed_boxes_and_masks_with_capacity(model):
    model.test_mask_on = False
    assert len(_check_stream(model, packed=True)) == 1
    model.test_mask_on, model.mask_format, model.packed_output_capacity = True, "rle", 128
    try:
        assert len(_check_stream(model, packed=True)) == 1
    finally:
        model.test_mask_on, model.mask_format, model.packed_output_capacity = False, "bitmask", None


def test_masks_and_semantic_maps(model):
    """The demo's configuration: a region prompt with instance masks and semantic maps through model(inputs)."""
    model.test_mask_on, model.semantic_on = True, True
    try:
        assert len(_check_stream(model)) == 1
    finally:
        model.test_mask_on, model.semantic_on = False, False


def test_phrase_prompt_with_region_captures_on_second_call(built):
    m = build_model(VLF_SPEC)
    synth.fill_state_dict(m)
    m = m.to(DEV).eval()
    m.engine_dtype = torch.float16
    m.set_model_language(_TextByContent())
    m.test_mask_on = False
    assert len(_check_stream(m, first_graph_call=1, prompt="text", text_prompt="red car,person,traffic light")) == 1


def test_packed_region_adds_no_host_synchronisation(model):
    model.test_mask_on, model.use_cuda_graphs = False, True
    model._graph_cache.clear()
    inputs = [dict(x, image=x["image"].to(DEV), mask_prompt=x["mask_prompt"].to(DEV)) for x in _inputs(0, 0)]
    for _ in range(2):
        model.forward_packed(inputs)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = model.forward_packed(inputs)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert len(_region_graphs(model)) == 1
    model.use_cuda_graphs = False
    _same_instances(parallel.unpack_packed(out), parallel.unpack_packed(model.forward_packed(inputs)))


def test_predictor_with_two_masks_replays_one_graph(model):
    from ape_b200.engine.defaults import DefaultPredictor, ResizeShortestEdge

    model.test_mask_on = False
    model._graph_cache.clear()
    pred = DefaultPredictor(model, aug=ResizeShortestEdge(64, 64))
    g = np.random.default_rng(3)
    img = g.integers(0, 256, (45, 60, 3), dtype=np.uint8)
    masks = [np.zeros((45, 60), dtype=np.uint8), np.zeros((45, 60), dtype=np.uint8)]
    masks[0][5:30, 10:50] = 255
    masks[1][30:45, 0:20] = 255
    for mask in masks + masks[:1]:
        model.use_cuda_graphs = True
        got = pred(img, mask_prompt=mask)
        model.use_cuda_graphs = False
        want = pred(img, mask_prompt=mask)
        _same_instances([got], [want])
        assert len(want["instances"]) > 0
    assert len(_region_graphs(model)) == 1
