"""GPU: one CUDA graph per padded shape, not per image size.  The MINI model (64^2 pad) in fp16 over a stream of distinct image sizes
inside its pad, revisiting the first: `use_cuda_graphs` captures a single "forward" graph, and every call's logits, boxes and
detections equal the eager 16-bit call at the same size bit for bit.  The same for boxes-only `forward_packed`, for two images of
different sizes per batch, and for `model(inputs)` with instance masks and semantic maps (the graph ends at the mask logits).
`forward_packed` with instance masks keeps the sizes in its key: its mask stage sizes its launches from host ints."""
import pytest
import torch

from ape_b200 import configs, parallel
from ape_b200.modeling import build_model
from oracle import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
STREAM = [(56, 64), (64, 64), (33, 17), (1, 64), (64, 1), (40, 48), (56, 64)]  # 6 distinct sizes, the first revisited


@pytest.fixture(scope="module")
def model(built):
    m = build_model(configs.MINI)
    synth.fill_state_dict(m)
    m = m.to(DEV).eval()
    m.engine_dtype = torch.float16
    return m


def _inputs(sizes, seed):
    return [{"image": synth.image(h, w, seed=seed + i), "height": 2 * h, "width": 2 * w} for i, (h, w) in enumerate(sizes)]


def _forward_graphs(model):
    return [k for k in model._graph_cache if k[0][0] == "forward"]


def _run(model, inputs, graphs, packed=False):
    model.use_cuda_graphs = graphs
    out = model.forward_packed(inputs).clone() if packed else model(inputs)
    lo = model.last_outputs
    return out, lo["pred_logits"].clone(), lo["pred_boxes"].clone()


def _same_instances(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        for k in set(x) | set(y):
            if k == "instances":
                i, j = x[k], y[k]
                assert i.image_size == j.image_size and len(i) == len(j)
                assert torch.equal(i.pred_boxes.tensor, j.pred_boxes.tensor) and torch.equal(i.scores, j.scores)
                assert torch.equal(i.pred_classes, j.pred_classes)
                if i.has("pred_masks") or j.has("pred_masks"):
                    assert torch.equal(i.pred_masks, j.pred_masks)
            elif torch.is_tensor(x[k]):
                assert torch.equal(x[k], y[k]), k
            else:
                assert x[k] == y[k], k


def _check_stream(model, batches, packed=False):
    model._graph_cache.clear()
    n = 0
    for step, sizes in enumerate(batches):
        inputs = _inputs(sizes, seed=step)
        got, logits, boxes = _run(model, inputs, True, packed)
        want, elogits, eboxes = _run(model, inputs, False, packed)
        assert torch.equal(logits, elogits) and torch.equal(boxes, eboxes), f"graph differs from eager at {sizes}"
        if packed:
            _same_instances(parallel.unpack_packed(got), parallel.unpack_packed(want))
        else:
            _same_instances(got, want)
        n += sum(len(o["instances"]) for o in (parallel.unpack_packed(want) if packed else want))
    assert n > 0
    return _forward_graphs(model)


def test_one_graph_for_a_stream_of_sizes(model):
    model.test_mask_on = False
    assert len(_check_stream(model, [[s] for s in STREAM])) == 1


def test_one_graph_for_packed_boxes(model):
    model.test_mask_on = False
    assert len(_check_stream(model, [[s] for s in STREAM], packed=True)) == 1


def test_one_graph_for_mixed_sizes_in_a_batch(model):
    model.test_mask_on = False
    batches = [[STREAM[i], STREAM[(i + 3) % len(STREAM)]] for i in range(len(STREAM))]
    assert len(_check_stream(model, batches)) == 1
    assert len(_check_stream(model, batches, packed=True)) == 1


def test_one_graph_with_masks_and_semantic_maps(model):
    model.test_mask_on, model.semantic_on = True, True
    try:
        assert len(_check_stream(model, [[s] for s in STREAM[:4]] + [[STREAM[0]]])) == 1
    finally:
        model.test_mask_on, model.semantic_on = False, False


def test_packed_masks_keep_one_graph_per_size(model):
    model.test_mask_on = True
    model.mask_format = "rle"
    try:
        model._graph_cache.clear()
        model.use_cuda_graphs = True
        for sizes in ([STREAM[0]], [STREAM[2]], [STREAM[3]], [STREAM[0]]):
            model.forward_packed(_inputs(sizes, 0))
        assert len(_forward_graphs(model)) == 3
    finally:
        model.test_mask_on, model.mask_format, model.use_cuda_graphs = False, "bitmask", False
