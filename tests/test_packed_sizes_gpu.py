"""GPU: the packed result stages with the image and output sizes held on the device (`ops.*_dev`, `model.packed_output_capacity`).

Kernel level: each device-size entry point gives its host-int counterpart's bytes (mask slots, semantic slots and info words,
panoptic ids, counts and slots) at 1 x 1, 1 x W, H x 1, odd sizes, sizes equal to the capacity and a small size inside a large
capacity, for fp32 / fp16 / bf16 logits, with the capacity buffers holding stale bytes; one captured graph replayed over a stream of
sizes equals the host-int calls at each size.  Model level: the MINI model in fp16 with a capacity captures one "forward" graph over
a stream of sizes, and `unpack_packed` of its results equals the default (per-size, eager) mode byte for byte; an output past the
capacity takes the per-size key; bad capacities are rejected."""
import pytest
import torch

from ape_b200 import configs, ops, parallel
from oracle import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PAD = (64, 64)          # padded image
LOGIT_HW = (16, 16)     # mask logit grid
Q, K, TOPK, N_CLS, N_THING = 12, 8, 6, 9, 4
SIZES = [((64, 64), (1, 1)), ((64, 64), (1, 37)), ((64, 64), (41, 1)), ((33, 17), (67, 35)), ((64, 48), (96, 96)),
         ((1, 1), (5, 3)), ((7, 64), (96, 11))]  # (image, output) pairs; 96 = the capacity
CAP = 96
SENTINEL = 0x5A


def _stale(nbytes):
    """Leave nbytes of sentinel bytes in the caching allocator, so that the next allocation of that size starts with them."""
    t = torch.full((nbytes,), SENTINEL, dtype=torch.uint8, device=DEV)
    del t


def _logits(dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(Q, *LOGIT_HW, generator=g) * 3).to(DEV, dtype).contiguous()


def _dims(img, out):
    return torch.tensor([img[0], img[1], out[0], out[1]], dtype=torch.int32, device=DEV)


def _rows(img, out, seed, B=1):
    """Selection rows [B, TOPK, 13] as forward_packed writes them: boxes in image pixels, nk = TOPK - 2 kept."""
    g = torch.Generator().manual_seed(seed)
    rows = torch.zeros((B, TOPK, 13))
    for b in range(B):
        ih, iw = img[b] if B > 1 else img
        oh, ow = out[b] if B > 1 else out
        xy = torch.rand(TOPK, 2, generator=g) * torch.tensor([iw, ih]) * 0.7
        wh = torch.rand(TOPK, 2, generator=g) * torch.tensor([iw, ih]) * 0.5 + 0.5
        rows[b, :, 0:2], rows[b, :, 2:4] = xy, xy + wh
        rows[b, :, 4] = torch.rand(TOPK, generator=g)
        rows[b, :, 6] = torch.randperm(Q, generator=g)[:TOPK].float()
        rows[b, :, 7], rows[b, :, 8] = TOPK, TOPK - 2
        rows[b, :, 9:13] = torch.tensor([ih, iw, oh, ow], dtype=torch.float32)
    return rows.to(DEV).contiguous()


def _stage_inputs(dtype, img, out, seed):
    """Device inputs of the three stages of one image: selection rows, kept queries and class weights, scores, classes."""
    g = torch.Generator().manual_seed(seed)
    scores = torch.rand(K, generator=g)
    scores[1] = float("-inf")
    return dict(rows=_rows(img, out, seed), qi=torch.randperm(Q, generator=g)[:K].to(DEV),
                cls=torch.softmax(torch.randn(K, N_CLS, generator=g), -1).to(DEV, torch.float16 if dtype == torch.float32 else dtype),
                scores=scores.to(DEV), classes=torch.randint(0, N_CLS, (K,), generator=g, dtype=torch.int32).to(DEV))


def _stages(logits, x, img, out, dims=None, stale=True):
    """(mask rows, semantic slot, semantic info, counts, panoptic slot, label map, panoptic ids) of one image from host ints, or
    from dims (the maps are then the capacity buffers: flat, the real map first).  No host synchronisation (graph-capturable)."""
    masks = ops.mask_pack(logits[None].contiguous(), x["rows"], [out], PAD, 2048) if dims is None else \
        ops.mask_pack_dev(logits[None].contiguous(), x["rows"], dims[None].contiguous(), PAD, 2048, CAP)
    slot = torch.full((1, 4096), SENTINEL, dtype=torch.uint8, device=DEV)
    info = torch.full((1, 3), -7, dtype=torch.int32, device=DEV)
    if dims is None:
        label, _ = ops.semseg_label(logits, x["qi"], x["cls"], PAD, img, out)
        ops.semseg_pack([label], N_CLS, slot, info)
    else:
        if stale:
            _stale(8 * CAP * CAP)
        label = ops.semseg_label_dev(logits, x["qi"], x["cls"], PAD, dims, CAP)
        ops.semseg_pack_dev(label[None], dims[None].contiguous(), CAP, N_CLS, slot, info)
    if dims is None:
        ids, counts = ops.panoptic_winners(logits, x["qi"], x["scores"], PAD, img, out, 0.3)
    else:
        if stale:
            _stale(4 * CAP * CAP)
        ids, counts = ops.panoptic_winners_dev(logits, x["qi"], x["scores"], PAD, dims, CAP, 0.3)
    pan = torch.full((ops.panoptic_slot_bytes_needed(K, (CAP, CAP)),), SENTINEL, dtype=torch.uint8, device=DEV)
    if dims is None:
        ops.panoptic_pack(ids, counts, x["classes"], N_CLS, N_THING, True, 0.4, pan)
    else:
        ops.panoptic_pack_dev(ids, counts, x["classes"], N_CLS, N_THING, True, 0.4, dims, CAP, pan)
    return masks, slot, info, counts, pan, label.flatten(), ids.flatten()


def _equal(got, want, out):
    """The slots, info words and counts byte for byte; the maps over the output's out_h * out_w pixels."""
    n = out[0] * out[1]
    for x, y in zip(got[:5], want[:5]):
        assert torch.equal(x, y)
    for x, y in zip(got[5:], want[5:]):
        assert torch.equal(x[:n], y[:n])


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("case", range(len(SIZES)))
def test_device_sizes_equal_host_sizes(built, dtype, case):
    img, out = SIZES[case]
    logits = _logits(dtype, case)
    x = _stage_inputs(dtype, img, out, case)
    want = _stages(logits, x, img, out)
    got = _stages(logits, x, img, out, _dims(img, out))
    _equal(got, want, out)
    assert int(want[2][0, 0]) in (ops.SEM_SLOT_CODES, ops.SEM_SLOT_MAP)


def test_mask_pack_dev_batch_of_two_sizes(built):
    logits = torch.stack([_logits(torch.float16, 1), _logits(torch.float16, 2)]).contiguous()
    img, out = [(33, 17), (64, 64)], [(67, 35), (1, 96)]
    rows = _rows(img, out, 3, B=2)
    dims = torch.tensor([list(i) + list(o) for i, o in zip(img, out)], dtype=torch.int32, device=DEV)
    assert torch.equal(ops.mask_pack_dev(logits, rows, dims, PAD, 2048, CAP), ops.mask_pack(logits, rows, out, PAD, 2048))


def test_sizes_are_clamped(built):
    """Sizes are clamped, the image to [1, pad] and the output to [1, capacity]: values change, addresses stay in the buffers."""
    logits = _logits(torch.float16, 5)
    bad = _dims((500, 0), (CAP + 40, -3))
    good = _dims((PAD[0], 1), (CAP, 1))
    x = _stage_inputs(torch.float16, PAD, (CAP, 1), 5)
    _equal(_stages(logits, x, PAD, (CAP, 1), bad), _stages(logits, x, PAD, (CAP, 1), good), (CAP, 1))


def test_one_graph_replays_every_size(built):
    logits = _logits(torch.float16, 9)
    dims = _dims(*SIZES[0])
    x = _stage_inputs(torch.float16, *SIZES[0], 9)  # static inputs: the rows carry the sizes too
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _stages(logits, x, *SIZES[0], dims)  # warm-up
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = _stages(logits, x, *SIZES[0], dims, stale=False)
    for step, (img, out) in enumerate(SIZES[::-1] + SIZES):
        fresh = _stage_inputs(torch.float16, img, out, 20 + step)
        for k in x:
            x[k].copy_(fresh[k])
        dims.copy_(_dims(img, out))
        graph.replay()
        _equal(outs, _stages(logits, fresh, img, out), out)


def test_bad_capacities_are_rejected(built):
    for cap in (0, -1, 1.5, True, ops.PACKED_CAPACITY_MAX + 1, "64"):
        with pytest.raises(ValueError):
            ops.check_capacity(cap)


# ---- the model ---------------------------------------------------------------------------------------------------------------
STREAM = [(56, 64), (64, 64), (33, 17), (1, 64), (64, 1), (40, 48), (56, 64)]


@pytest.fixture(scope="module")
def mini(built):
    from ape_b200.modeling import build_model

    m = build_model(configs.MINI)
    synth.fill_state_dict(m)
    m = m.to(DEV).eval()
    return m


_SAVED = ("panoptic_on", "semantic_on", "instance_on", "test_mask_on", "engine_dtype", "use_cuda_graphs", "mask_format",
          "packed_output_capacity")


@pytest.fixture
def model(mini):
    saved = {k: getattr(mini, k) for k in _SAVED}
    stuff = dict(mini.dataset_stuff)
    name = mini.dataset_names[0]
    mini.dataset_stuff[name] = ([f"c{i}" for i in range(6)], [f"c{i}" for i in range(6, 12)], "thing+stuff")
    mini.set_eval_dataset(name)
    mini.engine_dtype = torch.float16
    yield mini
    for k, v in saved.items():
        setattr(mini, k, v)
    mini.dataset_stuff = stuff
    mini.set_eval_dataset("")
    mini._graph_cache.clear()


def _inputs(sizes, seed):
    return [{"image": synth.image(h, w, seed=seed + i), "height": 2 * h + 1, "width": w + 3} for i, (h, w) in enumerate(sizes)]


def _forward_graphs(model):
    return [k for k in model._graph_cache if k[0][0] == "forward"]


def _unpacked(model, inputs, graphs, cap):
    model.use_cuda_graphs, model.packed_output_capacity = graphs, cap
    return parallel.unpack_packed(model.forward_packed(inputs))


def _same(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert set(g) == set(w)
        if "instances" in w:
            a, b = g["instances"], w["instances"]
            assert torch.equal(a.pred_boxes.tensor, b.pred_boxes.tensor) and torch.equal(a.scores, b.scores)
            assert torch.equal(a.pred_classes, b.pred_classes)
            if hasattr(b, "pred_masks_rle"):
                assert [r["counts"] for r in a.pred_masks_rle] == [r["counts"] for r in b.pred_masks_rle]
        if "sem_seg_rle" in w:
            assert g["sem_seg_rle"] == w["sem_seg_rle"]
        if "panoptic_seg" in w:
            assert torch.equal(g["panoptic_seg"][0], w["panoptic_seg"][0]) and g["panoptic_seg"][1] == w["panoptic_seg"][1]


BRANCHES = {"masks": (True, False, False), "semantic": (False, True, False), "panoptic": (False, False, True),
            "all": (True, True, True)}


@pytest.mark.parametrize("branches", list(BRANCHES))
def test_model_one_graph_equals_default_mode(model, branches):
    model.test_mask_on, model.semantic_on, model.panoptic_on = BRANCHES[branches]
    model.mask_format = "rle"
    model._graph_cache.clear()
    batches = [[s] for s in STREAM] + [[STREAM[i], STREAM[(i + 3) % len(STREAM)]] for i in range(3)]
    n = 0
    for step, sizes in enumerate(batches):
        inputs = _inputs(sizes, step)
        got = _unpacked(model, inputs, True, 160)
        _same(got, _unpacked(model, inputs, False, None))
        _same(_unpacked(model, inputs, False, 160), got)  # eager capacity mode runs the same kernels
        n += sum(len(o["instances"]) for o in got if "instances" in o)
    assert len(_forward_graphs(model)) == 2  # one per padded batch shape: B = 1 and B = 2
    assert n > 0 or branches != "masks"


def test_model_output_past_capacity_takes_the_per_size_key(model):
    model.test_mask_on, model.semantic_on, model.panoptic_on = True, True, True
    model.mask_format = "rle"
    model._graph_cache.clear()
    small, large = _inputs([STREAM[0]], 0), _inputs([STREAM[2]], 1)
    large[0]["height"] = 200  # past C = 160
    for inputs in (small, large, small):
        _same(_unpacked(model, inputs, True, 160), _unpacked(model, inputs, False, None))
    keys = _forward_graphs(model)
    assert len(keys) == 2
    sel = [k[0][5][7] for k in keys]
    assert sorted(len(s) for s in sel) == [5, 6]  # (sizes ...) and (None, None, ..., C)


def test_model_rejects_bad_capacities(model):
    model.test_mask_on = True
    for cap in (0, -5, 2.0, True, ops.PACKED_CAPACITY_MAX + 1):
        model.packed_output_capacity = cap
        with pytest.raises(ValueError, match="capacity"):
            model.forward_packed(_inputs([STREAM[0]], 0))
