"""GPU: panoptic slots built on the device (csrc/panoptic.cu ape_panoptic_pack, ops.panoptic_pack) and the panoptic form of
`forward_packed`.  The segment kernel reproduces postprocess._segments decision for decision on random areas (ratios exactly at the
overlap threshold, zero areas, many repeats of one stuff class, K up to APE_PANOPTIC_MAX_K, thousands of classes); the stage
(panoptic_winners + panoptic_pack) gives postprocess_panoptic_winners' map element for element, since both read the same winners
kernel; and for MINI `unpack_packed(model.forward_packed(x))` carries `model(x)`'s panoptic_seg unchanged."""
import numpy as np
import pytest
import torch

from ape_b200 import _lib, configs, ops, parallel
from ape_b200.modeling.postprocess import _query_scores, _segments, postprocess_panoptic_winners
from oracle import synth
from test_panoptic_merge_gpu import CFG, N_CLS, N_THING, PADDED, _inputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _decode(slot):
    """(header int32 [8], table int32 [K, 3], map int32 [H, W]) of a slot copied to the host."""
    raw = slot.cpu().numpy()
    hdr = raw[:32].view(np.int32)
    K, H, W = int(hdr[4]), int(hdr[2]), int(hdr[3])
    table = raw[32:32 + 12 * K].view(np.int32).reshape(K, 3)
    return hdr, table, raw[32 + 12 * K:32 + 12 * K + 2 * H * W].view(np.uint16).astype(np.int32).reshape(H, W), raw


def _stats(K, num_classes, num_things, seed):
    """mask_area, inter_area, original_area, classes [K] (numpy int64) built to hit the decisions' edges."""
    g = np.random.default_rng(seed)
    orig = g.integers(1, 60, K)
    area = g.integers(1, 60, K)
    inter = np.minimum(area, g.integers(0, 60, K))
    kind = g.integers(0, 6, K)
    m = g.integers(1, 20, K)
    exact = kind == 0  # ratio exactly at the threshold (2/5 at 0.4), and one pixel under it
    area[exact], orig[exact] = 2 * m[exact], 5 * m[exact]
    under = kind == 1
    area[under], orig[under] = 2 * m[under] - 1, 5 * m[under]
    zero = kind == 2  # one of the three areas is 0
    which = g.integers(0, 3, K)
    area[zero & (which == 0)] = 0
    orig[zero & (which == 1)] = 0
    inter[zero & (which == 2)] = 0
    inter[(kind != 2) & (inter == 0)] = 1
    classes = g.integers(0, num_classes, K)
    stuff_lo = min(num_things, num_classes - 1)
    classes[g.random(K) < 0.35] = stuff_lo  # many repeats of one stuff class
    classes[g.random(K) < 0.1] = num_classes - 1
    return area, inter, orig, classes


def _pack_stats(area, inter, orig, classes, num_classes, num_things, stuff_first, thr, hw=None, offset=0):
    K = len(area)
    counts = torch.from_numpy(np.stack([area, inter, orig]).astype(np.int32)).to(DEV)
    cls = torch.from_numpy(classes.astype(np.int32)).to(DEV)
    H, W = hw if hw is not None else (int(np.ceil((K + 1) / 64)), 64)
    g = torch.Generator().manual_seed(K)
    ids = (torch.randperm(H * W, generator=g) % (K + 1) - 1).to(torch.int32).view(H, W).to(DEV)  # every query, and -1
    need = ops.panoptic_slot_bytes_needed(K, (H, W))
    buf = torch.full((need + 64 + offset,), 0xAB, dtype=torch.uint8, device=DEV)
    slot = buf[offset:offset + need + 60]
    ops.panoptic_pack(ids, counts, cls, num_classes, num_things, stuff_first, thr, slot)
    return slot, ids, buf


@pytest.mark.parametrize("K", [0, 1, 300, 4096])
@pytest.mark.parametrize("num_classes", [20, 5000])
@pytest.mark.parametrize("stuff_first", [False, True])
def test_segments_match_the_reference_loop(K, num_classes, stuff_first):
    num_things = num_classes // 2
    for seed, thr in ((K, 0.4), (K + 1, 0.8)):
        area, inter, orig, classes = _stats(K, num_classes, num_things, seed)
        stats = torch.from_numpy(np.stack([area, orig, inter, classes]).astype(np.int64))
        lut, info = _segments(stats, range(num_things), num_things, stuff_first, thr)
        slot, ids, buf = _pack_stats(area, inter, orig, classes, num_classes, num_things, stuff_first, thr, offset=4 * (seed % 4))
        hdr, table, seg, raw = _decode(slot)
        H, W = ids.shape
        S = len(info)
        assert hdr.tolist() == [1, S, H, W, K, 32 + 12 * K + 2 * H * W, 0, 0]
        assert [{"id": int(i), "isthing": bool(t), "category_id": int(c)} for i, t, c in table[:S]] == info
        assert not table[S:].any()
        want = torch.cat([torch.zeros(1, dtype=torch.int32), lut])[ids.cpu().long() + 1]  # lut[ids], 0 where ids is -1
        assert torch.equal(torch.from_numpy(seg), want)
        assert not raw[32 + 12 * K + 2 * H * W:].any()  # the slot's tail is zeroed
        whole = buf.cpu().numpy()
        off = 4 * (seed % 4)
        assert (whole[:off] == 0xAB).all() and (whole[off + slot.numel():] == 0xAB).all()  # nothing outside the slot
        if K >= 300:
            assert S > 0 and any(not e["isthing"] for e in info)


def test_threshold_is_compared_in_double():
    """2/5 at 0.4 keeps the query (Python's int / int is a correctly rounded double); in fp32 0.4 rounds up and would drop it."""
    area, inter, orig, classes = (np.array([2, 3]), np.array([2, 3]), np.array([5, 5]), np.array([0, 1]))
    slot, _, _ = _pack_stats(area, inter, orig, classes, 4, 2, False, 0.4)
    hdr, table, _, _ = _decode(slot)
    assert hdr[1] == 2 and table[:2, 0].tolist() == [1, 2]


def test_graph_replay_equals_eager():
    area, inter, orig, classes = _stats(300, 40, 20, 5)
    K = 300
    counts = torch.from_numpy(np.stack([area, inter, orig]).astype(np.int32)).to(DEV)
    cls = torch.from_numpy(classes.astype(np.int32)).to(DEV)
    ids = (torch.arange(40 * 64, device=DEV) % (K + 1) - 1).to(torch.int32).view(40, 64)
    n = ops.panoptic_slot_bytes_needed(K, (40, 64)) + 16
    slot = torch.empty(n, dtype=torch.uint8, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.panoptic_pack(ids, counts, cls, 40, 20, True, 0.4, slot)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.panoptic_pack(ids, counts, cls, 40, 20, True, 0.4, slot)
    eager = torch.empty_like(slot)
    for seed in (6, 7):
        area, inter, orig, classes = _stats(K, 40, 20, seed)
        counts.copy_(torch.from_numpy(np.stack([area, inter, orig]).astype(np.int32)))
        cls.copy_(torch.from_numpy(classes.astype(np.int32)))
        slot.fill_(0xAB)
        graph.replay()
        ops.panoptic_pack(ids, counts, cls, 40, 20, True, 0.4, eager)
        torch.cuda.synchronize()
        assert torch.equal(slot, eager)


def test_bad_arguments_are_rejected():
    ids = torch.zeros((8, 8), dtype=torch.int32, device=DEV)
    counts = torch.zeros((3, 4), dtype=torch.int32, device=DEV)
    cls = torch.zeros(4, dtype=torch.int32, device=DEV)
    ws = torch.empty(int(_lib.lib.ape_panoptic_pack_workspace_bytes(4, 10)), dtype=torch.uint8, device=DEV)
    slot = torch.zeros(32 + 48 + 128 + 8, dtype=torch.uint8, device=DEV)
    s = _lib.current_stream_ptr()
    ok = dict(ids=ids.data_ptr(), K=4, nc=10, oh=8, ow=8, slot=slot.data_ptr(), n=slot.numel())

    def call(**kw):
        a = dict(ok, **kw)
        return _lib.lib.ape_panoptic_pack(a["ids"], counts.data_ptr(), cls.data_ptr(), a["K"], a["nc"], 5, 0, 0.4, a["oh"], a["ow"],
                                          ws.data_ptr(), a["slot"], a["n"], s)

    assert call() == 0
    torch.cuda.synchronize()
    for bad in (dict(K=-1), dict(K=4097), dict(nc=-1), dict(oh=0), dict(n=slot.numel() - 12), dict(n=slot.numel() - 2),
                dict(slot=slot.data_ptr() + 2), dict(ids=ids.data_ptr() + 4), dict(ids=None)):
        assert call(**bad) != 0, bad
        assert _lib.lib.ape_last_error()
    with pytest.raises(RuntimeError, match="bytes needed"):
        ops.panoptic_pack(ids, counts, cls, 10, 5, False, 0.4, slot[:200])
    with pytest.raises(RuntimeError):
        ops.panoptic_pack(ids, counts[:, :3], cls, 10, 5, False, 0.4, slot)


# ---- the stage: panoptic_winners + panoptic_pack against postprocess_panoptic_winners ------------------------------------------
_INPUTS = {}


def _cached_inputs(K, dtype):
    key = (K, dtype)
    if key not in _INPUTS:
        _INPUTS.clear()
        _INPUTS[key] = _inputs(K, dtype, seed=K + 100)
    return _INPUTS[key]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("K", [1, 12, 300, 900])
@pytest.mark.parametrize("out", [(480, 640), (1024, 768), (2048, 1536)])
def test_stage_matches_postprocess_panoptic_winners(out, K, dtype):
    logits, qi, mask_cls = _cached_inputs(K, dtype)
    img = (1000, 760)
    stuff_first = K % 2 == 0
    seg_ref, info_ref = postprocess_panoptic_winners(mask_cls, logits, qi, PADDED, img, out[0], out[1], range(N_THING), N_THING,
                                                     stuff_first, CFG)
    scores, labels, keep = _query_scores(mask_cls, CFG)
    ids, counts = ops.panoptic_winners(logits, qi, torch.where(keep, scores, float("-inf")), PADDED, img, out, CFG["prob"])
    slot = torch.full((ops.panoptic_slot_bytes_needed(K, out) + 1024,), 0xAB, dtype=torch.uint8, device=DEV)
    ops.panoptic_pack(ids, counts, labels.to(torch.int32), N_CLS, N_THING, stuff_first, CFG["overlap_threshold"], slot)
    seg, info = parallel._panoptic_from_slot(slot.cpu().numpy())
    print(f"  {dtype} K={K} {out}: {len(info)} segments")
    assert torch.equal(seg, seg_ref.cpu())
    assert info == info_ref
    if K >= 12:
        assert len(info) > 0


# ---- the model: forward_packed against model(inputs) ---------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mini():
    from ape_b200.modeling import build_model

    m = build_model(configs.MINI)
    synth.fill_state_dict(m)
    return m.to(DEV)


_SAVED = ("panoptic_on", "semantic_on", "instance_on", "test_mask_on", "panoptic_post_nms", "engine_dtype", "use_cuda_graphs",
          "panoptic_slot_bytes", "sem_seg_format")


@pytest.fixture
def model(mini):
    saved = {k: getattr(mini, k) for k in _SAVED}
    stuff = dict(mini.dataset_stuff)
    name = mini.dataset_names[0]
    mini.dataset_stuff[name] = ([f"c{i}" for i in range(6)], [f"c{i}" for i in range(6, 12)], "thing+stuff")
    mini.set_eval_dataset(name)
    yield mini
    for k, v in saved.items():
        setattr(mini, k, v)
    mini.dataset_stuff = stuff
    mini.set_eval_dataset("")


def _batch(seed):
    return [{"image": synth.image(56, 64, seed=seed), "height": 112, "width": 90},
            {"image": synth.image(48, 64, seed=seed + 50)}]


def _same_instances(a, b):
    ia, ib = a["instances"], b["instances"]
    assert torch.equal(ia.pred_boxes.tensor, ib.pred_boxes.tensor) and torch.equal(ia.scores, ib.scores)
    assert torch.equal(ia.pred_classes, ib.pred_classes) and torch.equal(ia.query_index, ib.query_index)
    if hasattr(ia, "pred_masks_rle") or hasattr(ib, "pred_masks_rle"):
        assert [r["counts"] for r in ia.pred_masks_rle] == [r["counts"] for r in ib.pred_masks_rle]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("graphs", [True, False], ids=["graphs", "eager"])
@pytest.mark.parametrize("semantic", [True, False], ids=["sem", "nosem"])
@pytest.mark.parametrize("masks", [True, False], ids=["masks", "boxes"])
@pytest.mark.parametrize("post_nms", [True, False], ids=["post_nms", "all_queries"])
def test_model_packed_panoptic_equals_model(model, post_nms, masks, semantic, graphs, dtype):
    model.panoptic_on, model.semantic_on, model.test_mask_on = True, semantic, masks
    model.panoptic_post_nms, model.engine_dtype, model.use_cuda_graphs = post_nms, dtype, graphs
    for seed in (1, 2):  # the second call replays the captured graph
        inp = _batch(seed)
        model.panoptic_on = True
        packed = model.forward_packed(inp)
        Q = model.num_queries
        K = model.test_topk_per_image if post_nms else Q
        sem_bytes = model.sem_seg_slot_bytes if semantic else 0
        assert packed.dtype == torch.uint8 and packed.dim() == 2
        hdr = packed[:, :32].cpu().numpy().view(np.int32)
        assert (hdr[:, 7] == model.panoptic_slot_bytes).all()
        assert packed.shape[1] == 32 + int(hdr[0, 0]) * int(hdr[0, 1]) + sem_bytes + model.panoptic_slot_bytes
        got = parallel.unpack_packed(packed)
        want = model(inp)
        assert len(got) == len(want) == 2
        for g, w in zip(got, want):
            seg, info = g["panoptic_seg"]
            wseg, winfo = w["panoptic_seg"]
            assert seg.device.type == "cpu" and torch.equal(seg, wseg.cpu())
            assert info == winfo
            pan = packed.shape[1] - model.panoptic_slot_bytes
            assert int(packed[0, pan + 16:pan + 20].cpu().numpy().view(np.int32)[0]) == K
        # instances and semantic codes are those of the packed form without panoptic
        model.panoptic_on = False
        plain = parallel.unpack_packed(model.forward_packed(inp))
        for g, p in zip(got, plain):
            _same_instances(g, p)
            assert ("sem_seg_rle" in g) == semantic == ("sem_seg_rle" in p)
            if semantic:
                assert g["sem_seg_rle"] == p["sem_seg_rle"]


def test_model_errors_and_entity(model):
    inp = _batch(3)
    model.panoptic_on, model.engine_dtype = True, torch.float32
    with pytest.raises(ValueError, match="16-bit engine_dtype"):
        model.forward_packed(inp)
    model.engine_dtype = torch.float16
    model.panoptic_slot_bytes = 32 + 12 * model.test_topk_per_image + 2 * 112 * 90 - 4
    with pytest.raises(ValueError, match=r"image 0 \(112 x 90.*needs \d+ bytes.*panoptic_slot_bytes"):
        model.forward_packed(inp)
    model.panoptic_slot_bytes = 1 << 16
    out = parallel.unpack_packed(model.forward_packed(inp))
    assert all("panoptic_seg" in o for o in out)
    name = model.dataset_names[0]
    model.dataset_stuff[name] = ([f"c{i}" for i in range(6)], [], None)  # entity "thing": the branch is off
    model.set_eval_dataset(name)
    assert model.eval_dataset_entity == "thing"
    packed = model.forward_packed(inp)
    pan = packed.shape[1] - model.panoptic_slot_bytes
    assert not packed[:, pan:].any()  # flag 0 and nothing else
    out = parallel.unpack_packed(packed)
    assert all("panoptic_seg" not in o for o in out)
    assert all("panoptic_seg" not in o for o in model(inp))
