"""GPU: semantic label maps as run-length codes (csrc/label_rle.cu).  `ops.label_map_rle` against the oracle's restatement of
cocoapi (oracle/rle.py) label by label, byte for byte; the packed slot (`ops.semseg_pack`) in its three kinds; and at model level
`unpack_packed(forward_packed(inputs))` against `model(inputs)` with `sem_seg_format = "rle"` on the MINI spec."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _voronoi(h, w, n, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[:h, :w]
    seeds = rng.random((n, 2)) * [h, w]
    d = (yy[None] - seeds[:, 0, None, None]) ** 2 + (xx[None] - seeds[:, 1, None, None]) ** 2
    return rng.integers(0, 1203, n)[d.argmin(0)].astype(np.int64)


def _maps():
    rng = np.random.default_rng(0)
    m = {"random": rng.integers(0, 20, (97, 131)), "smooth": _voronoi(300, 400, 30, 1), "single": np.full((64, 48), 7),
         "1x1": np.array([[65535]]), "1xW": rng.integers(0, 3, (1, 77)), "Hx1": rng.integers(0, 3, (45, 1)),
         "odd": rng.integers(0, 4, (33, 65)), "big": _voronoi(2048, 1536, 30, 2), "N1": np.zeros((50, 70)),
         "N5000": (rng.permutation(128 * 160) % 5000 * 13).reshape(128, 160)}  # 5000 distinct labels up to 64987
    first = np.full((40, 30), 3)
    first[0, 0] = 11  # a label present only at pixel 0
    m["first_pixel"] = first
    last = np.full((40, 30), 3)
    last[-1, -1] = 0  # ... and only at the last pixel
    m["last_pixel"] = last
    wrap = np.zeros((16, 6), np.int64)
    wrap[:, 1::2] = 5  # every change of label falls exactly on a column wrap
    m["column_wrap"] = wrap
    return {k: np.asarray(v, np.int64) for k, v in m.items()}


def _want(L):
    from oracle import rle as R

    return [(int(c), R.encode((L == c).astype(np.uint8))["counts"]) for c in np.unique(L)]


@pytest.mark.parametrize("name", list(_maps()))
def test_label_map_rle_matches_cocoapi(built, name):
    from ape_b200 import ops

    L = _maps()[name]
    got = ops.label_map_rle(torch.from_numpy(L).to(DEV))
    assert all(e["segmentation"]["size"] == list(L.shape) for e in got)
    assert [(e["label"], e["segmentation"]["counts"]) for e in got] == _want(L)
    if name == "N5000":
        assert len(got) == 5000
    assert np.array_equal(ops.label_map_from_rle(got), L)


def test_two_runs_give_identical_output(built):
    from ape_b200 import ops

    L = torch.from_numpy(np.random.default_rng(3).integers(0, 300, (512, 384))).to(DEV)
    a, b = ops.label_map_rle(L), ops.label_map_rle(L)
    assert a == b


def test_out_of_range_labels_are_rejected(built):
    from ape_b200 import ops

    for v in (-1, 65536):
        L = torch.zeros((9, 7), dtype=torch.int64, device=DEV)
        L[4, 3] = v
        with pytest.raises(RuntimeError, match="outside"):
            ops.label_map_rle(L)


def test_semseg_pack_kinds(built):
    """A slot holds the codes when they fit, else the map as uint16, else nothing (kind 3); a graph replay writes the same bytes."""
    from ape_b200 import ops

    maps = [_voronoi(120, 90, 8, 5), np.random.default_rng(6).integers(0, 1203, (61, 47))]
    labels = [torch.from_numpy(L).to(DEV) for L in maps]
    for slot, kinds in ((1 << 20, (1, 1)), (16384, (1, 2)), (4000, (1, 3))):
        slots = torch.full((2, slot + 4), 7, dtype=torch.uint8, device=DEV)[:, :slot]
        info = torch.empty((2, 3), dtype=torch.int32, device=DEV)
        ops.semseg_pack(labels, 1203, slots, info)
        inf = info.cpu().tolist()
        assert tuple(k for k, _, _ in inf) == kinds, (slot, inf)
        raw = slots.cpu().numpy()
        for L, (kind, n, P), s in zip(maps, inf, raw):
            assert P == len(np.unique(L))
            if kind == 1:
                got = ops._label_rle_table(s[:n], P, *L.shape)
                assert [(e["label"], e["segmentation"]["counts"]) for e in got] == _want(L)
            elif kind == 2:
                assert n == 2 * L.size and np.array_equal(s[:n].view(np.uint16).reshape(L.shape), L)
            else:
                assert n > slot
            assert not s[n if kind != 3 else 0:].any()  # the rest of the slot is zero
    graph = torch.cuda.CUDAGraph()
    slots = torch.empty((2, 16384), dtype=torch.uint8, device=DEV)
    info = torch.empty((2, 3), dtype=torch.int32, device=DEV)
    ops.semseg_pack(labels, 1203, slots, info)
    torch.cuda.synchronize()
    eager = slots.clone()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph):
            ops.semseg_pack(labels, 1203, slots, info)
    slots.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(slots, eager)


@pytest.fixture(scope="module")
def mini():
    from ape_b200 import configs
    from ape_b200.modeling import build_model
    from oracle import synth

    m = build_model(configs.MINI)
    synth.fill_state_dict(m)
    return m.to(DEV).eval()


def _images(B, seed):
    from oracle import synth

    sizes = [(56, 64, 112, 128), (48, 60, 95, 131)][:B]
    return [{"image": synth.image(h, w, seed=seed + i), "height": oh, "width": ow} for i, (h, w, oh, ow) in enumerate(sizes)]


def _codes(rle):
    return [(e["label"], e["segmentation"]["size"], e["segmentation"]["counts"]) for e in rle]


@pytest.mark.parametrize("masks,graphs,dtype,slot", [
    (True, True, torch.float16, None), (True, False, torch.float16, None), (False, True, torch.float16, None),
    (False, False, torch.bfloat16, None), (True, True, torch.float16, 28672), (False, False, torch.float16, 28672)])
def test_forward_packed_semantic_equals_the_model(built, mini, masks, graphs, dtype, slot):
    from ape_b200 import parallel

    model = mini
    saved = (model.semantic_on, model.test_mask_on, model.engine_dtype, model.use_cuda_graphs, model.sem_seg_slot_bytes)
    try:
        model.semantic_on, model.test_mask_on = True, masks
        model.engine_dtype, model.use_cuda_graphs = dtype, graphs
        model.mask_format, model.sem_seg_format = "rle", "rle"
        if slot is not None:
            model.sem_seg_slot_bytes = slot  # the 112 x 128 map as uint16, exactly: longer codes travel as the map (kind 2)
        for seed in (3, 4):  # the second call replays the graphs captured by the first
            inputs = _images(2, seed)
            want = model(inputs)
            packed = model.forward_packed(inputs)
            kinds = packed[:, :32].contiguous().view(torch.int32)[:, 2].tolist()
            got = parallel.unpack_packed(packed)
            model.semantic_on = False  # the form without the semantic branch: same boxes and masks
            plain = parallel.unpack_packed(model.forward_packed(inputs))
            model.semantic_on = True
            print(f"  masks={masks} graphs={graphs} {dtype} slot={slot} seed {seed}: kinds {kinds}, "
                  f"{[len(o['sem_seg_rle']) for o in want]} labels")
            for k, w in zip(kinds, want):
                need = sum(12 + len(e["segmentation"]["counts"]) for e in w["sem_seg_rle"])
                assert k == (1 if need <= (slot or model.sem_seg_slot_bytes) else 2), (k, need)
            for g, w, p in zip(got, want, plain):
                assert _codes(g["sem_seg_rle"]) == _codes(w["sem_seg_rle"])
                gi, pi = g["instances"], p["instances"]
                assert torch.equal(gi.pred_boxes.tensor, pi.pred_boxes.tensor) and torch.equal(gi.scores, pi.scores)
                assert torch.equal(gi.pred_classes, pi.pred_classes)
                if masks:
                    assert [r["counts"] for r in gi.pred_masks_rle] == [r["counts"] for r in pi.pred_masks_rle]
                L = w["sem_seg_label"].cpu().numpy()
                assert _codes(w["sem_seg_rle"]) == [(c, list(L.shape), s) for c, s in _want(L)]
    finally:
        model.semantic_on, model.test_mask_on, model.engine_dtype, model.use_cuda_graphs, model.sem_seg_slot_bytes = saved
        model.mask_format, model.sem_seg_format = "bitmask", "maps"


def test_forward_packed_semantic_rejects_fp32(built, mini):
    model = mini
    model.semantic_on = True
    try:
        with pytest.raises(ValueError, match="16-bit"):
            model.forward_packed(_images(1, 0))
    finally:
        model.semantic_on = False


def test_map_slot_is_encoded_on_the_receiving_side(built):
    """A slot that carries the map as uint16 (ops.semseg_pack's choice for codes longer than the slot) unpacks to the codes of
    label_map_rle, encoded on the device of the receiving rank."""
    from ape_b200 import ops, parallel

    L = np.random.default_rng(9).integers(0, 1203, (61, 47))
    rows = torch.zeros((5, 13))
    rows[:, 9:13] = torch.tensor([61.0, 47.0, 61.0, 47.0])
    det = rows.numpy().view(np.uint8).reshape(-1)
    slot = 2 * L.size + 2
    slots = torch.zeros((1, slot), dtype=torch.uint8, device=DEV)
    info = torch.empty((1, 3), dtype=torch.int32, device=DEV)
    ops.semseg_pack([torch.from_numpy(L).to(DEV)], 1203, slots, info)
    kind, n, P = info[0].tolist()
    assert kind == 2 and n == 2 * L.size
    hdr = np.array([5, 52, kind, n, 61, 47, P, 0], np.int32).view(np.uint8)
    packed = torch.from_numpy(np.concatenate([hdr, det, slots[0].cpu().numpy()])[None]).to(DEV)
    got = parallel.unpack_packed(packed)[0]["sem_seg_rle"]
    assert [(e["label"], e["segmentation"]["counts"]) for e in got] == _want(L)
