"""CPU: the panoptic form of `forward_packed` (a 32-byte header per image whose word 7 is the panoptic slot's size, the image's
detection rows, its semantic slot, its panoptic slot) through `parallel.unpack_packed` on hand-built tensors, alone, with a
semantic slot, with mask rows and with the branch off; a semantic-only tensor (word 7 = 0) still decodes as before; one gloo gather
of the panoptic form between two processes; and the errors forward_packed raises before it runs anything."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import ROOT


def _pan_slot(seed, K=7, hw=(30, 40), on=True, spare=44):
    """One panoptic slot (numpy uint8) with a random map of S <= K segments and K table rows; returns (slot, map, segments_info)."""
    rng = np.random.default_rng(seed)
    H, W = hw
    S = min(K, 5)
    info = [{"id": i + 1, "isthing": bool(rng.integers(2)), "category_id": int(rng.integers(0, 60))} for i in range(S)]
    seg = rng.integers(0, S + 1, size=hw).astype(np.int32)
    need = 32 + 12 * K + 2 * H * W
    buf = np.zeros(need + spare, np.uint8)
    if on:
        buf[:32] = np.array([1, S, H, W, K, need, 0, 0], np.int32).view(np.uint8)
        table = np.zeros((K, 3), np.int32)
        for r, e in enumerate(info):
            table[r] = [e["id"], int(e["isthing"]), e["category_id"]]
        buf[32:32 + 12 * K] = table.reshape(-1).view(np.uint8)
        buf[32 + 12 * K:need] = seg.astype(np.uint16).reshape(-1).view(np.uint8)
    return buf, torch.from_numpy(seg), info


def _with_panoptic(packed, pan):
    """A [1, 32 + topk * R + SEM] tensor of the semantic form with `pan` appended and header word 7 set to its size."""
    buf = np.concatenate([packed.numpy(), pan[None]], axis=1)
    buf[0, 28:32] = np.array([pan.size], np.int32).view(np.uint8)
    return torch.from_numpy(buf)


def _det(masks, seed=5):
    from test_mask_pack_cpu import _packed

    packed_masks, rows, _ = _packed(seed, 4)
    det = packed_masks[0].numpy() if masks else rows[0].numpy().view(np.uint8).reshape(rows.shape[1], 52)
    return det, (packed_masks if masks else rows)


def _same_instances(got, want):
    gi, wi = got["instances"], want["instances"]
    assert got["num_candidates"] == want["num_candidates"]
    assert torch.equal(gi.pred_boxes.tensor, wi.pred_boxes.tensor) and torch.equal(gi.scores, wi.scores)
    assert torch.equal(gi.pred_classes, wi.pred_classes) and torch.equal(gi.query_index, wi.query_index)


@pytest.mark.parametrize("masks", [False, True])
@pytest.mark.parametrize("semantic", [False, True])
def test_panoptic_slot_round_trip(masks, semantic):
    sys.path.insert(0, ROOT)
    from ape_b200 import parallel
    from oracle import rle as R
    from test_semseg_pack_cpu import _label_map, _semantic_packed

    det, plain = _det(masks)
    L = _label_map(1)
    sem = _semantic_packed(1, det, 1, L) if semantic else _semantic_packed(1, det, 0, slot=0)
    pan, seg, info = _pan_slot(3)
    got = parallel.unpack_packed(_with_panoptic(sem, pan))[0]
    _same_instances(got, parallel.unpack_packed(plain)[0])
    if masks:
        want = parallel.unpack_packed(plain)[0]["instances"].pred_masks_rle
        assert [r["counts"] for r in got["instances"].pred_masks_rle] == [r["counts"] for r in want]
    if semantic:
        rle = got["sem_seg_rle"]
        assert [e["label"] for e in rle] == np.unique(L).tolist()
        for e in rle:
            assert e["segmentation"]["counts"] == R.encode((L == e["label"]).astype(np.uint8))["counts"]
    else:
        assert "sem_seg_rle" not in got
    got_seg, got_info = got["panoptic_seg"]
    assert got_seg.dtype == torch.int32 and got_seg.device.type == "cpu" and torch.equal(got_seg, seg)
    assert got_info == info and all(type(e["isthing"]) is bool and type(e["id"]) is int for e in got_info)


def test_panoptic_slot_with_no_segment():
    sys.path.insert(0, ROOT)
    from ape_b200 import parallel
    from test_semseg_pack_cpu import _semantic_packed

    det, _ = _det(False)
    pan, _, _ = _pan_slot(4, K=0)  # K = 0 table rows, S = 0, an all-zero map
    seg, info = parallel.unpack_packed(_with_panoptic(_semantic_packed(1, det, 0, slot=0), pan))[0]["panoptic_seg"]
    assert info == [] and tuple(seg.shape) == (30, 40) and not seg.any()


def test_branch_off_adds_no_key():
    sys.path.insert(0, ROOT)
    from ape_b200 import parallel
    from test_semseg_pack_cpu import _semantic_packed

    det, plain = _det(False)
    pan, _, _ = _pan_slot(5, on=False)
    got = parallel.unpack_packed(_with_panoptic(_semantic_packed(1, det, 0, slot=0), pan))[0]
    assert "panoptic_seg" not in got and "sem_seg_rle" not in got
    _same_instances(got, parallel.unpack_packed(plain)[0])


def test_semantic_only_form_is_unchanged():
    """Word 7 = 0: no panoptic slot; the semantic slot runs to the end of the row, as before panoptic maps were packed."""
    sys.path.insert(0, ROOT)
    from ape_b200 import parallel
    from oracle import rle as R
    from test_semseg_pack_cpu import _label_map, _semantic_packed

    det, _ = _det(False)
    L = _label_map(2)
    packed = _semantic_packed(2, det, 1, L)
    assert int(packed[0, 28:32].numpy().view(np.int32)[0]) == 0
    got = parallel.unpack_packed(packed)[0]
    assert "panoptic_seg" not in got
    assert [e["segmentation"]["counts"] for e in got["sem_seg_rle"]] == \
        [R.encode((L == c).astype(np.uint8))["counts"] for c in np.unique(L)]


def test_images_with_different_outputs_in_one_tensor():
    sys.path.insert(0, ROOT)
    from ape_b200 import parallel
    from test_semseg_pack_cpu import _semantic_packed

    det, _ = _det(False)
    a, seg_a, info_a = _pan_slot(6, hw=(30, 40), spare=2 * 400)
    b, seg_b, info_b = _pan_slot(7, hw=(20, 30), spare=2 * 400 + 2 * (1200 - 600))
    assert a.size == b.size
    packed = torch.cat([_with_panoptic(_semantic_packed(1, det, 0, slot=0), a), _with_panoptic(_semantic_packed(2, det, 0, slot=0), b)])
    (sa, ia), (sb, ib) = (o["panoptic_seg"] for o in parallel.unpack_packed(packed))
    assert torch.equal(sa, seg_a) and ia == info_a and torch.equal(sb, seg_b) and ib == info_b


def test_forward_packed_rejects_before_running(built):
    """A model off CUDA (or in fp32) cannot build the slot on the device; a slot too small for an output is named with its bytes."""
    sys.path.insert(0, ROOT)
    from ape_b200 import configs
    from ape_b200.modeling import build_model

    m = build_model(configs.MINI)
    name = m.dataset_names[0]
    m.dataset_stuff = {name: ([f"c{i}" for i in range(6)], [f"c{i}" for i in range(6, 12)], "thing+stuff")}
    m.set_eval_dataset(name)
    m.panoptic_on = True
    inp = [{"image": torch.zeros(3, 32, 32, dtype=torch.uint8), "height": 64, "width": 48}]
    with pytest.raises(ValueError, match="16-bit engine_dtype"):
        m.forward_packed(inp)
    m.dataset_stuff = {}
    with pytest.raises(RuntimeError, match="dataset_stuff"):
        m.forward_packed(inp)
    from ape_b200 import ops

    assert ops.panoptic_slot_bytes_needed(300, (1024, 768)) == 32 + 12 * 300 + 2 * 1024 * 768
    assert ops.panoptic_slot_bytes_needed(1024, (1024, 1024)) <= m.panoptic_slot_bytes


def _gather_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from ape_b200 import parallel
    from test_semseg_pack_cpu import _label_map, _semantic_packed

    det, _ = _det(False, seed=rank)
    pan, _, _ = _pan_slot(20 + rank)
    out = parallel.gather_packed(_with_panoptic(_semantic_packed(rank, det, 1, _label_map(10 + rank)), pan), dst=0)
    if rank == 0:
        q.put([(o["instances"].pred_classes.tolist(), [e["label"] for e in o["sem_seg_rle"]], o["panoptic_seg"][0].numpy(),
                o["panoptic_seg"][1]) for o in out])
    else:
        assert out is None
    dist.barrier()
    dist.destroy_process_group()


def test_gather_of_the_panoptic_layout_over_gloo():
    """One gather of the 2-D uint8 tensor: rank 0 gets both ranks' detections, label codes and panoptic maps, unchanged."""
    sys.path.insert(0, ROOT)
    from test_semseg_pack_cpu import _label_map

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33100 + os.getpid() % 2000
    procs = [ctx.Process(target=_gather_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = q.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert len(res) == 2
    for rank in range(2):
        det, plain = _det(False, seed=rank)
        _, seg, info = _pan_slot(20 + rank)
        classes, labels, got_seg, got_info = res[rank]
        from ape_b200 import parallel

        assert classes == parallel.unpack_packed(plain)[0]["instances"].pred_classes.tolist()
        assert labels == np.unique(_label_map(10 + rank)).tolist()
        assert np.array_equal(got_seg, seg.numpy()) and got_info == info
