"""CPU: the semantic form of `forward_packed` (a 32-byte header per image, the image's detection rows, its semantic slot) through
`parallel.unpack_packed` on hand-built tensors, `ops.label_map_from_rle` against the oracle's restatement of cocoapi's
run-length code (oracle/rle.py), and one gloo gather of the semantic form between two processes.  Slots that carry the map as
uint16 are encoded by the device kernel on the receiving side; the GPU tests cover them."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import ROOT

SLOT = 4096


def _label_map(seed, h=30, w=40, n=5):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[:h, :w]
    seeds = rng.random((n, 2)) * [h, w]
    d = (yy[None] - seeds[:, 0, None, None]) ** 2 + (xx[None] - seeds[:, 1, None, None]) ** 2
    return (rng.permutation(20)[:n][d.argmin(0)]).astype(np.int64)


def _codes_body(L):
    """The codes body of a slot: P x (int32 label, character offset, length), then the characters."""
    from oracle import rle as R

    labels = np.unique(L)
    codes = [R.encode((L == c).astype(np.uint8))["counts"] for c in labels]
    table, off = [], 0
    for c, s in zip(labels, codes):
        table += [int(c), off, len(s)]
        off += len(s)
    return np.array(table, np.int32).view(np.uint8).tobytes() + b"".join(codes), labels, codes


def _semantic_packed(seed, det, kind, L=None, slot=SLOT):
    """[1, 32 + topk * R + slot] uint8 around the detection rows `det` [topk, R] (uint8) with a semantic slot of `kind`."""
    topk, R = det.shape
    body, P = b"", 0
    oh, ow = (30, 40) if L is None else L.shape
    if kind == 1:
        body, labels, _ = _codes_body(L)
        P = len(labels)
    n = len(body) if kind == 1 else 2 * oh * ow if kind == 3 else 0
    hdr = np.array([topk, R, kind, n, oh, ow, P, 0], np.int32).view(np.uint8)
    buf = np.zeros((1, 32 + topk * R + slot), np.uint8)
    buf[0, :32] = hdr
    buf[0, 32:32 + topk * R] = det.reshape(-1)
    buf[0, 32 + topk * R:32 + topk * R + len(body)] = np.frombuffer(body, np.uint8)
    if kind == 0:
        buf[0, 32 + topk * R:] = 0
    return torch.from_numpy(buf)


def _box_rows(seed, topk=5, nk=3):
    from test_mask_pack_cpu import _packed

    _, rows, _ = _packed(seed, nk, topk=topk)
    return rows


@pytest.mark.parametrize("masks", [False, True])
def test_codes_slot_round_trip(masks):
    sys.path.insert(0, ROOT)
    from ape_b200 import parallel
    from oracle import rle as R
    from test_mask_pack_cpu import _packed

    packed_masks, rows, _ = _packed(5, 4)
    det = packed_masks[0].numpy() if masks else rows[0].numpy().view(np.uint8).reshape(rows.shape[1], 52)
    L = _label_map(1)
    got = parallel.unpack_packed(_semantic_packed(1, det, 1, L))[0]
    want = parallel.unpack_packed(packed_masks if masks else rows)[0]
    gi, wi = got["instances"], want["instances"]
    assert got["num_candidates"] == want["num_candidates"]
    assert torch.equal(gi.pred_boxes.tensor, wi.pred_boxes.tensor) and torch.equal(gi.scores, wi.scores)
    assert torch.equal(gi.pred_classes, wi.pred_classes) and torch.equal(gi.query_index, wi.query_index)
    if masks:
        assert [r["counts"] for r in gi.pred_masks_rle] == [r["counts"] for r in wi.pred_masks_rle]
    rle = got["sem_seg_rle"]
    assert [e["label"] for e in rle] == np.unique(L).tolist()
    for e in rle:
        assert e["segmentation"]["size"] == [30, 40]
        assert e["segmentation"]["counts"] == R.encode((L == e["label"]).astype(np.uint8))["counts"]


def test_entity_gated_slot_adds_nothing():
    sys.path.insert(0, ROOT)
    from ape_b200 import parallel

    rows = _box_rows(2)
    det = rows[0].numpy().view(np.uint8).reshape(rows.shape[1], 52)
    got = parallel.unpack_packed(_semantic_packed(2, det, 0))[0]
    assert "sem_seg_rle" not in got
    assert torch.equal(got["instances"].pred_boxes.tensor, parallel.unpack_packed(rows)[0]["instances"].pred_boxes.tensor)


def test_slot_that_holds_nothing_raises():
    sys.path.insert(0, ROOT)
    from ape_b200 import parallel

    rows = _box_rows(3)
    det = rows[0].numpy().view(np.uint8).reshape(rows.shape[1], 52)
    ok = _semantic_packed(3, det, 1, _label_map(3))
    bad = _semantic_packed(3, det, 3, slot=ok.shape[1] - 32 - 5 * 52)
    with pytest.raises(ValueError, match=r"image 1 .*2400 bytes.*sem_seg_slot_bytes"):
        parallel.unpack_packed(torch.cat([ok, bad], 0))


def test_label_map_from_rle_round_trips():
    sys.path.insert(0, ROOT)
    from ape_b200 import ops
    from oracle import rle as R

    rng = np.random.default_rng(0)
    maps = [_label_map(4), rng.integers(0, 7, (13, 9)), np.full((5, 6), 3), np.zeros((1, 1), np.int64),
            rng.integers(0, 5000, (17, 1))]
    L = np.zeros((8, 8), np.int64)
    L[-1, -1] = 9
    maps.append(L)
    for L in maps:
        L = np.asarray(L, np.int64)
        rle = [{"label": int(c), "segmentation": R.encode((L == c).astype(np.uint8))} for c in np.unique(L)]
        back = ops.label_map_from_rle(rle)
        assert back.dtype == np.int64 and back.shape == L.shape
        assert np.array_equal(back, L)


def _gather_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from ape_b200 import parallel

    rows = _box_rows(rank)
    det = rows[0].numpy().view(np.uint8).reshape(rows.shape[1], 52)
    out = parallel.gather_packed(_semantic_packed(rank, det, 1, _label_map(10 + rank)), dst=0)
    if rank == 0:
        q.put([(o["instances"].pred_classes.tolist(), [(e["label"], e["segmentation"]["counts"]) for e in o["sem_seg_rle"]])
               for o in out])
    else:
        assert out is None
    dist.barrier()
    dist.destroy_process_group()


def test_gather_of_the_semantic_layout_over_gloo():
    """One gather of the 2-D uint8 tensor: rank 0 gets both ranks' detections and label codes, unchanged."""
    sys.path.insert(0, ROOT)
    from ape_b200 import parallel

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31100 + os.getpid() % 2000
    procs = [ctx.Process(target=_gather_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = q.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert len(res) == 2
    for rank in range(2):
        rows = _box_rows(rank)
        det = rows[0].numpy().view(np.uint8).reshape(rows.shape[1], 52)
        want = parallel.unpack_packed(_semantic_packed(rank, det, 1, _label_map(10 + rank)))[0]
        classes, codes = res[rank]
        assert classes == want["instances"].pred_classes.tolist()
        assert codes == [(e["label"], e["segmentation"]["counts"]) for e in want["sem_seg_rle"]]
