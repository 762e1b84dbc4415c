"""CPU: the byte layout of `forward_packed` with instance masks (13 fp32 columns, slot word, fixed-size slot) through
`parallel.unpack_packed`, the bits form of a slot, and one gloo gather of the uint8 tensor between two processes.  The slots are
built with the oracle's restatement of cocoapi's run-length code (oracle/rle.py)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import ROOT

SLOT = 512


def _packed(seed, nk, topk=5, size=(60, 80), out=(30, 40), slot=SLOT):
    """uint8 [1, topk, 60 + slot] with character slots for the first nk rows; slot 1 has a box that is empty after the rescale.
    Rows past nk carry junk that must be ignored.  Returns (packed, fp32 rows, {slot: mask})."""
    from oracle import rle as R

    g = torch.Generator().manual_seed(seed)
    rows = torch.zeros(topk, 13)
    h, w = size
    oh, ow = out
    x1, y1 = torch.rand(topk, generator=g) * w * 0.5, torch.rand(topk, generator=g) * h * 0.5
    rows[:, 0], rows[:, 1] = x1, y1
    rows[:, 2], rows[:, 3] = x1 + 4 + torch.rand(topk, generator=g) * w * 0.5, y1 + 4 + torch.rand(topk, generator=g) * h * 0.5
    rows[1, 2] = rows[1, 0]                                      # zero width: dropped with its mask
    rows[:, 4] = torch.linspace(0.9, 0.5, topk)
    rows[:, 5] = torch.arange(topk, dtype=torch.float32) + 10 * seed
    rows[:, 6] = torch.arange(topk, dtype=torch.float32) * 3
    rows[:, 7], rows[:, 8] = 17 + seed, nk
    rows[:, 9:13] = torch.tensor([float(h), float(w), float(oh), float(ow)])
    buf = np.zeros((1, topk, 60 + slot), np.uint8)
    buf[0, :, :52] = rows.numpy().view(np.uint8).reshape(topk, 52)
    rng = np.random.default_rng(seed)
    masks = {}
    for k in range(topk):
        if k >= nk:  # junk past the kept count
            buf[0, k, 52:60] = np.array([1, 9], np.int32).view(np.uint8)
            buf[0, k, 60:] = rng.integers(0, 256, slot)
            continue
        if k == 1:
            continue  # kind 0: the receiver drops this detection anyway
        m = rng.random((oh, ow)) < 0.02
        counts = R.counts_to_string(R.encode_counts(m))
        assert len(counts) <= slot
        buf[0, k, 52:60] = np.array([1, len(counts)], np.int32).view(np.uint8)
        buf[0, k, 60:60 + len(counts)] = np.frombuffer(counts, np.uint8)
        masks[k] = m
    return torch.from_numpy(buf), rows[None], masks


def test_layout_round_trip():
    sys.path.insert(0, ROOT)
    from ape_b200 import parallel
    from oracle import rle as R

    for nk in (0, 1, 4):
        packed, rows, masks = _packed(3, nk)
        got = parallel.unpack_packed(packed)[0]
        want = parallel.unpack_packed(rows)[0]  # the boxes-only layout of the same rows
        gi, wi = got["instances"], want["instances"]
        assert got["num_candidates"] == want["num_candidates"] == 20
        assert len(gi) == len(wi) == max(nk - (1 if nk > 1 else 0), 0)
        assert torch.equal(gi.pred_boxes.tensor, wi.pred_boxes.tensor) and torch.equal(gi.scores, wi.scores)
        assert torch.equal(gi.pred_classes, wi.pred_classes) and torch.equal(gi.query_index, wi.query_index)
        kept = [k for k in range(nk) if k != 1]
        assert len(gi.pred_masks_rle) == len(kept)
        for k, rle in zip(kept, gi.pred_masks_rle):
            assert rle["size"] == [30, 40]
            assert rle["counts"] == R.encode(masks[k])["counts"]
            assert np.array_equal(R.decode(rle), masks[k].astype(np.uint8))


def test_bits_slot_decodes_to_the_mask():
    sys.path.insert(0, ROOT)
    from ape_b200 import parallel

    rng = np.random.default_rng(0)
    for S in (128, 8):
        m = rng.random((S, S)) < 0.3
        slot = np.packbits(m.reshape(-1), bitorder="little")
        assert slot.size == S * S // 8
        assert torch.equal(parallel.unpack_mask_bits(slot.tobytes()), torch.from_numpy(m))
    # the kernel's order: pixel y * S + x is bit (x & 7) of byte (y * S + x) >> 3
    slot = np.zeros(2048, np.uint8)
    slot[(5 * 128 + 9) >> 3] = 1 << ((5 * 128 + 9) & 7)
    m = parallel.unpack_mask_bits(slot)
    assert m.sum() == 1 and bool(m[5, 9])


def _gather_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    sys.path.insert(0, ROOT)
    from ape_b200 import parallel

    packed, _, _ = _packed(rank, 3 + rank)
    out = parallel.gather_packed(packed, dst=0)
    if rank == 0:
        q.put([(len(o["instances"]), o["instances"].pred_classes.tolist(), [r["counts"] for r in o["instances"].pred_masks_rle])
               for o in out])
    else:
        assert out is None
    dist.barrier()
    dist.destroy_process_group()


def test_gather_of_the_mask_layout_over_gloo():
    """One gather of the uint8 tensor: rank 0 gets both ranks' detections and run-length codes, unchanged."""
    sys.path.insert(0, ROOT)
    from ape_b200 import parallel

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29100 + os.getpid() % 2000
    procs = [ctx.Process(target=_gather_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = q.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank in range(2):
        want = parallel.unpack_packed(_packed(rank, 3 + rank)[0])[0]["instances"]
        n, classes, counts = res[rank]
        assert n == len(want) == 2 + rank and classes == want.pred_classes.tolist()
        assert counts == [r["counts"] for r in want.pred_masks_rle]
