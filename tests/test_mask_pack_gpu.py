"""GPU: instance masks in the packed device results (ape_mask_pack, `forward_packed` with `test_mask_on`) against the host-
synchronised path they replace: `ops.mask_crop_and_resize` + detector_postprocess's rescale and clip + `ops.paste_masks_rle`, and
at model level `model(inputs)` with `mask_format = "rle"`.  Character slots must equal those codes byte for byte; bits slots must
hold the 128 x 128 mask and re-encode to the same bytes."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _logits(B, Q, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B * Q, 1, max(h // 8, 2), max(w // 8, 2), generator=g)
    return (F.interpolate(x, size=(h, w), mode="bicubic", align_corners=False)[:, 0] * 4.0).view(B, Q, h, w).contiguous().to(DEV)


def _rows(B, topk, Q, image_sizes, out_sizes, nks, seed):
    """Selection rows [B, topk, 13] with random boxes: some partly outside the image, some empty once clipped (a zero-width box
    and a box entirely right of the image).  Rows past nk hold valid but different values that must not be read."""
    g = torch.Generator().manual_seed(seed)
    rows = torch.zeros(B, topk, 13)
    for b, ((h, w), (oh, ow), nk) in enumerate(zip(image_sizes, out_sizes, nks)):
        c = torch.rand(topk, 2, generator=g) * torch.tensor([w, h])
        wh = torch.rand(topk, 2, generator=g) * torch.tensor([w, h]) * 0.7 + 1.0
        box = torch.cat([c - wh / 2, c + wh / 2], 1)
        if topk > 3:
            box[1, 2] = box[1, 0]                                                # zero width
            box[2] = torch.tensor([w + 3.0, 1.0, w + 9.0, h / 2])                # right of the image: empty after the clip
            box[3] = torch.tensor([-10.0, -10.0, w + 10.0, h + 10.0])            # over every edge
        rows[b, :, :4] = box
        rows[b, :, 4] = torch.rand(topk, generator=g)
        rows[b, :, 5] = torch.randint(0, 50, (topk,), generator=g).float()
        rows[b, :, 6] = torch.randint(0, Q, (topk,), generator=g).float()
        rows[b, :, 7], rows[b, :, 8] = 1000.0, float(nk)
        rows[b, :, 9:13] = torch.tensor([float(h), float(w), float(oh), float(ow)])
    return rows.to(DEV)


def _reference(logits, rows, out_sizes, padded_hw):
    """The path of `model(inputs)`: crop the kept queries, rescale and clip as detector_postprocess, drop empty boxes, paste and
    encode.  Per image: (indices of the kept slots, their codes)."""
    from ape_b200 import ops

    res = []
    for b, (oh, ow) in enumerate(out_sizes):
        r = rows[b]
        nk = int(r[0, 8])
        h, w = float(r[0, 9]), float(r[0, 10])
        box = r[:nk, :4].clone()
        box[:, 0::2] *= ow / w
        box[:, 1::2] *= oh / h
        box = torch.stack((box[:, 0].clamp(min=0, max=ow), box[:, 1].clamp(min=0, max=oh), box[:, 2].clamp(min=0, max=ow),
                           box[:, 3].clamp(min=0, max=oh)), dim=-1)
        keep = ((box[:, 2] - box[:, 0]) > 0) & ((box[:, 3] - box[:, 1]) > 0)
        crop = ops.mask_crop_and_resize(logits[b], r[:nk, 6].to(torch.int64), r[:nk, :4], padded_hw, 128)
        res.append((keep.nonzero()[:, 0].tolist(), crop[keep], ops.paste_masks_rle(crop[keep], box[keep], (oh, ow), 0.5)))
    return res


def _check(out, logits, rows, out_sizes, padded_hw, slot):
    """Every slot against the reference; returns the number of character and bits slots."""
    from ape_b200 import ops, parallel

    topk = rows.shape[1]
    assert out.dtype == torch.uint8 and tuple(out.shape) == (rows.shape[0], topk, ops.MASK_PACK_HEAD + slot)
    host = out.cpu()
    assert torch.equal(host[..., :52].contiguous().view(torch.float32), rows.cpu())
    words = host[..., 52:60].contiguous().view(torch.int32)
    n = {ops.MASK_SLOT_CHARS: 0, ops.MASK_SLOT_BITS: 0}
    for b, (kept, crop, rles) in enumerate(_reference(logits, rows, out_sizes, padded_hw)):
        for k in range(topk):
            kind, ln = int(words[b, k, 0]), int(words[b, k, 1])
            body = host[b, k, 60:]
            if k not in kept:
                assert kind == ops.MASK_SLOT_EMPTY and ln == 0 and not body.any(), (b, k)
                continue
            j = kept.index(k)
            assert not body[ln:].any()
            if kind == ops.MASK_SLOT_CHARS:
                assert bytes(body[:ln].numpy()) == rles[j]["counts"], (b, k)
            else:
                assert kind == ops.MASK_SLOT_BITS and ln == 2048 and len(rles[j]["counts"]) > slot, (b, k, kind)
                assert torch.equal(parallel.unpack_mask_bits(body[:ln].numpy()), crop[j].cpu()), (b, k)
            n[kind] += 1
        got = parallel.unpack_packed(out[b:b + 1])[0]["instances"]
        assert [r["counts"] for r in got.pred_masks_rle] == [r["counts"] for r in rles]
        assert all(r["size"] == [out_sizes[b][0], out_sizes[b][1]] for r in got.pred_masks_rle)
    return n[ops.MASK_SLOT_CHARS], n[ops.MASK_SLOT_BITS]


@pytest.mark.parametrize("out_hw", [(1, 1), (480, 640), (1024, 768), (777, 1333), (4000, 3000)])
@pytest.mark.parametrize("nk", ["0", "1", "topk"])
def test_slots_equal_the_host_path(built, out_hw, nk):
    from ape_b200 import ops

    topk, Q = 24, 60
    logits = _logits(1, Q, 256, 256, seed=out_hw[0])
    rows = _rows(1, topk, Q, [(1024, 768)], [out_hw], [{"0": 0, "1": 1, "topk": topk}[nk]], seed=out_hw[1])
    out = ops.mask_pack(logits, rows, [out_hw], (1024, 1024), 4096)
    chars, bits = _check(out, logits, rows, [out_hw], (1024, 1024), 4096)
    print(f"  {out_hw} nk={nk}: {chars} character slots, {bits} bits slots")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
def test_both_slot_kinds_give_the_same_codes(built, dtype):
    """Two images of different sizes; a 2048-byte slot sends the long codes as bits, a 64 KiB slot sends every code as
    characters: unpacked, both are the reference's codes."""
    from ape_b200 import parallel, ops

    topk, Q = 40, 80
    sizes, outs = [(1024, 768), (600, 1000)], [(2048, 1536), (300, 500)]
    logits = _logits(2, Q, 256, 256, seed=5).to(dtype)
    rows = _rows(2, topk, Q, sizes, outs, [topk, 31], seed=6)
    counts = {}
    for slot in (2048, 65536):
        out = ops.mask_pack(logits, rows, outs, (1024, 1024), slot)
        chars, bits = _check(out, logits, rows, outs, (1024, 1024), slot)
        print(f"  slot {slot}: {chars} character slots, {bits} bits slots")
        assert chars > 0 and (bits > 0) == (slot == 2048)
        counts[slot] = [[r["counts"] for r in o["instances"].pred_masks_rle] for o in parallel.unpack_packed(out)]
    assert counts[2048] == counts[65536]


def test_graph_replay_and_no_host_synchronisation(built):
    from ape_b200 import ops

    topk, Q = 30, 50
    outs = [(1024, 768), (480, 640)]
    inputs = [(_logits(2, Q, 256, 256, seed=s), _rows(2, topk, Q, [(1024, 768), (960, 1280)], outs, [topk, 17], seed=s))
              for s in (1, 2)]
    static_l, static_r = inputs[0][0].clone(), inputs[0][1].clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.mask_pack(static_l, static_r, outs, (1024, 1280), 4096)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        static_out = ops.mask_pack(static_l, static_r, outs, (1024, 1280), 4096)
    for logits, rows in reversed(inputs):
        static_l.copy_(logits)
        static_r.copy_(rows)
        g.replay()
        assert torch.equal(static_out, ops.mask_pack(logits, rows, outs, (1024, 1280), 4096))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = ops.mask_pack(inputs[1][0], inputs[1][1], outs, (1024, 1280), 4096)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    _check(out, inputs[1][0], inputs[1][1], outs, (1024, 1280), 4096)


def test_arguments_are_checked(built):
    from ape_b200 import ops

    logits = _logits(1, 10, 32, 32, seed=0)
    rows = _rows(1, 4, 10, [(128, 128)], [(64, 64)], [4], seed=0)
    with pytest.raises(RuntimeError, match="slot"):
        ops.mask_pack(logits, rows, [(64, 64)], (128, 128), 1024)  # cannot hold the 2048 bytes of bits
    with pytest.raises(RuntimeError, match="slot"):
        ops.mask_pack(logits, rows, [(64, 64)], (128, 128), 4098)
    with pytest.raises(RuntimeError, match="output size"):
        ops.mask_pack(logits, rows, [(0, 64)], (128, 128), 4096)
    with pytest.raises(RuntimeError, match="rows"):
        ops.mask_pack(logits, rows.double(), [(64, 64)], (128, 128), 4096)


# ---- model level ---------------------------------------------------------------------------------------------------------
def _model(spec_name):
    import copy

    from ape_b200 import configs
    from ape_b200.modeling import build_model
    from oracle import synth

    if spec_name == "MINI":
        model = build_model(configs.MINI)
        synth.fill_state_dict(model)
    else:  # APE-L_D with bench.py's weights and score threshold (about 500 candidates of 1203 names x 900 queries)
        spec = copy.deepcopy(configs.APE_L_D)
        spec["test_score_thresh"] = 0.0123
        model = build_model(spec, num_text=1203)
        synth.fill_state_dict(model)
        synth.suppress_invalid_anchor_logits(model)
    model = model.to(DEV).eval()
    model.test_mask_on = True
    model.mask_format = "rle"
    return model


def _same(got, want):
    from ape_b200 import parallel

    got = parallel.unpack_packed(got)
    assert len(got) == len(want)
    for g, w in zip(got, want):
        g, w = g["instances"], w["instances"]
        assert g.image_size == w.image_size and len(g) == len(w)
        assert torch.equal(g.pred_boxes.tensor, w.pred_boxes.tensor) and torch.equal(g.scores, w.scores)
        assert torch.equal(g.pred_classes, w.pred_classes) and torch.equal(g.query_index, w.query_index)
        assert [r["size"] for r in g.pred_masks_rle] == [r["size"] for r in w.pred_masks_rle]
        assert [r["counts"] for r in g.pred_masks_rle] == [r["counts"] for r in w.pred_masks_rle]
    return sum(len(o["instances"]) for o in want)


def _images(spec_name, B, seed):
    from oracle import synth

    if spec_name == "MINI":
        sizes = [(56, 64, 112, 128), (48, 60, 95, 131)][:B]
    else:
        sizes = [(1024, 768, 1024, 768), (768, 1024, 600, 800)][:B]
    return [{"image": synth.image(h, w, seed=seed + i), "height": oh, "width": ow} for i, (h, w, oh, ow) in enumerate(sizes)]


@pytest.mark.parametrize("spec_name,dtype,graphs,B", [
    ("MINI", torch.float16, True, 1), ("MINI", torch.float16, False, 2), ("MINI", torch.bfloat16, True, 2),
    ("MINI", torch.bfloat16, False, 1), ("MINI", torch.float32, False, 2),
    ("APE_L_D", torch.float16, True, 1), ("APE_L_D", torch.bfloat16, False, 1), ("APE_L_D", torch.float16, True, 2)])
def test_forward_packed_equals_the_model(built, spec_name, dtype, graphs, B):
    model = _model(spec_name)
    model.engine_dtype, model.use_cuda_graphs = dtype, graphs
    for seed in (3, 4):  # the second call replays the graphs captured by the first
        inputs = _images(spec_name, B, seed)
        want = model(inputs)
        n = _same(model.forward_packed(inputs), want)
        print(f"  {spec_name} {dtype} graphs={graphs} B={B} seed {seed}: {n} detections with masks")
        assert n > 0


def test_packed_masks_add_no_host_synchronisation(built):
    """After warm-up, with the images already on the device: if the boxes-only `forward_packed` runs under
    set_sync_debug_mode("error"), so must the one with masks; the mask stage alone runs under it in any case (above)."""
    model = _model("MINI")
    model.engine_dtype, model.use_cuda_graphs = torch.float16, True
    inputs = [dict(x, image=x["image"].to(DEV)) for x in _images("MINI", 2, 9)]
    results = {}
    for masks in (False, True):
        model.test_mask_on = masks
        for _ in range(2):
            model.forward_packed(inputs)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            model.forward_packed(inputs)
            results[masks] = None
        except RuntimeError as e:
            results[masks] = str(e).splitlines()[0]
        finally:
            torch.cuda.set_sync_debug_mode("default")
    print(f"  boxes only: {results[False] or 'no synchronisation'}; with masks: {results[True] or 'no synchronisation'}")
    if results[False] is None:
        assert results[True] is None


def _nccl_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    sys.path.insert(0, ROOT)
    import torch.distributed as dist

    torch.cuda.set_device(rank)
    global DEV
    DEV = f"cuda:{rank}"
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(DEV))
    from ape_b200 import parallel

    model = _model("MINI")
    model.engine_dtype, model.use_cuda_graphs = torch.float16, True
    inputs = _images("MINI", 2, 20 + 2 * rank)
    want = model(inputs)
    q.put(("want", rank, [[(o["instances"].pred_boxes.tensor.tolist(), o["instances"].pred_classes.tolist(),
                            [r["counts"] for r in o["instances"].pred_masks_rle]) for o in want]]))
    out = parallel.gather_packed(model.forward_packed(inputs), dst=0)
    if rank == 0:
        q.put(("got", 0, [[(o["instances"].pred_boxes.tensor.tolist(), o["instances"].pred_classes.tolist(),
                            [r["counts"] for r in o["instances"].pred_masks_rle]) for o in out]]))
    else:
        assert out is None
    dist.barrier()
    dist.destroy_process_group()


def test_two_gpu_gather_carries_the_masks(built):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 visible GPUs for an NCCL gather between two processes")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + os.getpid() % 2000
    procs = [ctx.Process(target=_nccl_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    msgs = [q.get(timeout=600) for _ in range(3)]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    want = {r: v[0] for k, r, v in msgs if k == "want"}
    got = [v[0] for k, _, v in msgs if k == "got"][0]
    assert got == want[0] + want[1]
