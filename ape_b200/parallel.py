"""Multi-GPU plumbing of the detection path: images shard one (or B/G) per GPU with no data-path
collective; the only exchange is ONE gather of fixed-shape packed detections per batch
(SURVEY.md §8e).  It replaces the reference's pickled `comm.gather(self._predictions, dst=0)` over a
gloo side group (ape/evaluation/lvis_evaluation.py:103-104) with a single tensor collective on the
job's own process group (NCCL over NVLink/NVSwitch on GPUs, gloo in the CPU tests)."""
from typing import List, Optional

import torch
import torch.distributed as dist

from .structures import Boxes, Instances

PACK_WIDTH = 8  # x1, y1, x2, y2, score, class, image_height, image_width


def shard(items: List, rank: int, world: int) -> List:
    """Contiguous, balanced split of a batch across ranks (rank r gets items [lo_r, hi_r))."""
    n = len(items)
    lo = (n * rank) // world
    hi = (n * (rank + 1)) // world
    return items[lo:hi]


def pack_detections(instances: List[Instances], max_det: int, device) -> torch.Tensor:
    """[len(instances), max_det + 1, PACK_WIDTH] fp32: row 0 holds the count, rows 1.. the detections."""
    out = torch.zeros((len(instances), max_det + 1, PACK_WIDTH), dtype=torch.float32, device=device)
    for i, inst in enumerate(instances):
        k = min(len(inst), max_det)
        out[i, 0, 0] = k
        if k:
            out[i, 1:k + 1, 0:4] = inst.pred_boxes.tensor[:k].to(device)
            out[i, 1:k + 1, 4] = inst.scores[:k].to(device)
            out[i, 1:k + 1, 5] = inst.pred_classes[:k].to(device=device, dtype=torch.float32)
        out[i, 0, 6], out[i, 0, 7] = float(inst.image_size[0]), float(inst.image_size[1])
    return out


def unpack_detections(packed: torch.Tensor) -> List[Instances]:
    res = []
    packed = packed.cpu()
    for p in packed:
        k = int(p[0, 0])
        res.append(Instances((int(p[0, 6]), int(p[0, 7])), pred_boxes=Boxes(p[1:k + 1, 0:4].clone()),
                             scores=p[1:k + 1, 4].clone(), pred_classes=p[1:k + 1, 5].to(torch.int64)))
    return res


def gather_detections(instances: List[Instances], max_det: int, device, dst: int = 0,
                      group: Optional[dist.ProcessGroup] = None) -> Optional[List[Instances]]:
    """One collective: every rank contributes the same number of images (pad with empty Instances if needed).
    Returns the concatenated per-image results on `dst` (rank order = image order), None elsewhere."""
    packed = pack_detections(instances, max_det, device)
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return unpack_detections(packed)
    world = dist.get_world_size(group)
    if dist.get_rank(group) == dst:
        bufs = [torch.empty_like(packed) for _ in range(world)]
        dist.gather(packed, bufs, dst=dst, group=group)
        return unpack_detections(torch.cat(bufs, 0))
    dist.gather(packed, None, dst=dst, group=group)
    return None


# ---- device-side path: no host round trip before the collective ---------------------------------------------------
def unpack_packed(packed: torch.Tensor) -> List[dict]:
    """Rows of `DeformableDETRSegmVL.forward_packed` (any device) -> the reference's output list [{"instances": Instances}] on
    the host: the kept detections rescaled to the requested output size, clipped, empty boxes dropped (detectron2
    detector_postprocess).  One device->host copy for everything.
    fp32 [images, topk, 13]: boxes only.  uint8 [images, topk, 60 + slot] (instance masks): the same 13 columns as bytes, and
    `pred_masks_rle` = [{"size": [H, W], "counts": bytes}] per kept detection, as `model(inputs)` returns with
    `mask_format = "rle"`.  A slot that holds its mask as bits is pasted and encoded here (`ops.paste_masks_rle`).
    uint8 [images, 32 + topk * R + slot] (semantic label maps): per image a header of 8 int32 (topk, R, semantic slot kind,
    bytes used, output height, width, labels present, 0), its rows in one of the forms above (R = 52: the 13 fp32 columns), then
    its semantic slot; the dicts gain `sem_seg_rle` as `model(inputs)` returns it with `sem_seg_format = "rle"` (none when the
    dataset's entity turned the branch off).  A slot that holds the map as uint16 is encoded here (`ops.label_map_rle`); a slot
    that holds nothing raises ValueError."""
    if packed.dtype == torch.uint8 and packed.dim() == 2:
        return _unpack_packed_semantic(packed)
    if packed.dtype == torch.uint8:
        return _unpack_packed_masks(packed)
    host = packed.to("cpu")
    return [_unpack_rows(p)[0] for p in host]


def _unpack_rows(p: torch.Tensor):
    """One image's [topk, 13] rows -> ({"instances", "num_candidates"}, indices of the kept slots)."""
    nk = int(p[0, 8])
    h, w, oh, ow = (float(v) for v in p[0, 9:13])
    r = p[:nk]
    b = r[:, :4].clone()
    if h > 0 and w > 0:
        b[:, 0::2] *= ow / w
        b[:, 1::2] *= oh / h
    b = torch.stack((b[:, 0].clamp(min=0, max=ow), b[:, 1].clamp(min=0, max=oh), b[:, 2].clamp(min=0, max=ow),
                     b[:, 3].clamp(min=0, max=oh)), dim=-1)
    keep = ((b[:, 2] - b[:, 0]) > 0) & ((b[:, 3] - b[:, 1]) > 0)
    return ({"instances": Instances((int(oh), int(ow)), pred_boxes=Boxes(b[keep]), scores=r[keep, 4].clone(),
                                    pred_classes=r[keep, 5].to(torch.int64), query_index=r[keep, 6].to(torch.int64)),
             "num_candidates": int(p[0, 7])}, keep.nonzero()[:, 0].tolist())


MASK_PACK_HEAD = 60  # = ops.MASK_PACK_HEAD: 13 fp32 columns, int32 slot kind, int32 slot length
MASK_SLOT_CHARS, MASK_SLOT_BITS = 1, 2  # = ops.MASK_SLOT_*


def unpack_mask_bits(slot_bytes) -> torch.Tensor:
    """The bits form of mask slots (pixel y * S + x at byte >> 3, bit & 7): [..., S*S/8] bytes -> bool [..., S, S]."""
    import numpy as np

    a = np.frombuffer(bytes(slot_bytes), dtype=np.uint8) if isinstance(slot_bytes, (bytes, bytearray)) else np.asarray(slot_bytes)
    S = int(round((8 * a.shape[-1]) ** 0.5))
    bits = np.unpackbits(a, axis=-1, bitorder="little")[..., : S * S]
    return torch.from_numpy(bits.reshape(a.shape[:-1] + (S, S)).astype(bool))


def _unpack_packed_masks(packed: torch.Tensor, device=None) -> List[dict]:
    host = packed.to("cpu")
    rows = host[..., :52].contiguous().view(torch.float32)                     # [images, topk, 13]
    words = host[..., 52:MASK_PACK_HEAD].contiguous().view(torch.int32).numpy()  # [images, topk, 2]: kind, length
    raw = host.numpy()
    out = []
    for i in range(host.shape[0]):
        res, kept = _unpack_rows(rows[i])
        inst = res["instances"]
        size = [inst.image_size[0], inst.image_size[1]]
        rles, bits = [], []
        for j, k in enumerate(kept):
            kind, n = int(words[i, k, 0]), int(words[i, k, 1])
            if kind == MASK_SLOT_CHARS:
                rles.append({"size": size, "counts": raw[i, k, MASK_PACK_HEAD:MASK_PACK_HEAD + n].tobytes()})
                continue
            if kind != MASK_SLOT_BITS:
                raise ValueError(f"unpack_packed: image {i} slot {k} is kept but holds no mask (kind {kind})")
            rles.append(None)
            bits.append((j, k, n))
        if bits:  # masks that travelled as bits: pasted and encoded with the kernels `model(inputs)` uses
            from . import ops

            n = bits[0][2]
            masks = unpack_mask_bits(raw[i, [k for _, k, _ in bits], MASK_PACK_HEAD:MASK_PACK_HEAD + n])
            dev = device if device is not None else packed.device if packed.is_cuda else torch.device("cuda")
            boxes = inst.pred_boxes.tensor[[j for j, _, _ in bits]]
            for (j, _, _), rle in zip(bits, ops.paste_masks_rle(masks.to(dev), boxes.to(dev), inst.image_size, 0.5)):
                rles[j] = rle
        inst.pred_masks_rle = rles
        out.append(res)
    return out


SEM_PACK_HEAD = 32  # = ops.SEM_PACK_HEAD
SEM_SLOT_NONE, SEM_SLOT_CODES, SEM_SLOT_MAP, SEM_SLOT_OVER = 0, 1, 2, 3  # = ops.SEM_SLOT_*


def _unpack_packed_semantic(packed: torch.Tensor) -> List[dict]:
    import numpy as np

    host = packed.to("cpu")
    raw = host.numpy()
    dev = packed.device if packed.is_cuda else torch.device("cuda")
    out = []
    for i in range(raw.shape[0]):
        topk, R, kind, n, oh, ow, P, _ = raw[i, :SEM_PACK_HEAD].view(np.int32).tolist()
        det = host[i, SEM_PACK_HEAD:SEM_PACK_HEAD + topk * R].reshape(1, topk, R)
        if R == 4 * 13:
            res = _unpack_rows(det[0].contiguous().view(torch.float32))[0]
        else:
            res = _unpack_packed_masks(det, dev)[0]
        slot = raw[i, SEM_PACK_HEAD + topk * R:]
        if kind == SEM_SLOT_CODES:
            from . import ops

            res["sem_seg_rle"] = ops._label_rle_table(slot[:n], P, oh, ow)
        elif kind == SEM_SLOT_MAP:
            from . import ops

            label = torch.from_numpy(slot[:2 * oh * ow].view(np.uint16).astype(np.int64).reshape(oh, ow))
            res["sem_seg_rle"] = ops.label_map_rle(label.to(dev))
        elif kind != SEM_SLOT_NONE:
            raise ValueError(f"unpack_packed: the semantic label map of image {i} ({oh} x {ow}) needs {n} bytes and did not fit its "
                             f"slot of {slot.size} bytes; raise model.sem_seg_slot_bytes")
        out.append(res)
    return out


def gather_packed(packed: torch.Tensor, dst: int = 0, group: Optional[dist.ProcessGroup] = None) -> Optional[List[dict]]:
    """ONE collective on the packed DEVICE tensor (NCCL gather on the compute stream; gloo in the CPU tests): non-destination
    ranks neither copy to the host nor synchronise.  Returns the per-image results of all ranks on `dst`, None elsewhere."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return unpack_packed(packed)
    world = dist.get_world_size(group)
    if dist.get_rank(group) == dst:
        buf = torch.empty((world,) + tuple(packed.shape), dtype=packed.dtype, device=packed.device)
        dist.gather(packed, list(buf.unbind(0)), dst=dst, group=group)
        return unpack_packed(buf.flatten(0, 1))
    dist.gather(packed, None, dst=dst, group=group)
    return None
