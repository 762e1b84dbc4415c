"""Panoptic merging of mask predictions (`DeformableDETRSegmVL._postprocess_panoptic`,
ape/modeling/ape_deta/deformable_detr_segm_vl.py:919-998), device-agnostic and without per-segment host round trips.

The reference walks the kept queries in a Python loop and calls `.item()` three times per query (areas of three masks).
Here the three areas of every query come from two `bincount`s over the per-pixel argmax, ONE small device->host copy
brings them over, the (inherently sequential, tiny) segment-id bookkeeping runs on those K-element arrays, and a lookup
table paints the segment ids.  Same decisions, same ids, same `segments_info`.

`postprocess_panoptic_winners` is the same merge for 16-bit engine mode on CUDA: one kernel (csrc/panoptic.cu) resamples
the mask logits per pixel and yields the winners and the three areas directly, so no [K, H, W] stack is formed."""
from typing import Dict, Iterable, List, Tuple

import torch
import torch.nn.functional as F


def _query_scores(mask_cls: torch.Tensor, cfg: Dict, col_ok=None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """(scores, labels, keep) of all K queries: the class scores and labels the merge ranks them by, and the queries above
    object_mask_threshold (on the sigmoid scores, before the transform_eval softmax).  col_ok: bool [N], the class columns of a
    padded prompt; the others never win the maximum and take no part in the softmax."""
    sig = mask_cls.sigmoid()
    if col_ok is not None:
        sig = sig.masked_fill(~col_ok, float("-inf"))
    scores, labels = sig.max(-1)
    keep = scores > cfg["object_mask_threshold"]
    if cfg["transform_eval"]:
        scores, labels = F.softmax(sig / cfg["pano_temp"], dim=-1).max(-1)
    return scores, labels, keep


def _segments(stats: torch.Tensor, thing_ids: Iterable[int], num_thing_classes: int, stuff_first_is_things: bool,
              overlap_threshold: float) -> Tuple[torch.Tensor, List[Dict]]:
    """The segment-id bookkeeping of the reference's loop over the kept queries.  stats: host int64 [4, K] = (mask_area,
    original_area, inter_area, class) per kept query -> (lut int32 [K]: segment id of each query's pixels, 0 = none,
    segments_info)."""
    thing_ids = set(int(t) for t in thing_ids)
    lut = [0] * int(stats.shape[1])
    segments_info, stuff_memory, current = [], {}, 0
    for k, (area, orig, inter, pred_class) in enumerate(zip(*stats.tolist())):  # Python ints: no tensor indexing per query
        isthing = pred_class in thing_ids
        if area > 0 and orig > 0 and inter > 0:
            if area / orig < overlap_threshold:
                continue
            if not isthing:
                if pred_class in stuff_memory:
                    lut[k] = stuff_memory[pred_class]
                    continue
                stuff_memory[pred_class] = current + 1
            current += 1
            lut[k] = current
            if not isthing and stuff_first_is_things:
                pred_class = pred_class - num_thing_classes + 1
            segments_info.append({"id": current, "isthing": bool(isthing), "category_id": int(pred_class)})
    return torch.tensor(lut, dtype=torch.int32), segments_info


def postprocess_panoptic(mask_cls: torch.Tensor, mask_pred: torch.Tensor, image_size: Tuple[int, int], height: int,
                         width: int, thing_ids: Iterable[int], num_thing_classes: int, stuff_first_is_things: bool,
                         cfg: Dict) -> Tuple[torch.Tensor, List[Dict]]:
    """mask_cls [K, N_t] class logits and mask_pred [K, H, W] mask logits (padded-image resolution) of the queries kept
    for one image -> (panoptic_seg int32 [height, width], segments_info).  cfg: prob, pano_temp, transform_eval,
    object_mask_threshold, overlap_threshold (the reference's `panoptic_configs`)."""
    prob = cfg["prob"]
    # sem_seg_postprocess: crop to the unpadded size, bilinear resize to the output size
    m = mask_pred[:, : image_size[0], : image_size[1]].expand(1, -1, -1, -1)
    m = F.interpolate(m, size=(height, width), mode="bilinear", align_corners=False)[0]
    scores, labels, keep = _query_scores(mask_cls, cfg)
    m = m.sigmoid()
    cur_scores, cur_classes, cur_masks = scores[keep], labels[keep], m[keep]
    K = int(cur_classes.shape[0])
    panoptic_seg = torch.zeros((height, width), dtype=torch.int32, device=m.device)
    if K == 0:
        return panoptic_seg, []
    cur_mask_ids = (cur_scores.view(-1, 1, 1) * cur_masks).argmax(0)                      # [h, w] winner per pixel
    winner_prob = torch.gather(cur_masks, 0, cur_mask_ids[None])[0]                        # mask prob of the winner
    solid = winner_prob >= prob                                                            # winner is also >= prob there
    mask_area = torch.bincount(cur_mask_ids.flatten(), minlength=K)                        # (cur_mask_ids == k).sum()
    inter_area = torch.bincount(cur_mask_ids[solid], minlength=K)                          # ((ids == k) & (m_k >= prob)).sum()
    original_area = (cur_masks >= prob).flatten(1).sum(1)                                  # (m_k >= prob).sum()
    stats = torch.stack([mask_area, original_area, inter_area, cur_classes.to(mask_area.dtype)]).cpu()  # the one D2H
    lut, segments_info = _segments(stats, thing_ids, num_thing_classes, stuff_first_is_things, cfg["overlap_threshold"])
    painted = lut.to(m.device)[cur_mask_ids]
    panoptic_seg = torch.where(solid, painted, panoptic_seg)
    return panoptic_seg, segments_info


def postprocess_panoptic_winners(mask_cls: torch.Tensor, mask_logits: torch.Tensor, query_index: torch.Tensor,
                                 padded_hw: Tuple[int, int], image_size: Tuple[int, int], height: int, width: int,
                                 thing_ids: Iterable[int], num_thing_classes: int, stuff_first_is_things: bool,
                                 cfg: Dict) -> Tuple[torch.Tensor, List[Dict]]:
    """postprocess_panoptic(mask_cls, F.interpolate(mask_logits[query_index][None].float(), padded_hw, mode="bilinear")[0],
    image_size, height, width, ...) without the mask stacks: mask_logits [Q, h, w] CUDA (fp32 / fp16 / bf16), query_index
    [K] int64, mask_cls [K, N_t].  `ops.panoptic_winners` finds every pixel's winner and the three areas of every query;
    queries under object_mask_threshold get the score -inf, which leaves them out without compacting the query list on the
    device.  The counts, classes and keep mask come over in ONE device->host copy; the bookkeeping is postprocess_panoptic's."""
    from .. import ops

    scores, labels, keep = _query_scores(mask_cls, cfg)
    ids, counts = ops.panoptic_winners(mask_logits, query_index, torch.where(keep, scores, float("-inf")), padded_hw,
                                       image_size, (height, width), cfg["prob"])
    stats = torch.cat([counts, labels.to(torch.int32)[None], keep.to(torch.int32)[None]]).cpu().long()  # the one D2H
    kept = stats[4].nonzero()[:, 0]
    mask_area, inter_area, original_area, classes = stats[:4, kept]
    lut, segments_info = _segments(torch.stack([mask_area, original_area, inter_area, classes]), thing_ids, num_thing_classes,
                                   stuff_first_is_things, cfg["overlap_threshold"])
    table = torch.zeros(int(query_index.numel()) + 1, dtype=torch.int32)  # table[1 + k]: segment id of query k; table[0] = 0
    table[1 + kept] = lut
    ids.add_(1)                                                             # -1 (not solid) -> 0
    panoptic_seg = torch.index_select(table.to(ids.device), 0, ids.view(-1)).view(height, width)
    return panoptic_seg, segments_info
