"""Meta-architecture of the engine: `DeformableDETRSegmVL`, its fusion-free subclass `DeformableDETRSegm` (+ `SomeThing`).

Mirror of ape/modeling/ape_deta/deformable_detr_segm_vl.py:33-164 (constructor), :166-726
(forward, inference branch), :728-750 (mask features), :759-810 (inference), :846-872
(pre/post-process), ape/modeling/ape_deta/deformable_detr.py:22-296 (base constructor),
ape/modeling/ape_deta/fast_rcnn.py:97-201 (threshold + class-aware NMS + top-k) and
ape/modeling/ape_deta/ape_deta.py:20-40 (`SomeThing`).  Same constructor keywords, same
`forward(batched_inputs, do_postprocess)` contract (list of dicts in, list of dicts with
"instances" out, results on CPU), same parameter names incl. the shared `class_embed` /
`bbox_embed` aliases under `transformer.decoder`.

Scope (SURVEY.md §8): inference (boxes, instance masks, semantic and panoptic maps) for "name", "phrase" / "text" and
"expression" prompts.  Training and mask prompts raise NotImplementedError (next rows of §8f) — loudly, never silently."""
import copy
import math
from typing import Dict, List

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F
import torchvision

from .. import ops
from ..layers import VisionLanguageAlign
from ..layers.common import MLP, ConvNorm, box_cxcywh_to_xyxy, inverse_sigmoid
from ..structures import Boxes, Instances


class PositionEmbeddingSine(nn.Module):
    """detrex PositionEmbeddingSine (SURVEY.md Appendix B)."""

    def __init__(self, num_pos_feats=64, temperature=10000, scale=2 * math.pi, eps=1e-6, offset=0.0, normalize=False):
        super().__init__()
        self.num_pos_feats, self.temperature, self.normalize = num_pos_feats, temperature, normalize
        self.scale, self.eps, self.offset = scale, eps, offset

    def dim_t(self, device):
        """The frequency table [num_pos_feats] fp32; ops.pad_geometry takes it from here, so its rounding is torch's."""
        dim_t = torch.arange(self.num_pos_feats, dtype=torch.float32, device=device)
        return self.temperature ** (2 * torch.div(dim_t, 2, rounding_mode="floor") / self.num_pos_feats)

    def forward(self, mask):
        not_mask = ~mask
        y = not_mask.cumsum(1, dtype=torch.float32)
        x = not_mask.cumsum(2, dtype=torch.float32)
        if self.normalize:
            y = (y + self.offset) / (y[:, -1:, :] + self.eps) * self.scale
            x = (x + self.offset) / (x[:, :, -1:] + self.eps) * self.scale
        dim_t = self.dim_t(mask.device)
        px = x[:, :, :, None] / dim_t
        py = y[:, :, :, None] / dim_t
        B, H, W = mask.shape
        px = torch.stack((px[:, :, :, 0::2].sin(), px[:, :, :, 1::2].cos()), dim=4).view(B, H, W, -1)
        py = torch.stack((py[:, :, :, 0::2].sin(), py[:, :, :, 1::2].cos()), dim=4).view(B, H, W, -1)
        return torch.cat((py, px), dim=3).permute(0, 3, 1, 2)


class ChannelMapper(nn.Module):
    """detrex ChannelMapper: per level `convs.{i}.conv` (1x1, bias) + `convs.{i}.norm` (GroupNorm)."""

    class _ConvNormAct(nn.Module):
        def __init__(self, cin, cout, kernel_size, norm_layer):
            super().__init__()
            self.conv = nn.Conv2d(cin, cout, kernel_size, padding=(kernel_size - 1) // 2)
            self.norm = norm_layer

        def forward(self, x):
            return self.norm(self.conv(x))

    def __init__(self, input_shapes, in_features, out_channels, kernel_size=1, norm_layer=None, num_outs=None, **kw):
        super().__init__()
        if num_outs is not None and num_outs != len(in_features):
            raise NotImplementedError("ape_b200.ChannelMapper: extra output levels are not used by APE")
        self.in_features = in_features
        self.convs = nn.ModuleList([self._ConvNormAct(input_shapes[f].channels, out_channels, kernel_size,
                                                      copy.deepcopy(norm_layer)) for f in in_features])

    def forward(self, inputs):
        first = inputs[self.in_features[0]]
        if first.is_cuda and first.dtype in (torch.float16, torch.bfloat16) and \
                all(c.conv.kernel_size == (1, 1) and isinstance(c.norm, nn.GroupNorm) for c in self.convs):
            # engine path: 1x1 conv = wgmma GEMM over tokens, GroupNorm kernel on the token-major layout, written
            # straight into its slice of the flattened [B, S, C] tensor the transformer consumes
            # (deformable_transformer_vl.py:435-452 flattens + concatenates the levels): no concat copy.
            xs = [inputs[f] for f in self.in_features]
            B = first.shape[0]
            hw = [int(x.shape[2]) * int(x.shape[3]) for x in xs]
            Cout = self.convs[0].conv.out_channels
            flat = torch.empty((B, sum(hw), Cout), dtype=first.dtype, device=first.device)
            outs, start = [], 0
            for conv, x, n in zip(self.convs, xs, hw):
                _, C, H, W = x.shape
                tok = x.permute(0, 2, 3, 1).reshape(B * H * W, C)  # free when x is channels_last (engine backbone)
                w, b = ops.packed(conv.conv, tok.dtype)
                y = ops.linear_tc(tok, w.view(w.shape[0], -1), b)
                gw, gb = ops.packed(conv.norm, tok.dtype)
                dst = flat[:, start:start + n]
                ops.groupnorm_nhwc(y.view(B, n, -1), gw, gb, conv.norm.num_groups, conv.norm.eps, out=dst)
                outs.append(dst.view(B, H, W, Cout).permute(0, 3, 1, 2))
                start += n
            self.last_flat = flat
            return tuple(outs)
        self.last_flat = None
        return tuple(self.convs[i](inputs[f]) for i, f in enumerate(self.in_features))


def fast_rcnn_inference_single_image(boxes, scores, image_shape, score_thresh, nms_thresh, topk_per_image):
    """fast_rcnn.py:97-201 (hard-NMS branch).  Returns (boxes, scores, classes, query indices)."""
    valid = torch.isfinite(boxes).all(dim=1) & torch.isfinite(scores).all(dim=1)
    if not valid.all():
        boxes, scores = boxes[valid], scores[valid]
    scores = scores[:, :-1]
    h, w = image_shape
    boxes = torch.stack((boxes[:, 0].clamp(min=0, max=w), boxes[:, 1].clamp(min=0, max=h),
                         boxes[:, 2].clamp(min=0, max=w), boxes[:, 3].clamp(min=0, max=h)), dim=-1)
    filter_mask = scores > score_thresh
    filter_inds = filter_mask.nonzero()
    boxes = boxes[filter_inds[:, 0]]
    scores = scores[filter_mask]
    if boxes.is_cuda:
        keep = ops.batched_nms(boxes.float(), scores, filter_inds[:, 1], nms_thresh)
    else:  # host tensors (fp32 parity runs without a GPU): the library the reference itself calls
        keep = torchvision.ops.batched_nms(boxes.float(), scores, filter_inds[:, 1], nms_thresh)
    if topk_per_image >= 0:
        keep = keep[:topk_per_image]
    boxes, scores, filter_inds = boxes[keep], scores[keep], filter_inds[keep]
    return boxes, scores, filter_inds[:, 1], filter_inds[:, 0]


def detector_postprocess(result: Instances, out_h, out_w, mask_format="bitmask"):
    """detectron2 detector_postprocess for box fields: rescale, clip, drop empty boxes.  mask_format "rle": the pasted masks leave
    as COCO run-length codes (`pred_masks_rle`: what the evaluators turn every mask into right away) instead of [N,H,W] booleans."""
    sx, sy = out_w / result.image_size[1], out_h / result.image_size[0]
    b = result.pred_boxes.tensor.clone()
    b[:, 0::2] *= sx
    b[:, 1::2] *= sy
    b = torch.stack((b[:, 0].clamp(min=0, max=out_w), b[:, 1].clamp(min=0, max=out_h),
                     b[:, 2].clamp(min=0, max=out_w), b[:, 3].clamp(min=0, max=out_h)), dim=-1)
    keep = ((b[:, 2] - b[:, 0]) > 0) & ((b[:, 3] - b[:, 1]) > 0)
    extra = {k: v[keep] for k, v in result.get_fields().items() if k not in ("pred_boxes", "scores", "pred_classes")}
    if "pred_masks" in extra:  # ROIMasks(pred_masks[:, 0]).to_bitmasks(boxes, H, W, 0.5): paste into the rescaled boxes
        if mask_format == "rle" and extra["pred_masks"].is_cuda:
            extra["pred_masks_rle"] = ops.paste_masks_rle(extra.pop("pred_masks")[:, 0], b[keep], (out_h, out_w), 0.5)
        else:
            extra["pred_masks"] = paste_masks_in_image(extra["pred_masks"][:, 0], b[keep], (out_h, out_w), 0.5)
    return Instances((out_h, out_w), pred_boxes=Boxes(b[keep]), scores=result.scores[keep],
                     pred_classes=result.pred_classes[keep], **extra)


def bitmasks_crop_and_resize(masks, boxes, mask_size):
    """detectron2 BitMasks.crop_and_resize: ROIAlign((S,S), scale 1, sampling_ratio 0, aligned=True) over the
    boolean masks as float, then >= 0.5."""
    from torchvision.ops import roi_align

    batch_inds = torch.arange(len(boxes), device=masks.device).to(dtype=boxes.dtype)[:, None]
    rois = torch.cat([batch_inds, boxes], dim=1)
    out = roi_align(masks.to(torch.float32)[:, None], rois, (mask_size, mask_size), 1.0, 0, True).squeeze(1)
    return out >= 0.5


def paste_masks_in_image(masks, boxes, image_shape, threshold=0.5):
    """detectron2.layers.mask_ops.paste_masks_in_image (`_do_paste_mask` with bilinear grid_sample, align_corners=False):
    masks [N, S, S] (probabilities) pasted into boxes [N, 4] of an (H, W) image -> bool [N, H, W]."""
    N = len(masks)
    img_h, img_w = int(image_shape[0]), int(image_shape[1])
    if N == 0:
        return masks.new_empty((0, img_h, img_w), dtype=torch.bool)
    if masks.is_cuda:  # ape_mask_paste: the sampling grid lives in registers (the library path below is the host route)
        return ops.paste_masks_in_image(masks, boxes, (img_h, img_w), threshold)
    out = torch.zeros((N, img_h, img_w), device=masks.device, dtype=torch.bool)
    chunk = max(1, int((1 << 30) // (img_h * img_w * 4)))  # GPU_MEM_LIMIT of 1 GiB, as detectron2
    for i0 in range(0, N, chunk):
        m = masks[i0:i0 + chunk, None].float()
        b = boxes[i0:i0 + chunk]
        x0, y0, x1, y1 = torch.split(b, 1, dim=1)
        img_y = torch.arange(0, img_h, device=masks.device, dtype=torch.float32) + 0.5
        img_x = torch.arange(0, img_w, device=masks.device, dtype=torch.float32) + 0.5
        img_y = (img_y - y0) / (y1 - y0) * 2 - 1
        img_x = (img_x - x0) / (x1 - x0) * 2 - 1
        gx = img_x[:, None, :].expand(len(b), img_h, img_w)
        gy = img_y[:, :, None].expand(len(b), img_h, img_w)
        grid = torch.stack([gx, gy], dim=3)
        pasted = F.grid_sample(m, grid.to(m.dtype), align_corners=False)[:, 0]
        out[i0:i0 + chunk] = pasted >= threshold
    return out


def sem_seg_postprocess(result, img_size, output_height, output_width):
    """detectron2 sem_seg_postprocess: crop to the unpadded size, bilinear resize (align_corners=False)."""
    result = result[:, : img_size[0], : img_size[1]].expand(1, -1, -1, -1)
    return F.interpolate(result, size=(output_height, output_width), mode="bilinear", align_corners=False)[0]


def get_stuff_score(box_cls, thing_classes, stuff_classes, entity):
    """deformable_detr_segm_vl.py:1251-1271 (thing / stuff overlap case keeps all classes, as the clone there)."""
    if entity == "thing+stuff" and stuff_classes and stuff_classes[0] == "things" and not set(thing_classes) & set(stuff_classes):
        n = len(thing_classes)
        s0, _ = box_cls[..., :n].min(dim=2, keepdim=True)
        return torch.cat([s0, box_cls[..., n:]], dim=2)
    return box_cls.clone()


class _Criterion(nn.Module):
    """Inference-only stand-in for DeformableCriterion entries of the `criterion` list."""

    loss_class_type = "focal_loss"

    def __init__(self, num_classes):
        super().__init__()
        self.num_classes = num_classes


class DeformableDETRSegmVL(nn.Module):
    def __init__(
        self,
        # DeformableDETRSegmVL (deformable_detr_segm_vl.py:63-90)
        instance_on: bool = True, semantic_on: bool = False, panoptic_on: bool = False, freeze_detr=False,
        input_shapes=None, mask_in_features=None, mask_encode_level=0, stuff_dataset_learn_thing: bool = True,
        stuff_prob_thing: float = -1.0, name_prompt_fusion_type: str = "none", name_prompt_fusion_text=None,
        test_mask_on: bool = True, semantic_post_nms: bool = True, panoptic_post_nms: bool = True,
        aux_mask: bool = False, panoptic_configs=None,
        # DeformableDETR (deformable_detr.py:52-88)
        backbone=None, position_embedding=None, neck=None, transformer=None, embed_dim=256, num_classes=80,
        num_queries=900, criterion=None, pixel_mean=(123.675, 116.280, 103.530), pixel_std=(58.395, 57.120, 57.375),
        aux_loss=True, with_box_refine=False, as_two_stage=False, select_box_nums_for_evaluation=100,
        select_box_nums_for_evaluation_list=None, input_format="RGB", vis_period=0, output_dir=None,
        dataset_names=(), dataset_metas=(), dataset_prompts=None, embed_dim_language=512,
        text_feature_batch_repeat=True, text_feature_bank=False, text_feature_bank_reset=False,
        text_feature_bank_random_size=False, text_feature_reduce_type="last",
        text_feature_reduce_before_fusion=True, expression_cumulative_gt_class=True, test_nms_thresh=0.7,
        test_score_thresh=0.0, last_class_embed_use_mlp=False, openset_classifier="VisionLanguageAlign",
        vocabulary=None,
    ):
        super().__init__()
        if not (with_box_refine and as_two_stage) or openset_classifier != "VisionLanguageAlign" or aux_mask \
                or last_class_embed_use_mlp:
            raise NotImplementedError("ape_b200: only the two-stage, box-refine, VisionLanguageAlign configuration")
        self.backbone, self.position_embedding, self.neck, self.transformer = backbone, position_embedding, neck, transformer
        if neck is None and hasattr(backbone, "flat_output"):
            # no neck (APE-L_B / L_C, …_lsj1024_cp_720k.py:53): the backbone's levels are the encoder input, so its engine
            # path writes them straight into the flattened [B, S, C] buffer the encoder consumes
            backbone.flat_output = True
        self.num_queries, self.num_classes = num_queries, num_classes
        self.embed_dim_language = embed_dim_language
        nd = transformer.decoder.num_layers
        cls = VisionLanguageAlign(embed_dim, embed_dim_language)
        box = MLP(embed_dim, embed_dim, 4, 3)
        nn.init.constant_(box.layers[-1].weight.data, 0)
        nn.init.constant_(box.layers[-1].bias.data, 0)
        self.class_embed = nn.ModuleList([copy.deepcopy(cls) for _ in range(nd + 1)])
        self.bbox_embed = nn.ModuleList([copy.deepcopy(box) for _ in range(nd + 1)])
        self.criterion = nn.ModuleList(criterion if criterion is not None else [_Criterion(num_classes)])
        # shared with the decoder, exactly as deformable_detr.py:158-200 (aliases appear in state_dict)
        transformer.decoder.bbox_embed = self.bbox_embed
        transformer.decoder.class_embed = self.class_embed
        bias_value = -math.log((1 - 0.01) / 0.01)
        transformer.decoder.class_embed[-1] = nn.Linear(embed_dim, 1)
        transformer.decoder.class_embed[-1].bias.data = torch.ones(1) * bias_value
        if transformer.proposal_ambiguous:
            transformer.decoder.bbox_embed_ambiguous = nn.ModuleList(
                [copy.deepcopy(self.bbox_embed[-1]) for _ in range(transformer.proposal_ambiguous)])
            transformer.decoder.class_embed_ambiguous = nn.ModuleList(
                [copy.deepcopy(self.class_embed[-1]) for _ in range(transformer.proposal_ambiguous)])

        self.aux_loss, self.with_box_refine, self.as_two_stage = aux_loss, with_box_refine, as_two_stage
        self.select_box_nums_for_evaluation = select_box_nums_for_evaluation
        self.select_box_nums_for_evaluation_list = select_box_nums_for_evaluation_list
        self.test_topk_per_image = select_box_nums_for_evaluation
        self.test_nms_thresh, self.test_score_thresh = test_nms_thresh, test_score_thresh
        self.input_format = input_format
        self.register_buffer("pixel_mean", torch.tensor(pixel_mean).view(-1, 1, 1), False)
        self.register_buffer("pixel_std", torch.tensor(pixel_std).view(-1, 1, 1), False)
        self.dataset_names = list(dataset_names)
        self.dataset_prompts = dataset_prompts
        # class-name vocabulary per dataset (the reference reads detectron2's MetadataCatalog,
        # deformable_detr.py:232-262; the engine takes the lists directly)
        self.vocabulary = vocabulary if vocabulary is not None else {}
        self.dataset_name_to_idx = {k: i for i, k in enumerate(self.dataset_names)}
        self.eval_dataset_id = -1
        self.eval_dataset_entity = ""
        self.text_feature_bank, self.text_feature_bank_reset = text_feature_bank, text_feature_bank_reset
        self.text_feature_batch_repeat = text_feature_batch_repeat
        self.text_feature_reduce_before_fusion = text_feature_reduce_before_fusion
        if text_feature_bank:
            bank = torch.zeros((len(self.criterion), max(c.num_classes for c in self.criterion), embed_dim_language))
            self.register_buffer("features_phrase_bank", bank, False)

        self.instance_on, self.semantic_on, self.panoptic_on = instance_on, semantic_on, panoptic_on
        self.test_mask_on = test_mask_on
        # "bitmask": `pred_masks` [N,H,W] booleans as the reference returns them; "rle": `pred_masks_rle`, COCO run-length codes
        # computed on the device from the 128 x 128 masks (what the evaluators encode every mask into: d3_evaluation.py:466-468),
        # 314 MB of booleans per 300 detections at 1024^2 that are never written or copied
        self.mask_format = "bitmask"
        # bytes per detection slot for the run-length code of a mask in `forward_packed` (a code that does not fit travels as
        # the 128 x 128 mask's 2048 bytes of bits and is encoded on the receiving side); a multiple of 4, at least 2048
        self.mask_slot_bytes = 4096
        # "maps": `sem_seg` [N_classes, H, W] fp32 scores as the reference returns them; "label": `sem_seg_label` int64 [H, W] (the
        # first argmax over classes of that map, all SemSegEvaluator keeps) and `sem_seg_score` fp32 [H, W] (its value).  On CUDA
        # with a 16-bit engine_dtype the map is never formed (csrc/semseg.cu: 5 GB per image at 1203 classes and 1024^2)
        self.sem_seg_format = "maps"
        # "rle" adds `sem_seg_rle` to what "label" returns: one cocoapi run-length code per label present (ops.label_map_rle), what
        # SemSegEvaluator.process encodes the map into.  `sem_seg_slot_bytes`: the semantic slot per image of `forward_packed`
        # (codes, or the map as uint16 when they do not fit: the default holds any map up to 1024 x 1024 exactly); a multiple of 4
        self.sem_seg_slot_bytes = 1 << 21
        # the panoptic slot per image of `forward_packed`: a 32-byte header, 12 bytes per query of the merge and the map as uint16
        # (ops.panoptic_pack); the default holds any output up to 1024 x 1024 with up to 1024 queries.  A multiple of 4
        self.panoptic_slot_bytes = (1 << 21) + (1 << 14)
        # None, or an int C: `forward_packed` calls whose image and output sizes all fit C x C run the packed mask / semantic /
        # panoptic stages on sizes held on the device (ops.*_dev), so `use_cuda_graphs` captures one graph per padded shape and
        # configuration for them instead of one per combination of sizes.  Larger outputs take the per-size path
        self.packed_output_capacity = None
        self.semantic_post_nms = semantic_post_nms
        self.panoptic_post_nms = panoptic_post_nms
        self.panoptic_configs = panoptic_configs if panoptic_configs is not None else {
            "prob": 0.1, "pano_temp": 0.06, "transform_eval": True, "object_mask_threshold": 0.01, "overlap_threshold": 0.4}
        self.stuff_prob_thing = stuff_prob_thing
        # (thing_classes, stuff_classes) per dataset for the semantic branch; the reference reads them from detectron2's
        # MetadataCatalog (deformable_detr.py:244-262).  None = "thing" entity over the dataset's vocabulary.
        self.dataset_stuff = {}
        self.input_shapes, self.mask_in_features, self.mask_encode_level = input_shapes, mask_in_features, mask_encode_level
        hidden = transformer.embed_dim
        in_ch = input_shapes[mask_in_features[0]].channels
        self.lateral_conv = ConvNorm(in_ch, hidden, 1, bias=False, norm=nn.GroupNorm(32, hidden))
        self.output_conv = ConvNorm(hidden, hidden, 3, padding=1, bias=False, norm=nn.GroupNorm(32, hidden), activation=F.relu)
        self.mask_conv = ConvNorm(hidden, hidden, 1, bias=False)
        self.mask_embed = MLP(hidden, hidden, hidden, 3)
        self.name_prompt_fusion_type = name_prompt_fusion_type
        self.name_prompt_fusion_text = name_prompt_fusion_text
        if name_prompt_fusion_type == "zero":
            self.name_prompt_fusion_feature = nn.Parameter(torch.zeros(1, 1, embed_dim_language), requires_grad=False)
        elif name_prompt_fusion_type == "learnable":
            self.name_prompt_fusion_feature = nn.Parameter(torch.randn(1, 1, embed_dim_language))
        else:
            self.name_prompt_fusion_feature = None
        self.model_language = None
        self._text_cache = {}
        # Numeric mode of the engine.  Parameters stay fp32 (checkpoint precision); with a 16-bit
        # engine_dtype the backbone runs on libape_b200's tensor-core kernels and the remaining library
        # ops run under autocast — the reference's own eval recipe casts the whole model to fp16
        # (tools/train_net.py:641-642).  float32 = strict-parity mode on fp32 library kernels.
        self.engine_dtype = torch.float32
        self.profile_stages = False   # record CUDA-event stage times of the last forward in self.stage_ms
        self.use_cuda_graphs = False  # capture the static stages once per padded shape and prompt configuration (16-bit engine mode)
        import collections

        self._geo_cache, self._graph_cache = {}, collections.OrderedDict()
        self.graph_cache_size = 8  # captured graphs kept (LRU)
        # static-shape final selection (one host sync per batch) for up to this many (query, class) pairs above the
        # score threshold; more than that falls back to the dynamic path.  0 disables.
        self.static_inference_cap = 8192

    # -- plumbing ----------------------------------------------------------------------------------
    @property
    def device(self):
        return self.pixel_mean.device

    def set_model_language(self, model_language):
        # kept out of the module tree like the reference (ape_deta.py:31-33 deletes its own handle)
        object.__setattr__(self, "model_language", model_language)

    def set_eval_dataset(self, dataset_name):
        """deformable_detr.py:524-549."""
        for d in self.dataset_names:
            if sum([dd in dataset_name for dd in d.split("+")]):
                self.eval_dataset_id = self.dataset_name_to_idx[d]
                self.eval_dataset_entity = self._dataset_entity(d)
                break
        else:
            self.eval_dataset_id = -1
            self.eval_dataset_entity = ""

    def _dataset_entity(self, name):
        """deformable_detr.py:246-262: "thing+stuff" / "thing" / "stuff" from the class lists of the dataset
        (`model.dataset_stuff[name] = (thing_classes, stuff_classes[, entity[, thing_ids]])`; the reference reads MetadataCatalog)."""
        info = self.dataset_stuff.get(name)
        if info is None:
            return "thing"
        if len(info) > 2 and info[2]:
            return info[2]
        things, stuff = info[0], info[1]
        return "thing+stuff" if things and stuff else "stuff" if stuff else "thing"

    def _detector_box_cls(self, box_cls):
        """Class columns the instance branch may use (:575-593): thing classes only.  Disjoint thing / stuff vocabularies keep
        the first len(thing_classes) columns; overlapping ones (one list a subset of the other) keep the thing ids and set the
        rest to -inf."""
        d = self.eval_dataset_id
        if not (0 <= d < len(self.dataset_names)):
            return box_cls
        info = self.dataset_stuff.get(self.dataset_names[d])
        if info is None or not info[0]:
            return box_cls
        things, stuff = list(info[0]), list(info[1] or [])
        if things and stuff and (set(things) <= set(stuff) or set(stuff) <= set(things)):
            ids = list(info[3]) if len(info) > 3 and info[3] is not None else list(range(len(things)))
            out = torch.full_like(box_cls, float("-inf"))
            idx = torch.as_tensor(ids, dtype=torch.long, device=box_cls.device)
            out[..., idx] = box_cls[..., idx]
            return out
        return box_cls[..., : len(things)]

    def preprocess_image(self, batched_inputs):
        """:846-855 + ImageList.from_tensors with padding_constraints square_size (pads AFTER normalising)."""
        sq = self.backbone.padding_constraints.get("square_size", 0)
        imgs = [x["image"].to(self.device, non_blocking=True) for x in batched_inputs]
        sizes = [(int(im.shape[-2]), int(im.shape[-1])) for im in imgs]
        H = max(s[0] for s in sizes) if sq <= 0 else sq
        W = max(s[1] for s in sizes) if sq <= 0 else sq
        div = int(self.backbone.padding_constraints.get("size_divisiblity", 0) or 0)  # (sic) detectron2's key
        if sq <= 0 and div > 1:  # ImageList.from_tensors rounds the batch shape up to the size divisibility
            H, W = -(-H // div) * div, -(-W // div) * div
        for (h, w) in sizes:
            if h > H or w > W:
                raise ValueError(f"ape_b200: image of {h}x{w} does not fit the {H}x{W} padded batch (square_size={sq}); "
                                 "resize it first (ResizeShortestEdge in the reference's predictor)")
        batch = torch.zeros((len(imgs), 3, H, W), dtype=self.pixel_mean.dtype, device=self.device)
        masks = torch.ones((len(imgs), H, W), dtype=self.pixel_mean.dtype, device=self.device)
        for i, im in enumerate(imgs):
            h, w = sizes[i]
            batch[i, :, :h, :w] = (im.to(self.pixel_mean.dtype) - self.pixel_mean) / self.pixel_std
            masks[i, :h, :w] = 0
        return batch, masks, sizes

    # -- text routing (:166-360) -------------------------------------------------------------------
    def _text_features(self, batched_inputs):
        dataset_id = self.eval_dataset_id
        if dataset_id >= 0:
            prompt = self.dataset_prompts[dataset_id]
        elif "prompt" in batched_inputs[0]:
            prompt = batched_inputs[0]["prompt"]
        else:
            prompt = "name"
        if prompt == "expression":  # (:184-193) referring expressions: one box per image, texts from `expressions`
            for x in batched_inputs:
                if not isinstance(x["expressions"], list):
                    x["expressions"] = [x["expressions"]]
                assert all(isinstance(xx, str) and len(xx) > 0 for xx in x["expressions"])
            self.test_topk_per_image = 1
        else:
            self.test_topk_per_image = self.select_box_nums_for_evaluation
        if self.select_box_nums_for_evaluation_list is not None:
            self.test_topk_per_image = self.select_box_nums_for_evaluation_list[dataset_id]
        text_list = None
        if prompt == "expression":
            text_list = [xx for x in batched_inputs for xx in x["expressions"]]  # (:289-290)
        if prompt == "text":
            texts = [x["text_prompt"] for x in batched_inputs]
            text_list = [x.strip() for x in ",".join(texts).split(",")]
            text_list = [x for x in text_list if len(x) > 0]
            prompt = "phrase" if any(x.count(" ") >= 1 for x in text_list) else "name"
        bs = len(batched_inputs)
        if prompt == "name":
            if text_list:
                cache = False
            elif dataset_id >= 0:
                text_list, cache = list(self.vocabulary[self.dataset_names[dataset_id]]), True
            else:
                text_list = []
                for d in self.dataset_names:
                    text_list += list(self.vocabulary[d])
                text_list, cache = text_list[:1203], True  # (:249-251)
            key = tuple(text_list)
            if cache and key in self._text_cache:
                features_l = self._text_cache[key]
            else:
                kw = {"need_hidden": False} if getattr(self.model_language, "pack_prompts", False) else {}
                features_l = self.model_language.forward_text(text_list, cache=cache, **kw)["last_hidden_state_eot"]
                if cache:
                    self._text_cache[key] = features_l
            if cache and features_l.device != self.device:  # keep cached vocabularies resident on the device
                features_l = features_l.to(self.device)
                self._text_cache[key] = features_l
            features_l = features_l.to(self.device).unsqueeze(0).repeat(bs, 1, 1)
            if self.name_prompt_fusion_text is not None and self.name_prompt_fusion_text[dataset_id]:
                fusion = features_l
            elif self.name_prompt_fusion_feature is not None:
                fusion = self.name_prompt_fusion_feature.repeat(bs, 1, 1)
            else:
                fusion = None
            return prompt, features_l, fusion
        # phrase / expression (:284-337)
        if not text_list:
            raise NotImplementedError("ape_b200: phrase prompts need `text_prompt` (or `expressions`) at inference")
        # a text tower that packs its prompts by length reads out the end-of-text rows alone when told that nothing else is wanted
        kw = {"need_hidden": False} if getattr(self.model_language, "pack_prompts", False) else {}
        features_l = self.model_language.forward_text(text_list, **kw)["last_hidden_state_eot"].to(self.device)
        if self.text_feature_bank and not self.text_feature_bank_reset and 0 <= dataset_id < len(self.dataset_names):
            n = self.criterion[dataset_id].num_classes
            features_l = torch.cat([features_l, self.features_phrase_bank[dataset_id]], dim=0)[: max(len(text_list), n)]
            self.features_phrase_bank[dataset_id, :n] = features_l[:n]
        elif self.text_feature_bank and self.text_feature_bank_reset:
            n = self.criterion[dataset_id].num_classes
            features_l = torch.cat([features_l.to(self.features_phrase_bank.dtype),
                                    self.features_phrase_bank[dataset_id] * 0], dim=0)[: max(len(text_list), n)]
        features_l = features_l.unsqueeze(0).repeat(bs, 1, 1)
        fusion = features_l
        if self.name_prompt_fusion_feature is not None:
            fusion = fusion + 0.0 * self.name_prompt_fusion_feature
        return prompt, features_l, fusion

    # -- forward -------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, batched_inputs: List[Dict], do_postprocess=True):
        if self.training:
            raise NotImplementedError("ape_b200 is an inference engine (SURVEY.md §8f row 4)")
        marks = [] if self.profile_stages else None

        def mark(name):
            if marks is not None:
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                marks.append((name, e))

        mark("start")
        prompt, features_l, fusion = self._text_features(batched_inputs)
        images, img_masks, image_sizes = self.preprocess_image(batched_inputs)
        mark("preprocess")
        low = self.engine_dtype != torch.float32
        # CUDA: the padded shape's geometry here; the per-size part (ops.pad_geometry, from `sizes` on the device) below, or
        # at the start of the captured graph, which therefore serves every image size inside the padded shape
        sizes = self._sizes_tensor(image_sizes) if images.is_cuda else None
        geo = self._padded_geometry(images.shape) if images.is_cuda else self._geometry(images.shape, image_sizes, img_masks)
        mask_prompt_flatten = self._mask_prompt(batched_inputs, images.shape, geo) if "mask_prompt" in batched_inputs[0] else None
        graphs = low and self.use_cuda_graphs and self._graph_prompt(prompt, fusion) and mask_prompt_flatten is None
        need_masks = self.semantic_on or self.panoptic_on or (self.instance_on and self.test_mask_on)
        with torch.autocast("cuda", dtype=self.engine_dtype, enabled=low):
            if graphs and not self.profile_stages:
                # encode -> select -> decode in ONE graph: the selection is written with static shapes and no host
                # synchronisation (transformer.select_proposals), so nothing between the image upload and the final
                # thresholding touches the host
                # the final selection (threshold, class-aware NMS, top-k: static shapes) rides in the same graph when boxes are
                # all that is asked for; its configuration is part of the graph key
                sel, const, dims = None, (geo, prompt), None
                # forward_packed with instance masks: the mask stage (csrc/mask_post.cu, ape_mask_pack) follows the selection in
                # the graph; the output sizes and the slot size join the key
                # with semantic_on the semantic stage (ape_label_rle_pack) follows too, and its configuration joins the key; so
                # does the panoptic stage (ape_panoptic_winners + ape_panoptic_pack) with panoptic_on
                packed = do_postprocess == "packed"
                packed_masks = packed and self.instance_on and self.test_mask_on
                packed_sem = self._packed_semantic_config() if packed and self.semantic_on else None
                packed_pan = self._packed_panoptic_config() if packed and self.panoptic_on else None
                if do_postprocess in (True, "packed") and (not need_masks or packed_masks or packed_sem or packed_pan) and \
                        self.static_inference_cap > 0 and self.test_topk_per_image >= 0 and self.num_queries <= 1024:
                    ent = self.eval_dataset_entity
                    sel = (bool(getattr(self, "_static_overflowed", False)), float(self.test_score_thresh),
                           float(self.test_nms_thresh), int(self.test_topk_per_image), int(self.static_inference_cap),
                           self.eval_dataset_id, bool(self.instance_on and not (ent and "thing" not in ent)))
                    const = (geo, prompt, sel)
                    if packed_masks or packed_sem or packed_pan:
                        mask_slot = int(self.mask_slot_bytes) if packed_masks else None
                        cap = self._packed_capacity(batched_inputs, image_sizes)
                        if cap is None:
                            # the packed mask / semantic / panoptic stages size their grids and workspaces from host ints (ape_mask_pack's
                            # output sizes and row width, the label-map GEMM and ape_panoptic_winners at the output resolution), so
                            # their graphs keep the image and output sizes in the key: one graph per combination of sizes
                            sel += ((tuple(image_sizes), self._output_sizes(batched_inputs, image_sizes), mask_slot, packed_sem,
                                     packed_pan),)
                            const = (geo, prompt, sel, self._size_columns(batched_inputs, image_sizes))
                        else:
                            # capacity mode: the stages read the sizes from `dims`, a graph input like `sizes`; the key holds C
                            sel += ((None, None, mask_slot, packed_sem, packed_pan, cap),)
                            const = (geo, prompt, sel)
                            dims = self._dims_tensor(batched_inputs, image_sizes)
                # the image sizes are a graph input like the image: the key holds the padded shape, not the sizes
                (memory, output_memory, enc_cls, enc_coord, features, feats, topk, box_cls, box_pred, inter_states,
                 init_reference, inter_references, mask_logits, graph_pack) = self._graphed(
                    ("forward", prompt, tuple(images.shape), tuple(features_l.shape), need_masks, sel),
                    self._stage_all, (images, fusion, features_l, sizes, dims), const)
                self.transformer.last_topk_proposals = topk
                mark("encode")
                mark("select")
            else:
                if graphs:
                    memory, fusion_out, output_memory, enc_cls, enc_coord, features, feats, mask_features, geo = self._graphed(
                        ("encode", tuple(images.shape), need_masks), self._stage_encode_sized, (images, fusion, sizes), (geo,))
                else:
                    if images.is_cuda:
                        geo = self._geometry(images.shape, image_sizes, sizes=sizes)
                    memory, fusion_out, output_memory, enc_cls, enc_coord, features, feats, mask_features = \
                        self._stage_encode(images, fusion, geo, mask_prompt_flatten)
                mark("encode")
                topk = self.transformer.stage_select(enc_cls, enc_coord, geo)
                self.transformer.last_topk_proposals = topk
                mark("select")
                features_l = self._mix_text(prompt, features_l, fusion_out)
                if graphs:
                    # memory / output_memory / enc_coord are the encode graph's static outputs: constants of this graph
                    box_cls, box_pred, inter_states, init_reference, inter_references, mask_logits = self._graphed(
                        ("decode", memory.data_ptr(), tuple(features_l.shape), need_masks), self._stage_decode,
                        (topk, features_l), (memory, output_memory, enc_coord, geo, mask_features))
                else:
                    box_cls, box_pred, inter_states, init_reference, inter_references, mask_logits = self._stage_decode(
                        topk, features_l, memory, output_memory, enc_coord, geo, mask_features)
        if not (graphs and not self.profile_stages):
            graph_pack = None
        self.last_outputs = dict(pred_logits=box_cls, pred_boxes=box_pred, memory=memory, inter_states=inter_states,
                                 init_reference=init_reference, inter_references=inter_references,
                                 features=features, neck=feats)
        mask_pred = mask_logits if need_masks else None  # [B, Q, h, w] logits of the last decoder level
        self.last_outputs["pred_masks"] = mask_pred
        mark("decode")
        if do_postprocess == "raw":  # logits / boxes stay on the device, no selection here
            return box_cls, box_pred, image_sizes
        if do_postprocess == "packed":  # forward_packed: the selection computed INSIDE the captured graph when there is one
            return box_cls, box_pred, image_sizes, graph_pack, mask_pred, tuple(images.shape[-2:])
        # the three branches are gated by the entity of the evaluated dataset (:575-577, :628-630, :671-673)
        ent = self.eval_dataset_entity
        instance_on = self.instance_on and not (ent and "thing" not in ent)
        semantic_on = self.semantic_on and not (ent and "stuff" not in ent)
        panoptic_on = self.panoptic_on and not (ent and "thing+stuff" not in ent)
        det_cls = self._detector_box_cls(box_cls) if instance_on else box_cls
        results = None
        if do_postprocess and box_cls.is_cuda and self.static_inference_cap > 0 and not need_masks:
            # CPU Instances, one host sync; `graph_pack` = the selection already computed inside the CUDA graph
            results = self._inference_static(det_cls, box_pred, image_sizes, first_pack=graph_pack)
        if results is None:
            results = self.inference(det_cls, box_pred, image_sizes)
        padded_hw = tuple(images.shape[-2:])
        if instance_on and self.test_mask_on:
            for b, r in enumerate(results):  # (:588-603) masks of the kept queries only (bilinear resize is per channel)
                if mask_pred.is_cuda:  # upsample > 0 as bits + ROIAlign over the bits (csrc/mask_post.cu): no fp32 full-size maps
                    m = ops.mask_crop_and_resize(mask_pred[b].contiguous(), r.query_index, r.pred_boxes.tensor, padded_hw, 128)
                else:
                    m = F.interpolate(mask_pred[b, r.query_index][None].float(), size=padded_hw, mode="bilinear", align_corners=False)[0]
                    m = bitmasks_crop_and_resize(m.sigmoid() > 0.5, r.pred_boxes.tensor.to(m.device), 128)
                r.pred_masks = m.unsqueeze(1).to(torch.float32)
        if not do_postprocess:
            return results, None, None
        out = []
        for r, inp, size in zip(results, batched_inputs, image_sizes):
            h, w = inp.get("height", size[0]), inp.get("width", size[1])
            out.append({"instances": detector_postprocess(r, h, w, getattr(self, "mask_format", "bitmask")).to("cpu")} if instance_on else {})
        # the semantic / panoptic branches select queries with the same threshold + NMS + top-k as the instance branch; when their
        # class logits are the instance branch's (no thing-class slicing, no "things" stuff column) the kept queries are reused
        # instead of running the selection two more times (ADVICE round 1)
        shared_keep = [r.query_index for r in results] if (instance_on and det_cls is box_cls and results is not None) else None
        if semantic_on:
            for o, sem in zip(out, self._semantic(box_cls, box_pred, mask_pred, image_sizes, padded_hw, batched_inputs, shared_keep)):
                o.update(sem)
        if panoptic_on:
            for o, pan in zip(out, self._panoptic(box_cls, box_pred, mask_pred, image_sizes, padded_hw, batched_inputs, shared_keep)):
                o["panoptic_seg"] = pan
        mark("inference")
        if marks is not None:
            torch.cuda.synchronize()
            self.stage_ms = {n: marks[i - 1][1].elapsed_time(e) for i, (n, e) in enumerate(marks) if i > 0}
        return out

    # -- stages (static shapes, no host synchronisation: CUDA-graph capturable) -----------------------------
    def _level_shapes(self, batch_shape):
        levels = self.neck.in_features if self.neck is not None else self.backbone._out_features  # (:375-378)
        strides = [self.backbone._out_feature_strides[f] for f in levels]
        H, W = batch_shape[-2], batch_shape[-1]
        return [(-(-H // s), -(-W // s)) for s in strides]

    def _geometry(self, batch_shape, image_sizes, img_masks=None, sizes=None):
        """Padding masks, sine position embeddings (:375-392) and the transformer's geometric constants for one batch.  CUDA:
        the padded shape's part (`_padded_geometry`) and the per-size part from ops.pad_geometry over `sizes` (int32 [B, 2] on
        the device; uploaded from image_sizes when None).  Elsewhere: the torch restatement over the pixel masks img_masks."""
        shapes = self._level_shapes(batch_shape)
        if self.device.type != "cuda":
            masks = [F.interpolate(img_masks[None], size=sh).to(torch.bool).squeeze(0) for sh in shapes]
            pos = [self.position_embedding(m).to(torch.float32) for m in masks]
            return self.transformer.geometry(shapes, masks, pos)
        if sizes is None:
            sizes = self._sizes_tensor(image_sizes)
        return self._size_geometry(self._padded_geometry(batch_shape), sizes, self._has_padding(batch_shape, shapes, image_sizes))

    def _padded_geometry(self, batch_shape):
        """The geometry that depends only on the padded shape (level shapes, start indices, level ids, the sine table),
        cached per padded shape: few keys whatever the image sizes."""
        H, W = int(batch_shape[-2]), int(batch_shape[-1])
        key = (H, W, str(self.device))
        geo = self._geo_cache.get(key)
        if geo is None:
            geo = self.transformer.padded_geometry(self._level_shapes(batch_shape), self.device)
            geo.update(padded_hw=(H, W), dim_t=self.position_embedding.dim_t(self.device))
            if len(self._geo_cache) > 16:
                self._geo_cache.clear()
            self._geo_cache[key] = geo
        return geo

    def _size_geometry(self, padded, sizes, has_padding):
        return self.transformer.size_geometry(padded, sizes, padded["padded_hw"], padded["dim_t"], self.position_embedding,
                                              self.engine_dtype, has_padding)

    def _sizes_tensor(self, image_sizes):
        """The image sizes as int32 [B, 2] (h, w) on the device, cached per sizes (read-only): a repeated size costs no upload, a
        new one is copied from pinned memory without a host synchronisation."""
        key = (tuple((int(h), int(w)) for h, w in image_sizes), str(self.device))
        cache = self.__dict__.setdefault("_sizes_dev", {})
        sizes = cache.get(key)
        if sizes is None:
            if len(cache) > 64:
                cache.clear()
            sizes = cache[key] = torch.tensor(key[0], dtype=torch.int32, pin_memory=True).to(self.device, non_blocking=True)
        return sizes

    @staticmethod
    def _has_padding(batch_shape, shapes, image_sizes):
        """bool(mask_flatten.any()) of the torch geometry, from the host sizes: a level has padding when the nearest source
        pixel of its last row or column (F.interpolate: min(floor(i * (float)in / out), in - 1) in fp32) lies outside the image."""
        def src(n_in, n_out):
            return min(int(np.floor(np.float32(n_out - 1) * (np.float32(n_in) / np.float32(n_out)))), n_in - 1)
        H, W = int(batch_shape[-2]), int(batch_shape[-1])
        return any(src(H, hl) >= h or src(W, wl) >= w for hl, wl in shapes for h, w in image_sizes)

    def _mask_prompt(self, batched_inputs, batch_shape, geo):
        """:394-412: region prompts.  Per-image masks padded like the image (ImageList.from_tensors), an all-zero batch means
        "everywhere" (set to 255), resized bilinearly to every level and thresholded by `.to(bool)`; flattened like the features
        (deformable_transformer_vl.py:465-470).  Proposals outside the prompt are disabled in the two-stage selection."""
        H, W = batch_shape[-2], batch_shape[-1]
        mp = torch.zeros((len(batched_inputs), H, W), dtype=self.pixel_mean.dtype, device=self.device)
        for i, x in enumerate(batched_inputs):
            m = x["mask_prompt"].to(self.device).to(self.pixel_mean.dtype)
            mp[i, : m.shape[-2], : m.shape[-1]] = m
        if mp.sum() == 0:
            mp[...] = 255
        levels = [F.interpolate(mp[None], size=sh, mode="bilinear").to(torch.bool).squeeze(0) for sh in geo["shapes"]]
        return torch.cat([m.flatten(1) for m in levels], 1)

    def _stage_encode(self, images, fusion, geo, mask_prompt_flatten=None):
        features = self.backbone(images.to(self.engine_dtype))
        if self.neck is not None:
            feats = self.neck({f: features[f] for f in self.neck.in_features})
            flat = getattr(self.neck, "last_flat", None)
        else:  # (:375-378) the levels are the backbone's output dict in order
            feats = tuple(features.values())
            flat = getattr(self.backbone, "last_flat", None)
        memory, fusion_out, output_memory, enc_cls, enc_coord = self.transformer.stage_encode(
            feats, geo, fusion, mask_prompt_flatten=mask_prompt_flatten, feat_flatten=flat)
        mask_features = None
        if self.semantic_on or self.panoptic_on or (self.instance_on and self.test_mask_on):
            mask_features = self.maskdino_mask_features(memory, features, geo)
        return memory, fusion_out, output_memory, enc_cls, enc_coord, features, feats, mask_features

    @staticmethod
    def _graph_prompt(prompt, fusion):
        """Prompts whose step is captured in a CUDA graph: one fusion token ("name" prompts), so the encoder's launch sequence
        does not depend on the text."""
        return fusion is not None and fusion.shape[1] == 1

    @staticmethod
    def _mix_text(prompt, features_l, fusion_out):
        if prompt == "name":
            if fusion_out is not None:
                features_l = 1.0 * features_l + 0.0 * fusion_out.float()  # (:446)
            return features_l
        return 0.0 * features_l + 1.0 * fusion_out.float()  # (:448)

    def _stage_encode_sized(self, images, fusion, sizes, padded):
        """_stage_encode after the per-size geometry, for the encode graph of the profiling split; the geometry is returned too,
        because selection and the decode graph read it."""
        geo = self._size_geometry(padded, sizes, True)
        return self._stage_encode(images, fusion, geo) + (geo,)

    def _stage_all(self, images, fusion, features_l, sizes, dims, padded, prompt, sel=None, size_columns=None):
        # inside a graph the padding mask is always passed: an all-false mask gives the values of None (masked_fill with no
        # true entry changes nothing), so one graph serves padded and unpadded sizes alike
        geo = self._size_geometry(padded, sizes, True)
        memory, fusion_out, output_memory, enc_cls, enc_coord, features, feats, mask_features = self._stage_encode(images, fusion, geo)
        topk = self.transformer.stage_select(enc_cls, enc_coord, geo)
        features_l = self._mix_text(prompt, features_l, fusion_out)
        box_cls, box_pred, inter_states, init_reference, inter_references, mask_logits = self._stage_decode(
            topk, features_l, memory, output_memory, enc_coord, geo, mask_features)
        pack = None
        if sel is not None:  # (class-wise path?, thresholds ..., instance branch on?) — see forward()
            det_cls = self._detector_box_cls(box_cls) if sel[6] else box_cls
            pack = self._select_device(det_cls, box_pred, sizes, sel[0])
            if len(sel) > 7:  # sel[7] = (image sizes, output sizes, mask slot bytes or None, semantic / panoptic configuration[, C])
                image_sizes, out_sizes, mask_slot, sem, pan = sel[7][:5]
                cap = sel[7][5] if len(sel[7]) > 5 else None
                if cap is not None:  # capacity mode: the size columns come from the device sizes (exact in fp32)
                    size_columns = dims.to(torch.float32)
                pack = self._pack_rows(pack, size_columns, box_cls, box_pred, mask_logits, sizes, image_sizes, tuple(images.shape[-2:]),
                                       sel[0], out_sizes, mask_slot, sem, pan, dims=dims, cap=cap)
        return (memory, output_memory, enc_cls, enc_coord, features, feats, topk, box_cls, box_pred, inter_states,
                init_reference, inter_references, mask_logits, pack)

    def _stage_decode(self, topk, features_l, memory, output_memory, enc_coord, geo, mask_features=None):
        inter_states, init_reference, inter_references = self.transformer.stage_decode(
            memory, output_memory, enc_coord, topk, geo)
        states16 = inter_states  # decoder outputs are LayerNorm outputs in the engine dtype
        inter_states, init_reference, inter_references = inter_states.float(), init_reference.float(), inter_references.float()
        # only the last decoder level feeds inference (:514-523); levels 0..n-2 are aux outputs
        lvl = inter_states.shape[0] - 1
        reference = init_reference if lvl == 0 else inter_references[lvl - 1]
        with torch.autocast("cuda", enabled=False):
            if states16.dtype in (torch.float16, torch.bfloat16):
                # engine: query x text logits and the box MLP on the tensor cores (fp32 accumulation, fp32 outputs)
                box_cls = self.class_embed[lvl](states16[lvl], features_l.float())
                box_pred = (self.bbox_embed[lvl](states16[lvl], out_dtype=torch.float32) + inverse_sigmoid(reference)).sigmoid()
            else:
                box_cls = self.class_embed[lvl](inter_states[lvl], features_l.float())
                box_pred = (self.bbox_embed[lvl](inter_states[lvl]) + inverse_sigmoid(reference)).sigmoid()
        mask_logits = None
        if mask_features is not None:
            # (:507-517) only the last level's masks reach inference (the other levels are added times 0.0)
            mf = mask_features
            if states16.dtype in (torch.float16, torch.bfloat16) and mf.dtype == states16.dtype and mf.shape[1] % 8 == 0:
                # engine: einsum("bqc,bchw->bqhw") = one wgmma GEMM per image over the token-major mask features
                # (fp32 accumulation, fp32 logits: their sign decides the mask)
                B, C, mh, mw = mf.shape
                tok = mf.permute(0, 2, 3, 1).reshape(B, mh * mw, C)  # free: the engine's mask features are channels_last
                emb = self.mask_embed(states16[lvl])
                mask_logits = torch.stack([ops.linear_tc(emb[b].contiguous(), tok[b], out_dtype=torch.float32)
                                           for b in range(B)]).view(B, -1, mh, mw)
            else:
                mask_logits = torch.einsum("bqc,bchw->bqhw", self.mask_embed(inter_states[lvl].to(mf.dtype)), mf)
        return box_cls, box_pred, inter_states, init_reference, inter_references, mask_logits

    def _graphed(self, key, fn, tensor_args, const_args):
        """Run fn(*tensor_args, *const_args) through a CUDA graph captured once per key: inputs are copied into
        static buffers, the replay reuses the captured launch sequence (about 2 000 kernel launches per image
        otherwise dominate the wall clock).  Outputs are static buffers, valid until the next replay of `key`."""
        # the ViT's opt-in FP8 mode is part of the captured launch sequence: one graph per mode
        key = (key, self.engine_dtype, bool(getattr(getattr(self.backbone, "net", None), "fp8_linears", False)))
        entry = self._graph_cache.get(key)
        if entry is not None:
            self._graph_cache.move_to_end(key)
        if entry is None:
            # bounded cache, each graph with a private memory pool: the image sizes are an input, but prompts, batch shapes,
            # selection settings and the packed stages' output sizes still make keys; evict the least recently used
            while len(self._graph_cache) >= self.graph_cache_size:
                self._graph_cache.popitem(last=False)
            static_in = [None if t is None else t.clone() for t in tensor_args]  # None: no fusion input (DeformableDETRSegm)
            # autocast's weight-cast cache must be off while capturing: cached casts would be freed when the
            # autocast region ends while the graph still reads them
            with torch.autocast("cuda", dtype=self.engine_dtype, cache_enabled=False):
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    for _ in range(2):  # warm-up: packs weights, fills caches, sets kernel attributes
                        fn(*static_in, *const_args)
                torch.cuda.current_stream().wait_stream(side)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    static_out = fn(*static_in, *const_args)
            entry = (graph, static_in, static_out, const_args)  # const_args: the graph owns the geometry tensors it reads
            self._graph_cache[key] = entry
        graph, static_in, static_out = entry[:3]
        for dst, src in zip(static_in, tensor_args):
            if dst is not None:
                dst.copy_(src)
        graph.replay()
        return static_out

    def maskdino_mask_features(self, memory, features, geo):
        """:728-750: p2 -> 1x1 conv + GroupNorm, + encoder memory of the mask_encode_level (bilinearly resized to p2),
        3x3 conv + GroupNorm + ReLU, 1x1 conv -> [B, C, h, w]."""
        lvl = self.mask_encode_level
        shapes = geo["shapes"]
        start = sum(h * w for h, w in shapes[:lvl])
        h, w = shapes[lvl]
        p2 = features[self.mask_in_features[0]]
        if memory.is_cuda and memory.dtype in (torch.float16, torch.bfloat16) and p2.dtype == memory.dtype \
                and isinstance(self.lateral_conv.norm, nn.GroupNorm) and p2.shape[1] % 8 == 0:
            # engine: token-major throughout; the two 1x1 convolutions are wgmma GEMMs, GroupNorm is the repo's kernel, the
            # memory slice of the encode level is already token-major (no permute); the 3x3 convolution is the library's
            from .backbone import _conv_weights

            B, C, H2, W2 = p2.shape
            dt = memory.dtype
            tok = p2.permute(0, 2, 3, 1).reshape(B * H2 * W2, C)
            y = ops.linear_tc(tok, _conv_weights(self.lateral_conv, dt))
            gw, gb = ops.packed(self.lateral_conv.norm, dt)
            x = ops.groupnorm_nhwc(y.view(B, H2 * W2, -1), gw, gb, self.lateral_conv.norm.num_groups, self.lateral_conv.norm.eps)
            hid = x.shape[-1]
            if (h, w) == (H2, W2):  # same stride: the bilinear resize (:737-742) is the identity
                x = x + memory[:, start:start + h * w]
            else:
                enc = memory[:, start:start + h * w].permute(0, 2, 1).reshape(B, hid, h, w)
                x = x + F.interpolate(enc, size=(H2, W2), mode="bilinear", align_corners=False).permute(0, 2, 3, 1).reshape(B, H2 * W2, hid)
            from .backbone import conv3x3_tokens

            z = conv3x3_tokens(self.output_conv, x.reshape(B * H2 * W2, hid), B, H2, W2, getattr(self.backbone, "conv3x3_engine", False))
            gw, gb = ops.packed(self.output_conv.norm, dt)
            z = ops.groupnorm_nhwc(z.view(B, H2 * W2, hid), gw, gb, self.output_conv.norm.num_groups, self.output_conv.norm.eps)
            z = F.relu(z)
            mf = ops.linear_tc(z.view(B * H2 * W2, hid), _conv_weights(self.mask_conv, dt))
            return mf.view(B, H2, W2, -1).permute(0, 3, 1, 2)  # NCHW view over token-major (channels_last) memory
        enc = memory[:, start:start + h * w].permute(0, 2, 1).reshape(memory.shape[0], -1, h, w)
        x = self.lateral_conv(features[self.mask_in_features[0]])
        x = x + F.interpolate(enc.to(x.dtype), size=x.shape[-2:], mode="bilinear", align_corners=False)
        return self.mask_conv(self.output_conv(x))

    def _semantic(self, box_cls, box_pred, mask_pred, image_sizes, padded_hw, batched_inputs, shared_keep=None):
        """Semantic branch (:628-666, `_postprocess_semantic` :875-918): class scores of the queries that survive the
        detection NMS, softmax(sigmoid / 0.06) over classes, times the sigmoid masks at padded-image resolution.  One dict per
        image: {"sem_seg"} or, with sem_seg_format "label", {"sem_seg_label", "sem_seg_score"} (see __init__)."""
        fmt = getattr(self, "sem_seg_format", "maps")
        if fmt not in ("maps", "label", "rle"):
            raise ValueError(f"ape_b200: sem_seg_format must be 'maps', 'label' or 'rle' (got {fmt!r})")
        if fmt == "rle":
            self.sem_seg_format = "label"
            try:
                outs = self._semantic(box_cls, box_pred, mask_pred, image_sizes, padded_hw, batched_inputs, shared_keep)
            finally:
                self.sem_seg_format = "rle"
            for o in outs:
                o["sem_seg_rle"] = ops.label_map_rle(o["sem_seg_label"])
            return outs
        name = self.dataset_names[self.eval_dataset_id] if self.dataset_names else None
        things, stuff, entity = self.dataset_stuff.get(name, (None, None, "thing"))
        sem_cls = get_stuff_score(box_cls, things or [], stuff or [], entity)
        outs = []
        if self.semantic_post_nms and shared_keep is not None and sem_cls.shape == box_cls.shape:  # plain clone of the same logits
            keep = shared_keep
        elif self.semantic_post_nms:
            keep = [r.query_index for r in self.inference(sem_cls, box_pred, image_sizes)]
        else:
            keep = [torch.arange(sem_cls.shape[1], device=sem_cls.device)] * sem_cls.shape[0]
        for b, (qi, size, inp) in enumerate(zip(keep, image_sizes, batched_inputs)):
            cls = F.softmax(sem_cls[b, qi].float().sigmoid() / 0.06, dim=-1)
            h, w = inp.get("height", size[0]), inp.get("width", size[1])
            class0 = None  # (:655-664) the "things" column of a stuff dataset is a constant
            if entity == "stuff" and stuff and stuff[0] == "things" and self.stuff_prob_thing > 0:
                class0 = math.log(self.stuff_prob_thing / (1 - self.stuff_prob_thing))
            engine = self.engine_dtype in (torch.float16, torch.bfloat16) and mask_pred.is_cuda
            if fmt == "label" and engine:
                # engine: resample the kept masks once at the output size and take the class argmax in the GEMM epilogue
                # (csrc/semseg.cu); the [N, H, W] map below is never formed
                label, score = ops.semseg_label(mask_pred[b].contiguous(), qi, cls.to(self.engine_dtype), padded_hw, size, (h, w),
                                                class0)
                outs.append({"sem_seg_label": label, "sem_seg_score": score})
                continue
            if engine and len(qi) > 0:
                # engine: einsum("qc,qhw->chw") (757 GFLOP at K = 300 kept queries x 1203 names x 1024^2) as ONE wgmma GEMM:
                # the resize runs channels_last so that the sigmoid masks come out pixel-major [H*W, K] = the K-major operand
                dt = self.engine_dtype
                K = len(qi)
                Kp = (K + 7) // 8 * 8
                mp = mask_pred[b, qi][None].float()
                if Kp != K:
                    mp = torch.cat([mp, mp.new_zeros(1, Kp - K, *mp.shape[-2:])], 1)
                mp = mp.contiguous(memory_format=torch.channels_last)
                m = F.interpolate(mp, size=padded_hw, mode="bilinear", align_corners=False).sigmoid()
                m = m.permute(0, 2, 3, 1).reshape(-1, Kp).to(dt)                               # [H*W, Kp]
                ct = torch.zeros((cls.shape[1], Kp), dtype=dt, device=cls.device)
                ct[:, :K] = cls.t().to(dt)                                                      # [N, Kp] (zero weight on the padding)
                result = ops.linear_tc(ct, m, out_dtype=torch.float32).view(cls.shape[1], *padded_hw)
            else:
                m = F.interpolate(mask_pred[b, qi][None].float(), size=padded_hw, mode="bilinear", align_corners=False)[0].sigmoid()
                result = torch.einsum("qc,qhw->chw", cls, m)  # stays on the GPU (the reference moves >1000 classes to the CPU, :896-898)
            sem = sem_seg_postprocess(result, size, h, w)
            if class0 is not None:
                sem[0, ...] = class0
            if fmt == "label":  # the reference definition of the label map (first maximal class, as torch.argmax)
                outs.append({"sem_seg_label": sem.argmax(0), "sem_seg_score": sem.amax(0)})
            else:
                outs.append({"sem_seg": sem})
        return outs

    def _panoptic(self, box_cls, box_pred, mask_pred, image_sizes, padded_hw, batched_inputs, shared_keep=None):
        """Panoptic branch (:671-696): queries that survive the detection NMS, merged by
        `postprocess.postprocess_panoptic` (the reference's `_postprocess_panoptic`, :919-998, without its per-segment
        host round trips).  Needs the thing / stuff split of the evaluated dataset in `self.dataset_stuff`.  On CUDA with a
        16-bit engine_dtype, `postprocess.postprocess_panoptic_winners` makes the same merge from one kernel over the logits
        (csrc/panoptic.cu) and the [K, H, W] mask stacks are never formed."""
        from .postprocess import postprocess_panoptic, postprocess_panoptic_winners

        name = self.dataset_names[self.eval_dataset_id] if self.dataset_names else None
        if name not in self.dataset_stuff:
            raise RuntimeError(f"ape_b200: panoptic_on needs model.dataset_stuff[{name!r}] = (thing_classes, stuff_classes, entity)")
        things, stuff, _ = self.dataset_stuff[name]
        things, stuff = list(things or []), list(stuff or [])
        thing_ids = range(len(things))  # contiguous ids of the thing classes (metadata.thing_dataset_id_to_contiguous_id.values())
        if self.panoptic_post_nms and shared_keep is not None:
            keep = shared_keep
        elif self.panoptic_post_nms:
            keep = [r.query_index for r in self.inference(box_cls, box_pred, image_sizes)]
        else:
            keep = [torch.arange(box_cls.shape[1], device=box_cls.device)] * box_cls.shape[0]
        engine = self.engine_dtype in (torch.float16, torch.bfloat16) and mask_pred.is_cuda
        stuff_first = bool(stuff) and stuff[0] == "things"
        outs = []
        for b, (qi, size, inp) in enumerate(zip(keep, image_sizes, batched_inputs)):
            h, w = inp.get("height", size[0]), inp.get("width", size[1])
            if engine:
                outs.append(postprocess_panoptic_winners(box_cls[b, qi].float(), mask_pred[b].contiguous(), qi, padded_hw, size, h,
                                                         w, thing_ids, len(things), stuff_first, self.panoptic_configs))
                continue
            m = F.interpolate(mask_pred[b, qi][None].float(), size=padded_hw, mode="bilinear", align_corners=False)[0]
            outs.append(postprocess_panoptic(box_cls[b, qi].float(), m, size, h, w, thing_ids, len(things), stuff_first,
                                             self.panoptic_configs))
        return outs

    def _inference_static(self, box_cls, box_pred, image_sizes, first_pack=None):
        """`inference` (:759-810 + fast_rcnn.py:97-201) with static shapes and ONE device->host copy + synchronisation per
        batch instead of four per image.  Two device paths, chosen by the number n of (query, class) pairs above the score
        threshold (as torchvision's batched_nms switches strategy by size):
          n <= static_inference_cap: pairs compacted with nonzero_static (same row-major order as `.nonzero()`), class-aware
             NMS with the coordinate-offset trick on the padded list (true count passed on the device), first top-k kept;
          n  > static_inference_cap (test_score_thresh 0.0 with a 1203-name vocabulary: 1.08 M pairs): per-class NMS over the
             shared per-query boxes (`ops.nms_classwise`, torchvision's `_batched_nms_vanilla` semantics), top-k of the
             surviving scores.  Memory is bounded by Q^2 bits whatever the vocabulary size."""
        cap, topk = int(self.static_inference_cap), int(self.test_topk_per_image)
        if topk < 0 or box_cls.shape[1] > 1024:
            return None
        classwise = bool(getattr(self, "_static_overflowed", False))
        sizes = None
        for attempt in range(2):
            if not (attempt == 0 and first_pack is not None) and sizes is None:
                sizes = self._sizes_tensor(image_sizes)
            dev_pack = first_pack if (attempt == 0 and first_pack is not None) else \
                self._select_device(box_cls, box_pred, sizes, classwise)
            host = dev_pack.to("cpu")  # the one synchronising copy
            over = any(int(host[b, 0, 7].item()) > cap for b in range(len(image_sizes)))
            if over == classwise:
                break
            classwise = over  # wrong path for this batch: run the other one (and start with it next time)
        self._static_overflowed = classwise
        results = []
        for b, (h, w) in enumerate(image_sizes):
            p = host[b]
            nk = int(p[0, 8].item())
            p = p[:nk]
            results.append(Instances((h, w), pred_boxes=Boxes(p[:, :4].contiguous()), scores=p[:, 4].contiguous(),
                                     pred_classes=p[:, 5].to(torch.int64), query_index=p[:, 6].to(torch.int64)))
        return results

    def _select_device(self, box_cls, box_pred, sizes, classwise):
        """Device half of `_inference_static`: [B, topk, 9] fp32 = (x1, y1, x2, y2, score, class, query index, number of
        candidates, number kept) per detection slot; static shapes, no host synchronisation (CUDA-graph / NCCL friendly)."""
        cap, topk = int(self.static_inference_cap), int(self.test_topk_per_image)
        # sizes: int32 [B, 2] (h, w) on the device (a graph input), so the fp32 scaling and clamp below read them from device memory
        hw = sizes.to(device=box_cls.device, dtype=torch.float32)
        zero = hw.new_zeros(())
        packs = []
        for b in range(box_cls.shape[0]):
            h, w = hw[b, 0], hw[b, 1]
            scores = box_cls[b].float().sigmoid().contiguous()                              # [Q, N] (bg column dropped again, :772)
            xyxy = box_cxcywh_to_xyxy(box_pred[b].float())
            boxes = torch.stack((xyxy[:, 0] * w, xyxy[:, 1] * h, xyxy[:, 2] * w, xyxy[:, 3] * h), dim=-1)
            valid = torch.isfinite(boxes).all(dim=1) & torch.isfinite(scores).all(dim=1)     # fast_rcnn.py:120-123
            qmap = valid.cumsum(0) - 1                                                       # row index after the filter
            boxes = torch.stack((boxes[:, 0].clamp(min=zero, max=w), boxes[:, 1].clamp(min=zero, max=h),
                                 boxes[:, 2].clamp(min=zero, max=w), boxes[:, 3].clamp(min=zero, max=h)), dim=-1).contiguous()
            mask = (scores > self.test_score_thresh) & valid[:, None]
            n = mask.sum().to(torch.int32).reshape(1)
            Q, N = scores.shape
            if classwise:
                k = min(topk, Q * N)
                surv = ops.nms_classwise(boxes, scores, self.test_score_thresh, self.test_nms_thresh,
                                         row_valid=valid.to(torch.uint8))                   # [N, Q], -inf = gone
                topv, topi = torch.topk(surv.flatten(), k)                                  # descending score
                c, q = topi // Q, topi % Q
                nk = torch.isfinite(topv).sum().to(torch.float32)
                pack = torch.cat([boxes[q], topv[:, None], c[:, None].float(), qmap[q, None].float(),
                                  torch.stack([n[0].float(), nk]).expand(k, 2)], dim=1)
                if k < topk:
                    pack = torch.cat([pack, pack.new_zeros(topk - k, 9)], 0)
                packs.append(pack)
                continue
            flat = torch.nonzero_static(mask.flatten(), size=cap, fill_value=0)[:, 0]
            slot_ok = torch.arange(cap, device=flat.device) < n
            q, c = flat // N, flat % N
            cb = boxes[q]
            cs = torch.where(slot_ok, scores.flatten()[flat], scores.new_full((), float("-inf")))
            # batched_nms: boxes + class * (max coordinate over the candidates + 1), scores sorted descending
            mx = torch.where(slot_ok[:, None], cb, cb.new_full((), float("-inf"))).max()
            nb = cb + (c.to(cb) * (mx + 1))[:, None]
            order = cs.sort(0, descending=True)[1]
            keep, _ = ops.nms_sorted_mask(nb.index_select(0, order).contiguous(), self.test_nms_thresh, n_valid=n)
            pos = torch.nonzero_static(keep, size=topk, fill_value=0)[:, 0]
            nk = keep.sum().clamp(max=topk).to(torch.float32)
            sel = order[pos]
            packs.append(torch.cat([cb[sel], cs[sel, None], c[sel, None].float(), qmap[q[sel], None].float(),
                                    torch.stack([n[0].float(), nk]).expand(topk, 2)], dim=1))  # [topk, 9]
        return torch.stack(packs)

    def forward_packed(self, batched_inputs):
        """Detections as ONE device tensor, without touching the host: the multi-GPU path hands it straight to one NCCL gather
        on the compute stream (ape_b200.parallel.gather_packed) and only the destination rank copies to the host.
        Boxes only: fp32 [B, topk, 13], the 9 columns of `_select_device` + image height / width and requested output height /
        width.  With `instance_on and test_mask_on`: uint8 [B, topk, 60 + mask_slot_bytes], those 13 columns as bytes, then
        each kept mask as a COCO run-length code in a slot of fixed size (`ops.mask_pack`); `parallel.unpack_packed` turns
        either into what `model(inputs)` returns (with `mask_format = "rle"` for masks).  The selection path (candidate list
        vs class-wise NMS) is the one the last host-synchronised forward found appropriate; the packed rows carry the candidate
        count so the receiver can tell if that choice was wrong for an image (count > static_inference_cap on the
        candidate-list path).
        With `semantic_on`: uint8 [B, 32 + topk * R + sem_seg_slot_bytes] per image, a header of 8 int32 (topk, R, semantic slot
        kind, its bytes used, output height, width, labels present, 0), then that image's rows of either form above (R = 52, or 60 +
        mask_slot_bytes), then its semantic label map as one run-length code per label (`ops.semseg_pack`): `unpack_packed` adds
        `sem_seg_rle` as `model(inputs)` returns it with `sem_seg_format = "rle"`.  Needs a 16-bit engine_dtype on CUDA.
        With `panoptic_on`: the same 2-D form with a panoptic slot of `panoptic_slot_bytes` at the end of each image's row, whose
        size is header word 7 (0 in every other form; without semantic_on the semantic slot is empty, kind 0).  The slot holds a
        header of 8 int32 (1, or 0 when the dataset's entity turns the branch off; segments S; output height, width; table rows
        Kt = topk with panoptic_post_nms, else num_queries; bytes used; 0; 0), Kt rows of int32 (id, isthing, category_id) of
        which the first S are the segments, then the panoptic map as uint16 (`ops.panoptic_pack`): `unpack_packed` adds
        `panoptic_seg` as `model(inputs)` returns it.  Needs a 16-bit engine_dtype on CUDA; an output whose slot would not fit
        raises ValueError before anything runs."""
        masks = self.instance_on and self.test_mask_on
        sem = self._packed_semantic_config() if self.semantic_on else None
        pan = self._packed_panoptic_config() if self.panoptic_on else None
        if sem is not None and not (self.engine_dtype in (torch.float16, torch.bfloat16) and self.device.type == "cuda"):
            raise ValueError("ape_b200: forward_packed with semantic_on needs a CUDA model with a 16-bit engine_dtype (the semantic "
                             "label map is built by ops.semseg_label); use model(inputs) with sem_seg_format = 'rle' instead")
        if pan is not None:
            self._check_panoptic_slot(pan, batched_inputs)
        box_cls, box_pred, image_sizes, pack, mask_pred, padded_hw = self.forward(batched_inputs, do_postprocess="packed")
        if pack is not None and (masks or sem is not None or pan is not None):
            return pack.clone()  # the stages ran in the graph; their buffer is rewritten by the next replay
        if pack is None:  # no graph for this call (fp32 mode, phrase prompts ...): the same selection, eagerly
            ent = self.eval_dataset_entity
            det_cls = self._detector_box_cls(box_cls) if (self.instance_on and not (ent and "thing" not in ent)) else box_cls
            pack = self._select_device(det_cls, box_pred, self._sizes_tensor(image_sizes), bool(getattr(self, "_static_overflowed", False)))
        cols = self._size_columns(batched_inputs, image_sizes, pack.device)
        if masks or sem is not None or pan is not None:
            # capacity mode runs the kernels the graph runs, so the two agree by construction
            cap = self._packed_capacity(batched_inputs, image_sizes)
            dims = self._dims_tensor(batched_inputs, image_sizes) if cap is not None else None
            return self._pack_rows(pack, cols, box_cls, box_pred, mask_pred, self._sizes_tensor(image_sizes), tuple(image_sizes), padded_hw,
                                   bool(getattr(self, "_static_overflowed", False)), self._output_sizes(batched_inputs, image_sizes),
                                   int(self.mask_slot_bytes) if masks else None, sem, pan, dims=dims, cap=cap)
        return torch.cat([pack, cols[:, None, :].expand(-1, pack.shape[1], -1)], dim=2)

    @staticmethod
    def _output_sizes(batched_inputs, image_sizes):
        return tuple((int(inp.get("height", h)), int(inp.get("width", w))) for (h, w), inp in zip(image_sizes, batched_inputs))

    def _size_columns(self, batched_inputs, image_sizes, device=None):
        """[B, 4] fp32 (image height, width, output height, width) on the device, cached per geometry: no pageable upload per call."""
        device = self.device if device is None else device
        rows = tuple((float(h), float(w), float(oh), float(ow))
                     for (h, w), (oh, ow) in zip(image_sizes, self._output_sizes(batched_inputs, image_sizes)))
        cache = self.__dict__.setdefault("_packed_extra", {})
        extra = cache.get((rows, str(device)))
        if extra is None:
            if len(cache) > 64:
                cache.clear()
            extra = cache[(rows, str(device))] = torch.tensor(rows, dtype=torch.float32).to(device)
        return extra

    def _packed_capacity(self, batched_inputs, image_sizes):
        """model.packed_output_capacity when it is set and every image and output size of the call fits C x C, else None.
        ValueError for a capacity that is not an int in [1, ops.PACKED_CAPACITY_MAX]."""
        cap = self.packed_output_capacity
        if cap is None:
            return None
        cap = ops.check_capacity(cap)
        sizes = list(image_sizes) + list(self._output_sizes(batched_inputs, image_sizes))
        return cap if all(h <= cap and w <= cap for h, w in sizes) else None

    def _dims_tensor(self, batched_inputs, image_sizes):
        """(image h, w, output h, w) as int32 [B, 4] on the device, cached per sizes like _sizes_tensor: capacity mode's graph input."""
        rows = tuple((int(h), int(w), int(oh), int(ow))
                     for (h, w), (oh, ow) in zip(image_sizes, self._output_sizes(batched_inputs, image_sizes)))
        key = (rows, str(self.device))
        cache = self.__dict__.setdefault("_dims_dev", {})
        dims = cache.get(key)
        if dims is None:
            if len(cache) > 64:
                cache.clear()
            dims = cache[key] = torch.tensor(rows, dtype=torch.int32, pin_memory=True).to(self.device, non_blocking=True)
        return dims

    def _packed_semantic_config(self):
        """Everything the packed semantic stage reads from the model, as a graph-key tuple: (slot bytes, branch on for the
        evaluated dataset, semantic_post_nms, class-0 constant or None, thing classes, stuff classes, entity)."""
        ent = self.eval_dataset_entity
        name = self.dataset_names[self.eval_dataset_id] if self.dataset_names else None
        things, stuff, entity = self.dataset_stuff.get(name, (None, None, "thing"))
        class0 = None  # as _semantic (:655-664)
        if entity == "stuff" and stuff and stuff[0] == "things" and self.stuff_prob_thing > 0:
            class0 = math.log(self.stuff_prob_thing / (1 - self.stuff_prob_thing))
        slot = int(self.sem_seg_slot_bytes)
        if slot < 16 or slot % 4:
            raise ValueError(f"ape_b200: sem_seg_slot_bytes must be a multiple of 4 of at least 16 (got {slot})")
        return (slot, not (ent and "stuff" not in ent), bool(self.semantic_post_nms), class0, tuple(things or ()), tuple(stuff or ()),
                entity)

    def _packed_panoptic_config(self):
        """Everything the packed panoptic stage reads from the model, as a graph-key tuple: (slot bytes, branch on for the
        evaluated dataset, panoptic_post_nms, thing classes, stuff classes, prob, pano_temp, transform_eval,
        object_mask_threshold, overlap_threshold)."""
        ent = self.eval_dataset_entity
        on = not (ent and "thing+stuff" not in ent)
        name = self.dataset_names[self.eval_dataset_id] if self.dataset_names else None
        if on and name not in self.dataset_stuff:  # as _panoptic
            raise RuntimeError(f"ape_b200: panoptic_on needs model.dataset_stuff[{name!r}] = (thing_classes, stuff_classes, entity)")
        things, stuff = self.dataset_stuff.get(name, (None, None))[:2]
        if not (self.engine_dtype in (torch.float16, torch.bfloat16) and self.device.type == "cuda"):
            raise ValueError("ape_b200: forward_packed with panoptic_on needs a CUDA model with a 16-bit engine_dtype (the panoptic "
                             "map is built by ops.panoptic_winners); use model(inputs) instead")
        slot = int(self.panoptic_slot_bytes)
        if slot < ops.PAN_PACK_HEAD or slot % 4:
            raise ValueError(f"ape_b200: panoptic_slot_bytes must be a multiple of 4 of at least {ops.PAN_PACK_HEAD} (got {slot})")
        c = self.panoptic_configs
        return (slot, bool(on), bool(self.panoptic_post_nms), tuple(things or ()), tuple(stuff or ()), float(c["prob"]),
                float(c["pano_temp"]), bool(c["transform_eval"]), float(c["object_mask_threshold"]), float(c["overlap_threshold"]))

    def _check_panoptic_slot(self, pan, batched_inputs):
        """ValueError, before anything is enqueued, when an image's panoptic map would not fit the slot: its size depends only on
        the output size and the number of queries of the merge."""
        slot, on, post_nms = pan[:3]
        if not on:
            return
        if post_nms:  # the top-k that _text_features is about to set for this call
            d = self.eval_dataset_id
            prompt = self.dataset_prompts[d] if d >= 0 else batched_inputs[0].get("prompt", "name")
            K = 1 if prompt == "expression" else int(self.select_box_nums_for_evaluation)
            if self.select_box_nums_for_evaluation_list is not None:
                K = int(self.select_box_nums_for_evaluation_list[d])
        else:
            K = int(self.num_queries)
        if K > ops.APE_PANOPTIC_MAX_K:
            raise ValueError(f"ape_b200: forward_packed merges at most {ops.APE_PANOPTIC_MAX_K} queries per panoptic map (got {K})")
        for i, inp in enumerate(batched_inputs):
            h, w = inp["image"].shape[-2:]
            oh, ow = int(inp.get("height", h)), int(inp.get("width", w))
            need = ops.panoptic_slot_bytes_needed(K, (oh, ow))
            if need > slot:
                raise ValueError(f"ape_b200: the panoptic map of image {i} ({oh} x {ow}, {K} queries) needs {need} bytes; "
                                 f"model.panoptic_slot_bytes is {slot}")

    def _pack_rows(self, pack, size_columns, box_cls, box_pred, mask_logits, sizes, image_sizes, padded_hw, classwise, out_sizes,
                   mask_slot, sem, pan=None, dims=None, cap=None):
        """Selection rows [B, topk, 9] + size columns -> what forward_packed returns: fp32 [B, topk, 13] rows, or uint8
        [B, topk, 60 + mask_slot] with the kept masks' run-length codes (mask_slot not None); with a semantic configuration
        (`_packed_semantic_config`) or a panoptic one (`_packed_panoptic_config`) each image's header, those rows as bytes, its
        semantic slot (empty without one) and its panoptic slot (none without one).  No host synchronisation.  With a capacity cap,
        the stages read the sizes from dims (int32 [B, 4] on the device) and image_sizes / out_sizes are not used."""
        rows = torch.cat([pack, size_columns[:, None, :].expand(-1, pack.shape[1], -1)], dim=2)
        if mask_slot is not None:
            if cap is not None:
                rows = ops.mask_pack_dev(mask_logits.contiguous(), rows, dims, padded_hw, mask_slot, cap)
            else:
                rows = ops.mask_pack(mask_logits.contiguous(), rows, out_sizes, padded_hw, mask_slot)
        if sem is None and pan is None:
            return rows
        B, topk = rows.shape[0], rows.shape[1]
        det = rows.contiguous().view(torch.uint8).reshape(B, -1)
        R = det.shape[1] // max(topk, 1)
        sem_bytes = sem[0] if sem is not None else 0
        pan_bytes = pan[0] if pan is not None else 0
        out = torch.empty((B, ops.SEM_PACK_HEAD + det.shape[1] + sem_bytes + pan_bytes), dtype=torch.uint8, device=rows.device)
        out[:, ops.SEM_PACK_HEAD:ops.SEM_PACK_HEAD + det.shape[1]] = det
        info = torch.zeros((B, 3), dtype=torch.int32, device=rows.device)  # kind, bytes used, labels present
        if sem is not None:
            self._pack_semantic(sem, out[:, ops.SEM_PACK_HEAD + det.shape[1]:ops.SEM_PACK_HEAD + det.shape[1] + sem_bytes], info, pack,
                                box_cls, box_pred, mask_logits, sizes, image_sizes, padded_hw, classwise, out_sizes, dims, cap)
        if pan is not None:
            self._pack_panoptic(pan, out[:, out.shape[1] - pan_bytes:], pack, box_cls, box_pred, mask_logits, sizes, image_sizes,
                                padded_hw, classwise, out_sizes, dims, cap)
        hdr = torch.zeros((B, 8), dtype=torch.int32, device=rows.device)
        hdr[:, 0], hdr[:, 1] = topk, R
        hdr[:, 2:4] = info[:, 0:2]
        hdr[:, 4:6] = size_columns[:, 2:4].to(torch.int32)
        hdr[:, 6] = info[:, 2]
        hdr[:, 7] = pan_bytes
        out[:, :ops.SEM_PACK_HEAD] = hdr.view(torch.uint8)
        return out

    def _pack_semantic(self, sem, slots, info, pack, box_cls, box_pred, mask_logits, sizes, image_sizes, padded_hw, classwise,
                       out_sizes, dims=None, cap=None):
        """The semantic slots [B, slot] of `_pack_rows` and their (kind, bytes used, labels present) in info [B, 3]."""
        slot, on, post_nms, class0, things, stuff, entity = sem
        B = slots.shape[0]
        if on:
            sem_cls = get_stuff_score(box_cls, list(things), list(stuff), entity)
            if post_nms and self.instance_on and not (self.eval_dataset_entity and "thing" not in self.eval_dataset_entity) and \
                    self._detector_box_cls(box_cls) is box_cls and sem_cls.shape == box_cls.shape:
                keep = pack  # _semantic reuses the instance branch's kept queries in this case
            elif post_nms:
                keep = self._select_device(sem_cls, box_pred, sizes, classwise)
            else:
                keep = None
            if cap is not None:
                labels = torch.stack([self._semantic_label_static(sem_cls[b], mask_logits[b], None if keep is None else keep[b], padded_hw,
                                                                  None, None, class0, dims[b], cap) for b in range(B)])
                ops.semseg_pack_dev(labels, dims, cap, sem_cls.shape[-1], slots, info)
                return
            labels = [self._semantic_label_static(sem_cls[b], mask_logits[b], None if keep is None else keep[b], padded_hw, image_sizes[b],
                                                  out_sizes[b], class0) for b in range(B)]
            ops.semseg_pack(labels, sem_cls.shape[-1], slots, info)
        else:
            slots.zero_()

    def _pack_panoptic(self, pan, slots, pack, box_cls, box_pred, mask_logits, sizes, image_sizes, padded_hw, classwise, out_sizes,
                       dims=None, cap=None):
        """The panoptic slots [B, slot] of `_pack_rows`: `_panoptic`'s merge with K = topk queries whatever the kept count (every
        query without panoptic_post_nms), no host synchronisation.  The rows of the selection at or past the kept count and the
        queries under object_mask_threshold get the score -inf, so they take no part (ops.panoptic_winners)."""
        from .postprocess import _query_scores

        slot, on, post_nms, things, stuff, prob, pano_temp, transform_eval, object_mask_threshold, overlap_threshold = pan
        if not on:
            slots.zero_()
            return
        cfg = {"prob": prob, "pano_temp": pano_temp, "transform_eval": transform_eval, "object_mask_threshold": object_mask_threshold}
        ent = self.eval_dataset_entity
        if post_nms and self.instance_on and not (ent and "thing" not in ent) and self._detector_box_cls(box_cls) is box_cls:
            keep = pack  # _panoptic reuses the instance branch's kept queries in this case
        elif post_nms:
            keep = self._select_device(box_cls, box_pred, sizes, classwise)
        else:
            keep = None
        B, Q = box_cls.shape[0], box_cls.shape[1]
        stuff_first = bool(stuff) and stuff[0] == "things"
        for b in range(B):
            if keep is None:
                qi, live = torch.arange(Q, device=box_cls.device), None
            else:
                qi = keep[b, :, 6].to(torch.int64).clamp(0, Q - 1)
                live = torch.arange(keep.shape[1], device=keep.device) < keep[b, :, 8].to(torch.int64)
            scores, labels, kept = _query_scores(box_cls[b, qi].float(), cfg)
            if live is not None:
                kept = kept & live
            scores = torch.where(kept, scores, float("-inf"))
            if cap is not None:
                ids, counts = ops.panoptic_winners_dev(mask_logits[b].contiguous(), qi, scores, padded_hw, dims[b], cap, prob)
                ops.panoptic_pack_dev(ids, counts, labels.to(torch.int32), box_cls.shape[-1], len(things), stuff_first, overlap_threshold,
                                      dims[b], cap, slots[b])
                continue
            ids, counts = ops.panoptic_winners(mask_logits[b].contiguous(), qi, scores, padded_hw, image_sizes[b], out_sizes[b], prob)
            ops.panoptic_pack(ids, counts, labels.to(torch.int32), box_cls.shape[-1], len(things), stuff_first, overlap_threshold,
                              slots[b])

    def _semantic_label_static(self, sem_cls, mask_logits, keep, padded_hw, size, out_hw, class0, dims=None, cap=None):
        """`_semantic`'s label map of one image with K = topk queries whatever the kept count (no host synchronisation): the
        rows of `keep` ([topk, 9] selection rows, None = every query) at or past the kept count get zero class weights, so the
        class GEMM adds exact zeros for them.  With a capacity cap the sizes are dims ([4] on the device) and the map is
        ops.semseg_label_dev's [cap * cap] buffer."""
        Q = sem_cls.shape[0]
        if keep is None:
            qi, live = torch.arange(Q, device=sem_cls.device), None
        else:
            qi = keep[:, 6].to(torch.int64).clamp(0, Q - 1)
            live = torch.arange(keep.shape[0], device=keep.device) < keep[:, 8].to(torch.int64)
        cls = F.softmax(sem_cls[qi].float().sigmoid() / 0.06, dim=-1)
        if live is not None:
            cls = torch.where(live[:, None], cls, cls.new_zeros(()))
        if cap is not None:
            return ops.semseg_label_dev(mask_logits.contiguous(), qi, cls.to(self.engine_dtype), padded_hw, dims, cap, class0)
        label, _ = ops.semseg_label(mask_logits.contiguous(), qi, cls.to(self.engine_dtype), padded_hw, size, out_hw, class0)
        return label

    def inference(self, box_cls, box_pred, image_sizes):
        """:759-810 + fast_rcnn.py:40-95.  CUDA: the static-shape selection above (device results; bounded memory for any
        vocabulary size); CPU: the literal per-image sequence."""
        if box_cls.is_cuda and self.static_inference_cap > 0:
            res = self._inference_static(box_cls, box_pred, image_sizes)
            if res is not None:
                return [r.to(box_cls.device) for r in res]
        results = []
        zeros = torch.zeros((box_cls.size(1), 1), device=box_cls.device, dtype=box_cls.dtype)
        for b, (h, w) in enumerate(image_sizes):
            scores = torch.cat((box_cls[b].sigmoid(), zeros), dim=1)
            scale = torch.tensor([w, h, w, h], dtype=box_pred.dtype, device=box_pred.device)
            boxes = box_cxcywh_to_xyxy(box_pred[b]) * scale
            bx, sc, cl, qi = fast_rcnn_inference_single_image(boxes.float(), scores.float(), (h, w), self.test_score_thresh,
                                                              self.test_nms_thresh, self.test_topk_per_image)
            results.append(Instances((h, w), pred_boxes=Boxes(bx), scores=sc, pred_classes=cl, query_index=qi))
        return results


class DeformableDETRSegm(DeformableDETRSegmVL):
    """ape/modeling/ape_deta/deformable_detr_segm.py (APE-L_A): the model of DeformableDETRSegmVL without vision-language
    fusion, over DeformableDetrTransformer.  Same constructor keywords and forward contract.  Text features of every prompt
    type go straight to the classifier (no fusion input to the encoder, no `features_l` mix), and region prompts
    (`mask_prompt`) are not read, as in the reference.  The step is captured in a CUDA graph for "name" prompts: the text
    enters only the classifier, so the graph key on the shape of the text features covers it."""

    def _text_features(self, batched_inputs):
        prompt, features_l, _ = super()._text_features(batched_inputs)
        return prompt, features_l, None

    def _mask_prompt(self, batched_inputs, batch_shape, geo):
        return None

    @staticmethod
    def _graph_prompt(prompt, fusion):
        return prompt == "name"

    @staticmethod
    def _mix_text(prompt, features_l, fusion_out):
        return features_l


class SomeThing(nn.Module):
    """ape_deta.py:20-40."""

    def __init__(self, model_vision, model_language, **kwargs):
        super().__init__()
        self.model_vision = model_vision
        self.model_vision.set_model_language(model_language)

    def forward(self, batched_inputs, do_postprocess=True):
        return self.model_vision(batched_inputs, do_postprocess=do_postprocess)

    def set_eval_dataset(self, dataset_name):
        self.model_vision.set_eval_dataset(dataset_name)
