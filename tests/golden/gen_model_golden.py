"""Generates tests/golden/model_mini_*.npz by running the REFERENCE model (unmodified files from
/root/reference under oracle/refshim.py) on the MINI spec with name-derived synthetic weights
(oracle/synth.py).  Build container only:   python tests/golden/gen_model_golden.py

Recorded per case: backbone pyramid, neck outputs, encoder memory, two-stage outputs and the
selected proposal indices, decoder states / references, logits, boxes and the final detections
(boxes, scores, classes, kept query indices) — the boundary tensors of SURVEY.md §8(a) rows
a4-a18."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from ape_b200 import configs  # noqa: E402
from oracle import ref_model, synth  # noqa: E402

CASES = {
    # name: (list of (h, w, out_h, out_w), text_prompt or None)
    "single": ([(48, 64, 96, 128)], None),
    "batch2": ([(64, 64, 64, 64), (40, 56, 80, 112)], None),
    "phrase": ([(64, 48, 64, 48)], "red apple,a dog on grass,tall tree"),
    # referring expressions (prompt "expression": texts from `expressions`, one box per image; :184-193, :289-290)
    "expression": ([(64, 56, 128, 112)], ["the red apple on the left", "a dog"]),
    # region prompt (`mask_prompt`, deformable_detr_segm_vl.py:394-412): proposals only inside the rectangle (y0, y1, x0, x1)
    "maskprompt": ([(64, 64, 64, 64)], None, (8, 40, 16, 56)),
}


def main(only=None):
    spec = configs.MINI
    model, names = ref_model.build_reference_model(spec)
    synth.fill_state_dict(model)
    cap = {}

    def hook(name):
        def f(mod, inp, out):
            cap[name] = out
        return f

    model.backbone.register_forward_hook(hook("backbone"))
    model.neck.register_forward_hook(hook("neck"))
    model.transformer.register_forward_hook(hook("transformer"))
    model.transformer.encoder.register_forward_hook(hook("encoder"))
    for i, layer in enumerate(model.transformer.encoder.vl_layers):
        layer.register_forward_hook(hook(f"vlf{i}"))

    for cname, case in CASES.items():
        sizes, text = case[0], case[1]
        rect = case[2] if len(case) > 2 else None
        if only and cname != only:
            continue
        inputs = []
        for i, (h, w, oh, ow) in enumerate(sizes):
            d = {"image": synth.image(h, w, seed=i), "height": oh, "width": ow}
            if rect is not None:
                mp = torch.zeros(h, w)
                mp[rect[0]:rect[1], rect[2]:rect[3]] = 1.0
                d["mask_prompt"] = mp
            if isinstance(text, list):
                d["prompt"] = "expression"
                d["expressions"] = list(text)
            elif text is not None:
                d["prompt"] = "text"
                d["text_prompt"] = text
            inputs.append(d)
        cap.clear()
        # record the proposal indices the reference really selected: it gathers the chosen boxes with
        # torch.gather(enc_outputs_coord_unact, 1, topk_proposals[..., None].repeat(1, 1, 4))
        # (deformable_transformer_vl.py:627-629)
        gathered = []
        orig_gather = torch.gather

        def spy(inp, dim, index, *a, **k):
            if index.dim() == 3 and index.shape[-1] == 4 and index.shape[1] == spec["num_queries"]:
                gathered.append(index[..., 0].clone())
            return orig_gather(inp, dim, index, *a, **k)

        torch.gather = spy
        try:
            with torch.no_grad():
                out = model(inputs)
        finally:
            torch.gather = orig_gather
        (inter_states, init_reference, inter_references, enc_cls, enc_coord_unact, anchors, memory, feats_l) = cap["transformer"]
        assert len(gathered) == 1
        topk = gathered[0]
        assert torch.equal(orig_gather(enc_coord_unact, 1, topk.unsqueeze(-1).repeat(1, 1, 4)).sigmoid(), init_reference)
        # large per-token tensors are stored for every 4th token / channel only (fixture size)
        rec = {f"backbone.{k}": v[:, ::4] for k, v in cap["backbone"].items()}
        rec.update({f"neck.{i}": v[:, ::8] for i, v in enumerate(cap["neck"])})
        rec.update(memory=memory[:, ::4], inter_states=inter_states, init_reference=init_reference,
                   inter_references=inter_references, enc_outputs_class=enc_cls,
                   enc_outputs_coord_unact=enc_coord_unact, topk_proposals=topk)
        for i in range(len(model.transformer.encoder.vl_layers)):
            rec[f"vlf{i}.v"] = cap[f"vlf{i}"][0][:, ::8]
            rec[f"vlf{i}.l"] = cap[f"vlf{i}"][1]
        for b, o in enumerate(out):
            inst = o["instances"]
            rec[f"det{b}.boxes"] = inst.pred_boxes.tensor
            rec[f"det{b}.scores"] = inst.scores
            rec[f"det{b}.classes"] = inst.pred_classes
        # logits/boxes of the last decoder level, recomputed exactly as deformable_detr_segm_vl.py:485-503
        np.savez_compressed(os.path.join(HERE, f"model_mini_{cname}.npz"),
                            **{k: v.detach().cpu().numpy() for k, v in rec.items()})
        print(cname, {k: tuple(v.shape) for k, v in rec.items() if k.startswith(("memory", "inter_states", "det", "topk"))})


def main_masks():
    """model_mini_masks.npz: the same MINI model with test_mask_on / semantic_on (SURVEY.md 8(a) rows a17, a19, a20):
    mask logits of the last decoder level, pasted instance masks (bit-packed) and the semantic map."""
    spec = configs.MINI
    model, names = ref_model.build_reference_model(spec, test_mask_on=True, semantic_on=True)
    synth.fill_state_dict(model)
    cap = {}
    orig = model.maskdino_mask_features

    def spy(*a, **k):
        cap["mask_features"] = orig(*a, **k)
        return cap["mask_features"]

    model.maskdino_mask_features = spy
    orig_interp = torch.nn.functional.interpolate
    import ape.modeling.ape_deta.deformable_detr_segm_vl as segm  # the module object refshim loaded

    def interp_spy(x, *a, **k):  # first 4-D call with num_queries channels is `mask_pred` (:563-566)
        if x.dim() == 4 and x.shape[1] == spec["num_queries"] and "pred_masks" not in cap:
            cap["pred_masks"] = x.clone()
        return orig_interp(x, *a, **k)

    segm.F.interpolate = interp_spy
    sizes = [(48, 64, 96, 128)]
    inputs = [{"image": synth.image(h, w, seed=i), "height": oh, "width": ow} for i, (h, w, oh, ow) in enumerate(sizes)]
    try:
        with torch.no_grad():
            out = model(inputs)
    finally:
        segm.F.interpolate = orig_interp
    inst = out[0]["instances"]
    rec = {"mask_features": cap["mask_features"][:, ::8], "pred_masks": cap["pred_masks"],
           "det0.boxes": inst.pred_boxes.tensor, "det0.scores": inst.scores, "det0.classes": inst.pred_classes,
           "det0.masks_packed": torch.from_numpy(np.packbits(inst.pred_masks.numpy().astype(np.uint8), axis=-1)),
           "det0.masks_shape": torch.tensor(inst.pred_masks.shape), "sem_seg": out[0]["sem_seg"]}
    np.savez_compressed(os.path.join(HERE, "model_mini_masks.npz"), **{k: v.detach().cpu().numpy() for k, v in rec.items()})
    print("masks", {k: tuple(v.shape) for k, v in rec.items()})


def main_ti():
    """model_ti_1024.npz — BASELINE.json configs[0]: APE-Ti (vit_eva02.py backbone), one image padded to 1024^2,
    80-name vocabulary, "name" prompt, pytorch_attn=True / SDPA-math on CPU.  The image is 768 x 1024 so that a
    quarter of the square is padding (masks, valid ratios).  Per-token tensors are stored sub-sampled."""
    import time

    spec = configs.APE_TI
    n_text = 80
    model, names = ref_model.build_reference_model(spec, num_text=n_text)
    synth.fill_state_dict(model)
    model.test_score_thresh = 0.0
    cap = {}
    model.backbone.register_forward_hook(lambda m, i, o: cap.__setitem__("backbone", o))
    model.transformer.register_forward_hook(lambda m, i, o: cap.__setitem__("transformer", o))
    gathered = []
    orig_gather = torch.gather

    def spy(inp, dim, index, *a, **k):
        if index.dim() == 3 and index.shape[-1] == 4 and index.shape[1] == spec["num_queries"]:
            gathered.append(index[..., 0].clone())
        return orig_gather(inp, dim, index, *a, **k)

    torch.gather = spy
    t0 = time.time()
    try:
        with torch.no_grad():
            out = model([{"image": synth.image(768, 1024, seed=11), "height": 384, "width": 512}])
    finally:
        torch.gather = orig_gather
    print(f"reference APE-Ti forward on CPU: {time.time() - t0:.1f} s")
    (inter_states, init_reference, inter_references, enc_cls, enc_coord_unact, anchors, memory, feats_l) = cap["transformer"]
    inst = out[0]["instances"]
    rec = {f"backbone.{k}": v[:, ::16, ::4, ::4] for k, v in cap["backbone"].items()}
    rec.update(memory=memory[:, ::128, ::4], enc_outputs_class=enc_cls[:, ::16], topk_proposals=gathered[0],
               init_reference=init_reference, inter_states_last=inter_states[-1][:, ::3], inter_references_last=inter_references[-1],
               **{"det0.boxes": inst.pred_boxes.tensor, "det0.scores": inst.scores, "det0.classes": inst.pred_classes})
    np.savez_compressed(os.path.join(HERE, "model_ti_1024.npz"), **{k: v.detach().cpu().numpy() for k, v in rec.items()})
    print("ti", {k: tuple(v.shape) for k, v in rec.items()})


def main_ld():
    """model_ld_1024.npz — BASELINE.json configs[1]: the real APE-L_D architecture (ViT-L 24 blocks, 6+6 deformable
    layers, 900 queries), one 1024 x 768 image padded to 1024^2, 1203-name vocabulary, "name" prompt, boxes only, run by
    the REFERENCE's own files on the CPU (pytorch_attn=True / SDPA-math, fp32).  This is the pin of the benchmarked
    configuration: the GPU tests compare the fp32 path AND the shipped 16-bit CUDA-graph engine with it stage by stage.
    Per-token tensors are stored sub-sampled (fixture size); indices, boxes and detections in full.
    Detections are recorded twice: with the config's own test_score_thresh (0.0: all 1.08 M (query, class) pairs go
    through class-aware NMS) and with a threshold placed at the 500th highest score (the bench's selection load)."""
    import time

    spec = configs.APE_L_D
    n_text = 1203
    model, names = ref_model.build_reference_model(spec, num_text=n_text)
    synth.fill_state_dict(model)
    synth.suppress_invalid_anchor_logits(model)  # invalid anchors score at the prior, as with trained weights
    cap = {}
    model.backbone.register_forward_hook(lambda m, i, o: cap.__setitem__("backbone", o))
    model.neck.register_forward_hook(lambda m, i, o: cap.__setitem__("neck", o))
    model.transformer.register_forward_hook(lambda m, i, o: cap.__setitem__("transformer", o))
    for i, layer in enumerate(model.transformer.encoder.vl_layers):
        layer.register_forward_hook(lambda m, inp, o, i=i: cap.__setitem__(f"vlf{i}", o))
    for i, layer in enumerate(model.transformer.encoder.layers):
        layer.register_forward_hook(lambda m, inp, o, i=i: cap.__setitem__(f"enc{i}", o))
    gathered = []
    orig_gather = torch.gather

    def spy(inp, dim, index, *a, **k):
        if index.dim() == 3 and index.shape[-1] == 4 and index.shape[1] == spec["num_queries"]:
            gathered.append(index[..., 0].clone())
        return orig_gather(inp, dim, index, *a, **k)

    orig_inf = model.inference

    def inf_spy(box_cls, box_pred, image_sizes, *a, **k):
        cap["box_cls"], cap["box_pred"], cap["image_sizes"] = box_cls.clone(), box_pred.clone(), image_sizes
        return orig_inf(box_cls, box_pred, image_sizes, *a, **k)

    model.inference = inf_spy
    torch.gather = spy
    t0 = time.time()
    try:
        with torch.no_grad():
            out = model([{"image": synth.image(1024, 768, seed=0), "height": 1024, "width": 768}])
    finally:
        torch.gather = orig_gather
    print(f"reference APE-L_D forward on CPU: {time.time() - t0:.1f} s")
    (inter_states, init_reference, inter_references, enc_cls, enc_coord_unact, anchors, memory, feats_l) = cap["transformer"]
    inst = out[0]["instances"]
    rec = {f"backbone.{k}": v[:, ::16, ::8, ::8] for k, v in cap["backbone"].items()}  # sampled: the file stays under 1 MB
    rec.update({f"neck.{i}": v[:, ::16, ::8, ::8] for i, v in enumerate(cap["neck"])})
    for i in range(spec["enc_layers"]):
        rec[f"vlf{i}.v"] = cap[f"vlf{i}"][0][:, ::2048, ::4]
        rec[f"vlf{i}.l"] = cap[f"vlf{i}"][1][:, ::2048, ::4]
        rec[f"enc{i}"] = cap[f"enc{i}"][:, ::2048, ::4]
    box_cls, box_pred = cap["box_cls"], cap["box_pred"]
    top = torch.topk(box_cls.flatten(), 4096)
    rec.update(memory=memory[:, ::512, ::4], enc_outputs_class=enc_cls[:, ::16], enc_outputs_coord_unact=enc_coord_unact[:, ::16],
               topk_proposals=gathered[0], init_reference=init_reference,
               inter_references=inter_references, pred_logits=box_cls[:, :, ::32], pred_boxes=box_pred,
               pred_logits_top_values=top.values, pred_logits_top_index=top.indices,
               **{"det0.boxes": inst.pred_boxes.tensor, "det0.scores": inst.scores, "det0.classes": inst.pred_classes})
    # second selection load: threshold at the 500th highest score (between two distinct score values)
    sc = box_cls.flatten().sigmoid()
    s = torch.unique(sc).flip(0)  # distinct values, descending
    k = int((sc > s[499]).sum())  # at least 499 candidates; the threshold sits between two distinct values
    thr = float((s[499].double() + s[500].double()) / 2)
    print(f"thresholded selection: {int((sc > thr).sum())} candidates above {thr:.6f}")
    model.test_score_thresh = thr
    with torch.no_grad():
        res, finds = orig_inf(box_cls, box_pred, cap["image_sizes"])
    r = res[0]
    rec.update(**{"det_thr.thresh": torch.tensor(thr), "det_thr.boxes": r.pred_boxes.tensor, "det_thr.scores": r.scores,
                  "det_thr.classes": r.pred_classes, "det_thr.query_index": finds[0]})
    np.savez_compressed(os.path.join(HERE, "model_ld_1024.npz"), **{k: v.detach().cpu().numpy() for k, v in rec.items()})
    print("ld", {k: tuple(v.shape) for k, v in rec.items()})


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "ld":
        main_ld()
    elif len(sys.argv) > 1 and sys.argv[1] in CASES:
        main(only=sys.argv[1])
    elif len(sys.argv) > 1 and sys.argv[1] == "ti":
        main_ti()
    elif len(sys.argv) > 1 and sys.argv[1] == "masks":
        main_masks()
    else:
        main()
        main_masks()
