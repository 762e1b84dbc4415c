"""GPU: every form of the instance-mask and panoptic pixel kernels (csrc/mask_post.cu, csrc/panoptic.cu) against the float64
oracle of oracle/mask_chain.py, exactly at every pixel the oracle calls certain, on the adversarial inputs of that module: box
edges on texels, boxes past every side of the image, degenerate and sub-pixel boxes, partial bit words, 1-wide grids, exact
ties (upsampled values of exactly 0, roi averages and paste values of exactly 0.5, p of exactly 0.5 at prob 0.5, duplicate
queries).  Each case prints its number of uncertain pixels and asserts it below the bound, so that no case passes vacuously.

One-line mutations of the kernels this file catches (the first test to fail):
  mask_binarize_kernel  `v > 0.f` -> `v >= 0.f`                  test_crop_and_resize_dyadic_ties
                        `y0 < h - 1` -> `y0 < h`                  test_crop_and_resize[production-*]
  mask_roialign_kernel  `y_low >= Hp - 1` -> `y_low > Hp - 1`     test_crop_and_resize[production-*]
                        `y > (float)Hp` -> `y >= (float)Hp`       test_crop_and_resize_dyadic_ties
  paste_px              `v >= threshold` -> `v > threshold`       test_paste_and_its_run_length_form
                        `x_w < S` -> `x_w < S - 1`                test_paste_and_its_run_length_form
  panoptic_winners      `s > best` -> `s >= best`                 test_panoptic_dyadic_ties (the duplicate query)
                        `best_p >= prob` -> `best_p > prob`       test_panoptic_dyadic_ties (p == 0.5 at prob 0.5)
                        resize2 columns over Wp, not img_w        test_panoptic_crop_edge
`max(grid_h * grid_w, 1)` -> `grid_h * grid_w` in mask_roialign_kernel changes no output: a product <= 0 means a grid count
<= 0, so no sample runs, and 0 / 0 = NaN >= 0.5 is false like 0 / 1."""
import pytest
import torch

from ape_b200 import ops
from oracle import mask_chain as MC
from oracle import rle as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# Bounds on the share of pixels the oracle leaves uncertain, per case, at about 1.5 x what the seeded inputs give (the count depends
# on the inputs and the oracle only, not on the kernel).  Observed: crop 3.5e-4 (production), 4.6e-3 (odd), 4.5e-4 (partial
# words), 0 (1-wide grids, dyadic); paste <= 5.4e-6 (large), 0 (small, 1-wide, dyadic); mask_pack_dev slots <= 1.4e-3; panoptic
# <= 2.7e-5, 0 (dyadic).  The larger shares are pixels whose real-number value is exactly 0.5 (a roi average of bits, a paste
# half way between two texels) at sample positions that fp32 rounds, for example the 13 / 53 scale of the odd case or the 1.25
# box scale of the packed case: there the reference's own rounding decides, and no oracle can say which way.
BOUND = 1e-4
CROP_BOUND = {"production": 5e-4, "odd": 7e-3, "partial-words": 7e-4, "1x1": 0, "1xN": 0, "Nx1": 0}
PASTE_BOUND = {(480, 640): 1e-5, (1024, 768): 1e-5, (2048, 1536): 1e-5, (37, 53): 0, (1, 640): 0, (480, 1): 0}
PACK_BOUND = 2e-3


def _agree(what, got, on, cert, bound=BOUND):
    got, on, cert = got.to(DEV), on.to(DEV), cert.to(DEV)
    n_unc = int((~cert).sum())
    wrong = int(((got != on) & cert).sum())
    print(f"  {what}: {n_unc} uncertain of {cert.numel()} pixels ({n_unc / cert.numel():.1e}), {wrong} certain pixels differ")
    assert wrong == 0, what
    assert n_unc <= bound * cert.numel(), what


CROP = {  # name: (h, w, Hp, Wp, S, K)
    "production": (256, 256, 1024, 1024, 128, 23),
    "odd": (13, 21, 53, 83, 28, 12),
    "partial-words": (40, 47, 160, 189, 32, 24),
    "1x1": (1, 1, 37, 45, 16, 12),
    "1xN": (1, 30, 17, 120, 16, 12),
    "Nx1": (30, 1, 120, 17, 16, 12),
}


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("name", list(CROP))
def test_crop_and_resize(built, name, dtype):
    h, w, Hp, Wp, S, K = CROP[name]
    Q = K + 5
    logits = MC.smooth_logits(Q, h, w, seed=h * w, dtype=dtype)
    if h == 1 or w == 1:
        logits = torch.randn(logits.shape, generator=torch.Generator().manual_seed(3)).to(dtype)
    index = torch.randperm(Q, generator=torch.Generator().manual_seed(1))[:K]
    boxes = MC.edge_boxes(Hp, Wp, S, seed=2, n=K)
    got = ops.mask_crop_and_resize(logits.to(DEV), index.to(DEV), boxes.to(DEV), (Hp, Wp), S)
    on, cert = MC.crop_and_resize(logits.to(DEV)[index.to(DEV)], boxes, (Hp, Wp), S)
    _agree(f"crop {name} {dtype}", got, on, cert, CROP_BOUND[name])


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=["fp32", "fp16", "bf16"])
def test_crop_and_resize_dyadic_ties(built, dtype):
    """Upsampled values of exactly 0 are off; roi averages of exactly 0.5 are on; samples on y = Hp and y = -1 count."""
    L, boxes, padded, S = MC.dyadic_crop_case()
    got = ops.mask_crop_and_resize(L.to(DEV, dtype), torch.arange(len(L), device=DEV), boxes.to(DEV), padded, S)
    on, cert = MC.crop_and_resize(L.to(DEV), boxes, padded, S)
    _agree(f"crop dyadic {dtype}", got, on, cert, 0)


PASTE = [(480, 640), (1024, 768), (2048, 1536), (37, 53), (1, 640), (480, 1)]


def _paste_masks(S=128):
    """Masks for MC.paste_boxes: all ones in the whole-image box and in the box past every side, all zeros in the boxes that touch
    only the last row and the last column, smooth shapes elsewhere (the degenerate boxes included)."""
    masks = MC.smooth_logits(17, S, S, seed=9) > 0
    masks[0:2] = True
    masks[4:6] = False
    return masks


@pytest.mark.parametrize("hw", PASTE)
def test_paste_and_its_run_length_form(built, hw):
    masks = _paste_masks()
    boxes = MC.paste_boxes(*hw, seed=hw[0] + hw[1], n=len(masks))
    if hw == (2048, 1536):
        boxes[8:] = boxes[8:] * torch.tensor([3.0, 3.0, 3.0, 3.0])  # upsampling pastes (boxes wider than the mask)
    on, cert = MC.paste(masks.to(DEV), torch.ones_like(masks, device=DEV), boxes, hw)
    got = ops.paste_masks_in_image(masks.to(DEV), boxes.to(DEV), hw)
    bound = PASTE_BOUND[hw]
    _agree(f"paste {hw}", got, on, cert, bound)
    rles = ops.paste_masks_rle(masks.to(DEV), boxes.to(DEV), hw)
    dec = torch.from_numpy(__import__("numpy").stack([R.decode(r) for r in rles])).bool()
    _agree(f"paste_rle {hw}", dec, on, cert, bound)


def test_paste_dyadic_ties(built):
    """Column 16 of a 128-wide box at x = 16.5 samples ixf = -0.5 with weight exactly 1/2: on (the threshold is >= 0.5)."""
    masks, boxes, hw = MC.dyadic_paste_case()
    on, cert = MC.paste(masks.to(DEV), torch.ones_like(masks, device=DEV), boxes, hw)
    assert on[0, 20:140, 16].all()
    _agree("paste dyadic", ops.paste_masks_in_image(masks.to(DEV), boxes.to(DEV), hw), on, cert, 0)
    import numpy as np

    dec = torch.from_numpy(np.stack([R.decode(r) for r in ops.paste_masks_rle(masks.to(DEV), boxes.to(DEV), hw)])).bool()
    _agree("paste_rle dyadic", dec, on, cert, 0)


def test_mask_pack_dev_slots(built):
    """One image through ops.mask_pack_dev at a capacity: every kept slot, decoded (characters or bits), equals the oracle's crop
    and paste of the same rows."""
    from ape_b200 import parallel

    Q, h, w, Hp, Wp, S, topk, cap = 40, 64, 64, 256, 256, 128, 12, 320
    ih, iw, oh, ow = 240, 200, 300, 250
    logits = MC.smooth_logits(Q, h, w, seed=5, dtype=torch.float16)
    boxes = MC.edge_boxes(ih, iw, S, seed=3, n=topk)
    rows = torch.zeros((1, topk, 13))
    rows[0, :, :4] = boxes
    rows[0, :, 4] = 0.5
    rows[0, :, 6] = torch.randperm(Q, generator=torch.Generator().manual_seed(4))[:topk].float()
    rows[0, :, 8] = topk - 2  # the last two slots hold nothing
    rows[0, :, 9:13] = torch.tensor([ih, iw, oh, ow]).float()
    sizes = torch.tensor([[ih, iw, oh, ow]], dtype=torch.int32, device=DEV)
    out = ops.mask_pack_dev(logits[None].to(DEV).contiguous(), rows.to(DEV), sizes, (Hp, Wp), 4096, cap, S).cpu()
    planes = logits.to(DEV)[rows[0, :, 6].long().to(DEV)]
    c_on, c_cert = MC.crop_and_resize(planes, boxes, (Hp, Wp), S)
    sx, sy = torch.tensor(ow / iw, dtype=torch.float64).float(), torch.tensor(oh / ih, dtype=torch.float64).float()
    pb = torch.stack([(boxes[:, 0] * sx).clamp(0, ow), (boxes[:, 1] * sy).clamp(0, oh), (boxes[:, 2] * sx).clamp(0, ow),
                      (boxes[:, 3] * sy).clamp(0, oh)], 1)
    live = ((pb[:, 2] - pb[:, 0]) > 0) & ((pb[:, 3] - pb[:, 1]) > 0) & (torch.arange(topk) < topk - 2)
    p_on, p_cert = MC.paste(c_on, c_cert, pb, (oh, ow))
    kinds = out[0, :, 52:60].contiguous().view(torch.int32)
    n_chars = 0
    for k in range(topk):
        kind, n = int(kinds[k, 0]), int(kinds[k, 1])
        if not live[k]:
            assert kind == 0, k
            continue
        body = out[0, k, ops.MASK_PACK_HEAD:ops.MASK_PACK_HEAD + n].numpy()
        if kind == ops.MASK_SLOT_CHARS:
            n_chars += 1
            got = torch.from_numpy(R.decode({"size": [oh, ow], "counts": body.tobytes()})).bool()
            _agree(f"mask_pack_dev slot {k} (characters)", got, p_on[k], p_cert[k], PACK_BOUND)
        else:
            assert kind == ops.MASK_SLOT_BITS, k
            _agree(f"mask_pack_dev slot {k} (bits)", parallel.unpack_mask_bits(body), c_on[k], c_cert[k], PACK_BOUND)
    assert n_chars > 0


# ---- panoptic -------------------------------------------------------------------------------------------------------------
def _panoptic_check(what, logits, index, scores, padded, img, out, prob, bound=BOUND):
    o = MC.panoptic(logits, index, scores, padded, img, out, prob)
    ids, counts = ops.panoptic_winners(logits, index.to(DEV), scores.to(DEV), padded, img, out, prob)
    _agree(f"{what} ids", ids.long(), o["ids"], o["ids_certain"], bound)
    c = counts.long()
    inside = (c >= o["lo"]) & (c <= o["hi"])
    print(f"    counts: {o['unsure_pairs']} uncertain (pixel, query) pairs; widest bound {int((o['hi'] - o['lo']).max()) if c.numel() else 0}")
    assert inside.all(), (what, inside.logical_not().nonzero()[:5].tolist())
    return o


@pytest.mark.parametrize("K,img,out", [(1, (1024, 768), (1024, 768)), (300, (1024, 768), (480, 640)),
                                       (300, (600, 1000), (2048, 1536)), (900, (1024, 1024), (1024, 1024)),
                                       (300, (1024, 768), (1, 640)), (300, (1024, 768), (480, 1))])
def test_panoptic_winners(built, K, img, out):
    logits = MC.panoptic_logits(K + 7, 256, 256, seed=K + out[1]).to(DEV, torch.float16)
    index, scores = MC.panoptic_queries(K + 7, K, seed=K)
    o = _panoptic_check(f"panoptic K={K} {img} -> {out}", logits, index.to(DEV), scores.to(DEV), (1024, 1024), img, out, 0.1)
    if K >= 3:  # the repeat of query 0 and the -inf query win nowhere
        assert o["hi"][0, 1] == 0 and (o["hi"][:, 2] == 0).all()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_panoptic_winners_dtypes(built, dtype):
    logits = MC.panoptic_logits(107, 256, 256, seed=11).to(DEV, dtype)
    index, scores = MC.panoptic_queries(107, 100, seed=3)
    _panoptic_check(f"panoptic {dtype}", logits, index.to(DEV), scores.to(DEV), (1024, 1024), (1000, 900), (700, 560), 0.3)


def test_panoptic_dyadic_ties(built):
    """p == 0.5 exactly at prob 0.5 is solid; of two identical queries the lower index wins."""
    L, index, scores, padded, img, out, prob = MC.dyadic_panoptic_case()
    o = _panoptic_check("panoptic dyadic", L.to(DEV), index.to(DEV), scores.to(DEV), padded, img, out, prob, 0)
    assert torch.equal(o["lo"], o["hi"]) and o["count"][1, 0] == o["count"][0, 0] > 0 and o["count"][0, 1] == 0


def test_panoptic_crop_edge(built):
    """resize2 reads the image crop only: the last output column of an upsampled crop sits beyond the crop's last column."""
    L, index, scores, padded, img, out, prob = MC.crop_edge_panoptic_case()
    o = _panoptic_check("panoptic crop edge", L.to(DEV), index.to(DEV), scores.to(DEV), padded, img, out, prob, 0)
    assert (o["ids"][:, -1] == 0).all()


def test_panoptic_winners_dev(built):
    logits = MC.panoptic_logits(307, 256, 256, seed=17).to(DEV, torch.float16)
    index, scores = MC.panoptic_queries(307, 300, seed=17)
    img, out, cap = (1000, 800), (700, 560), 1024
    o = MC.panoptic(logits, index.to(DEV), scores.to(DEV), (1024, 1024), img, out, 0.1)
    sizes = torch.tensor([img[0], img[1], out[0], out[1]], dtype=torch.int32, device=DEV)
    ids, counts = ops.panoptic_winners_dev(logits, index.to(DEV), scores.to(DEV), (1024, 1024), sizes, cap, 0.1)
    _agree("panoptic_winners_dev ids", ids[:out[0] * out[1]].view(out).long(), o["ids"], o["ids_certain"])
    assert ((counts.long() >= o["lo"]) & (counts.long() <= o["hi"])).all()


def test_postprocess_panoptic_winners_segments(built):
    """segments_info of postprocess_panoptic_winners equals the reference loop on the oracle's areas whenever no area bound
    straddles the zero-area or overlap_threshold decision; at least one of the seeds must be decisive, so that the comparison
    happens."""
    from ape_b200.modeling.postprocess import postprocess_panoptic_winners

    n_cls, n_thing, K = 20, 10, 120
    cfg = {"prob": 0.1, "pano_temp": 0.06, "transform_eval": True, "object_mask_threshold": 0.01, "overlap_threshold": 0.4}
    img, out = (1024, 768), (480, 640)
    compared = 0
    for seed in range(3):
        logits = MC.panoptic_logits(K + 7, 256, 256, seed=seed).to(DEV, torch.float16)
        qi = torch.randperm(K + 7, generator=torch.Generator().manual_seed(seed))[:K].to(DEV)
        mask_cls = (torch.randn(K, n_cls, generator=torch.Generator().manual_seed(seed)) * 2).to(DEV)
        seg, info = postprocess_panoptic_winners(mask_cls, logits, qi, (1024, 1024), img, out[0], out[1], range(n_thing), n_thing,
                                                 True, cfg)
        s, _ = mask_cls.sigmoid().max(-1)
        kept = (s > cfg["object_mask_threshold"]).nonzero()[:, 0]
        scores, labels = torch.softmax(mask_cls.sigmoid() / cfg["pano_temp"], -1).max(-1)
        o = MC.panoptic(logits, qi[kept], scores[kept], (1024, 1024), img, out, cfg["prob"])
        want = MC.segments(o["lo"].cpu(), o["hi"].cpu(), labels[kept].cpu(), range(n_thing), n_thing, True, cfg["overlap_threshold"])
        print(f"  seed {seed}: {len(kept)} kept, {len(info)} segments, oracle {'decisive' if want is not None else 'straddles'}")
        assert len(info) > 0
        if want is not None:
            assert info == want
            compared += 1
    assert compared > 0
