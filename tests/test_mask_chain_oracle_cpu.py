"""CPU: oracle/mask_chain.py pinned to the library calls it restates (F.interpolate, torchvision roi_align, grid_sample and the
panoptic argmax, in float32 on the host), the adversarial constructors checked for their properties, and the dyadic cases
proven exact (the oracle's formulas give bit-identical values in float32 and float64 there, so their ties are certain).

Bounds on the uncertain pixels: below 5e-3 of the pixels on the adversarial random cases, 0 on the dyadic ones.  The random
cases are uncertain mostly where the real-number value sits exactly on the threshold (roi averages of bits, pastes whose
texel positions are rationals with a period of a few pixels) but the fp32 one is rounded: there the reference itself decides
by its rounding."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import mask_chain as MC

RANDOM_BOUND = 5e-3


def _lib_crop(planes, boxes, padded_hw, S):
    from torchvision.ops import roi_align

    m = F.interpolate(planes[None].float(), size=padded_hw, mode="bilinear", align_corners=False)[0]
    m = (m.sigmoid() > 0.5).float()[:, None]
    rois = torch.cat([torch.arange(len(boxes), dtype=torch.float32)[:, None], boxes], 1)
    return roi_align(m, rois, (S, S), 1.0, 0, True)[:, 0] >= 0.5


def _lib_paste(masks, boxes, hw):
    H, W = hw
    x0, y0, x1, y1 = torch.split(boxes, 1, dim=1)
    gy = (torch.arange(H, dtype=torch.float32) + 0.5 - y0) / (y1 - y0) * 2 - 1
    gx = (torch.arange(W, dtype=torch.float32) + 0.5 - x0) / (x1 - x0) * 2 - 1
    grid = torch.stack([gx[:, None, :].expand(len(boxes), H, W), gy[:, :, None].expand(len(boxes), H, W)], dim=3)
    return F.grid_sample(masks[:, None].float(), grid, align_corners=False)[:, 0] >= 0.5


def _lib_panoptic(logits, index, scores, padded, img, out, prob):
    m = F.interpolate(logits[index][None].float(), size=padded, mode="bilinear", align_corners=False)[0]
    p = F.interpolate(m[None, :, :img[0], :img[1]], size=out, mode="bilinear", align_corners=False)[0].sigmoid()
    live = scores != float("-inf")
    s = torch.where(live[:, None, None], scores[:, None, None] * p, float("-inf"))
    win = s.argmax(0)
    solid = p.gather(0, win[None])[0] >= prob
    K = len(index)
    counts = torch.stack([torch.bincount(win.flatten(), minlength=K), torch.bincount(win[solid], minlength=K),
                          ((p >= prob) & live[:, None, None]).flatten(1).sum(1)])
    return torch.where(solid, win, -1), counts


def _agree(what, want, on, cert, bound):
    n_unc = int((~cert).sum())
    wrong = int(((want != on) & cert).sum())
    print(f"  {what}: {n_unc} uncertain of {cert.numel()} pixels, {wrong} certain pixels differ from the library")
    assert wrong == 0, what
    assert n_unc <= bound * cert.numel(), what
    return n_unc


CROP_CASES = {
    "production-fp32": dict(Q=30, h=256, w=256, Hp=1024, Wp=1024, S=128, K=6, dtype=torch.float32),
    "odd-fp16": dict(Q=12, h=13, w=21, Hp=53, Wp=83, S=28, K=12, dtype=torch.float16),
    "partial-words-bf16": dict(Q=10, h=40, w=47, Hp=160, Wp=189, S=32, K=12, dtype=torch.bfloat16),
    "1x1": dict(Q=4, h=1, w=1, Hp=37, Wp=45, S=16, K=12, dtype=torch.float32),
    "1xN": dict(Q=4, h=1, w=30, Hp=17, Wp=120, S=16, K=12, dtype=torch.float16),
    "Nx1": dict(Q=4, h=30, w=1, Hp=120, Wp=17, S=16, K=12, dtype=torch.float32),
}


@pytest.mark.parametrize("name", list(CROP_CASES))
def test_crop_oracle_matches_the_library(name):
    c = CROP_CASES[name]
    logits = MC.smooth_logits(c["Q"], c["h"], c["w"], seed=len(name), dtype=c["dtype"])
    if c["h"] == 1 or c["w"] == 1:
        logits = logits * 0 + torch.randn(logits.shape, generator=torch.Generator().manual_seed(3)).to(c["dtype"])
    index = torch.arange(c["K"]) % c["Q"]
    boxes = MC.edge_boxes(c["Hp"], c["Wp"], c["S"], seed=1, n=c["K"])
    planes = logits[index]
    on, cert = MC.binarize(planes, (c["Hp"], c["Wp"]))
    want_bits = F.interpolate(planes[None].float(), size=(c["Hp"], c["Wp"]), mode="bilinear", align_corners=False)[0].sigmoid() > 0.5
    _agree(f"{name} upsample", want_bits, on, cert, RANDOM_BOUND)
    on, cert = MC.roi_align(on, cert, boxes, c["S"])
    _agree(f"{name} crop", _lib_crop(planes, boxes, (c["Hp"], c["Wp"]), c["S"]), on, cert, RANDOM_BOUND)
    assert 0.02 < on.float().mean() < 0.98


@pytest.mark.parametrize("hw", [(120, 160), (37, 53), (1, 64), (64, 1), (300, 410)])
def test_paste_oracle_matches_grid_sample(hw):
    S = 128
    masks = MC.smooth_logits(12, S, S, seed=9) > 0
    masks[0:2] = True   # all ones in the whole-image box and in the box past every side
    masks[4:6] = False  # all zeros in the boxes on the last row and column
    boxes = MC.paste_boxes(*hw, seed=hw[0], n=12)
    on, cert = MC.paste(masks, torch.ones_like(masks), boxes, hw)
    _agree(f"paste {hw}", _lib_paste(masks, boxes, hw), on, cert, RANDOM_BOUND)


def test_dyadic_crop_is_exact_and_its_ties_decide():
    L, boxes, padded, S = MC.dyadic_crop_case()
    on, cert = MC.binarize(L, padded)
    assert cert.all()
    up = F.interpolate(L[None], size=padded, mode="bilinear", align_corners=False)[0]
    up64 = F.interpolate(L[None].double(), size=padded, mode="bilinear", align_corners=False)[0]
    assert torch.equal(up.double(), up64)                       # the fp32 upsample is exact
    zero = up64 == 0
    assert zero[0].all() and zero[2].any() and not zero[2].all()    # exact zeros, which must be off
    assert not on[zero].any()
    assert torch.equal(on, up > 0)
    crop_on, crop_cert = MC.roi_align(on, cert, boxes, S)
    assert crop_cert.all()
    want = _lib_crop(L, boxes, padded, S)
    assert torch.equal(crop_on, want)
    # the library's fp32 roi averages equal float64 ones, and some are exactly 0.5 (on)
    from torchvision.ops import roi_align

    rois = torch.cat([torch.arange(len(boxes), dtype=torch.float32)[:, None], boxes], 1)
    m = on.float()[:, None]
    a32 = roi_align(m, rois, (S, S), 1.0, 0, True)[:, 0]
    a64 = roi_align(m.double(), rois.double(), (S, S), 1.0, 0, True)[:, 0]
    half = a64 == 0.5
    assert half.any() and (a32[half] == 0.5).all() and crop_on[half].all()
    # samples exactly on y = Hp and on y = -1: the outside test is inclusive there
    ys = lambda b, p: (float(b[1]) - 0.5) + p + 0.5  # noqa: E731  (roi of S, one sample per bin)
    assert ys(boxes[4], S // 2) == padded[0] and ys(boxes[5], 7) == -1


def test_dyadic_paste_is_exact_and_its_ties_decide():
    masks, boxes, hw = MC.dyadic_paste_case()
    on, cert = MC.paste(masks, torch.ones_like(masks), boxes, hw)
    assert cert.all()
    want = _lib_paste(masks, boxes, hw)
    assert torch.equal(on, want)
    # column 16 of the box starting at 16.5: ixf = -0.5 exactly, weight 1/2 on column 0, so exactly 0.5: on
    gx = (torch.tensor(16.0) + 0.5 - boxes[0, 0]) / (boxes[0, 2] - boxes[0, 0]) * 2 - 1
    assert ((gx + 1) * 128 - 1) / 2 == -0.5
    assert on[0, 20:140, 16].all() and not on[0, 20:140, 15].any() and not on[1].any()
    H, W = hw
    x0, y0, x1, y1 = torch.split(boxes, 1, dim=1)
    gy = (torch.arange(H, dtype=torch.float64) + 0.5 - y0.double()) / (y1 - y0).double() * 2 - 1
    gxx = (torch.arange(W, dtype=torch.float64) + 0.5 - x0.double()) / (x1 - x0).double() * 2 - 1
    grid = torch.stack([gxx[:, None, :].expand(len(boxes), H, W), gy[:, :, None].expand(len(boxes), H, W)], dim=3)
    v64 = F.grid_sample(masks[:, None].double(), grid, align_corners=False)[:, 0]
    gy32 = (torch.arange(H, dtype=torch.float32) + 0.5 - y0) / (y1 - y0) * 2 - 1
    gx32 = (torch.arange(W, dtype=torch.float32) + 0.5 - x0) / (x1 - x0) * 2 - 1
    grid32 = torch.stack([gx32[:, None, :].expand(len(boxes), H, W), gy32[:, :, None].expand(len(boxes), H, W)], dim=3)
    v32 = F.grid_sample(masks[:, None].float(), grid32, align_corners=False)[:, 0]
    assert torch.equal(v32.double(), v64)
    assert (v64 == 0.5).sum() > 100


def test_edge_boxes_have_their_properties():
    Hp, Wp, S = 1024, 1024, 128
    b = MC.edge_boxes(Hp, Wp, S, seed=0)
    roi_w = (b[:, 2] - 0.5) - (b[:, 0] - 0.5)
    assert ((roi_w == S) | (roi_w == 2 * S)).sum() >= 2
    assert (roi_w > S).logical_and(roi_w == torch.nextafter(torch.tensor(float(S)), torch.tensor(1e9))).any()
    assert ((b[:, 2] - b[:, 0]) == 0).any() and ((b[:, 3] - b[:, 1]) == 0).any()
    assert ((b[:, 2] - b[:, 0]) < 1).any()
    assert (b[:, 0] < 0).any() and (b[:, 1] < 0).any() and (b[:, 2] > Wp).any() and (b[:, 3] > Hp).any()
    assert ((b[:, 1] == Hp - 1) & (b[:, 3] == Hp)).any() and ((b[:, 0] == Wp - 1) & (b[:, 2] == Wp)).any()
    assert ((b - 0.5).frac() == 0).any()                          # roi_start on a texel centre
    p = MC.paste_boxes(480, 640, seed=0)
    assert ((p[:, 2] == p[:, 0]) | (p[:, 3] == p[:, 1])).sum() >= 2 and (p[:, 0] < 0).any() and (p[:, 2] > 640).any()
    index, scores = MC.panoptic_queries(50, 10, seed=0)
    assert index[0] == index[1] and scores[0] == scores[1] and scores[2] == float("-inf")


def _check_panoptic(logits, index, scores, padded, img, out, prob, bound):
    o = MC.panoptic(logits, index, scores, padded, img, out, prob)
    ids, counts = _lib_panoptic(logits, index, scores, padded, img, out, prob)
    _agree(f"panoptic {tuple(img)} -> {tuple(out)} K={len(index)}", ids, o["ids"], o["ids_certain"], bound)
    assert ((counts >= o["lo"]) & (counts <= o["hi"])).all()
    return o


@pytest.mark.parametrize("K,img,out", [(1, (200, 256), (200, 256)), (12, (256, 200), (300, 170)), (40, (131, 173), (1, 97)),
                                       (40, (256, 256), (96, 1))])
def test_panoptic_oracle_matches_the_library(K, img, out):
    logits = MC.panoptic_logits(K + 5, 64, 64, seed=K)
    index, scores = MC.panoptic_queries(K + 5, K, seed=K)
    o = _check_panoptic(logits, index, scores, (256, 256), img, out, 0.1, RANDOM_BOUND)
    if K >= 3:
        assert o["hi"][:, 2].sum() == 0 and o["hi"][0, 1] == 0  # the -inf query and the repeat of query 0 never win
    assert (o["ids"] >= 0).any()


def test_dyadic_panoptic_is_exact_and_its_ties_decide():
    L, index, scores, padded, img, out, prob = MC.dyadic_panoptic_case()
    o = _check_panoptic(L, index, scores, padded, img, out, prob, 0)
    assert torch.equal(o["lo"], o["hi"])
    m = F.interpolate(L[index][None], size=padded, mode="bilinear", align_corners=False)[0]
    v = F.interpolate(m[None, :, :img[0], :img[1]], size=out, mode="bilinear", align_corners=False)[0]
    m64 = F.interpolate(L[index][None].double(), size=padded, mode="bilinear", align_corners=False)[0]
    v64 = F.interpolate(m64[None, :, :img[0], :img[1]], size=out, mode="bilinear", align_corners=False)[0]
    assert torch.equal(v.double(), v64)
    ids = o["ids"]
    assert (ids == 0).any() and (ids == 2).any() and not (ids == 1).any() and not (ids == 3).any()
    assert o["count"][1, 0] == o["count"][0, 0] > 0                # p == 0.5 exactly at prob 0.5: solid wherever query 0 wins
    assert o["count"][2, 0] == out[0] * out[1] == o["count"][2, 1]


def test_crop_edge_panoptic_case_tells_the_crop_from_the_pad():
    """The oracle, like the library, resizes the crop: the last output column stays on, and resizing the padded map instead
    would turn it off."""
    L, index, scores, padded, img, out, prob = MC.crop_edge_panoptic_case()
    o = _check_panoptic(L, index, scores, padded, img, out, prob, 0)
    assert (o["ids"][:, -1] == 0).all() and o["ids_certain"].all()
    m = F.interpolate(L[None], size=padded, mode="bilinear", align_corners=False)[0]
    assert m[0, 0, 599] == 2 and m[0, 0, 600] == -12
    wide = F.interpolate(m[None, :, :img[0], :img[1] + 1], size=(out[0], out[1] * (img[1] + 1) // img[1]), mode="bilinear",
                         align_corners=False)[0]
    src = (out[1] - 0.5) * img[1] / out[1] - 0.5  # the last column's source, 599.3: between 599 and 600 if read past the crop
    assert 599 < src < 600 and 0.7 * 2 + 0.3 * -12 < 0
