"""GPU: instance-mask post-processing kernels (csrc/mask_post.cu) against the library formulation of the same steps —
F.interpolate + sigmoid > 0.5 + torchvision roi_align (detectron2 BitMasks.crop_and_resize) and grid_sample
(detectron2 paste_masks_in_image) — which is what the reference runs (deformable_detr_segm_vl.py:569-603).  Outputs are
booleans: they must equal the float64 oracle (oracle/mask_chain.py) at every pixel it calls certain, i.e. only pixels whose
interpolated value sits within float rounding of the threshold may differ."""
import pytest
import torch
import torch.nn.functional as F

from oracle import mask_chain as MC

pytestmark = pytest.mark.gpu


def _library_crop(logits, index, boxes, padded_hw, S):
    from torchvision.ops import roi_align

    m = F.interpolate(logits[index][None].float(), size=padded_hw, mode="bilinear", align_corners=False)[0]
    m = (m.sigmoid() > 0.5).to(torch.float32)[:, None]
    rois = torch.cat([torch.arange(len(boxes), device=boxes.device, dtype=boxes.dtype)[:, None], boxes], dim=1)
    return roi_align(m, rois, (S, S), 1.0, 0, True).squeeze(1) >= 0.5


def _library_paste(masks, boxes, hw):
    img_h, img_w = hw
    x0, y0, x1, y1 = torch.split(boxes, 1, dim=1)
    img_y = (torch.arange(0, img_h, device=masks.device, dtype=torch.float32) + 0.5 - y0) / (y1 - y0) * 2 - 1
    img_x = (torch.arange(0, img_w, device=masks.device, dtype=torch.float32) + 0.5 - x0) / (x1 - x0) * 2 - 1
    gx = img_x[:, None, :].expand(len(boxes), img_h, img_w)
    gy = img_y[:, :, None].expand(len(boxes), img_h, img_w)
    return F.grid_sample(masks[:, None].float(), torch.stack([gx, gy], dim=3), align_corners=False)[:, 0] >= 0.5


def _smooth_logits(Q, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(Q, 1, h // 8, w // 8, generator=g)
    return F.interpolate(x, size=(h, w), mode="bicubic", align_corners=False)[:, 0].contiguous().cuda() * 4.0


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("h,w,Hp,Wp", [(64, 64, 256, 256), (48, 64, 192, 256), (256, 256, 1024, 1024)])
def test_crop_and_resize_matches_the_library_formulation(built, dtype, h, w, Hp, Wp):
    import ape_b200

    Q, K, S = 40, 23, 128 if Hp >= 1024 else 28
    logits = _smooth_logits(Q, h, w, seed=h + Wp).to(dtype)
    g = torch.Generator().manual_seed(1)
    index = torch.randperm(Q, generator=g)[:K].cuda()
    c = torch.rand(K, 2, generator=g) * torch.tensor([Wp, Hp])
    wh = torch.rand(K, 2, generator=g) * torch.tensor([Wp, Hp]) * 0.9 + 2.0
    boxes = torch.cat([(c - wh / 2), (c + wh / 2)], 1)
    boxes[:, 0::2] = boxes[:, 0::2].clamp(0, Wp)
    boxes[:, 1::2] = boxes[:, 1::2].clamp(0, Hp)
    boxes[0] = torch.tensor([0.0, 0.0, Wp, Hp])      # the whole image (largest sampling grid)
    boxes[1] = torch.tensor([3.25, 4.5, 5.0, 6.75])   # smaller than the output grid
    boxes = boxes.cuda()
    n0 = ape_b200._lib.launch_count()
    got = ape_b200.ops.mask_crop_and_resize(logits, index, boxes, (Hp, Wp), S)
    assert ape_b200._lib.launch_count() - n0 == 2
    want = _library_crop(logits, index, boxes, (Hp, Wp), S)
    assert got.dtype == torch.bool and got.shape == want.shape
    frac = (got != want).float().mean().item()
    on, cert = MC.crop_and_resize(logits[index], boxes, (Hp, Wp), S)
    wrong, unsure = int(((got != on) & cert).sum()), int((~cert).sum())
    print(f"  crop_and_resize {dtype} {h}x{w}->{Hp}x{Wp}: {frac * 100:.4f} % of the {got.numel()} mask pixels differ from the library path; "
          f"{unsure} uncertain for the oracle, {wrong} certain ones differ from it")
    assert wrong == 0 and unsure <= 5e-3 * got.numel() and 0.05 < got.float().mean().item() < 0.95


@pytest.mark.parametrize("hw", [(480, 640), (1024, 1024), (37, 53)])
def test_paste_matches_grid_sample(built, hw):
    import ape_b200

    g = torch.Generator().manual_seed(3)
    N, S = 17, 128
    masks = (_smooth_logits(N, S, S, seed=9) > 0)
    H, W = hw
    c = torch.rand(N, 2, generator=g) * torch.tensor([W, H])
    wh = torch.rand(N, 2, generator=g) * torch.tensor([W, H]) * 0.8 + 1.0
    boxes = torch.cat([(c - wh / 2), (c + wh / 2)], 1).cuda()
    boxes[0] = torch.tensor([0.0, 0.0, float(W), float(H)])
    got = ape_b200.ops.paste_masks_in_image(masks, boxes, hw)
    want = _library_paste(masks, boxes, hw)
    assert got.dtype == torch.bool and tuple(got.shape) == (N, H, W)
    frac = (got != want).float().mean().item()
    on, cert = MC.paste(masks, torch.ones_like(masks), boxes, hw)
    wrong, unsure = int(((got != on) & cert).sum()), int((~cert).sum())
    print(f"  paste {hw}: {frac * 100:.5f} % of the pixels differ from grid_sample; {unsure} uncertain for the oracle, {wrong} "
          f"certain ones differ from it")
    assert wrong == 0 and unsure <= 5e-3 * got.numel()
    assert torch.equal(ape_b200.ops.paste_masks_in_image(masks.float(), boxes, hw), got)  # 0 / 1 floats as detector_postprocess passes them
    assert ape_b200.ops.paste_masks_in_image(masks[:0], boxes[:0], hw).shape == (0, H, W)


@pytest.mark.parametrize("hw", [(480, 640), (1024, 1024), (37, 53), (300, 1)])
def test_paste_rle_decodes_to_the_dense_paste(built, hw):
    """ape_mask_paste_rle (run boundaries found on the device, column-major) against the dense paste kernel: the decoded run-length
    code IS the dense mask, and the code equals the oracle's encoding of it (cocoapi's rleEncode + rleToString restated)."""
    import ape_b200
    from oracle import rle as R

    g = torch.Generator().manual_seed(7)
    N, S = 19, 128
    masks = (_smooth_logits(N, S, S, seed=13) > 0)
    H, W = hw
    c = torch.rand(N, 2, generator=g) * torch.tensor([W, H])
    wh = torch.rand(N, 2, generator=g) * torch.tensor([W, H]) * 0.8 + 1.0
    boxes = torch.cat([(c - wh / 2), (c + wh / 2)], 1).cuda()
    boxes[0] = torch.tensor([0.0, 0.0, float(W), float(H)])          # the whole image
    boxes[1] = torch.tensor([-5.0, -5.0, W + 5.0, H + 5.0])           # first and last pixel inside the mask's support
    masks[2] = True                                                   # a solid box
    masks[3] = False                                                  # an empty mask: a single run of zeros
    dense = ape_b200.ops.paste_masks_in_image(masks, boxes, hw).cpu().numpy().astype("uint8")
    rles = ape_b200.ops.paste_masks_rle(masks, boxes, hw)
    assert len(rles) == N
    for n in range(N):
        assert rles[n]["size"] == [H, W]
        assert (R.decode(rles[n]) == dense[n]).all(), f"mask {n}"
        assert rles[n]["counts"] == R.encode(dense[n])["counts"]
    assert rles[3]["counts"] == R.counts_to_string([H * W])
    assert ape_b200.ops.paste_masks_rle(masks[:0], boxes[:0], hw) == []


def test_model_returns_run_length_masks_when_asked(built):
    """mask_format = "rle": `pred_masks_rle` of the detections decode to the `pred_masks` the default format returns."""
    from ape_b200 import configs
    from ape_b200.modeling import build_model
    from oracle import rle as R
    from oracle import synth

    spec = configs.MINI
    model = build_model(spec)
    synth.fill_state_dict(model)
    model = model.cuda().eval()
    model.test_mask_on = True
    img = synth.image(56, 64, seed=7)
    inp = [{"image": img, "height": 112, "width": 128}]
    want = model(inp)[0]["instances"]
    model.mask_format = "rle"
    got = model(inp)[0]["instances"]
    assert len(got) == len(want) > 0 and not got.has("pred_masks")
    assert torch.equal(got.pred_boxes.tensor, want.pred_boxes.tensor)
    for rle, m in zip(got.pred_masks_rle, want.pred_masks):
        assert rle["size"] == [112, 128]
        assert (torch.from_numpy(R.decode(rle)).bool() == m.cpu()).all()
