"""GPU: panoptic merging (ape_b200/modeling/postprocess.py; reference `_postprocess_panoptic`,
deformable_detr_segm_vl.py:919-998) on device tensors against the same function on host tensors, which
tests/test_panoptic_cpu.py pins to the reference's own function: same segments, same ids, same segment map up to the pixels
whose interpolated mask probability sits within float rounding of a decision boundary."""
import pytest
import torch

from ape_b200.modeling.postprocess import postprocess_panoptic
from oracle import mask_chain as MC

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed,K,n_cls,stuff_first", [(0, 12, 9, False), (1, 40, 7, True), (3, 100, 133, True)])
def test_device_equals_host(seed, K, n_cls, stuff_first):
    g = torch.Generator().manual_seed(seed)
    H = W = 256
    image_size, out_hw = (200, 240), (400, 480)
    mask_cls = torch.randn(K, n_cls, generator=g) * 2
    yy, xx = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
    c = torch.rand(K, 2, generator=g) * 220
    r = torch.rand(K, generator=g) * 60 + 10
    mask_pred = (r[:, None, None] - ((yy[None] - c[:, 0, None, None]) ** 2 + (xx[None] - c[:, 1, None, None]) ** 2).sqrt()) * 0.3
    mask_pred = mask_pred + torch.randn(K, H, W, generator=g) * 0.3
    n_thing = n_cls // 2
    cfg = dict(prob=0.5, pano_temp=0.06, transform_eval=True, object_mask_threshold=0.3, overlap_threshold=0.6)
    args = (image_size, out_hw[0], out_hw[1], range(n_thing), n_thing, stuff_first, cfg)
    want_seg, want_info = postprocess_panoptic(mask_cls, mask_pred, *args)
    seg, info = postprocess_panoptic(mask_cls.cuda(), mask_pred.cuda(), *args)
    assert seg.is_cuda and seg.dtype == torch.int32 and tuple(seg.shape) == out_hw
    assert info == want_info and len(info) > 0
    frac = (seg.cpu() != want_seg).float().mean().item()
    scores, _ = torch.softmax(mask_cls.sigmoid() / cfg["pano_temp"], -1).max(-1)
    kept = (mask_cls.sigmoid().max(-1)[0] > cfg["object_mask_threshold"]).nonzero()[:, 0]
    o = MC.panoptic(mask_pred.cuda(), kept.cuda(), scores[kept].cuda(), (H, W), image_size, out_hw, cfg["prob"])
    cert = o["ids_certain"].cpu()
    print(f"  panoptic K={K}: {len(info)} segments, {frac * 100:.4f} % of the pixels differ between device and host; "
          f"{o['unsure_pixels']} pixels uncertain for the float64 oracle")
    assert not ((seg.cpu() != want_seg) & cert).any()
    assert o["unsure_pixels"] <= 5e-3 * seg.numel()
