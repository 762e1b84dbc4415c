"""GPU: panoptic merging on the device without the [K, H, W] mask stacks (csrc/panoptic.cu, ops.panoptic_winners,
postprocess.postprocess_panoptic_winners, the engine path of DeformableDETRSegmVL._panoptic) against
postprocess.postprocess_panoptic, which tests/test_panoptic_cpu.py pins to the reference's own function: same segments_info, the
same map and the same three areas per query up to the pixels whose probability sits within float rounding of a decision."""
import pytest
import torch
import torch.nn.functional as F

from ape_b200 import _lib, configs, ops
from ape_b200.modeling.postprocess import postprocess_panoptic, postprocess_panoptic_winners
from oracle import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LIB = _lib.lib
CFG = {"prob": 0.1, "pano_temp": 0.06, "transform_eval": True, "object_mask_threshold": 0.01, "overlap_threshold": 0.4}
N_CLS, N_THING = 20, 10
PADDED = (1024, 1024)


def _inputs(K, dtype, seed, Q=None, hw=(256, 256)):
    """Overlapping blobs (as test_panoptic_gpu.py) as mask logits [Q, h, w] of `dtype`, K distinct query rows of them, and
    class logits [K, N_CLS]."""
    g = torch.Generator().manual_seed(seed)
    Q = K + 7 if Q is None else Q
    H, W = hw
    yy, xx = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
    c = torch.rand(Q, 2, generator=g) * torch.tensor([H, W]).float()
    r = torch.rand(Q, generator=g) * 50 + 8
    logits = torch.empty(Q, H, W)
    for i in range(0, Q, 64):  # in chunks: [Q, H, W] distance temporaries at Q = 900 are large
        d = ((yy[None] - c[i:i + 64, 0, None, None]) ** 2 + (xx[None] - c[i:i + 64, 1, None, None]) ** 2).sqrt()
        logits[i:i + 64] = (r[i:i + 64, None, None] - d) * 0.3 + torch.randn(d.shape, generator=g) * 0.3
    qi = torch.randperm(Q, generator=g)[:K]
    mask_cls = torch.randn(K, N_CLS, generator=g) * 2
    return logits.to(DEV, dtype), qi.to(DEV), mask_cls.to(DEV)


def _reference(logits, qi, mask_cls, img, out, cfg=CFG, stuff_first=False):
    """(ids, counts, kept) of the kept queries and postprocess_panoptic's (map, segments_info), from the fp32 upsample of the
    same logits to the padded size: the quantities postprocess_panoptic computes, spelled out."""
    m = F.interpolate(logits[qi][None].float(), size=PADDED, mode="bilinear", align_corners=False)[0]
    seg, info = postprocess_panoptic(mask_cls, m, img, out[0], out[1], range(N_THING), N_THING, stuff_first, cfg)
    scores, _ = mask_cls.sigmoid().max(-1)
    kept = (scores > cfg["object_mask_threshold"]).nonzero()[:, 0]
    scores, _ = F.softmax(mask_cls.sigmoid() / cfg["pano_temp"], dim=-1).max(-1)
    p = F.interpolate(m[:, :img[0], :img[1]][None], size=out, mode="bilinear", align_corners=False)[0][kept].sigmoid()
    del m
    K = len(kept)
    if K == 0:
        return torch.full(out, -1, device=DEV), torch.zeros((3, 0), dtype=torch.long, device=DEV), kept, scores, seg, info
    win = (scores[kept].view(-1, 1, 1) * p).argmax(0)
    solid = torch.gather(p, 0, win[None])[0] >= cfg["prob"]
    counts = torch.stack([torch.bincount(win.flatten(), minlength=K), torch.bincount(win[solid], minlength=K),
                          (p >= cfg["prob"]).flatten(1).sum(1)])
    ids = torch.where(solid, win, -1)
    return ids, counts, kept, scores, seg, info


def _check(logits, qi, mask_cls, img, out, what, cfg=CFG, stuff_first=False):
    ids_ref, counts_ref, kept, scores, seg_ref, info_ref = _reference(logits, qi, mask_cls, img, out, cfg, stuff_first)
    P = out[0] * out[1]
    ids, counts = ops.panoptic_winners(logits, qi[kept], scores[kept], PADDED, img, out, cfg["prob"])
    assert ids.dtype == torch.int32 and tuple(ids.shape) == tuple(out) and tuple(counts.shape) == (3, len(kept))
    id_frac = (ids != ids_ref).float().mean().item()
    count_err = (counts.long() - counts_ref).abs().max().item() if len(kept) else 0
    seg, info = postprocess_panoptic_winners(mask_cls, logits, qi, PADDED, img, out[0], out[1], range(N_THING), N_THING, stuff_first,
                                             cfg)
    seg_frac = (seg != seg_ref).float().mean().item()
    print(f"  {what}: K={len(kept)}, {len(info)} segments; ids differ on {id_frac:.2e}, map on {seg_frac:.2e} of the pixels; "
          f"max count error {count_err} = {count_err / P:.2e} of the pixels")
    assert seg.dtype == torch.int32 and seg.device == seg_ref.device and tuple(seg.shape) == tuple(out)
    assert info == info_ref
    assert id_frac < 1e-3 and seg_frac < 1e-3
    assert count_err <= 1e-3 * P
    return info


@pytest.mark.parametrize("K", [1, 12, 100, 300, 900])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=["fp32", "fp16", "bf16"])
def test_op_matches_reference(dtype, K):
    logits, qi, mask_cls = _inputs(K, dtype, seed=K)
    info = _check(logits, qi, mask_cls, (1024, 768), (1024, 768), f"{dtype} K={K}")
    assert len(info) > 0


@pytest.mark.parametrize("img", [(1024, 1024), (1024, 768), (600, 1000)])
@pytest.mark.parametrize("out", ["image", (480, 640), (2048, 1536)])
def test_op_geometry(img, out):
    out = img if out == "image" else out
    logits, qi, mask_cls = _inputs(300, torch.float16, seed=img[1] + out[1])
    info = _check(logits, qi, mask_cls, img, out, f"image {img}, output {out}", stuff_first=True)
    assert len(info) > 0


def test_op_bf16_small_image_upsampled_output():
    logits, qi, mask_cls = _inputs(100, torch.bfloat16, seed=3)
    _check(logits, qi, mask_cls, (600, 1000), (2048, 1536), "bf16 image 600 x 1000 -> 2048 x 1536")


def test_no_query_above_the_threshold():
    logits, qi, mask_cls = _inputs(50, torch.float16, seed=9)
    mask_cls = mask_cls - 30.0  # every sigmoid score below object_mask_threshold: K = 0 kept
    info = _check(logits, qi, mask_cls, (1024, 768), (480, 640), "no kept query")
    assert info == []
    ids, counts = ops.panoptic_winners(logits, qi[:0], torch.zeros(0, device=DEV), PADDED, (1024, 768), (480, 640), 0.1)
    assert tuple(counts.shape) == (3, 0) and (ids == -1).all()


def test_excluded_queries_take_no_part():
    """A score of -inf leaves a query out exactly as if it were not in the list."""
    logits, qi, mask_cls = _inputs(40, torch.float16, seed=11)
    scores = torch.rand(40, generator=torch.Generator(device=DEV).manual_seed(1), device=DEV)
    drop = torch.arange(40, device=DEV) % 3 == 1
    ids, counts = ops.panoptic_winners(logits, qi, torch.where(drop, float("-inf"), scores), PADDED, (1000, 900), (500, 450), 0.1)
    ids2, counts2 = ops.panoptic_winners(logits, qi[~drop], scores[~drop], PADDED, (1000, 900), (500, 450), 0.1)
    pos = (~drop).nonzero()[:, 0].int()
    assert torch.equal(ids, torch.where(ids2 >= 0, pos[ids2.clamp(min=0).long()], -1))
    assert torch.equal(counts[:, ~drop], counts2) and (counts[:, drop] == 0).all()


@pytest.fixture(scope="module")
def mini():
    from ape_b200.modeling import build_model

    m = build_model(configs.MINI)
    synth.fill_state_dict(m)
    return m.to(DEV)


@pytest.mark.parametrize("post_nms", [True, False])
def test_model_panoptic_matches_postprocess_panoptic(mini, post_nms):
    """MINI, fp16 engine, panoptic_on with a thing / stuff split: panoptic_seg against postprocess_panoptic applied to the same
    last_outputs and the same kept queries."""
    model = mini
    name = model.dataset_names[0]
    things, stuff = [f"c{i}" for i in range(6)], [f"c{i}" for i in range(6, 12)]
    saved = (model.panoptic_on, model.panoptic_post_nms, model.engine_dtype, dict(model.dataset_stuff))
    inp = [{"image": synth.image(56, 64, seed=4), "height": 112, "width": 90}]
    try:
        model.dataset_stuff[name] = (things, stuff, "thing+stuff")
        model.set_eval_dataset(name)
        model.panoptic_on, model.panoptic_post_nms, model.engine_dtype = True, post_nms, torch.float16
        out = model(inp)
        lo = model.last_outputs
        images, _, sizes = model.preprocess_image(inp)
        box_cls, box_pred, mask_pred = lo["pred_logits"], lo["pred_boxes"], lo["pred_masks"]
        if post_nms:
            qi = model.inference(box_cls, box_pred, sizes)[0].query_index
        else:
            qi = torch.arange(box_cls.shape[1], device=box_cls.device)
    finally:
        model.panoptic_on, model.panoptic_post_nms, model.engine_dtype, model.dataset_stuff = saved
        model.set_eval_dataset("")
    assert mask_pred.is_cuda
    seg, info = out[0]["panoptic_seg"]
    m = F.interpolate(mask_pred[0, qi][None].float(), size=tuple(images.shape[-2:]), mode="bilinear", align_corners=False)[0]
    seg_ref, info_ref = postprocess_panoptic(box_cls[0, qi].float(), m, sizes[0], 112, 90, range(6), 6, False, model.panoptic_configs)
    frac = (seg != seg_ref).float().mean().item()
    print(f"  MINI fp16 post_nms={post_nms}: {len(qi)} queries, {len(info)} segments, {frac:.2e} of the pixels differ")
    assert info == info_ref
    assert frac < 1e-3


def test_memory_stays_small():
    """K = 300, 1024^2 padded, 1024 x 768 output: the device path allocates a few int32 maps; the old path several [K, H, W] fp32
    stacks."""
    K, img, out = 300, (1024, 768), (1024, 768)
    logits, qi, mask_cls = _inputs(K, torch.float16, seed=21)
    args = (img, out[0], out[1], range(N_THING), N_THING, False, CFG)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    new = postprocess_panoptic_winners(mask_cls, logits, qi, PADDED, *args)
    torch.cuda.synchronize()
    grow_new = torch.cuda.max_memory_allocated() - base
    del new
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    m = F.interpolate(logits[qi][None].float(), size=PADDED, mode="bilinear", align_corners=False)[0]
    old = postprocess_panoptic(mask_cls, m, *args)
    del m
    torch.cuda.synchronize()
    grow_old = torch.cuda.max_memory_allocated() - base
    del old
    plane = out[0] * out[1] * 4
    print(f"  peak growth: device path {grow_new / 2**20:.1f} MiB ({grow_new / plane:.2f} x oh*ow*4), "
          f"old path {grow_old / 2**30:.2f} GiB")
    assert grow_new <= 4 * plane


def test_graph_replay_equals_eager():
    logits, qi, mask_cls = _inputs(120, torch.float16, seed=31)
    scores = torch.rand(120, generator=torch.Generator(device=DEV).manual_seed(2), device=DEV)
    args = (PADDED, (1000, 800), (700, 560), 0.1)
    static_logits = logits.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.panoptic_winners(static_logits, qi, scores, *args)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = ops.panoptic_winners(static_logits, qi, scores, *args)
    fresh, _, _ = _inputs(120, torch.float16, seed=32)
    for new in (fresh, logits):
        static_logits.copy_(new)
        graph.replay()
        eager = ops.panoptic_winners(new, qi, scores, *args)
        torch.cuda.synchronize()
        assert torch.equal(static[0], eager[0]) and torch.equal(static[1], eager[1])


def test_bad_arguments_are_rejected():
    logits = torch.zeros((4, 16, 16), device=DEV)
    index = torch.arange(3, device=DEV)
    scores = torch.ones(3, device=DEV)
    ids = torch.zeros((8, 8), dtype=torch.int32, device=DEV)
    counts = torch.zeros((3, 3), dtype=torch.int32, device=DEV)
    s = _lib.current_stream_ptr()
    ok = dict(K=3, h=16, w=16, Hp=32, Wp=32, ih=30, iw=20, oh=8, ow=8, ld=_lib.APE_DTYPE_F32)

    def call(**kw):
        a = dict(ok, **kw)
        return LIB.ape_panoptic_winners(logits.data_ptr(), index.data_ptr(), scores.data_ptr(), ids.data_ptr(), counts.data_ptr(),
                                        a["K"], a["h"], a["w"], a["Hp"], a["Wp"], a["ih"], a["iw"], a["oh"], a["ow"], 0.5, a["ld"], s)

    assert call() == 0
    torch.cuda.synchronize()
    for bad in (dict(ld=_lib.APE_DTYPE_E4M3), dict(K=-1), dict(K=4097), dict(ih=33), dict(iw=0), dict(oh=0), dict(h=0)):
        assert call(**bad) == -1, bad
        assert LIB.ape_last_error()
    with pytest.raises(RuntimeError):
        ops.panoptic_winners(logits, index, scores[:2], (32, 32), (30, 20), (8, 8), 0.5)
    with pytest.raises(RuntimeError):
        ops.panoptic_winners(logits, index, scores, (32, 32), (33, 20), (8, 8), 0.5)
    with pytest.raises(RuntimeError):
        ops.panoptic_winners(logits.cpu(), index, scores, (32, 32), (30, 20), (8, 8), 0.5)
