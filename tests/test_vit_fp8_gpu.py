"""GPU: the opt-in FP8 ViT-L backbone (`ViT(fp8_linears=True)`: e4m3 qkv and w12 GEMMs fed by the e4m3 LayerNorm) on APE-L_D
and APE-L_B at 1024^2, 1203 names, against the committed fp32 goldens of the reference (model_ld_1024.npz,
model_lb_1024.npz; tests/golden/gen_model_golden.py, gen_lb_golden.py), with the fp16 engine's errors beside it.

* Pyramid features: median and maximum |err| over the RMS of the golden, fp16 and fp16 + FP8.
* Detections: the share of the fp16 engine's top-100 detections that the FP8 run reproduces (same class, box IoU >= 0.9).
* The FP8 backbone calls no library GEMM, convolution or attention kernel, and its CUDA-graph replay equals eager.
* With fp8_linears back off, the outputs are bit-identical to a run that never used FP8.
Weights are name-derived synthetic (oracle/synth.py), so these are numerical checks, not accuracy on the released checkpoints."""
import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden
from ape_b200 import configs
from oracle import synth

pytestmark = [pytest.mark.gpu, pytest.mark.slow]
DEV = "cuda:0"
N_TEXT = 1203
TOP = 100
# Bounds set from the first measurement on an H100 80GB HBM3: median / max |err| over rms(golden) of the pyramid features
# (worst level) and the share of the fp16 engine's top-100 detections reproduced.  Measured, FP8 (fp16 beside it):
#   APE-L_D  median 6.1e-2 .. 7.1e-2 (7.0e-4 .. 8.7e-4), max 1.8e-1 .. 4.3e-1 (2.5e-3 .. 4.9e-3), reproduced 0.53
#   APE-L_B  median 8.1e-2 .. 1.09e-1 (1.0e-3 .. 1.3e-3), max 2.9e-1 .. 7.7e-1 (4.0e-3 .. 8.7e-3), reproduced 0.56
BOUNDS = {
    "ld": dict(median=0.1, max=0.65, reproduced=0.4),
    "lb": dict(median=0.15, max=1.1, reproduced=0.4),
}
SPECS = {"ld": (configs.APE_L_D, "model_ld_1024.npz"), "lb": (configs.APE_L_B, "model_lb_1024.npz")}


def err(name, got, want):
    got, want = got.float().cpu(), want.float().cpu()
    assert got.shape == want.shape, (name, got.shape, want.shape)
    d = (got - want).abs()
    rms = want.pow(2).mean().sqrt().item() + 1e-12
    return d.median().item() / rms, d.max().item() / rms


@pytest.fixture(scope="module", params=sorted(SPECS))
def model(request):
    from ape_b200.modeling import build_model

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    spec, golden = SPECS[request.param]
    m = build_model(spec, num_text=N_TEXT)
    synth.fill_state_dict(m)
    synth.suppress_invalid_anchor_logits(m)
    m = m.to(DEV)
    yield request.param, m, load_golden(golden)
    del m
    torch.cuda.empty_cache()


def _run(m, fp8, graphs=True, seed=0):
    m.backbone.net.fp8_linears = fp8
    m.engine_dtype = torch.float16
    m.use_cuda_graphs = graphs
    try:
        inp = [{"image": synth.image(1024, 768, seed=seed), "height": 1024, "width": 768}]
        out = m(inp)
        if graphs:  # second call = graph replay
            out = m(inp)
        feats = {k: v.clone() for k, v in m.last_outputs["features"].items()}
        return out[0]["instances"], feats, m.last_outputs["pred_logits"].clone()
    finally:
        m.engine_dtype, m.use_cuda_graphs = torch.float32, False
        m.backbone.net.fp8_linears = False


def _box_iou(a, b):
    lt = torch.max(a[:, None, :2], b[None, :, :2])
    rb = torch.min(a[:, None, 2:], b[None, :, 2:])
    inter = (rb - lt).clamp_min(0).prod(-1)
    area = lambda x: (x[:, 2:] - x[:, :2]).clamp_min(0).prod(-1)
    return inter / (area(a)[:, None] + area(b)[None, :] - inter + 1e-9)


def _reproduced(ref, got):
    """Share of ref's top-TOP detections with a detection of got of the same class and box IoU >= 0.9."""
    rb, rc = ref.pred_boxes.tensor[:TOP].float(), ref.pred_classes[:TOP]
    gb, gc = got.pred_boxes.tensor.float(), got.pred_classes
    iou = _box_iou(rb, gb)
    ok = ((iou >= 0.9) & (rc[:, None] == gc[None, :])).any(1)
    return ok.float().mean().item()


def test_fp8_features_and_detections(model):
    name, m, g = model
    inst16, f16, _ = _run(m, fp8=False)
    inst8, f8, _ = _run(m, fp8=True)
    b = BOUNDS[name]
    print(f"\n== APE-L_{name[1:].upper()} 1024^2: pyramid error over rms(fp32 golden), fp16 | fp16 + FP8 qkv / w12")
    rec = {}
    for k in ("p2", "p3", "p4", "p5", "p6"):
        med16, max16 = err(k, f16[k][:, ::16, ::8, ::8], g[f"backbone.{k}"])
        rec[k] = err(k, f8[k][:, ::16, ::8, ::8], g[f"backbone.{k}"])
        print(f"  {k}: median {med16:.3e} | {rec[k][0]:.3e}   max {max16:.3e} | {rec[k][1]:.3e}")
    share = _reproduced(inst16, inst8)
    print(f"  fp16 top-{TOP} detections reproduced by FP8 (same class, IoU >= 0.9): {share:.3f}")
    for k, (med8, max8) in rec.items():
        assert med8 < b["median"] and max8 < b["max"], (k, med8, max8)
    assert share >= b["reproduced"]


def test_fp8_backbone_runs_no_library_kernels(model, monkeypatch):
    import ape_b200

    _, m, _ = model

    def forbidden(*a, **k):
        raise AssertionError("library kernel called on the FP8 backbone path")

    for mod, fn in ((F, "linear"), (F, "conv2d"), (F, "conv_transpose2d"), (F, "scaled_dot_product_attention"),
                    (torch, "matmul")):
        monkeypatch.setattr(mod, fn, forbidden)
    img = torch.randn(1, 3, 1024, 1024, generator=torch.Generator().manual_seed(8)).to(DEV, torch.float16)
    m.backbone.net.fp8_linears = True
    try:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            n0 = ape_b200._lib.launch_count()
            feats = m.backbone(img)
            torch.cuda.synchronize()
            launched = ape_b200._lib.launch_count() - n0
    finally:
        m.backbone.net.fp8_linears = False
    assert sorted(feats) == ["p2", "p3", "p4", "p5", "p6"] and launched > 24 * 8
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert any("gemm_fp8_kernel" in n for n in names) and any("layernorm_e4m3_kernel" in n for n in names)
    library = [n for n in names if "ape::" not in n and any(s in n.lower() for s in (
        "cublas", "cutlass", "gemm", "gemv", "xmma", "flash", "cudnn", "fmha", "efficient_attention"))]
    assert not library, sorted(set(library))[:5]


def test_fp8_graph_replay_equals_eager_and_off_restores_outputs(model):
    _, m, _ = model
    _, f_off, logits_off = _run(m, fp8=False, graphs=False)
    inst_e, f_e, logits_e = _run(m, fp8=True, graphs=False)
    m.backbone.net.fp8_linears = True
    m.engine_dtype, m.use_cuda_graphs = torch.float16, True
    try:
        for seed in (0, 3, 0):  # capture, then replays with a different image in between
            out = m([{"image": synth.image(1024, 768, seed=seed), "height": 1024, "width": 768}])
        logits_g = m.last_outputs["pred_logits"].clone()
    finally:
        m.engine_dtype, m.use_cuda_graphs = torch.float32, False
        m.backbone.net.fp8_linears = False
    assert torch.equal(logits_g, logits_e), "CUDA graph replay differs from eager (FP8)"
    assert torch.equal(out[0]["instances"].pred_classes, inst_e.pred_classes)
    assert not torch.equal(logits_e, logits_off)  # the FP8 path did run
    _, f_back, logits_back = _run(m, fp8=False, graphs=False)
    assert torch.equal(logits_back, logits_off)
    assert all(torch.equal(f_back[k], f_off[k]) for k in f_off)
