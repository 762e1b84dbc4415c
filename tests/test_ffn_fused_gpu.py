"""GPU: the fused FFN kernel (ape_ffn_fused: x + relu(x W1^T + b1) W2^T + b2 in one launch) against the two-GEMM path it
replaces (bit for bit) and an fp32 torch reference; argument checks; the model's FFNs take it."""
import threading

import pytest
import torch

from ape_b200 import _lib, ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = [torch.float16, torch.bfloat16]
VARIANTS = {"single": 1, "cluster": 2}


def _operands(M, F, dtype, seed=0, E=256):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(M, E, device=DEV, generator=g).to(dtype)
    w1 = (torch.randn(F, E, device=DEV, generator=g) * E ** -0.5).to(dtype)
    b1 = torch.randn(F, device=DEV, generator=g) * 0.5
    w2 = (torch.randn(E, F, device=DEV, generator=g) * F ** -0.5).to(dtype)
    b2 = torch.randn(E, device=DEV, generator=g) * 0.5
    return x, w1, b1, w2, b2


def _two_gemm(x, w1, b1, w2, b2):
    h = ops.linear_tc(x, w1, b1, act="relu")
    return ops.linear_tc(h, w2, b2, residual=x, out_dtype=torch.float32)


@pytest.mark.parametrize("variant", sorted(VARIANTS))
@pytest.mark.parametrize("F", [64, 128, 2048])
@pytest.mark.parametrize("M", [1, 127, 900, 19000, 87296])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_bit_identical_to_two_gemms(dtype, M, F, variant):
    x, w1, b1, w2, b2 = _operands(M, F, dtype, seed=M + F)
    want = _two_gemm(x, w1, b1, w2, b2)
    got = ops.ffn_fused(x, w1, b1, w2, b2, variant=VARIANTS[variant])
    torch.cuda.synchronize()
    assert got.dtype == torch.float32 and got.shape == (M, 256)
    assert torch.equal(got, want), f"max |diff| {(got - want).abs().max().item():.3e}"


@pytest.mark.parametrize("M,F", [(900, 2048), (19000, 128), (4096, 2048)])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_matches_fp32_reference(dtype, M, F):
    x, w1, b1, w2, b2 = _operands(M, F, dtype, seed=7)
    h = torch.relu(x.float() @ w1.float().T + b1).to(dtype).float()  # the hidden activation is 16-bit, as in the model
    want = x.float() + h @ w2.float().T + b2
    got = ops.ffn_fused(x, w1, b1, w2, b2)
    rel = (got - want).norm() / want.norm()
    assert rel < 1e-4, f"relative error {rel.item():.2e}"


def test_no_bias_and_strided_rows():
    x, w1, _, w2, _ = _operands(300, 192, torch.float16, seed=3)
    xs = torch.zeros(300, 264, device=DEV, dtype=torch.float16)[:, :256]
    xs.copy_(x)
    out = torch.zeros(300, 258, device=DEV)[:, :256]
    ops.ffn_fused(xs, w1, None, w2, None, out=out)
    assert torch.equal(out, _two_gemm(x, w1, None, w2, None))


@pytest.mark.parametrize("variant", sorted(VARIANTS))
@pytest.mark.parametrize("M", [1, 127, 900])
def test_rows_past_m_are_not_written(M, variant):
    x, w1, b1, w2, b2 = _operands(M, 128, torch.bfloat16, seed=11)
    big = torch.full((M + 300, 256), 1234.5, device=DEV)
    ops.ffn_fused(x, w1, b1, w2, b2, out=big[:M], variant=VARIANTS[variant])
    torch.cuda.synchronize()
    assert torch.all(big[M:] == 1234.5)
    assert torch.equal(big[:M], _two_gemm(x, w1, b1, w2, b2))


def _call(x, ldx, w1, ldw1, b1, w2, ldw2, b2, out, ldo, M, E, F, dtype, variant=0):
    p = lambda t: None if t is None else (t if isinstance(t, int) else t.data_ptr())  # noqa: E731
    return _lib.lib.ape_ffn_fused(p(x), ldx, p(w1), ldw1, p(b1), p(w2), ldw2, p(b2), p(out), ldo, M, E, F, dtype, variant,
                                  _lib.current_stream_ptr())


def test_bad_arguments_are_rejected():
    F16 = _lib.APE_DTYPE_F16
    x, w1, b1, w2, b2 = _operands(256, 128, torch.float16)
    out = torch.empty(256, 256, device=DEV)
    ok = (x, 256, w1, 256, b1, w2, 128, b2, out, 256, 256, 256, 128, F16)
    assert _call(*ok) == 0
    bad = {
        "E != 256": dict(E=128),
        "F % 64": dict(F=96),
        "F = 0": dict(F=0),
        "fp32 operands": dict(dtype=_lib.APE_DTYPE_F32),
        "misaligned x": dict(x=x.data_ptr() + 2),
        "misaligned w2": dict(w2=w2.data_ptr() + 8),
        "x pitch": dict(ldx=260),
        "w1 pitch": dict(ldw1=252),
        "out pitch": dict(ldo=257),
        "misaligned out": dict(out=out.data_ptr() + 4),
        "misaligned bias": dict(b1=b1.data_ptr() + 4),
        "null x": dict(x=None),
        "variant": dict(variant=3),
    }
    names = ["x", "ldx", "w1", "ldw1", "b1", "w2", "ldw2", "b2", "out", "ldo", "M", "E", "F", "dtype", "variant"]
    rcs = {}

    def reject_all():  # on a thread of its own: ape_last_error() is per thread, and this one's text dies with it
        torch.cuda.set_device(DEV)
        for what, change in bad.items():
            rcs[what] = _call(**{**dict(zip(names, ok + (0,))), **change})

    t = threading.Thread(target=reject_all)
    t.start()
    t.join()
    assert set(rcs) == set(bad)
    for what, rc in rcs.items():
        assert rc < 0, f"{what}: accepted"
    assert rcs["E != 256"] == -2 and rcs["F % 64"] == -2
    with pytest.raises(RuntimeError, match="one dtype"):
        ops.ffn_fused(x, w1.to(torch.bfloat16), b1, w2, b2)
    with pytest.raises(RuntimeError, match="w1 must be"):
        ops.ffn_fused(x, w1, b1, w2.T.contiguous(), b2)
    torch.cuda.synchronize()
    assert torch.equal(out, _two_gemm(x, w1, b1, w2, b2))  # the rejected calls wrote nothing


def test_model_ffns_take_the_fused_kernel():
    import copy

    from ape_b200 import configs
    from ape_b200.modeling import build_model
    from oracle import synth

    spec = copy.deepcopy(configs.MINI)
    spec["ffn_dim"] = 192  # a width no other GEMM of the MINI model has
    model = build_model(spec)
    synth.fill_state_dict(model)
    model = model.to(DEV)
    inputs = [{"image": synth.image(64, 64, seed=3), "height": 64, "width": 64}]
    model.engine_dtype = torch.float16
    try:
        ops.PROFILE_EVENTS = []
        eager = model(inputs)
        torch.cuda.synchronize()
        tags = [t for (t, _, _) in ops.PROFILE_EVENTS]
        ops.PROFILE_EVENTS = None
        le = model.last_outputs["pred_logits"].clone()
        model.use_cuda_graphs = True
        for _ in range(2):  # capture, then replay
            out = model(inputs)
        lg = model.last_outputs["pred_logits"].clone()
    finally:
        ops.PROFILE_EVENTS = None
        model.engine_dtype, model.use_cuda_graphs = torch.float32, False
    F = spec["ffn_dim"]
    n_layers = spec["enc_layers"] + spec["dec_layers"]
    fused = [t for t in tags if t[0] == "ffn_fused"]
    assert len(fused) == n_layers and all(t[2:] == (256, F) for t in fused), fused
    ffn_gemms = [t for t in tags if t[0] == "gemm_tn" and (t[2], t[3]) in ((F, 256), (256, F))]
    assert not ffn_gemms, ffn_gemms
    torch.testing.assert_close(lg, le, rtol=0, atol=0)
    assert torch.equal(out[0]["instances"].pred_classes, eager[0]["instances"].pred_classes)
