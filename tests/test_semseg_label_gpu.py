"""Semantic label maps on the device (model.sem_seg_format = "label", csrc/semseg.cu + the class-argmax GEMM epilogue):
the operand resampler against F.interpolate -> sigmoid -> crop -> F.interpolate, the argmax epilogue against torch.argmax of an
fp32 matmul of the same 16-bit operands, the model's label output against the argmax of its "maps" output, memory, argument
rejection and CUDA-graph replay."""
import math

import pytest
import torch
import torch.nn.functional as F

from ape_b200 import _lib, ops
from ape_b200 import configs
from oracle import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LIB = _lib.lib


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _resample(logits, index, padded, img, out, dt, row0=0, rows=None, fill=7.0):
    """ape_semseg_resample of output rows [row0, row0 + rows) -> [rows * out_w, Kp] (filled with `fill` beforehand)."""
    K = index.numel()
    Kp = (K + 7) // 8 * 8
    rows = out[0] - row0 if rows is None else rows
    A = torch.full((rows * out[1], Kp), fill, dtype=dt, device=DEV)
    rc = LIB.ape_semseg_resample(logits.data_ptr(), index.data_ptr(), A.data_ptr(), Kp, K, logits.shape[1], logits.shape[2],
                                 padded[0], padded[1], img[0], img[1], out[0], out[1], row0, rows,
                                 _lib.dtype_code(logits.dtype), _lib.dtype_code(dt), _lib.current_stream_ptr())
    _lib.check(rc, "ape_semseg_resample")
    return A


def _ref_operand(logits, index, padded, img, out):
    m = F.interpolate(logits[index][None].float(), size=padded, mode="bilinear", align_corners=False)[0].sigmoid()
    a = F.interpolate(m[None, :, : img[0], : img[1]], size=out, mode="bilinear", align_corners=False)[0]
    return a.permute(1, 2, 0).reshape(-1, index.numel())


RESAMPLE_CASES = {  # K, logit grid, padded, image, output
    "down_300": (300, (256, 256), (1024, 1024), (1024, 768), (480, 640)),
    "up_7": (7, (256, 256), (1024, 1024), (1024, 768), (2048, 1536)),
    "odd_1": (1, (37, 53), (301, 299), (250, 201), (333, 177)),
    "odd_7": (7, (64, 48), (255, 257), (255, 190), (97, 101)),
}


@pytest.mark.parametrize("logit_dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("case", sorted(RESAMPLE_CASES))
def test_resampler_matches_interpolate_sigmoid_crop_interpolate(case, logit_dtype):
    K, hw, padded, img, out = RESAMPLE_CASES[case]
    Q = K + 5
    logits = (torch.randn((Q, *hw), generator=_gen(1), device=DEV) * 4).to(logit_dtype)
    index = torch.randperm(Q, generator=_gen(2), device=DEV)[:K]
    want = _ref_operand(logits, index, padded, img, out)
    for dt, tol in ((torch.float16, 1e-3), (torch.bfloat16, 4e-3)):  # one rounding of values in [0, 1] to the operand type
        A = _resample(logits, index, padded, img, out, dt)
        err = (A[:, :K].float() - want).abs().max().item()
        assert err <= tol, f"{case} {dt}: max|err| {err:.2e}"
        assert (A[:, K:] == 0).all(), "pad columns K..Kp must be zero"
    del want


def test_resampler_band_split_gives_the_same_bytes():
    K, hw, padded, img, out = 13, (64, 64), (512, 512), (500, 380), (300, 229)
    logits = torch.randn((20, *hw), generator=_gen(3), device=DEV).half()
    index = torch.arange(3, 3 + K, device=DEV)
    one = _resample(logits, index, padded, img, out, torch.float16)
    parts, r0 = [], 0
    for rows in (1, 77, 100, 122):
        parts.append(_resample(logits, index, padded, img, out, torch.float16, row0=r0, rows=rows))
        r0 += rows
    assert r0 == out[0]
    assert torch.equal(torch.cat(parts).view(torch.int16), one.view(torch.int16))


def _argmax(A, W, col_base=0, init=(float("-inf"), 0)):
    M, K = A.shape
    keys = torch.empty((M,), dtype=torch.int64, device=DEV)
    label = torch.empty((M,), dtype=torch.int64, device=DEV)
    score = torch.empty((M,), dtype=torch.float32, device=DEV)
    s = _lib.current_stream_ptr()
    _lib.check(LIB.ape_semseg_keys_init(keys.data_ptr(), M, init[0], init[1], s), "ape_semseg_keys_init")
    _lib.check(LIB.ape_gemm_tn_argmax(A.data_ptr(), A.stride(0), W.data_ptr(), W.stride(0), keys.data_ptr(), M, W.shape[0], K,
                                      col_base, _lib.dtype_code(A.dtype), s), "ape_gemm_tn_argmax")
    _lib.check(LIB.ape_semseg_keys_decode(keys.data_ptr(), M, label.data_ptr(), score.data_ptr(), s), "ape_semseg_keys_decode")
    return label, score


def _operands(M, N, K, dt, seed):
    A = torch.rand((M, K), generator=_gen(seed), device=DEV).to(dt)          # sigmoid-like pixel operand
    W = torch.rand((N, K), generator=_gen(seed + 1), device=DEV).to(dt)      # class weights
    return A, W


def _check_labels(label, score, ref):
    top2 = ref.topk(min(2, ref.shape[1]), dim=1).values
    mx = top2[:, 0]
    gap = (top2[:, 0] - top2[:, 1]) if ref.shape[1] > 1 else torch.full_like(mx, float("inf"))
    want = ref.argmax(1)
    clear = gap > 1e-4 * mx.abs()
    assert clear.float().mean().item() > 0.5, "test operands have too few well-separated maxima"
    assert torch.equal(label[clear], want[clear])
    assert ((label >= 0) & (label < ref.shape[1])).all()
    torch.testing.assert_close(score, mx, rtol=1e-5, atol=1e-5)
    # wherever the label differs, the value it picked is (within accumulation-order noise) also maximal
    torch.testing.assert_close(ref.gather(1, label[:, None])[:, 0], mx, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,N,K", [(384, 128, 64), (1000, 1203, 304), (517, 1, 24), (777, 2049, 72), (130, 300, 8)])
def test_argmax_epilogue_matches_torch_argmax(M, N, K, dt):
    A, W = _operands(M, N, K, dt, seed=M + N)
    label, score = _argmax(A, W)
    _check_labels(label, score, A.float() @ W.float().t())


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_argmax_exact_ties_resolve_to_the_lowest_class(dt):
    M, N, K = 700, 1500, 64
    A, W = _operands(M, N, K, dt, seed=11)
    W[:] = W * 0.5
    top = (torch.rand((K,), generator=_gen(12), device=DEV) + 1.0).to(dt)
    for c in (1499, 700, 21, 20, 300):  # same tile, same thread pair (20, 21), other tiles; the lowest must win everywhere
        W[c] = top
    label, score = _argmax(A, W)
    assert (label == 20).all()
    ref = A.float() @ W.float().t()
    torch.testing.assert_close(score, ref[:, 20], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_argmax_class0_constant(dt):
    M, N, K = 1000, 300, 40
    A, W = _operands(M, N, K, dt, seed=21)
    ref = A.float() @ W.float().t()
    c0 = ref.max(1).values.median().item()  # class 0 wins about half of the rows
    label, score = _argmax(A, W[1:], col_base=1, init=(c0, 0))
    full = torch.cat([torch.full((M, 1), c0, device=DEV), ref[:, 1:]], 1)
    frac0 = (label == 0).float().mean().item()
    assert 0.2 < frac0 < 0.8
    _check_labels(label, score, full)
    # a constant equal to a GEMM value loses nothing: class 0 is the lowest index
    label, _ = _argmax(A, W[1:] * 0, col_base=1, init=(0.0, 0))
    assert (label == 0).all()


def test_semseg_label_band_split_and_empty_selection():
    Q, hw, padded, img, out = 40, (64, 64), (512, 512), (480, 400), (300, 251)
    logits = torch.randn((Q, *hw), generator=_gen(31), device=DEV)
    qi = torch.arange(0, Q, 2, device=DEV)
    cls = torch.softmax(torch.randn((len(qi), 150), generator=_gen(32), device=DEV) * 3, -1).half()
    l1, s1 = ops.semseg_label(logits, qi, cls, padded, img, out)
    l2, s2 = ops.semseg_label(logits, qi, cls, padded, img, out, band_bytes=7 * out[1] * 24 * 2)  # 7-row bands
    assert torch.equal(l1, l2) and torch.equal(s1, s2)
    empty = qi[:0]
    l, s = ops.semseg_label(logits, empty, cls[:0], padded, img, out)
    assert (l == 0).all() and (s == 0).all()
    l, s = ops.semseg_label(logits, empty, cls[:0], padded, img, out, class0_const=-2.0)
    assert (l == 1).all() and (s == 0).all()


def _semantic_inputs(Q, N, hw, seed):
    g = torch.Generator().manual_seed(seed)
    box_cls = (torch.randn((1, Q, N), generator=g) * 2).to(DEV)
    box_pred = torch.rand((1, Q, 4), generator=g).to(DEV) * 0.5 + 0.25
    mask_pred = (torch.randn((1, Q, *hw), generator=g) * 4).to(DEV)
    return box_cls, box_pred, mask_pred


@pytest.fixture(scope="module")
def mini():
    from ape_b200.modeling import build_model

    torch.backends.cuda.matmul.allow_tf32 = False
    m = build_model(configs.MINI)
    synth.fill_state_dict(m)
    return m.to(DEV)


def _both_formats(model, args, dtype):
    model.engine_dtype = dtype
    try:
        model.sem_seg_format = "maps"
        maps = model._semantic(*args)
        model.sem_seg_format = "label"
        label = model._semantic(*args)
    finally:
        model.engine_dtype, model.sem_seg_format = torch.float32, "maps"
    return maps, label


def _compare(maps, label, bound, what):
    for m, l in zip(maps, label):
        sem = m["sem_seg"]
        assert set(l) == {"sem_seg_label", "sem_seg_score"} and l["sem_seg_label"].dtype == torch.int64
        assert l["sem_seg_label"].shape == sem.shape[1:] and l["sem_seg_label"].device == sem.device
        top2 = sem.topk(2, dim=0).values
        mx, gap = top2[0], top2[0] - top2[1]
        diff = l["sem_seg_label"] != sem.argmax(0)
        frac = diff.float().mean().item()
        print(f"{what}: {frac:.2e} of {diff.numel()} pixels take another class than the maps' argmax")
        assert (gap[diff] <= bound * mx.abs()[diff]).all(), "a disagreeing pixel has a clear maximum"
        assert ((l["sem_seg_score"] - mx).abs() <= bound * mx.abs() + 1e-6).all()


def _forward_label(model, inp, dtype):
    """A "label" forward of the MINI masks model, and the arguments that give its semantic branch the same inputs again."""
    model.test_mask_on, model.semantic_on = True, True
    model.engine_dtype, model.sem_seg_format = dtype, "label"
    try:
        out = model(inp)
        lo = model.last_outputs
        images, _, sizes = model.preprocess_image(inp)
        args = (lo["pred_logits"], lo["pred_boxes"], lo["pred_masks"], sizes, tuple(images.shape[-2:]), inp)
    finally:
        model.test_mask_on, model.semantic_on = False, False
        model.engine_dtype, model.sem_seg_format = torch.float32, "maps"
    return out, args


def test_model_fp32_label_is_the_argmax_of_the_map(mini):
    model = mini
    inp = [{"image": synth.image(48, 64, seed=0), "height": 96, "width": 128}]
    out, args = _forward_label(model, inp, torch.float32)
    assert "sem_seg" not in out[0] and "instances" in out[0]
    maps = model._semantic(*args)
    sem = maps[0]["sem_seg"]
    assert out[0]["sem_seg_label"].shape == sem.shape[1:]
    assert torch.equal(out[0]["sem_seg_label"], sem.argmax(0))
    assert torch.equal(out[0]["sem_seg_score"], sem.amax(0))


@pytest.mark.parametrize("dtype,bound", [(torch.float16, 2e-3), (torch.bfloat16, 2e-2)])
def test_model_16bit_label_agrees_with_maps(mini, dtype, bound):
    model = mini
    inp = [{"image": synth.image(56, 64, seed=2), "height": 112, "width": 90}]
    out, args = _forward_label(model, inp, dtype)
    assert "sem_seg" not in out[0] and out[0]["sem_seg_label"].shape == (112, 90)
    maps, label = _both_formats(model, args, dtype)
    assert torch.equal(label[0]["sem_seg_label"], out[0]["sem_seg_label"])
    _compare(maps, label, bound, f"MINI {dtype}")


@pytest.mark.parametrize("dtype,bound", [(torch.float16, 2e-3), (torch.bfloat16, 2e-2)])
def test_1203_classes_label_agrees_with_maps(mini, dtype, bound):
    """300 kept queries (semantic_post_nms off), 1203 classes, 256^2 logits, a 1024 x 768 image padded to 1024^2, output 480 x 640,
    with the stuff_prob_thing constant in class 0."""
    model = mini
    box_cls, box_pred, mask_pred = _semantic_inputs(300, 1203, (256, 256), seed=5)
    name = model.dataset_names[0] if model.dataset_names else None
    saved = (model.semantic_post_nms, model.eval_dataset_id, dict(model.dataset_stuff), model.stuff_prob_thing)
    try:
        model.semantic_post_nms = False
        if name is not None:  # a stuff dataset whose first class is "things": class 0 is the stuff_prob_thing constant
            model.eval_dataset_id = 0
            model.dataset_stuff[name] = (None, ["things"] + [f"s{i}" for i in range(1202)], "stuff")
            model.stuff_prob_thing = 0.55
        args = (box_cls, box_pred, mask_pred, [(1024, 768)], (1024, 1024), [{"height": 480, "width": 640}])
        maps, label = _both_formats(model, args, dtype)
    finally:
        model.semantic_post_nms, model.eval_dataset_id, model.dataset_stuff, model.stuff_prob_thing = saved
    if name is not None:
        assert (maps[0]["sem_seg"][0] == math.log(0.55 / 0.45)).all()
        print(f"class 0 (the constant) wins {(label[0]['sem_seg_label'] == 0).float().mean().item():.3f} of the pixels")
    _compare(maps, label, bound, f"1203 classes {dtype}")


def test_label_memory_stays_small():
    """N_t = 1203 at 1024^2: the map path writes a 5 GB [1203, 1024, 1024] fp32 map; the label path stays under 10 % of it."""
    Q, N = 300, 1203
    logits = (torch.randn((Q, 256, 256), generator=_gen(41), device=DEV) * 4).half()
    qi = torch.arange(Q, device=DEV)
    cls = torch.softmax(torch.randn((Q, N), generator=_gen(42), device=DEV), -1).half()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    label, score = ops.semseg_label(logits, qi, cls, (1024, 1024), (1024, 1024), (1024, 1024))
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    map_bytes = N * 1024 * 1024 * 4
    print(f"label path: {extra / 2**20:.1f} MiB above the inputs ({100 * extra / map_bytes:.1f} % of the map)")
    assert extra < 0.1 * map_bytes


def test_bad_arguments_are_rejected():
    logits = torch.zeros((4, 16, 16), device=DEV)
    index = torch.arange(3, device=DEV)
    A = torch.zeros((64, 16), dtype=torch.float16, device=DEV)
    s = _lib.current_stream_ptr()
    ok = dict(lda=8, K=3, h=16, w=16, Hp=32, Wp=32, ih=30, iw=20, oh=8, ow=8, row0=0, rows=8, ld=APE_F32, ad=APE_F16)

    def resample(**kw):
        a = dict(ok, **kw)
        return LIB.ape_semseg_resample(logits.data_ptr(), index.data_ptr(), A.data_ptr(), a["lda"], a["K"], a["h"], a["w"], a["Hp"],
                                       a["Wp"], a["ih"], a["iw"], a["oh"], a["ow"], a["row0"], a["rows"], a["ld"], a["ad"], s)

    assert resample() == 0
    torch.cuda.synchronize()
    for bad in (dict(ad=APE_F32), dict(ld=5), dict(lda=4), dict(lda=12), dict(ih=33), dict(K=0), dict(rows=9), dict(row0=-1),
                dict(oh=0)):
        rc = resample(**bad)
        assert rc < 0, bad
        assert LIB.ape_last_error()
    keys = torch.zeros((64,), dtype=torch.int64, device=DEV)
    W = torch.zeros((8, 16), dtype=torch.float16, device=DEV)

    def gemm(lda=16, N=8, K=16, col_base=0, dt=APE_F16, a_off=0):
        return LIB.ape_gemm_tn_argmax(A.data_ptr() + a_off, lda, W.data_ptr(), 16, keys.data_ptr(), 64, N, K, col_base, dt, s)

    for bad in (dict(dt=APE_F32), dict(lda=12), dict(K=24), dict(N=0), dict(col_base=-1), dict(a_off=2)):
        assert gemm(**bad) < 0, bad
    assert LIB.ape_semseg_keys_init(keys.data_ptr(), -1, 0.0, 0, s) < 0
    assert LIB.ape_semseg_keys_init(keys.data_ptr() + 4, 8, 0.0, 0, s) < 0
    with pytest.raises(RuntimeError):
        ops.semseg_label(logits, index, torch.zeros((3, 5), device=DEV), (32, 32), (30, 20), (8, 8))  # fp32 class weights
    with pytest.raises(RuntimeError):
        ops.semseg_label(logits, index, torch.zeros((3, 5), dtype=torch.float16, device=DEV), (32, 32), (33, 20), (8, 8))


APE_F32, APE_F16 = _lib.APE_DTYPE_F32, _lib.APE_DTYPE_F16


def test_graph_replay_equals_eager():
    Q, N = 60, 200
    logits = (torch.randn((Q, 64, 64), generator=_gen(51), device=DEV) * 4).half()
    qi = torch.arange(0, Q, 3, device=DEV)
    cls = torch.softmax(torch.randn((len(qi), N), generator=_gen(52), device=DEV) * 3, -1).half()
    args = (logits, qi, cls, (256, 256), (250, 200), (300, 240))
    eager = ops.semseg_label(*args, class0_const=0.01, band_bytes=64 * 240 * 24 * 2)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.semseg_label(*args, class0_const=0.01, band_bytes=64 * 240 * 24 * 2)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = ops.semseg_label(*args, class0_const=0.01, band_bytes=64 * 240 * 24 * 2)
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static[0], eager[0]) and torch.equal(static[1], eager[1])
