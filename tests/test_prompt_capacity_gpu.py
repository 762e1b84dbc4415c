"""GPU: `prompt_capacity` — name prompts of any length up to a capacity C replay one CUDA graph per padded shape.

Kernel: ops.linear_cols_dev (ape_gemm_tn_cols_dev) equals linear_tc(act="clamp", fp32 out) over the first n rows of the weight bit
for bit, writes -inf past them, and reads n from the device under capture: one graph, replayed with several n.

Model: MINI (and the fusion-free MINI_L_A) in fp16 and bf16 under `use_cuda_graphs`, over a seeded stream of `text_prompt` name
lists of 1 to 60 names (distinct counts, mixed image sizes inside the 64^2 pad).  With C = 64 the stream captures one "forward"
graph, and its logits (cut back to n), boxes, scores, classes and query indices equal a `prompt_capacity = None` run of the
same calls bit for bit: a logit column does not depend on the GEMM's N, and the padded columns (-inf) are never candidates, so the
compacted pairs keep their order.  Also: a negative test_score_thresh (where a padded column would otherwise pass), instance
masks + semantic maps through model(inputs) (`sem_seg` is [n, H, W]), `forward_packed` with masks and semantic maps under
`packed_output_capacity`, n > C on the per-n path, a cached vocabulary keeping its exact-n key, `DefaultPredictor`, and a
boxes-only `forward_packed` of a new prompt length without a host synchronisation."""
import zlib

import numpy as np
import pytest
import torch

from ape_b200 import configs, ops, parallel
from ape_b200.modeling import build_model
from oracle import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CAP = 64
DTYPES = [torch.float16, torch.bfloat16]


class _NamesOnDevice:
    """Text features seeded by each name's content, kept on the device (so a new prompt uploads nothing)."""

    def __init__(self, lang_dim):
        self.bank = torch.randn((4096, lang_dim), generator=torch.Generator().manual_seed(5)).to(DEV)

    def forward_text(self, text_list, cache=False, **kw):
        return {"last_hidden_state_eot": torch.stack([self.bank[zlib.crc32(t.encode()) % 4096] for t in text_list])}


def _model(spec, dtype):
    m = build_model(spec)
    synth.fill_state_dict(m)
    m = m.to(DEV).eval()
    m.engine_dtype = dtype
    m.set_model_language(_NamesOnDevice(spec["lang_dim"]))
    m.test_mask_on = False
    return m


@pytest.fixture(scope="module", params=DTYPES, ids=["fp16", "bf16"])
def model(built, request):
    return _model(configs.MINI, request.param)


def _stream(seed, count=8, lo=1, hi=60):
    """(image size, names) pairs: distinct name counts in [lo, hi], sizes inside the 64^2 pad."""
    g = np.random.default_rng(seed)
    counts = g.choice(np.arange(lo, hi + 1), size=count, replace=False)
    sizes = [(64, 64), (56, 64), (33, 17), (48, 40)]
    return [(sizes[i % len(sizes)], ",".join(f"thing{seed}_{i}_{j}" for j in range(int(n)))) for i, n in enumerate(counts)]


def _inputs(size, names, seed):
    h, w = size
    return [{"image": synth.image(h, w, seed=seed), "height": 2 * h, "width": 2 * w, "prompt": "text", "text_prompt": names}]


def _padded_graphs(model):
    return [k for k in model._graph_cache if k[0][0] == "forward" and k[0][6] is not None]


def _call(model, inputs, cap, packed=False):
    model.prompt_capacity, model.use_cuda_graphs = cap, True
    out = model.forward_packed(inputs).clone() if packed else model(inputs)
    return out, model.last_outputs["pred_logits"].clone(), model.last_outputs["pred_boxes"].clone()


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert set(x) == set(y)
        for k in x:
            if k == "instances":
                i, j = x[k], y[k]
                assert len(i) == len(j)
                assert torch.equal(i.pred_boxes.tensor, j.pred_boxes.tensor) and torch.equal(i.scores, j.scores)
                assert torch.equal(i.pred_classes, j.pred_classes)
                for f in ("pred_masks", "query_index"):
                    if i.has(f) or j.has(f):
                        assert torch.equal(getattr(i, f), getattr(j, f)), f
                if i.has("pred_masks_rle") or j.has("pred_masks_rle"):
                    assert [r["counts"] for r in i.pred_masks_rle] == [r["counts"] for r in j.pred_masks_rle]
            elif torch.is_tensor(x[k]):
                assert torch.equal(x[k], y[k]), k
            elif isinstance(x[k], list):
                assert [r["counts"] for r in x[k]] == [r["counts"] for r in y[k]], k
            else:
                assert x[k] == y[k], k


def _check_stream(model, seed, packed=False, check=None, n_graphs=1, stream=None):
    """Runs the stream with C = CAP (one capture per padded shape and size key), then with None, and compares call by call."""
    stream = stream or _stream(seed)
    try:
        model._graph_cache.clear()
        got = [_call(model, _inputs(size, names, seed + i), CAP, packed) for i, (size, names) in enumerate(stream)]
        assert len(_padded_graphs(model)) == n_graphs and len(model._graph_cache) == n_graphs, "one graph for every prompt length"
        n_det = 0
        for i, (size, names) in enumerate(stream):
            n = len(names.split(","))
            want = _call(model, _inputs(size, names, seed + i), None, packed)
            out, logits, boxes = got[i]
            assert logits.shape[-1] == n and torch.equal(logits, want[1]), f"logits differ at call {i} (n = {n})"
            assert torch.equal(boxes, want[2])
            a, b = (parallel.unpack_packed(out), parallel.unpack_packed(want[0])) if packed else (out, want[0])
            (check or _same)(a, b)
            n_det += sum(len(o["instances"]) for o in b)
            if not packed:
                assert all(bool((o["instances"].pred_classes < n).all()) for o in a)
        assert n_det > 0
    finally:
        model.prompt_capacity = None


# -- the kernel --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("M", [20, 900])
def test_cols_dev_matches_exact_gemm_and_replays(built, dtype, M):
    g = torch.Generator().manual_seed(M)
    C, K = 1536, 256
    x = (torch.randn((M, K), generator=g) * 2).to(DEV, dtype)
    w = torch.randn((C, K), generator=g).to(DEV, dtype)
    b = torch.randn((C,), generator=g).to(DEV)
    w[7] *= 1e4  # a clamped column
    n_dev = torch.zeros((1,), dtype=torch.int32, device=DEV)
    ops.linear_cols_dev(x, w, b, n_dev)  # warm-up outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ops.linear_cols_dev(x, w, b, n_dev)
    for n in (3, 1203, 1, C, 8):
        n_dev.fill_(n)
        graph.replay()
        want = ops.linear_tc(x, w[:n], b[:n].contiguous(), act="clamp", out_dtype=torch.float32)
        assert torch.equal(out[:, :n], want), f"n = {n}"
        assert torch.isneginf(out[:, n:]).all()
        eager = ops.linear_cols_dev(x, w, b, n_dev)
        assert torch.equal(eager, out)
    ref = (x.double() @ w[:n].double().t() + b[:n].double()).clamp(-50000, 50000)  # the last replay's n columns
    assert (out[:, :n].double() - ref).abs().max().item() < 1e-2 * ref.abs().max().item()
    with pytest.raises(RuntimeError, match="n_cols"):
        ops.linear_cols_dev(x, w, b, n_dev.long())


# -- the model -----------------------------------------------------------------------------------------------------------------
def test_name_prompt_stream_one_graph_bit_identical(model):
    _check_stream(model, 1)


def test_fusion_free_model(built):
    m = _model(configs.MINI_L_A, torch.float16)
    _check_stream(m, 2)


def test_negative_score_threshold_keeps_padding_out(model):
    """Every real pair is a candidate at a negative threshold; a padded column (score 0) would be one too if it were not masked.
    Both selection arms: the compacted list and (cap 1) the class-wise NMS."""
    thresh, cap = model.test_score_thresh, model.static_inference_cap
    try:
        model.test_score_thresh = -1.0
        _check_stream(model, 3)
        model.static_inference_cap, model._static_overflowed = 1, True
        _check_stream(model, 4)
    finally:
        model.test_score_thresh, model.static_inference_cap, model._static_overflowed = thresh, cap, False


def test_masks_and_semantic_maps(model):
    model.test_mask_on, model.semantic_on = True, True
    try:
        _check_stream(model, 5)
    finally:
        model.test_mask_on, model.semantic_on = False, False


def _rle_decode(seg):
    """cocoapi's compressed run-length string -> bool [H, W] (column-major runs, starting with a run of zeros)."""
    h, w = seg["size"]
    s, counts, p = seg["counts"], [], 0
    while p < len(s):
        x, k, more = 0, 0, True
        while more:
            c = s[p] - 48
            x |= (c & 0x1F) << (5 * k)
            more = bool(c & 0x20)
            p, k = p + 1, k + 1
            if not more and c & 0x10:
                x |= -1 << (5 * k)
        if len(counts) > 2:
            x += counts[-2]
        counts.append(x)
    m, pos, val = np.zeros(h * w, dtype=bool), 0, False
    for c in counts:
        m[pos:pos + c] = val
        pos, val = pos + c, not val
    return m.reshape(w, h).T


def _label_map(table):
    h, w = table[0]["segmentation"]["size"]
    out = np.full((h, w), -1, dtype=np.int64)
    for e in table:
        out[_rle_decode(e["segmentation"])] = e["label"]
    return out


def _packed_same(n_classes):
    """Detections bit for bit.  The packed semantic map comes from a softmax over C columns (the padding at exactly zero
    weight) instead of n, whose last bits may differ: every label is a real class (< n), and at least 99 % of the pixels carry the
    exact-n run's label."""
    def check(a, b):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            _same([{"instances": x["instances"]}], [{"instances": y["instances"]}])
            if "sem_seg_rle" in y:
                assert all(e["label"] < n_classes() for e in x["sem_seg_rle"])
                gm, wm = _label_map(x["sem_seg_rle"]), _label_map(y["sem_seg_rle"])
                assert (wm >= 0).all() and (gm >= 0).all()
                assert (gm == wm).mean() >= 0.99
            if "panoptic_seg" in y:
                (gm, gs), (wm, ws) = x["panoptic_seg"], y["panoptic_seg"]
                assert all(s["category_id"] < n_classes() for s in gs) and len(gs) > 0
                assert (gm == wm).float().mean().item() >= 0.99
    return check


def _check_packed(model, seed, n_graphs=1, lo=1):
    stream = _stream(seed, lo=lo)
    counts = iter([len(names.split(",")) for _, names in stream])
    state = {}

    def n_classes():
        return state["n"]

    check = _packed_same(n_classes)

    def wrapped(a, b):
        state["n"] = next(counts)
        check(a, b)

    _check_stream(model, seed, packed=True, check=wrapped, n_graphs=n_graphs, stream=stream)


def test_packed_masks_and_semantic_with_output_capacity(model):
    model.test_mask_on, model.semantic_on, model.mask_format, model.packed_output_capacity = True, True, "rle", 128
    try:
        _check_packed(model, 6)
    finally:
        model.test_mask_on, model.semantic_on, model.mask_format, model.packed_output_capacity = False, False, "bitmask", None


def test_packed_semantic_per_size_key(model):
    """Without packed_output_capacity the packed semantic stage takes ops.semseg_label at host sizes: one graph per image size
    (four in the stream), each serving every prompt length."""
    model.test_mask_on, model.semantic_on, model.mask_format = True, True, "rle"
    try:
        _check_packed(model, 7, n_graphs=4)
    finally:
        model.test_mask_on, model.semantic_on, model.mask_format = False, False, "bitmask"


def test_packed_panoptic(model):
    """The panoptic class choice and its transform_eval softmax over a padded prompt: thing / stuff lists of 6 + 6 classes, prompts
    of 12 to 60 names (the dataset's prompt type set to "text", so the names come from the call)."""
    name = model.dataset_names[0]
    saved = (dict(model.dataset_stuff), list(model.dataset_prompts))
    model.dataset_stuff[name] = ([f"c{i}" for i in range(6)], [f"c{i}" for i in range(6, 12)], "thing+stuff")
    model.dataset_prompts = ["text"] * len(model.dataset_names)
    model.set_eval_dataset(name)
    model.test_mask_on, model.panoptic_on, model.mask_format, model.packed_output_capacity = True, True, "rle", 128
    try:
        _check_packed(model, 8, lo=12)
    finally:
        model.test_mask_on, model.panoptic_on, model.mask_format, model.packed_output_capacity = False, False, "bitmask", None
        model.dataset_stuff, model.dataset_prompts = saved
        model.set_eval_dataset("")


def test_longer_prompt_and_cached_vocabulary_keep_exact_keys(model):
    """n > C takes the per-n key; a dataset vocabulary (cached) keeps its exact-n key with C set."""
    model._graph_cache.clear()
    try:
        names = ",".join(f"long{j}" for j in range(CAP + 5))
        out, logits, _ = _call(model, _inputs((64, 64), names, 0), CAP)
        assert logits.shape[-1] == CAP + 5 and not _padded_graphs(model)
        want = _call(model, _inputs((64, 64), names, 0), None)
        _same(out, want[0])
        model._graph_cache.clear()
        _call(model, [{"image": synth.image(64, 64, seed=0), "height": 64, "width": 64}], CAP)
        keys = [k for k in model._graph_cache if k[0][0] == "forward"]
        assert len(keys) == 1 and keys[0][0][6] is None and keys[0][0][3][1] == configs.MINI["num_classes"]
        model.prompt_capacity = 0
        with pytest.raises(ValueError, match="prompt_capacity"):
            model(_inputs((64, 64), "a,b", 0))
    finally:
        model.prompt_capacity = None


def test_predictor_replays_one_graph(model):
    from ape_b200.engine.defaults import DefaultPredictor, ResizeShortestEdge

    model._graph_cache.clear()
    pred = DefaultPredictor(model, aug=ResizeShortestEdge(64, 64))
    img = np.random.default_rng(3).integers(0, 256, (45, 60, 3), dtype=np.uint8)
    try:
        for names in ("person,car,dog", "cat", "person,car,dog,bus,bicycle,traffic_light", "cat"):
            model.prompt_capacity, model.use_cuda_graphs = CAP, True
            got = pred(img, text_prompt=names)
            model.prompt_capacity = None
            want = pred(img, text_prompt=names)
            _same([got], [want])
        assert len(_padded_graphs(model)) == 1
    finally:
        model.prompt_capacity = None


def test_packed_new_prompt_length_adds_no_host_synchronisation(model):
    model._graph_cache.clear()
    model.prompt_capacity, model.use_cuda_graphs = CAP, True
    try:
        img = synth.image(56, 64, seed=0).to(DEV)
        inp = lambda names: [{"image": img, "height": 56, "width": 64, "prompt": "text", "text_prompt": names}]  # noqa: E731
        for names in ("a,b,c", "a,b,c,d"):
            model.forward_packed(inp(names))
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            out = model.forward_packed(inp("p,q,r,s,t,u,v,w,x,y,z"))  # a length not seen before
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert len(_padded_graphs(model)) == 1
        model.prompt_capacity = None
        _same(parallel.unpack_packed(out), parallel.unpack_packed(model.forward_packed(inp("p,q,r,s,t,u,v,w,x,y,z"))))
    finally:
        model.prompt_capacity = None


# -- multi-token prompts: the folded fusion on a padded text ------------------------------------------------------------------
def _fold_operands(B, S, NH, N, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    v = torch.randn((B, S, 256), generator=g).to(DEV, dtype)
    qa = (torch.randn((B, NH, N, 256), generator=g) * 0.08).to(DEV, dtype)
    u = torch.randn((B, NH, N, 256), generator=g).to(DEV, dtype)
    qc = torch.randn((B, NH, N), generator=g).to(DEV)
    gamma, bias = torch.rand(256, generator=g).to(DEV), torch.randn(256, generator=g).to(DEV)
    return v, qa, u, qc, gamma, bias


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("C", [64, 256])
def test_fold_dev_matches_exact_n_and_replays(built, dtype, C):
    """ape_vlf_fold_vision_dev / ape_vlf_fold_pool_dev on a text padded to C tokens (garbage in the padding) against the exact-n
    entry points on the first n tokens: the vision side within one 16-bit rounding of the output scale, the pooled rows of
    real tokens likewise, the padding rows exactly zero; captured once and replayed with several n."""
    B, S, NH = 2, 700, 8
    v, qa, u, qc, gamma, bias = _fold_operands(B, S, NH, C, dtype, C)
    n_dev = torch.ones((1,), dtype=torch.int32, device=DEV)
    ops.vlf_fold_vision(v, qa, u, qc, gamma, bias, n_dev=n_dev)
    ops.vlf_fold_pool(v, qa, n_dev=n_dev)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ops.vlf_fold_vision(v, qa, u, qc, gamma, bias, n_dev=n_dev)
        pooled = ops.vlf_fold_pool(v, qa, n_dev=n_dev)
    tol = 2 ** -9 if dtype == torch.float16 else 2 ** -6
    for n in (3, C, 1, C - 5, 17):
        n_dev.fill_(n)
        graph.replay()
        want = ops.vlf_fold_vision(v, qa[:, :, :n].contiguous(), u[:, :, :n].contiguous(), qc[:, :, :n].contiguous(), gamma, bias)
        scale = want.float().abs().max().item()
        assert (out.float() - want.float()).abs().max().item() <= 2 * tol * scale, f"vision side, n = {n}"
        wp = ops.vlf_fold_pool(v, qa[:, :, :n].contiguous()).view(B, n, -1)
        gp = pooled.view(B, C, -1)
        assert (gp[:, :n].float() - wp.float()).abs().max().item() <= 2 * tol * wp.float().abs().max().item(), f"pool, n = {n}"
        assert (gp[:, n:] == 0).all()
    with pytest.raises(RuntimeError, match="n_dev"):
        ops.vlf_fold_pool(v, qa, n_dev=n_dev.long())


@pytest.fixture(scope="module")
def vlf(built):
    from test_prompt_graph_gpu import SPEC

    m = _model(SPEC, torch.float16)
    m.set_model_language(_NamesOnDevice(SPEC["lang_dim"]))
    return m


def _phrase_stream(seed, count=6):
    """1 to 16 phrases (with spaces: "phrase" prompts), distinct counts, mixed sizes."""
    g = np.random.default_rng(seed)
    counts = g.choice(np.arange(1, 17), size=count, replace=False)
    sizes = [(64, 64), (56, 64), (33, 17)]
    return [(sizes[i % len(sizes)], ",".join(f"red thing {seed} {i} {j}" for j in range(int(c)))) for i, c in enumerate(counts)]


def _close_run(model, stream, make_inputs, logit_tol, feat_tol):
    """C = CAP (one graph for the stream) against None (per-n eager or graph): the fused features (memory) and the logits within
    a 16-bit tolerance relative to their scale, and the kept detections identical (classes, query indices; the boxes, decoded
    from features that carry the fusion's 16-bit rounding, within 2e-3 relative)."""
    try:
        model._graph_cache.clear()
        got = []
        for i, (size, text) in enumerate(stream):
            model.prompt_capacity, model.use_cuda_graphs = CAP, True
            out = model(make_inputs(size, text, i))
            lo = model.last_outputs
            got.append((out, lo["pred_logits"].clone(), lo["memory"].clone()))
        assert len(_padded_graphs(model)) == 1 and len(model._graph_cache) == 1
        n_det = 0
        for i, (size, text) in enumerate(stream):
            model.prompt_capacity = None
            want = model(make_inputs(size, text, i))
            lo = model.last_outputs
            out, logits, memory = got[i]
            assert logits.shape == lo["pred_logits"].shape
            assert (logits - lo["pred_logits"]).abs().max().item() <= logit_tol * max(1.0, lo["pred_logits"].abs().max().item())
            assert (memory.float() - lo["memory"].float()).abs().max().item() <= feat_tol * lo["memory"].float().abs().max().item()
            for x, y in zip(out, want):
                i1, i2 = x["instances"], y["instances"]
                assert torch.equal(i1.pred_classes, i2.pred_classes) and torch.equal(i1.query_index, i2.query_index)
                torch.testing.assert_close(i1.pred_boxes.tensor, i2.pred_boxes.tensor, rtol=2e-3, atol=1e-3)
                n_det += len(i2)
        assert n_det > 0
    finally:
        model.prompt_capacity = None


def _phrase_inputs(size, text, seed):
    h, w = size
    return [{"image": synth.image(h, w, seed=seed), "height": h, "width": w, "prompt": "text", "text_prompt": text}]


def test_phrase_prompts_one_graph_within_tolerance(vlf):
    _close_run(vlf, _phrase_stream(1), _phrase_inputs, 2e-2, 2e-2)


def test_expression_prompts_one_graph_within_tolerance(vlf):
    def inputs(size, text, seed):
        h, w = size
        return [{"image": synth.image(h, w, seed=seed + k), "height": h, "width": w, "prompt": "expression",
                 "expressions": f"the {text.split(',')[0]} number {k}"} for k in range(2)]

    _close_run(vlf, _phrase_stream(2, count=4), inputs, 2e-2, 2e-2)


def test_fused_vocabulary_names_one_graph_within_tolerance(vlf):
    saved = vlf.name_prompt_fusion_text
    vlf.name_prompt_fusion_text = [True] * len(vlf.dataset_names)
    try:
        stream = [(size, ",".join(f"fv{i}_{j}" for j in range(n))) for i, ((size, _), n) in
                  enumerate(zip(_phrase_stream(3), (2, 9, 33, 5, 60, 14)))]
        _close_run(vlf, stream, _phrase_inputs, 2e-2, 2e-2)
    finally:
        vlf.name_prompt_fusion_text = saved


def test_fusion_free_model_phrases_bit_identical(built):
    """APE-L_A's classifier-only text: phrase prompts of 1 to 16 phrases now share one graph, equal to the per-n run bit for bit."""
    m = _model(configs.MINI_L_A, torch.float16)
    _check_stream(m, 9, stream=_phrase_stream(9))
