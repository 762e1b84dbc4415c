"""GPU: the per-image-size geometry built on the device (csrc/geometry.cu ape_pad_geometry, ops.pad_geometry) against the torch
geometry it stands for: the pixel mask F.interpolate'd to every level, PositionEmbeddingSine and
DeformableDetrTransformerVL.geometry.  Padded 1024^2 and 1536^2 over the p2..p6 levels that APE-L_D's neck and APE-L_B's backbone
both feed the encoder, a four-level set, a padded shape that is not square (size_divisibility padding) and the MINI spec's 64^2 pad
whose last level is 1 x 1; one to four images of different sizes per batch, including the full pad, one-pixel-wide and
one-pixel-tall images and sizes that are no multiple of any stride.  Every output is compared with torch.equal."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from ape_b200 import _lib, configs, ops
from ape_b200.modeling import build_model
from ape_b200.modeling.detr import PositionEmbeddingSine

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
E = 256


@pytest.fixture(scope="module")
def transformer(built):
    return build_model(configs.MINI).transformer.to(DEV)


def _shapes(Hp, Wp, strides):
    return [(-(-Hp // s), -(-Wp // s)) for s in strides]


def _torch_geometry(tr, pe, Hp, Wp, shapes, sizes):
    """DeformableDETRSegmVL's geometry as the torch code builds it: pixel mask, nearest resize per level, sine embedding."""
    masks = torch.ones((len(sizes), Hp, Wp), dtype=torch.float32, device=DEV)
    for i, (h, w) in enumerate(sizes):
        masks[i, :h, :w] = 0
    lm = [F.interpolate(masks[None], size=sh).to(torch.bool).squeeze(0) for sh in shapes]
    pos = [pe(m).to(torch.float32) for m in lm]
    return tr.geometry(shapes, lm, pos)


def _sizes(Hp, Wp, B, seed):
    g = torch.Generator().manual_seed(seed)
    fixed = [(Hp, Wp), (Hp, 1), (1, Wp), (1, 1)]
    out = []
    for i in range(B):
        if seed % 2 == 0 and i < len(fixed):
            out.append(fixed[(i + seed // 2) % len(fixed)])
        else:  # sizes that are no multiple of any stride
            out.append((int(torch.randint(1, Hp + 1, (1,), generator=g)) | 1, int(torch.randint(1, Wp + 1, (1,), generator=g)) | 1))
    return [(min(h, Hp), min(w, Wp)) for h, w in out]


CASES = [  # (padded H, W, strides)
    (1024, 1024, (4, 8, 16, 32, 64)),
    (1536, 1536, (4, 8, 16, 32, 64)),
    (1024, 1024, (8, 16, 32, 64)),
    (800, 1344, (4, 8, 16, 32, 64)),
    (64, 64, (4, 8, 16, 32, 64)),
]


@pytest.mark.parametrize("Hp,Wp,strides", CASES)
@pytest.mark.parametrize("B", [1, 2, 3, 4])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
def test_equals_the_torch_geometry(transformer, Hp, Wp, strides, B, dtype):
    pe = PositionEmbeddingSine(num_pos_feats=E // 2, temperature=10000, normalize=True, offset=-0.5)
    shapes = _shapes(Hp, Wp, strides)
    lvl = torch.randn(len(shapes), E, generator=torch.Generator().manual_seed(B)).to(DEV)
    for seed in range(4):
        sizes = _sizes(Hp, Wp, B, seed)
        want = _torch_geometry(transformer, pe, Hp, Wp, shapes, sizes)
        got = ops.pad_geometry(torch.tensor(sizes, dtype=torch.int32, device=DEV), (Hp, Wp), shapes, pe.dim_t(DEV), lvl, dtype,
                               offset=pe.offset, eps=pe.eps, scale=pe.scale, want_pos=True)
        for k in ("mask_flatten", "valid_ratios", "reference_points", "output_proposals", "proposal_invalid"):
            assert got[k].dtype == want[k].dtype and got[k].shape == want[k].shape, k
            assert torch.equal(got[k], want[k]), f"{k} differs for sizes {sizes} in {Hp}x{Wp}"
        assert bool(want["mask_flatten"].any()) == (want["has_padding"])
        # pos: the same fp32 divisions and the precise sinf / cosf torch's kernels call
        assert torch.equal(got["pos_flatten"], want["pos_flatten"]), \
            f"pos differs for {sizes}: max {(got['pos_flatten'] - want['pos_flatten']).abs().max().item():.3g}"
        lvl_embed = torch.cat([lvl[i].view(1, 1, -1).expand(1, h * w, -1) for i, (h, w) in enumerate(shapes)], 1)
        assert torch.equal(got["pos_lvl"], (want["pos_flatten"] + lvl_embed).to(dtype)), "pos + level embedding differs"
        pad = transformer.padded_geometry(shapes, DEV)
        for k in ("spatial_shapes", "level_start_index", "level_ids"):
            assert torch.equal(pad[k], want[k]), k


def test_sizes_are_clamped_to_the_pad(transformer):
    """Sizes outside [1, Hp] x [1, Wp] change values only: they give the geometry of the clamped size."""
    shapes = _shapes(64, 64, (4, 8, 16, 32, 64))
    pe = PositionEmbeddingSine(num_pos_feats=E // 2, normalize=True, offset=-0.5)
    lvl = torch.zeros(len(shapes), E, device=DEV)
    run = lambda s: ops.pad_geometry(torch.tensor(s, dtype=torch.int32, device=DEV), (64, 64), shapes, pe.dim_t(DEV), lvl,  # noqa: E731
                                     torch.float16, pe.offset, pe.eps, pe.scale)
    got, want = run([[5000, 0], [-3, 70]]), run([[64, 1], [1, 64]])
    for k in want:
        if want[k] is not None:
            assert torch.equal(got[k], want[k]), k


def test_model_geometry_equals_the_torch_geometry(transformer, built):
    """DeformableDETRSegmVL._geometry on CUDA (padded part + ops.pad_geometry) against the torch restatement it kept for other
    devices, including has_padding at sizes where some levels have no padded row although the image is smaller than the pad."""
    model = build_model(configs.MINI).to(DEV)
    for sizes in ([(64, 64)], [(60, 64)], [(61, 64)], [(57, 63), (64, 64)], [(1, 64), (64, 1), (33, 17)]):
        geo = model._geometry((len(sizes), 3, 64, 64), sizes)
        want = _torch_geometry(model.transformer, model.position_embedding, 64, 64, geo["shapes"], sizes)
        assert geo["has_padding"] == want["has_padding"], sizes
        for k in ("mask_flatten", "valid_ratios", "reference_points", "output_proposals", "proposal_invalid", "level_ids"):
            assert torch.equal(geo[k], want[k]), (k, sizes)


def _call(sizes=1, B=1, Hp=64, Wp=64, level_hw=((16, 16),), L=None, dim_t=1, lvl=1, E=4, dtype=_lib.APE_DTYPE_F16, outs=True):
    """ape_pad_geometry through ctypes with valid buffers unless told otherwise (0 = a null pointer)."""
    t = lambda n, dt=torch.float32: torch.zeros(max(n, 1), dtype=dt, device=DEV)  # noqa: E731
    keep = [t(2 * max(B, 1), torch.int32), t(64), t(64), t(1 << 14, torch.uint8), t(1 << 14), t(1 << 14), t(64), t(1 << 14),
            t(1 << 14), t(1 << 14, torch.uint8)]
    p = [k.data_ptr() for k in keep]
    hw = (ctypes.c_int * (2 * len(level_hw)))(*[v for sh in level_hw for v in sh])
    rc = _lib.lib.ape_pad_geometry(p[0] if sizes else None, B, Hp, Wp, hw, len(level_hw) if L is None else L, p[1] if dim_t else None,
                                   p[2] if lvl else None, E, -0.5, 1e-6, 6.28, 1, p[3] if outs else None, p[4], dtype, None, p[6],
                                   p[7], p[8], p[9], _lib.current_stream_ptr())
    torch.cuda.synchronize()
    return rc, _lib.lib.ape_last_error().decode()


def test_invalid_arguments_are_rejected(built):
    assert _call()[0] == 0
    assert _call(B=0) == (-1, "pad_geometry: B=0")
    assert _call(L=0)[0] == -1 and _call(L=9)[0] == -1
    assert _call(level_hw=((65, 16),))[0] == -1 and "does not fit" in _call(level_hw=((65, 16),))[1]
    assert _call(level_hw=((16, 0),))[0] == -1
    assert _call(E=3)[0] == -1 and "even" in _call(E=3)[1]
    assert _call(dtype=_lib.APE_DTYPE_E4M3)[0] == -2
    for kw in ({"sizes": 0}, {"dim_t": 0}, {"lvl": 0}, {"outs": 0}):
        assert _call(**kw)[0] == -3, kw
    lvl = torch.zeros(5, E, device=DEV)
    dim_t = PositionEmbeddingSine(num_pos_feats=E // 2).dim_t(DEV)
    with pytest.raises(RuntimeError, match="int32"):
        ops.pad_geometry(torch.ones(1, 2, device=DEV), (64, 64), [(16, 16)], dim_t, lvl, torch.float16)
    with pytest.raises(RuntimeError, match="E/2"):
        ops.pad_geometry(torch.ones(1, 2, dtype=torch.int32, device=DEV), (64, 64), [(16, 16)], dim_t[:5], lvl, torch.float16)
    with pytest.raises(RuntimeError, match="does not fit"):
        ops.pad_geometry(torch.ones(1, 2, dtype=torch.int32, device=DEV), (64, 64), [(128, 16)], dim_t, lvl, torch.float16)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_zero_masked_rows_equals_masked_fill(built, dtype):
    """ops.zero_masked_rows_, which the deformable attention uses for the padding mask that a graph always passes: the masked_fill
    it replaces, on a row pitch wider than the rows, for all-false, all-true and random masks."""
    g = torch.Generator().manual_seed(0)
    base = torch.randn(3, 500, 264, generator=g).to(DEV, dtype)
    for mask in (torch.zeros(3, 500, dtype=torch.bool), torch.ones(3, 500, dtype=torch.bool), torch.rand(3, 500, generator=g) < 0.3):
        mask = mask.to(DEV)
        x = base.clone()[..., :256]
        want = x.masked_fill(mask[..., None], 0.0)
        got = ops.zero_masked_rows_(x, mask)
        assert got.data_ptr() == x.data_ptr() and torch.equal(got, want)
        assert torch.equal(base[..., 256:], x.as_strided(base.shape, base.stride())[..., 256:]), "wrote past the rows"
