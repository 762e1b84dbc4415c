"""CPU: the tap rule of the region-prompt kernel (ape_region_prompt, csrc/geometry.cu), restated in numpy, equals the torch
restatement of the reference (deformable_detr_segm_vl.py:394-412: prompts padded like the images, an all-zero batch set to 255,
F.interpolate(mode="bilinear") to every level, `.to(bool)`, flattened as the features) on the host.

The rule: token d of a level of n_out rows reads source rows t0 = trunc(src) and, when lambda = src - t0 is nonzero and
t0 < n_in - 1, t0 + 1, with src = max(fma(d + 0.5, (float)n_in / n_out, -0.5), 0) in fp32; columns alike.  A token is inside the
region when one of its taps is set, or when the whole batch is empty.  Swept over the padded shapes and levels of MINI, APE-Ti and
APE-L_D at 1024^2, a non-square pad, odd ratios (64 -> 13, 1024 -> 24, and 33 -> 13 / 65 -> 25, where the fused multiply-add
lands on an integer the unfused one misses), uint8 0/255, float 0/1 and random non-negative float prompts, single pixels,
one-pixel lines and rectangles touching the image edge and the padding.  Where the fused and the unfused source index read
different rows (or columns), the sweep adds prompts whose edge falls on each such row, so the two rules give different region
flags on it and the sweep pins the fused one.  The GPU tests compare the kernel with the same sweep."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from ape_b200 import configs

STRIDES = (4, 8, 16, 32, 64)


def levels(H, W):
    """The engine's level shapes of a padded (H, W) batch (DeformableDETRSegmVL._level_shapes)."""
    return [(-(-H // s), -(-W // s)) for s in STRIDES]


# (padded shape, level shapes, image sizes inside the pad)
GEOMETRIES = {
    "mini": ((64, 64), levels(64, 64), [(64, 64), (40, 56)]),
    "ape_ti": ((configs.APE_TI["backbone"]["square_pad"],) * 2, configs.level_shapes(configs.APE_TI), [(1024, 768)]),
    "ape_l_d": ((configs.APE_L_D["backbone"]["square_pad"],) * 2, configs.level_shapes(configs.APE_L_D), [(768, 1024)]),
    "nonsquare": ((800, 1344), levels(800, 1344), [(800, 1201), (613, 1344)]),
    "odd_64_13": ((64, 64), [(13, 13), (13, 29), (5, 7)], [(64, 64), (50, 37)]),
    "odd_1024_24": ((1024, 1024), [(24, 24), (24, 100)], [(1024, 1024)]),
    "fma_edge": ((33, 65), [(13, 25), (29, 47)], [(33, 65), (17, 30)]),
}


def taps(n_in, n_out, fused=True):
    """(t0, t1) int64 [n_out]: the two source indices of each destination index; t1 == t0 when the second tap has no weight.
    The fused multiply-add is exact in float64 (a 24-bit scale times a d + 0.5 of at most 15 bits) and rounded once; fused=False
    rounds the product and the difference separately (the rule the kernel must not follow)."""
    scale = np.float32(n_in) / np.float32(n_out)
    d = np.arange(n_out, dtype=np.float32) + np.float32(0.5)
    if fused:
        src = (np.float64(scale) * d.astype(np.float64) - 0.5).astype(np.float32)
    else:
        src = scale * d - np.float32(0.5)
    src = np.where(src < 0, np.float32(0), src)
    t0 = np.minimum(src.astype(np.int64), n_in - 1)
    lam = src - t0.astype(np.float32)
    t1 = np.where((lam != 0) & (t0 < n_in - 1), t0 + 1, t0)
    return t0, t1


def split_taps(n_in, n_out):
    """Source indices read by the fused rule and not the unfused one, or the other way round, for some destination index."""
    f0, f1 = taps(n_in, n_out)
    u0, u1 = taps(n_in, n_out, fused=False)
    out = set()
    for d in range(n_out):
        out |= {int(f0[d]), int(f1[d])} ^ {int(u0[d]), int(u1[d])}
    return sorted(out)


def region_np(nonzero, shapes, fused=True):
    """nonzero: bool [B, Hp, Wp].  The kernel's region flags bool [B, S] (fused=False: with the unfused source index)."""
    B, Hp, Wp = nonzero.shape
    if not nonzero.any():
        return np.ones((B, sum(h * w for h, w in shapes)), dtype=bool)
    out = []
    for h, w in shapes:
        r0, r1 = taps(Hp, h, fused)
        c0, c1 = taps(Wp, w, fused)
        m = np.zeros((B, h, w), dtype=bool)
        for r in (r0, r1):
            for c in (c0, c1):
                m |= nonzero[:, r[:, None], c[None, :]]
        out.append(m.reshape(B, -1))
    return np.concatenate(out, 1)


def region_torch(prompts, padded, shapes, device="cpu"):
    """The torch restatement of the reference: prompts padded into a zero fp32 batch, 255 everywhere when its sum is 0, bilinear
    to every level, `.to(bool)`, flattened level after level."""
    mp = torch.zeros((len(prompts),) + tuple(padded), dtype=torch.float32, device=device)
    for i, m in enumerate(prompts):
        mp[i, : m.shape[-2], : m.shape[-1]] = m.to(device=device, dtype=torch.float32)
    if mp.sum() == 0:
        mp[...] = 255
    return torch.cat([F.interpolate(mp[None], size=sh, mode="bilinear").to(torch.bool).squeeze(0).flatten(1) for sh in shapes], 1)


def padded_nonzero(prompts, padded, device="cpu"):
    """The engine's map: 1 where the prompt, cast to fp32, is nonzero; 0 elsewhere and in the padding."""
    out = torch.zeros((len(prompts),) + tuple(padded), dtype=torch.bool, device=device)
    for i, m in enumerate(prompts):
        out[i, : m.shape[-2], : m.shape[-1]] = m.to(device=device, dtype=torch.float32) != 0
    return out


def shapes_of(h, w, rng):
    """Binary prompts of an h x w image: single pixels (corners, centre, random), one-pixel lines, rectangles touching the image
    edge (and so the padding beyond it), the whole image."""
    out = []
    for (y, x) in [(0, 0), (h - 1, w - 1), (0, w - 1), (h - 1, 0), (h // 2, w // 2),
                   (int(rng.integers(h)), int(rng.integers(w)))]:
        m = np.zeros((h, w), dtype=bool)
        m[y, x] = True
        out.append(("pixel", m))
    for k in (0, h // 3, h - 1):
        m = np.zeros((h, w), dtype=bool)
        m[k, :] = True
        out.append(("row", m))
    for k in (0, w // 3, w - 1):
        m = np.zeros((h, w), dtype=bool)
        m[:, k] = True
        out.append(("column", m))
    for (y0, y1, x0, x1) in [(h // 2, h, w // 2, w), (0, max(1, h // 5), w // 3, w), (h // 4, h // 4 + 3, 0, 3),
                             (h // 3, 2 * h // 3, w // 3, 2 * w // 3)]:
        m = np.zeros((h, w), dtype=bool)
        m[y0:y1, x0:x1] = True
        out.append(("rect", m))
    out.append(("full", np.ones((h, w), dtype=bool)))
    return out


def split_edges(padded, shapes, h, w):
    """Prompts of an h x w image whose edge falls on a row or column where the fused and unfused taps differ (split_taps): that
    line alone, everything up to it and everything from it on."""
    out = {}
    for lh, lw in shapes:
        for axis, (n_in, n_out, n_img) in enumerate(((padded[0], lh, h), (padded[1], lw, w))):
            for k in split_taps(n_in, n_out):
                if k >= n_img:
                    continue
                for name, sl in (("line", slice(k, k + 1)), ("upto", slice(0, k + 1)), ("from", slice(k, n_img))):
                    m = np.zeros((h, w), dtype=bool)
                    if axis == 0:
                        m[sl, :] = True
                    else:
                        m[:, sl] = True
                    out[f"split-{'row' if axis == 0 else 'column'}{k}-{name}"] = m
    return list(out.items())


def as_prompt(m, kind, rng):
    """A binary shape as the prompt dtype a caller passes: uint8 0/255, float 0/1, random non-negative floats on the shape."""
    if kind == "u8":
        return torch.from_numpy(m.astype(np.uint8) * 255)
    if kind == "f01":
        return torch.from_numpy(m.astype(np.float32))
    v = rng.uniform(1e-3, 300.0, size=m.shape).astype(np.float32)
    v[rng.random(m.shape) < 0.5] = np.float32(1e-30)
    return torch.from_numpy(np.where(m, v, np.float32(0)))


def cases(geometry, seed=0):
    """(name, prompts) of one geometry: every shape and dtype per image size, one image per batch; then a batch of two with one
    empty prompt, and an all-empty batch."""
    padded, shapes, sizes = GEOMETRIES[geometry]
    rng = np.random.default_rng(seed)
    out = []
    for h, w in sizes:
        for name, m in shapes_of(h, w, rng) + split_edges(padded, shapes, h, w):
            for kind in ("u8", "f01", "rand"):
                out.append((f"{h}x{w}-{name}-{kind}", [as_prompt(m, kind, rng)]))
    h, w = sizes[-1]
    one = shapes_of(h, w, rng)[-2][1]
    out.append(("one-empty", [as_prompt(one, "u8", rng), torch.zeros((h, w), dtype=torch.uint8)]))
    out.append(("all-empty", [torch.zeros((h, w), dtype=torch.uint8), torch.zeros(sizes[0], dtype=torch.float32)]))
    return out


@pytest.mark.parametrize("geometry", sorted(GEOMETRIES))
def test_tap_rule_matches_bilinear_to_bool(geometry):
    padded, shapes, _ = GEOMETRIES[geometry]
    n = 0
    for name, prompts in cases(geometry):
        want = region_torch(prompts, padded, shapes).numpy()
        got = region_np(padded_nonzero(prompts, padded).numpy(), shapes)
        assert got.shape == want.shape
        bad = np.argwhere(got != want)
        assert len(bad) == 0, f"{geometry} {name}: {len(bad)} tokens differ, first {bad[:3].tolist()}"
        n += int(want.sum())
    assert n > 0


def test_empty_batch_rule():
    """Only an all-empty batch means "everywhere": one empty image beside a prompted one keeps no token."""
    padded, shapes, _ = GEOMETRIES["mini"]
    c = dict(cases("mini"))
    one = region_np(padded_nonzero(c["one-empty"], padded).numpy(), shapes)
    assert one[0].any() and not one[0].all() and not one[1].any()
    assert region_np(padded_nonzero(c["all-empty"], padded).numpy(), shapes).all()


def test_sweep_tells_fused_from_unfused():
    """Every level of the fma_edge geometry has cases whose region flags differ between the fused and the unfused rule, on rows
    and on columns, so a kernel with the unfused source index fails the sweep.  The other geometries have no such row."""
    padded, shapes, _ = GEOMETRIES["fma_edge"]
    starts = np.cumsum([0] + [h * w for h, w in shapes])
    hit = set()
    for name, prompts in cases("fma_edge"):
        nz = padded_nonzero(prompts, padded).numpy()
        diff = region_np(nz, shapes) != region_np(nz, shapes, fused=False)
        for l in range(len(shapes)):
            if diff[:, starts[l]:starts[l + 1]].any():
                hit.add((l, "row" if "-split-row" in name else "column" if "-split-column" in name else "other"))
    assert hit >= {(l, a) for l in range(len(shapes)) for a in ("row", "column")}, hit
    for g in GEOMETRIES:
        if g != "fma_edge":
            padded, shapes, _ = GEOMETRIES[g]
            assert not any(split_taps(padded[0], h) or split_taps(padded[1], w) for h, w in shapes), g


def test_fma_edge_is_exercised():
    """33 -> 13, row 6: the fused source index is 15.999999 (taps 15 and 16), the unfused one 16.0 (tap 16 alone); a prompt on
    row 15 alone tells the two apart, and the bilinear reference agrees with the fused rule."""
    t0, t1 = taps(33, 13)
    assert (t0[6], t1[6]) == (15, 16)
    m = torch.zeros((33, 65))
    m[15, :] = 1
    got = region_np(padded_nonzero([m], (33, 65)).numpy(), [(13, 25)]).reshape(13, 25)
    want = region_torch([m], (33, 65), [(13, 25)]).numpy().reshape(13, 25)
    assert got[6].all() and np.array_equal(got, want)


def test_bad_arguments_are_reported(built):
    """The C entry point checks the batch and level count before any launch (no device needed).  The calls run on a thread of
    their own: the error text is thread-local, so this thread's stays as it was."""
    import ctypes
    import threading

    from ape_b200 import _lib

    hw = (ctypes.c_int * 2)(16, 16)
    seen = []

    def run():
        for B, L in ((0, 1), (65536, 1), (1, 0)):
            rc = _lib.lib.ape_region_prompt(None, B, 64, 64, hw, L, *([None] * 7))
            seen.append((rc, _lib.lib.ape_last_error()))

    t = threading.Thread(target=run)
    t.start()
    t.join()
    assert [rc for rc, _ in seen] == [-1, -1, -1]
    assert b"B=0" in seen[0][1] and b"B=65536" in seen[1][1] and b"L=0" in seen[2][1]
