"""CPU: the row layout of the text tower's length-packed mode (ape_b200.modeling.text.pack_layout): every prompt sits in
exactly one tile of 128 rows, contiguous and in input order; `pos`, `seg_start`, `eot_row`, `src` and `rows` agree with one
another; the layout is a function of the lengths alone."""
import numpy as np
import pytest

CTX, TILE = 77, 128


def _check(lengths, lay):
    lens = np.asarray(lengths)
    N, M = len(lens), lay["tiles"] * TILE
    for k in ("src", "pos", "seg_start"):
        assert lay[k].shape == (M,) and lay[k].dtype == np.int32
    assert lay["eot_row"].shape == (N,) and lay["eot_row"].dtype == np.int64
    real = lay["pos"] >= 0
    assert real.sum() == lens.sum() == len(lay["rows"])
    # walk the rows: each prompt once, contiguous, in input order, never across a tile boundary
    r = np.flatnonzero(real)
    prompt, p = lay["src"][r] // CTX, lay["src"][r] % CTX
    assert np.array_equal(p, lay["pos"][r])
    starts = np.flatnonzero(p == 0)
    assert np.array_equal(prompt[starts], np.arange(N))                    # every prompt, once, in order
    assert np.array_equal(np.diff(np.append(starts, len(r))), lens)        # ... with all of its tokens
    first, last = r[starts], r[np.append(starts[1:], len(r)) - 1]
    assert np.array_equal(last - first, lens - 1)                          # contiguous rows
    assert np.array_equal(first // TILE, last // TILE)                     # inside one tile
    assert np.array_equal(lay["eot_row"], last)
    assert np.array_equal(lay["seg_start"][r], np.repeat(first % TILE, lens))
    pad = np.flatnonzero(~real)
    assert np.array_equal(lay["seg_start"][pad], pad % TILE) and not lay["src"][pad].any()
    # tail rows only: inside a tile no pad row precedes a real one
    for t in range(lay["tiles"]):
        k = real[t * TILE:(t + 1) * TILE]
        assert k[0] and not np.any(~k[:-1] & k[1:])
    assert np.array_equal(lay["rows"], r) and np.array_equal(lay["src"][lay["rows"]], np.repeat(np.arange(N) * CTX, lens) + p)
    # next-fit: a prompt opens a tile only when it did not fit behind its predecessor
    for i in np.flatnonzero(first % TILE == 0)[1:]:
        assert last[i - 1] % TILE + 1 + lens[i] > TILE


@pytest.mark.parametrize("n", [1, 2, 17, 300, 1203, 5000])
def test_random_length_sets(built, n):
    from ape_b200.modeling.text import pack_layout

    rng = np.random.default_rng(n)
    for hi in (8, 16, 77):
        lengths = rng.integers(2, hi + 1, size=n).tolist()
        lay = pack_layout(lengths, CTX)
        _check(lengths, lay)
        again = pack_layout(list(lengths), CTX)
        assert all(np.array_equal(lay[k], again[k]) for k in lay)          # deterministic


def test_edge_cases(built):
    from ape_b200.modeling.text import pack_layout

    lay = pack_layout([5], CTX)                                            # N = 1
    _check([5], lay)
    assert lay["tiles"] == 1 and lay["eot_row"].tolist() == [4]
    exact = [64, 32, 16, 8, 8]                                             # sums to exactly 128: one full tile, no pad row
    lay = pack_layout(exact + [3], CTX)
    _check(exact + [3], lay)
    assert lay["tiles"] == 2 and (lay["pos"][:128] >= 0).all() and lay["eot_row"][-1] == 130
    lay = pack_layout([77] * 9, CTX)                                       # one 77-token prompt per tile
    _check([77] * 9, lay)
    assert lay["tiles"] == 9 and lay["eot_row"].tolist() == [128 * i + 76 for i in range(9)]
    lay = pack_layout([77, 51, 52], CTX)                                   # 77 + 51 fill a tile, 52 does not fit behind them
    assert lay["tiles"] == 2 and lay["eot_row"].tolist() == [76, 127, 128 + 51]


def test_bad_lengths_are_rejected(built):
    from ape_b200.modeling.text import pack_layout

    for bad in ([], [0], [3, 78], [129]):
        with pytest.raises(ValueError, match="pack_layout"):
            pack_layout(bad, CTX)


def test_flag_is_off_by_default_and_reaches_the_tower(built):
    from ape_b200.modeling import EVA01CLIP, EVA02CLIP, TextTransformer

    cfg = dict(text_cfg=dict(context_length=77, vocab_size=100, width=64, heads=1, layers=1), embed_dim=32)
    assert TextTransformer.pack_prompts is False
    for cls, kw in ((EVA02CLIP, {}), (EVA01CLIP, dict(cache_dir=None))):
        clip = cls(**cfg, **kw)
        assert clip.pack_prompts is False and clip.net.text.pack_prompts is False
        clip = cls(pack_prompts=True, **cfg, **kw)
        assert clip.pack_prompts is True and clip.net.text.pack_prompts is True
        clip.pack_prompts = False
        assert clip.net.text.pack_prompts is False
