"""CPU: pins the oracle's port of the detection forward (oracle/ape_forward.py) against golden
tensors produced by the REFERENCE's own files run under oracle/refshim.py on the MINI spec
(tests/golden/gen_model_golden.py).  Weights are a pure function of (name, shape) (oracle/synth.py),
so only outputs are stored."""
import pytest
import torch

from conftest import load_golden
from ape_b200 import configs
from oracle import ape_forward as AF
from oracle import synth

CASES = {
    "single": ([(48, 64, 96, 128)], None),
    "batch2": ([(64, 64, 64, 64), (40, 56, 80, 112)], None),
    "phrase": ([(64, 48, 64, 48)], 3),
    "expression": ([(64, 56, 128, 112)], 2),  # two referring expressions, one box kept per image
}


def mini_state_dict():
    """Reference-named state_dict for the MINI spec, shapes taken from the golden generator's
    model; here rebuilt from the engine's own module tree (same names by construction)."""
    from ape_b200.modeling import build_model

    m = build_model(configs.MINI)
    synth.fill_state_dict(m)
    return {k: v.clone() for k, v in m.state_dict().items()}


@pytest.fixture(scope="module")
def sd():
    return mini_state_dict()


@pytest.mark.parametrize("case", sorted(CASES))
def test_port_matches_reference_golden(case, sd):
    spec = configs.MINI
    sizes, n_phrase = CASES[case]
    g = load_golden(f"model_mini_{case}.npz")
    images = [synth.image(h, w, seed=i) for i, (h, w, _, _) in enumerate(sizes)]
    outs = [(oh, ow) for (_, _, oh, ow) in sizes]
    n_text = n_phrase if n_phrase else spec["num_classes"]
    text = synth.text_features(8192, spec["lang_dim"])[:n_text]
    res, taps = AF.forward(images, outs, text, sd, spec, phrase=bool(n_phrase), topk=1 if case == "expression" else None)
    tol = dict(rtol=2e-4, atol=2e-4)
    for k in ("p2", "p3", "p4", "p5", "p6"):
        torch.testing.assert_close(taps[f"backbone.{k}"][:, ::4], g[f"backbone.{k}"], **tol)
    for i in range(5):
        torch.testing.assert_close(taps[f"neck.{i}"][:, ::8], g[f"neck.{i}"], **tol)
    for i in range(spec["enc_layers"]):
        torch.testing.assert_close(taps[f"vlf{i}.v"][:, ::8], g[f"vlf{i}.v"], **tol)
        torch.testing.assert_close(taps[f"vlf{i}.l"], g[f"vlf{i}.l"], **tol)
    torch.testing.assert_close(taps["memory"][:, ::4], g["memory"], **tol)
    # bit-exact requirement: selected proposal indices (deformable_transformer_vl.py:569-625).  Entries that are
    # padded / invalid proposals come from ties among zero scores in the reference's torch.topk (implementation-
    # defined order; the oracle fixes "lowest index first"), so exact equality is required on the valid ones.
    valid = (g["init_reference"] < 1).all(-1)
    assert torch.equal(taps["topk_proposals"][valid], g["topk_proposals"][valid])
    assert taps["topk_proposals"].shape == g["topk_proposals"].shape
    torch.testing.assert_close(taps["init_reference"], g["init_reference"], **tol)
    torch.testing.assert_close(taps["inter_states"], g["inter_states"], rtol=1e-3, atol=1e-3)
    torch.testing.assert_close(taps["inter_references"], g["inter_references"], **tol)
    for b, r in enumerate(res):
        assert torch.equal(r["classes"], g[f"det{b}.classes"])  # bit-exact: kept (query, class) pairs
        torch.testing.assert_close(r["scores"], g[f"det{b}.scores"], rtol=1e-3, atol=1e-5)
        torch.testing.assert_close(r["boxes"], g[f"det{b}.boxes"], rtol=1e-3, atol=1e-2)


def test_port_masks_and_semantic_match_reference_golden(sd):
    """SURVEY.md 8(a) rows a17 / a19 / a20 of the port against the reference's own outputs (model_mini_masks.npz)."""
    import numpy as np

    spec = configs.MINI
    g = load_golden("model_mini_masks.npz")
    text = synth.text_features(8192, spec["lang_dim"])[: spec["num_classes"]]
    res, taps = AF.forward([synth.image(48, 64, seed=0)], [(96, 128)], text, sd, spec, masks_on=True, semantic_on=True)
    torch.testing.assert_close(taps["mask_features"][:, ::8], g["mask_features"], rtol=2e-4, atol=2e-4)
    torch.testing.assert_close(taps["pred_masks"], g["pred_masks"], rtol=1e-3, atol=1e-3)
    r = res[0]
    assert torch.equal(r["classes"], g["det0.classes"])
    want = torch.from_numpy(np.unpackbits(g["det0.masks_packed"].numpy(), axis=-1)).bool()[..., : int(g["det0.masks_shape"][2])]
    assert r["masks"].shape == want.shape
    assert (r["masks"] != want).float().mean().item() < 1e-3
    torch.testing.assert_close(r["sem_seg"], g["sem_seg"], rtol=1e-3, atol=1e-3)


def test_port_matches_reference_golden_ape_ti():
    """BASELINE.json configs[0]: APE-Ti (vit_eva02.py backbone: fused qkv, packed SwiGLU, 14x14 windows over a padded
    grid), one 768 x 1024 image padded to 1024^2, 80 names, on the CPU — the oracle port against the reference's own
    output at the real architecture and size (tests/golden/gen_model_golden.py ti; about half a minute of host time)."""
    from ape_b200.modeling import build_model

    spec = configs.APE_TI
    g = load_golden("model_ti_1024.npz")
    m = build_model(spec, num_text=80)
    synth.fill_state_dict(m)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    text = synth.text_features(8192, spec["lang_dim"])[:80]
    res, taps = AF.forward([synth.image(768, 1024, seed=11)], [(384, 512)], text, sd, spec)
    tol = dict(rtol=1e-5, atol=1e-5)  # measured: 0.0 through the encoder (same ATen kernels in the same order)
    for k in ("p2", "p3", "p4", "p5", "p6"):
        torch.testing.assert_close(taps[f"backbone.{k}"][:, ::16, ::4, ::4], g[f"backbone.{k}"], **tol)
    torch.testing.assert_close(taps["memory"][:, ::128, ::4], g["memory"], **tol)
    torch.testing.assert_close(taps["enc_outputs_class"][:, ::16], g["enc_outputs_class"], **tol)
    # selected proposals: exact on the valid ones (ties among zero-score padding entries of the 16x16 level are
    # implementation-defined in the reference's torch.topk, see test_port_matches_reference_golden)
    valid = (g["init_reference"] < 1).all(-1) & torch.isfinite(g["init_reference"]).all(-1)
    assert valid.sum() >= 890
    assert torch.equal(taps["topk_proposals"][valid], g["topk_proposals"][valid])  # bit-exact index requirement
    same = (taps["topk_proposals"] == g["topk_proposals"])[0]
    torch.testing.assert_close(taps["inter_states"][-1][:, ::3][:, same[::3]], g["inter_states_last"][:, same[::3]],
                               rtol=5e-3, atol=5e-3)
    r = res[0]
    k = min(50, len(r["scores"]), len(g["det0.scores"]))
    torch.testing.assert_close(r["scores"][:k], g["det0.scores"][:k], rtol=1e-4, atol=1e-5)
    assert (r["classes"][:k] == g["det0.classes"][:k]).float().mean().item() > 0.9
