"""CPU: the DINO v1 oracle (oracle/vit_dino_v1.py, ViT-S/8 and ViT-B/8) against the live reference's golden
(tests/golden/vit_dino_v1_small.npz, oracle/make_golden_vit_dino_v1.py), which regenerates bit for bit where the
reference is present; the v1 block against ``transformers``' ViTLayer; the model names, patch sizes and the
LayerScale-free weight table of dino_tracker_b200/vit.py."""
import os

import numpy as np
import pytest
import torch

from oracle import ref_harness
from oracle import vit_dino_v1 as ov1

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "vit_dino_v1_small.npz")


@pytest.mark.parametrize("name", ["dino_vits8", "dino_vitb8"])
def test_v1_oracle_matches_reference_golden(name):
    """2 blocks at the real width, layer 1, one 36 x 50 frame: 5 x 7 tokens at patch 8, stride 7; tokens and keys."""
    from oracle import make_golden_vit_dino_v1 as mg
    g = dict(np.load(GOLDEN))
    sd, video = mg.case_state_dict(name), mg.case_video(name)
    _, dim, heads = ov1.CONFIGS[name]
    assert "blocks.0.ls1.gamma" not in sd and sd["pos_embed"].shape[1] == 1 + 28 * 28
    for facet in mg.FACETS:
        ref = g[f"{name}_{facet}"]
        mine = ov1.dino_features_video(video, sd, heads, mg.LAYER, facet=facet).numpy()
        assert mine.shape == ref.shape == (1, dim, 5, 7)
        assert np.abs(mine - ref).max() <= 1e-5 * np.abs(ref).max(), facet


@pytest.mark.skipif(not ref_harness.reference_available(), reason="the reference sources are not present")
def test_v1_golden_regenerates_bit_for_bit(tmp_path):
    pytest.importorskip("transformers")
    from oracle import make_golden_vit_dino_v1 as mg
    mg.main(out_dir=str(tmp_path))
    new, old = dict(np.load(tmp_path / "vit_dino_v1_small.npz")), dict(np.load(GOLDEN))
    assert sorted(new) == sorted(old)
    for k in old:
        assert new[k].dtype == old[k].dtype and new[k].tobytes() == old[k].tobytes(), k


@pytest.mark.parametrize("dim,heads,tokens", [(64, 1, 50), (128, 2, 222), (384, 6, 97)])
def test_v1_block_matches_transformers_vit_layer(dim, heads, tokens):
    pytest.importorskip("transformers")
    from oracle.make_golden_vit_dino_v1 import hf_vit_layer
    g = torch.Generator().manual_seed(11)
    depth = 2
    sd = ov1.random_state_dict(depth, dim, g, std=0.08)
    x = torch.randn(2, tokens, dim, generator=g)
    with torch.no_grad():
        ref, got = x, x
        for i in range(depth):
            out = hf_vit_layer(dim, heads, sd, i)(ref)
            ref = out[0] if isinstance(out, (tuple, list)) else out
            got = ov1.block_forward(got, sd, i, heads)
            assert (got - ref).abs().max().item() <= 2e-5 * max(1.0, ref.abs().max().item()), i


def test_model_names_and_patch_sizes():
    """The reference's get_patch_size (8 for names containing '8') and dims; the *16 names stay unknown."""
    from dino_tracker_b200 import vit
    assert vit.CONFIGS["dino_vits8"] == ov1.CONFIGS["dino_vits8"] == (12, 384, 6)
    assert vit.CONFIGS["dino_vitb8"] == ov1.CONFIGS["dino_vitb8"] == (12, 768, 12)
    assert [vit.patch_size(n) for n in ("dino_vits8", "dino_vitb8", "dinov2_vits14", "dinov2_vitg14")] == [8, 8, 14, 14]
    assert "dino_vits16" not in vit.CONFIGS and "dino_vitb16" not in vit.CONFIGS


def test_patch_mismatch_and_partial_layerscale_raise():
    """Checked before any device work: a patch that does not match the embedding's kernel, and LayerScale in some
    blocks only."""
    from dino_tracker_b200.vit import DinoV2Features
    sd = ov1.random_state_dict(2, 64, torch.Generator().manual_seed(1))
    with pytest.raises(ValueError, match="patch"):
        DinoV2Features(sd, heads=1, patch=14, device="cpu")
    sd["blocks.1.ls1.gamma"] = torch.ones(64)
    with pytest.raises(ValueError, match="LayerScale"):
        DinoV2Features(sd, heads=1, patch=8, device="cpu")


POS_CASES = [(197, 198), (198, 197), (198, 198), (476, 854), (36, 50)]   # 197 x 198: a 28 x 28 grid of a non-square frame


def test_pos_embed_rule_package_matches_v1_oracle():
    """The package's host-side interpolation, told whether the frame is square, and the v1 oracle's agree exactly; for a
    non-square frame with a 28 x 28 grid the table is resampled, for a square one it is returned as it is."""
    from dino_tracker_b200.vit import interpolate_pos_embed
    pos = torch.randn(1, 1 + 28 * 28, 64, generator=torch.Generator().manual_seed(3))
    for H, W in POS_CASES:
        n_h, n_w = 1 + (H - 8) // 7, 1 + (W - 8) // 7
        a = interpolate_pos_embed(pos, n_h, n_w, H == W)
        b = ov1.interpolate_pos_embed(pos, n_h, n_w, H, W)
        assert torch.equal(a, b), (H, W)
        assert (a is pos) == (H == W == 198)


@pytest.mark.skipif(not ref_harness.reference_available(), reason="the reference sources are not present")
def test_pos_embed_rule_matches_live_reference():
    """VitExtractor._fix_pos_enc(8, (7, 7)) from the live reference, called as dino's prepare_tokens calls it (w = H_img,
    h = W_img), against the package's interpolation."""
    from dino_tracker_b200.vit import interpolate_pos_embed
    ref_harness.install("cpu")
    from models.extractor import VitExtractor
    pos = torch.randn(1, 1 + 28 * 28, 64, generator=torch.Generator().manual_seed(4))
    fn = VitExtractor._fix_pos_enc(8, (7, 7))
    owner = type("M", (), {"pos_embed": pos})()
    for H, W in POS_CASES:
        n_h, n_w = 1 + (H - 8) // 7, 1 + (W - 8) // 7
        with torch.no_grad():
            ref = fn(owner, torch.zeros(1, 1 + n_h * n_w, 64), H, W)
        assert torch.equal(interpolate_pos_embed(pos, n_h, n_w, H == W), ref), (H, W)
