"""CPU: the oracle of ViT-g/14's SwiGLU feed-forward and of the query / key / value facets (oracle/vit_swiglu_facets.py)
against the live reference's goldens (tests/golden/vit_facets_small.npz, vit_g_small.npz; oracle/make_golden_vit_models.py)
and the SwiGLU block against ``transformers``' Dinov2Layer(use_swiglu_ffn=True); the C ABI additions against the header;
the host-side w12 interleave and facet names of dino_tracker_b200/vit.py."""
import os
import re

import numpy as np
import pytest
import torch

from oracle import synth
from oracle import vit_swiglu_facets as ovf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def test_facets_oracle_matches_reference_golden():
    """queries / keys / values at layers 0 and 1 through the live reference's qkv hook (dinov2_vits14 dims)."""
    from oracle import make_golden_vit_models as mgv
    cfg = mgv.FACETS_CASE
    g = dict(np.load(os.path.join(GOLDEN_DIR, "vit_facets_small.npz")))
    sd, video = mgv.case_state_dict(cfg, swiglu=False), mgv.case_video(cfg)
    for layer in cfg["layers"]:
        for facet in ("queries", "keys", "values"):
            ref = g[f"{facet}_{layer}"]
            mine = ovf.dino_features_video(video, sd, cfg["heads"], layer, facet=facet).numpy()
            assert mine.shape == ref.shape == (cfg["T"], cfg["dim"], 5, 7)
            assert np.abs(mine - ref).max() <= 1e-5 * np.abs(ref).max(), (facet, layer)


def test_vitg_oracle_matches_reference_golden():
    """dinov2_vitg14 (C = 1536 from the name, 24 heads), 2 SwiGLU blocks, layer 1: tokens and keys, on the stored
    seeded sample of entries and the float64 sums of the whole output."""
    from oracle import make_golden_vit_models as mgv
    cfg = mgv.G_CASE
    g = dict(np.load(os.path.join(GOLDEN_DIR, "vit_g_small.npz")))
    sd, video = mgv.case_state_dict(cfg, swiglu=True), mgv.case_video(cfg)
    for facet in ("tokens", "keys"):
        mine = ovf.dino_features_video(video, sd, cfg["heads"], cfg["layer"], facet=facet).numpy()
        assert mine.shape == tuple(g[f"{facet}_shape"]) == (1, 1536, 13, 17)
        idx = g[f"{facet}_idx"]
        assert np.array_equal(idx, mgv.sample_index(cfg, mine.size))
        scale = float(g[f"{facet}_absmax"])
        assert np.abs(mine.reshape(-1)[idx] - g[f"{facet}_vals"]).max() <= 1e-5 * scale, facet
        m64 = mine.astype(np.float64)
        s, sa = g[f"{facet}_sums"]
        assert abs(m64.sum() - s) <= 1e-5 * sa and abs(np.abs(m64).sum() - sa) <= 1e-6 * sa, facet
        assert abs(np.abs(mine).max() - scale) <= 1e-5 * scale


@pytest.mark.parametrize("dim,heads,tokens", [(64, 1, 50), (128, 2, 222), (192, 3, 97)])
def test_swiglu_block_matches_transformers_dinov2(dim, heads, tokens):
    pytest.importorskip("transformers")
    from oracle.make_golden_vit_models import hf_dinov2_swiglu_layer
    g = torch.Generator().manual_seed(7)
    depth = 2
    sd = ovf.random_state_dict(depth, dim, g, n_pos=4, std=0.08, swiglu=True)
    for i in range(depth):
        sd[f"blocks.{i}.ls1.gamma"] = 0.5 + torch.rand(dim, generator=g)
        sd[f"blocks.{i}.ls2.gamma"] = 0.5 + torch.rand(dim, generator=g)
    assert sd["blocks.0.mlp.w3.weight"].shape == (dim, ovf.swiglu_hidden(dim))
    x = torch.randn(2, tokens, dim, generator=g)
    with torch.no_grad():
        ref, got = x, x
        for i in range(depth):
            out = hf_dinov2_swiglu_layer(dim, heads, sd, i)(ref)
            ref = out[0] if isinstance(out, (tuple, list)) else out
            got = ovf.block_forward(got, sd, i, heads)
            assert (got - ref).abs().max().item() <= 2e-5 * max(1.0, ref.abs().max().item()), i


def test_swiglu_hidden_width_rule():
    """The hub's SwiGLUFFNFused: 4096 for ViT-g/14; 344 at D = 128 (2 Hd = 688 = 2 x 256 + 176: an N tail)."""
    assert ovf.swiglu_hidden(1536) == 4096 and ovf.swiglu_hidden(128) == 344
    assert ovf.CONFIGS["dinov2_vitg14"] == (40, 1536, 24)


def test_unknown_facet_raises():
    from dino_tracker_b200.vit import get_dino_features_video
    with pytest.raises(ValueError, match="facet attn not supported"):
        get_dino_features_video(torch.zeros(1, 3, 42, 56), facet="attn", state_dict={})
    with pytest.raises(ValueError, match="not supported"):
        ovf.vit_tokens(synth.random_video(1, 42, 56, seed=1), {}, 1, 0, facet="attn")


def test_w12_interleave_layout():
    """Rows 4q .. 4q+3 of the interleaved w12 (and bias) = x1[2q], x1[2q+1], x2[2q], x2[2q+1]."""
    from dino_tracker_b200.vit import interleave_w12
    hd, D = 344, 16
    w = torch.randn(2 * hd, D)
    b = torch.randn(2 * hd)
    wi, bi = interleave_w12(w), interleave_w12(b)
    x1, x2 = w[:hd], w[hd:]
    for q in (0, 1, hd // 2 - 1):
        assert torch.equal(wi[4 * q:4 * q + 4], torch.stack((x1[2 * q], x1[2 * q + 1], x2[2 * q], x2[2 * q + 1])))
        assert torch.equal(bi[4 * q:4 * q + 4], torch.stack((b[2 * q], b[2 * q + 1], b[hd + 2 * q], b[hd + 2 * q + 1])))
    assert torch.equal(wi.sort(0).values, w.sort(0).values)


def test_vit_config_abi_matches_header():
    """dinotrk_vit_config's fields in header order (swiglu_hidden and facet appended) and DINOTRK_VIT_SWIGLU."""
    from dino_tracker_b200 import _lib
    src = open(os.path.join(ROOT, "include", "dinotrk.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    body = re.search(r"typedef struct dinotrk_vit_config \{(.*?)\} dinotrk_vit_config;", src, flags=re.S).group(1)
    fields = [n.strip() for decl in body.split(";") if decl.strip() for n in decl.strip().removeprefix("int ").split(",")]
    assert fields == [f[0] for f in _lib.VitConfig._fields_]
    assert fields[-2:] == ["swiglu_hidden", "facet"]
    assert re.search(r"#define DINOTRK_VIT_SWIGLU 6\b", src)
    cfg = _lib.VitConfig(24, 1024, 16, 15, 14, 7, 0, 1, 1)    # positional callers: the appended fields stay 0
    assert cfg.swiglu_hidden == 0 and cfg.facet == 0
