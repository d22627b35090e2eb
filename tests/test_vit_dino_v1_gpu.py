"""GPU tests: DINO v1 ViT-S/8 and ViT-B/8 on the CUDA feature stage.

Stage: the residual epilogue without LayerScale (dinotrk_vit_stage PROJ / FC2 with ls = NULL, the forward's own launch
code) against float64 from the same fp16 operands, at both v1 widths, on one and two 854 x 476 frames (67 x 121 tokens
at patch 14: the stage's row count only), in CTA-pair and single-CTA mode, with tests/test_vit_layers_gpu.py's bound
gamma(K) (sum |a w| + |bias|) + half an fp32 ulp.  Its result must equal the LayerScale epilogue's with ls = 1 bit for bit.

Forward (DinoV2Features.from_name, patch 8 from the name) against the oracle (oracle/vit_dino_v1.py, pinned to the live
reference's golden and to transformers' ViTLayer): tokens and keys, last of 2 and 4 blocks, two frames of 854 x 476
(67 x 121 tokens, as at patch 14) and 856 x 480 (68 x 122 tokens, against 67 x 121 at patch 14), fp32 oracle on the GPU
(TF32 off).  Bar: max |diff| <= 5e-3 max |ref| and every token's cosine > 0.9999, as for the DINOv2 backbones
(test_vit_swiglu_facets_gpu.py): fp16 operands, fp32 accumulation.  Also the golden through get_dino_features_video,
whose weights are larger (std 0.05: a gain of ~1.4 per linear layer at D = 768); there the bar is 1e-2 max |ref|
(measured on an H100: 2.1e-3 for ViT-S/8, 6.1e-3 for ViT-B/8 tokens) with the same cosine bar."""
import os

import numpy as np
import pytest
import torch

from oracle import synth
from oracle import vit_dino_v1 as ov1
from test_vit_layers_gpu import CANARY, DEV, N1, _bits_equal, _check, _gemm64, _gen, _nan, _randn, _stage, gamma, half_ulp32
from test_vit_swiglu_facets_gpu import _compare

pytestmark = pytest.mark.gpu
PROJ, FC2 = 3, 5                   # DINOTRK_VIT_* of include/dinotrk.h
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vit_dino_v1_small.npz")


@pytest.mark.parametrize("stage", [PROJ, FC2])
@pytest.mark.parametrize("name,frames", [(n, f) for n in ov1.CONFIGS for f in (1, 2)])
def test_residual_stage_without_layerscale(name, frames, stage):
    _, D, heads = ov1.CONFIGS[name]
    K = D if stage == PROJ else 4 * D
    rows = frames * N1
    g = _gen("v1 residual", stage, D, frames)
    a = (_randn(g, rows, K, std=0.5) if stage == PROJ else torch.nn.functional.gelu(_randn(g, rows, K))).half()
    w = _randn(g, D, K, std=K ** -0.5).half()
    bias = _randn(g, D, std=0.05)
    x0 = _nan(rows + CANARY, D)
    x0[:rows] = _randn(g, rows, D)
    out = {}
    for pair in (True, False):
        x = x0.clone()
        _stage(stage, D, heads, frames, a, w, bias, None, (x,), pair)
        out[pair] = x
    acc, aabs = _gemm64(a, w)
    ref, scale = acc + bias.double(), aabs + bias.double().abs()
    label = f"{'proj' if stage == PROJ else 'fc2'} no-LS {name} x{frames}"
    for pair, x in out.items():
        xn = x[:rows].double()
        r = half_ulp32(xn)
        _check(f"{label} {'pair' if pair else 'single'}", xn - x0[:rows].double(), ref, gamma(K) * scale + r, K, scale, r)
        assert x[rows:].isnan().all(), f"{label} wrote rows past B * N1"
    assert _bits_equal(out[True], out[False]), f"{label}: CTA-pair and single-CTA results differ"
    ones = x0.clone()
    _stage(stage, D, heads, frames, a, w, bias, torch.ones(D, device=DEV), (ones,), True)
    assert _bits_equal(out[True], ones), f"{label}: differs from the LayerScale epilogue with ls = 1"


@pytest.mark.parametrize("H,W,grid", [(476, 854, (67, 121)), (480, 856, (68, 122))])
@pytest.mark.parametrize("name,depth,facet", [("dino_vits8", 4, "tokens"), ("dino_vits8", 2, "keys"),
                                              ("dino_vitb8", 2, "tokens"), ("dino_vitb8", 3, "keys")])
def test_full_frame_against_gpu_oracle(name, depth, facet, H, W, grid):
    import oracle
    from dino_tracker_b200.vit import DinoV2Features
    oracle.use_exact_fp32()
    _, dim, heads = ov1.CONFIGS[name]
    sd = ov1.random_state_dict(depth, dim, torch.Generator().manual_seed(19), std=0.02)
    video = synth.random_video(2, H, W, seed=20)
    ex = DinoV2Features.from_name(name, sd, layer=depth - 1, device=DEV, facet=facet)
    assert ex.patch == 8 and not ex.layerscale
    got = ex.features_chw(video).cpu()
    del ex
    assert got.shape[-2:] == grid
    sd_dev = {k: v.to(DEV) for k, v in sd.items()}
    with torch.no_grad():
        ref = ov1.dino_features_video(video.to(DEV), sd_dev, heads, depth - 1, facet=facet).cpu()
    _compare(f"{name} {facet} last of {depth} blocks, {W} x {H}", got, ref)


@pytest.mark.parametrize("attention", ["fused", "fused-single-cta", "materialized"])
@pytest.mark.parametrize("facet", ["tokens", "queries", "keys", "values"])
def test_small_forward_every_facet_and_mode(facet, attention):
    """dim 128, 2 heads, 2 blocks, three 98 x 126 frames at patch 8 (13 x 17 tokens), layer 1."""
    from dino_tracker_b200.vit import DinoV2Features
    sd = ov1.random_state_dict(2, 128, torch.Generator().manual_seed(21), std=0.05)
    video = synth.random_video(3, 98, 126, seed=22)
    ref = ov1.dino_features_video(video, sd, 2, 1, facet=facet)
    ex = DinoV2Features(sd, heads=2, layer=1, patch=8, device=DEV, facet=facet,
                        attention="fused" if attention.startswith("fused") else attention, cta_pairs=attention == "fused")
    _compare(f"v1 {facet} [{attention}]", ex.features_chw(video).cpu(), ref)


@pytest.mark.parametrize("name", list(ov1.CONFIGS))
def test_matches_reference_golden(name):
    """The live reference's get_dino_features_video with the dino:main stand-in (vit_dino_v1_small.npz): tokens and
    keys, layer 1 of 2 blocks, through this package's get_dino_features_video."""
    from dino_tracker_b200.vit import get_dino_features_video
    from oracle import make_golden_vit_dino_v1 as mg
    g = dict(np.load(GOLDEN))
    sd, video = mg.case_state_dict(name), mg.case_video(name)
    for facet in mg.FACETS:
        got = get_dino_features_video(video, name, facet=facet, layer=mg.LAYER, state_dict=sd)
        ref = torch.from_numpy(g[f"{name}_{facet}"])
        err, scale = (got - ref).abs().max().item(), ref.abs().max().item()
        cos = torch.nn.functional.cosine_similarity(got.flatten(2), ref.flatten(2), dim=1).min().item()
        print(f"golden {name} {facet}: max |diff| = {err:.3e} (max |ref| = {scale:.3f}), min token cosine = {cos:.6f}")
        assert got.shape == ref.shape and err <= 1e-2 * scale and cos > 0.9999


def test_non_square_frame_with_square_grid():
    """197 x 198 pixels give a 28 x 28 grid at patch 8, stride 7 (the hub table's own size).  The reference sends a
    non-square frame through the bicubic interpolation (models/extractor.py:62) and returns the table as it is for a
    square one (198 x 198).  The interpolation runs where the weights are, as in the reference on its default device, so
    the oracle runs on the GPU too (PyTorch's CUDA bicubic upsampling between equal sizes copies; on the CPU it resamples,
    tests/test_vit_dino_v1_oracle_cpu.py)."""
    from dino_tracker_b200.vit import DinoV2Features
    sd = ov1.random_state_dict(2, 128, torch.Generator().manual_seed(23), std=0.05)
    sd_dev = {k: v.to(DEV) for k, v in sd.items()}
    for H, W in ((197, 198), (198, 198)):
        video = synth.random_video(2, H, W, seed=24)
        ex = DinoV2Features(sd, heads=2, layer=1, patch=8, device=DEV)
        got = ex.features_chw(video).cpu()
        assert got.shape[-2:] == (28, 28)
        with torch.no_grad():
            ref = ov1.dino_features_video(video.to(DEV), sd_dev, 2, 1).cpu()
        _compare(f"v1 tokens {W} x {H}", got, ref)


# sha256 of a DINOv2 ViT-L/14 forward (3 blocks, LayerScale 0.5 + noise, two 854 x 476 frames) as the build before the
# LayerScale-free epilogue wrote it, on an H100: the LayerScale kernels must keep producing these bytes
VITL_SHA256 = {
    ("fused", True, "tokens"): "fd374ae607b9afb4163324a7ec7ee8c5eab4678583a6984bee6bd77b0d959c3c",
    ("fused", True, "keys"): "2dc35354cce9f164aeafcb33117a74454e6599b5d9a3cc6154c304cbc1b71296",
    ("fused", False, "tokens"): "fd374ae607b9afb4163324a7ec7ee8c5eab4678583a6984bee6bd77b0d959c3c",
    ("fused", False, "keys"): "2dc35354cce9f164aeafcb33117a74454e6599b5d9a3cc6154c304cbc1b71296",
    ("materialized", False, "tokens"): "69759ca12837079d43d44875cdcebaadddfc5fe1d545358da6964e53224a9dee",
    ("materialized", False, "keys"): "657078e30904815c3285b8b61d4b764550e1f1d0c5f6fa5a6c9ea7b685bf33e4",
}


@pytest.mark.parametrize("attention,pairs,facet", sorted(VITL_SHA256))
def test_dinov2_vitl_bytes_unchanged(attention, pairs, facet):
    import hashlib
    from dino_tracker_b200.vit import DinoV2Features
    from oracle import vit as ovit
    sd = ovit.random_state_dict(3, 1024, torch.Generator().manual_seed(5), n_pos=37, ls_init=0.5)
    video = synth.random_video(2, 476, 854, seed=6)
    ex = DinoV2Features.from_name("dinov2_vitl14", sd, layer=2, device=DEV, attention=attention, cta_pairs=pairs, facet=facet)
    got = ex(video).cpu()
    assert hashlib.sha256(got.numpy().tobytes()).hexdigest() == VITL_SHA256[(attention, pairs, facet)]
