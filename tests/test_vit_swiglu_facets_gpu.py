"""GPU tests: ViT-g/14's SwiGLU feed-forward and the query / key / value facets of the CUDA feature stage.

Stages (dinotrk_vit_stage, the forward's own launch code) against float64 from the same fp16 operands, at the ViT-g width
(D 1536, Hd 4096) and at a width with N and K tails (D 128, Hd 344: 2 Hd = 688 = 2 x 256 + 176, K = 344 = 5 x 64 + 24),
on one and two full 854 x 476 frames, in CTA-pair and single-CTA mode.  Bounds follow tests/test_vit_layers_gpu.py (same
pinned accumulation constant GAMMA_C).  The SwiGLU stage h = silu(a) b with a = acc1 + b1, b = acc2 + b2 is held to
    gamma(D) (|b silu'(a)| S1 + |silu(a)| S2) + |silu(a) b| SILU_REL(a) + half an fp16 ulp of h
where S1, S2 are sum |y w| + |bias| of the two halves and SILU_REL bounds the MUFU evaluation of silu (ex2.approx and
rcp.approx, each ~2^-22 relative, the rounded exponent argument |a| 2^-24 log 2, two fp32 multiplies).  Outputs start
NaN-filled with canary rows past `rows`; h is [rows][Hd] with no spare columns, so those rows also catch a write past Hd.

Forward (DinoV2Features) against the oracle (oracle/vit_swiglu_facets.py, pinned to the live reference's goldens and to
transformers' Dinov2Layer): SwiGLU and each facet at layer 0 and at the last layer, fused / fused-single-cta /
materialized; full frames at the ViT-g width (tokens, keys) and the ViT-L width (keys) against the fp32 oracle on the GPU;
both goldens; determinism and batch invariance."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from dino_tracker_b200 import _lib
from oracle import synth
from oracle import vit_swiglu_facets as ovf
from test_vit_layers_gpu import (CANARY, DEV, FRAME_H, FRAME_W, N1, _bits_equal, _check, _gemm64, _gen, _nan, _randn,
                                 gamma, half_ulp16, half_ulp32)

pytestmark = pytest.mark.gpu
FC2, SWIGLU = 5, 6                 # DINOTRK_VIT_* of include/dinotrk.h
SWIGLU_WIDTHS = {"vitg14": (1536, 24, 4096), "tails": (128, 2, 344)}
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

swiglu_shapes = pytest.mark.parametrize("width,frames", [(w, f) for w in SWIGLU_WIDTHS for f in (1, 2)])


def silu_rel(a):
    return 2.0 ** -21 + a.abs() * 2.0 ** -23


def _stage(stage, dim, heads, hd, frames, inp, w, p0, p1, out, pair):
    lib = _lib.load()
    cfg = _lib.VitConfig(1, dim, heads, 0, 14, 7, 0, 1, 1 if pair else 0, hd, 0)
    geom = _lib.make_geom(FRAME_H, FRAME_W)
    ws = torch.empty(4096, dtype=torch.uint8, device=DEV)
    _lib.check(lib.dinotrk_vit_stage(stage, ctypes.byref(cfg), ctypes.byref(geom), frames, _lib.ptr(inp), _lib.ptr(w),
                                     _lib.ptr(p0), _lib.ptr(p1), _lib.ptr(out), None, None, _lib.ptr(ws), ws.numel(),
                                     _lib.stream_ptr()), "vit_stage")
    torch.cuda.synchronize()


def _deinterleave(t):
    """[rows][2 Hd] in the interleaved column order -> x1 [rows][Hd], x2 [rows][Hd]."""
    q = t.reshape(t.shape[0], -1, 4)
    return q[..., :2].reshape(t.shape[0], -1), q[..., 2:].reshape(t.shape[0], -1)


@swiglu_shapes
def test_swiglu_stage(width, frames):
    """w12 GEMM with the SwiGLU epilogue: h = silu(x1) x2 straight from the accumulator, fp16 [rows][Hd]."""
    D, heads, hd = SWIGLU_WIDTHS[width]
    rows = frames * N1
    g = _gen("swiglu", D, frames)
    y = _randn(g, rows, D).half()
    w = _randn(g, 2 * hd, D, std=D ** -0.5).half()     # interleaved rows: the kernel never sees the hub layout
    bias = _randn(g, 2 * hd, std=0.05)
    out = {}
    for pair in (True, False):
        h = _nan(rows + CANARY, hd, dtype=torch.half)
        _stage(SWIGLU, D, heads, hd, frames, y, w, bias, None, h, pair)
        out[pair] = h
    acc, aabs = _gemm64(y, w)
    v, s = acc + bias.double(), aabs + bias.double().abs()
    del acc, aabs
    a, b = _deinterleave(v)
    s1, s2 = _deinterleave(s)
    del v, s
    sig = torch.sigmoid(a)
    silu = a * sig
    ref = silu * b
    dsilu = sig * (1 + a * (1 - sig))
    scale = (b * dsilu).abs() * s1 + silu.abs() * s2
    for pair, h in out.items():
        got = h[:rows]
        rest = ref.abs() * silu_rel(a) + half_ulp16(torch.maximum(ref.abs(), got.double().abs()))
        _check(f"swiglu {width} x{frames} {'pair' if pair else 'single'}", got, ref, gamma(D) * scale + rest, D, scale, rest)
        assert h[rows:].isnan().all(), "the SwiGLU stage wrote rows past B * N1 (or columns past Hd)"
    assert _bits_equal(out[True], out[False]), "swiglu: CTA-pair and single-CTA results differ"


@swiglu_shapes
def test_w3_stage(width, frames):
    """FC2 with K = swiglu_hidden (the SwiGLU MLP's w3) + bias, LayerScale and the residual add."""
    D, heads, hd = SWIGLU_WIDTHS[width]
    rows = frames * N1
    g = _gen("w3", D, frames)
    a = (torch.nn.functional.silu(_randn(g, rows, hd)) * _randn(g, rows, hd)).half()
    w = _randn(g, D, hd, std=hd ** -0.5).half()
    bias = _randn(g, D, std=0.05)
    ls = _randn(g, D, std=0.3)
    x0 = _nan(rows + CANARY, D)
    x0[:rows] = _randn(g, rows, D)
    out = {}
    for pair in (True, False):
        x = x0.clone()
        _stage(FC2, D, heads, hd, frames, a, w, bias, ls, x, pair)
        out[pair] = x
    acc, aabs = _gemm64(a, w)
    ls64 = ls.double()
    ref = ls64 * (acc + bias.double())
    scale = ls64.abs() * (aabs + bias.double().abs())
    for pair, x in out.items():
        xn = x[:rows].double()
        r = half_ulp32(xn)
        _check(f"w3 {width} x{frames} {'pair' if pair else 'single'}", xn - x0[:rows].double(), ref, gamma(hd) * scale + r,
               hd, scale, r)
        assert x[rows:].isnan().all(), "w3 wrote rows past B * N1"
    assert _bits_equal(out[True], out[False]), "w3: CTA-pair and single-CTA results differ"


def _state_dict(mlp, depth, dim, seed, std=0.05, n_pos=4):
    g = torch.Generator().manual_seed(seed)
    return ovf.random_state_dict(depth, dim, g, n_pos=n_pos, std=std, swiglu=mlp == "swiglu")


def _compare(label, got, ref):
    assert got.shape == ref.shape
    scale = ref.abs().max().item()
    err = (got - ref).abs().max().item()
    cos = torch.nn.functional.cosine_similarity(got.flatten(2), ref.flatten(2), dim=1).min().item()
    print(f"{label}: max |diff| = {err:.3e} (max |ref| = {scale:.3f}), min token cosine = {cos:.6f}")
    assert err <= 5e-3 * scale
    assert cos > 0.9999


FORWARD_CASES = ([("swiglu", "tokens", 0), ("swiglu", "tokens", 1)]
                 + [(mlp, f, layer) for mlp in ("gelu", "swiglu") for f in ("queries", "keys", "values") for layer in (0, 1)])


@pytest.mark.parametrize("attention", ["fused", "fused-single-cta", "materialized"])
@pytest.mark.parametrize("mlp,facet,layer", FORWARD_CASES)
def test_forward_matches_oracle(mlp, facet, layer, attention):
    """dim 128 (Hd 344 for SwiGLU), 2 heads, 2 blocks, three 98 x 126 frames; layer 0 and the last layer."""
    from dino_tracker_b200.vit import DinoV2Features
    sd = _state_dict(mlp, 2, 128, seed=3)
    video = synth.random_video(3, 98, 126, seed=4)
    ref = ovf.dino_features_video(video, sd, 2, layer, facet=facet)
    ex = DinoV2Features(sd, heads=2, layer=layer, device=DEV, attention="fused" if attention.startswith("fused") else attention,
                        cta_pairs=attention == "fused", facet=facet)
    assert ex.swiglu_hidden == (344 if mlp == "swiglu" else 0)
    _compare(f"{mlp} {facet}@{layer} [{attention}]", ex.features_chw(video).cpu(), ref)


@pytest.mark.parametrize("name,depth,facet", [("dinov2_vitg14", 2, "tokens"), ("dinov2_vitg14", 2, "keys"),
                                              ("dinov2_vitl14", 2, "keys")])
def test_full_frame_against_gpu_oracle(name, depth, facet):
    """Two 854 x 476 frames at the ViT-g width (SwiGLU, Hd 4096) and the ViT-L width, last of `depth` blocks, against
    the fp32 oracle on the GPU (TF32 off)."""
    import oracle
    from dino_tracker_b200.vit import DinoV2Features
    oracle.use_exact_fp32()
    _, dim, heads = ovf.CONFIGS[name]
    sd = _state_dict("swiglu" if name == "dinov2_vitg14" else "gelu", depth, dim, seed=9, std=0.02, n_pos=37)
    video = synth.random_video(2, FRAME_H, FRAME_W, seed=10)
    ex = DinoV2Features.from_name(name, sd, layer=depth - 1, device=DEV, facet=facet)
    got = ex.features_chw(video).cpu()
    del ex
    sd_dev = {k: v.to(DEV) for k, v in sd.items()}
    with torch.no_grad():
        ref = ovf.dino_features_video(video.to(DEV), sd_dev, heads, depth - 1, facet=facet).cpu()
    _compare(f"{name} {facet} full frame", got, ref)


def test_facets_match_reference_golden():
    """Queries / keys / values at layers 0 and 1 against the live reference's qkv hook (vit_facets_small.npz)."""
    from dino_tracker_b200.vit import get_dino_features_video
    from oracle import make_golden_vit_models as mgv
    cfg = mgv.FACETS_CASE
    g = dict(np.load(os.path.join(GOLDEN_DIR, "vit_facets_small.npz")))
    sd, video = mgv.case_state_dict(cfg, swiglu=False), mgv.case_video(cfg)
    for layer in cfg["layers"]:
        for facet in ("queries", "keys", "values"):
            got = get_dino_features_video(video, cfg["model_name"], facet=facet, layer=layer, state_dict=sd)
            _compare(f"golden {facet}@{layer}", got, torch.from_numpy(g[f"{facet}_{layer}"]))


def test_vitg_matches_reference_golden():
    """dinov2_vitg14 from a hub-keyed SwiGLU state dict (2 blocks, layer 1) through get_dino_features_video: tokens and
    keys against the live reference's stored sample (vit_g_small.npz)."""
    from dino_tracker_b200.vit import get_dino_features_video
    from oracle import make_golden_vit_models as mgv
    cfg = mgv.G_CASE
    g = dict(np.load(os.path.join(GOLDEN_DIR, "vit_g_small.npz")))
    sd, video = mgv.case_state_dict(cfg, swiglu=True), mgv.case_video(cfg)
    for facet in ("tokens", "keys"):
        got = get_dino_features_video(video, cfg["model_name"], facet=facet, layer=cfg["layer"], state_dict=sd).numpy()
        assert got.shape == tuple(g[f"{facet}_shape"])
        scale = float(g[f"{facet}_absmax"])
        err = np.abs(got.reshape(-1)[g[f"{facet}_idx"]] - g[f"{facet}_vals"]).max()
        print(f"ViT-g {facet} vs reference golden: max |diff| = {err:.3e} (max |ref| = {scale:.3f})")
        assert err <= 5e-3 * scale
        assert abs(np.abs(got.astype(np.float64)).sum() / g[f"{facet}_sums"][1] - 1) <= 1e-3


@pytest.mark.parametrize("mlp,facet", [("swiglu", "tokens"), ("gelu", "keys")])
def test_deterministic_and_batch_invariant(mlp, facet):
    from dino_tracker_b200.vit import DinoV2Features
    sd = _state_dict(mlp, 2, 128, seed=5)
    video = synth.random_video(5, 98, 126, seed=6)
    ex = DinoV2Features(sd, heads=2, layer=1, device=DEV, facet=facet)
    a = ex(video).clone()
    b = ex(video).clone()
    assert torch.equal(a, b), f"non-deterministic: {(a - b).abs().max().item()}"
    c = ex(video[1:4]).clone()
    assert torch.equal(a[1:4], c), f"batch-dependent: {(a[1:4] - c).abs().max().item()}"


def test_swiglu_shape_mismatch_raises():
    from dino_tracker_b200.vit import DinoV2Features
    sd = _state_dict("swiglu", 2, 128, seed=7)
    sd["blocks.1.mlp.w3.weight"] = sd["blocks.1.mlp.w3.weight"][:, :336]
    with pytest.raises(ValueError, match="block 1"):
        DinoV2Features(sd, heads=2, device=DEV)
