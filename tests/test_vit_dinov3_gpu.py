"""GPU tests: DINOv3 ViTs and DINOv2 with registers on the CUDA feature stage.

Stage: the qkv GEMM with the rotary epilogue (dinotrk_vit_stage_ext, the forward's own launch code) at D = 1024 on one and
two 854 x 476 frames at patch 16 / stride 8 (58 x 105 tokens + cls + 4 registers: N1 = 6095 rows, odd, patches from row
5), CTA pairs and single CTAs, against float64 from the same fp16 operands and the same fp32 (cos, sin) table.  The bound
is test_vit_layers_gpu.py's qkv bound over both members of a pair (|cos|, |sin| <= 1), plus the rotation's two fp32
roundings.  Prefix rows must come out unrotated, v untouched by RoPE.

Forward (DinoV3Features / DinoV2Features with registers) against the oracle (oracle/vit_dinov3.py, cross-checked against
transformers on the CPU), with test_vit_swiglu_facets_gpu.py's bars: tokens and the three facets at layer 0 and the last
layer, R = 4 and 0, GELU and gated MLP (hidden 344: N and K tails), fused on CTA pairs, fused on single CTAs and TF32
materialised; ViT-L/16 widths at 854 x 476, stride 8 and 16, against the fp32 oracle on the GPU; the transformers golden;
determinism and batch invariance."""
import ctypes
import os

import numpy as np
import pytest
import torch

from dino_tracker_b200 import _lib
from oracle import synth
from oracle import vit_dinov3 as ov3
from oracle import vit_swiglu_facets as ovf
from test_vit_layers_gpu import CANARY, DEV, QSCALE, U24, _bits_equal, _check, _gemm64, _gen, _nan, _randn, gamma, half_ulp16
from test_vit_swiglu_facets_gpu import _compare

pytestmark = pytest.mark.gpu
QKV = 2                            # DINOTRK_VIT_QKV
FRAME_H, FRAME_W = 476, 854
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vit_dinov3_small.npz")


@pytest.mark.parametrize("frames", [1, 2])
def test_rope_qkv_stage(frames):
    from dino_tracker_b200.vit import rope_table
    D, heads, R = 1024, 16, 4
    geom = _lib.make_geom(FRAME_H, FRAME_W, 16, 8, 35)
    h, w = geom.h, geom.w
    P, pre = h * w, 1 + R
    N1 = P + pre
    assert (h, w, N1) == (58, 105, 6095)
    rows, BH, N1p8 = frames * N1, frames * heads, (N1 + 7) // 8 * 8
    g = _gen("rope-qkv", D, frames)
    y = _randn(g, rows, D).half()
    wq = _randn(g, 3 * D, D, std=D ** -0.5).half()
    bias = _randn(g, 3 * D, std=0.05)
    bias[D:2 * D] = 0                                   # DINOv3 has no key bias
    table = rope_table(h, w, 100.0, DEV)
    cfg = _lib.VitConfig(1, D, heads, 0, 16, 8, 0, 1, 1)
    wt = _lib.VitWeights()
    wt.rope, wt.n_registers = table.data_ptr(), R
    lib = _lib.load()
    res = {}
    for pair in (True, False):
        cfg.gemm_pair = 1 if pair else 0
        q, k = _nan(BH * N1 * 64 + CANARY, dtype=torch.half), _nan(BH * N1 * 64 + CANARY, dtype=torch.half)
        vT = _nan(BH * 64 * N1p8 + CANARY, dtype=torch.half)
        ws = torch.empty(4096, dtype=torch.uint8, device=DEV)
        _lib.check(lib.dinotrk_vit_stage_ext(QKV, ctypes.byref(cfg), ctypes.byref(wt), ctypes.byref(geom), frames, _lib.ptr(y),
                                             _lib.ptr(wq), _lib.ptr(bias), None, _lib.ptr(q), _lib.ptr(k), _lib.ptr(vT),
                                             _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "vit_stage_ext")
        torch.cuda.synchronize()
        res[pair] = (q, k, vT)
    acc, aabs = _gemm64(y, wq)
    ref, scale = acc + bias.double(), aabs + bias.double().abs()
    del acc, aabs
    # (cos, sin) per row: identity on the prefix rows
    cs = torch.zeros(N1, 32, 2, dtype=torch.float64, device=DEV)
    cs[:, :, 0] = 1
    cs[pre:] = table.double()
    cs = cs.repeat(frames, 1, 1)[:, None]             # [rows][1][32][2]

    def rotated(lo, sc):
        t = ref[:, lo:lo + D].reshape(rows, heads, 32, 2)
        s = scale[:, lo:lo + D].reshape(rows, heads, 32, 2)
        a, b, c, si = t[..., 0], t[..., 1], cs[..., 0], cs[..., 1]
        out = torch.stack((a * c - b * si, b * c + a * si), dim=-1)
        s2 = (s[..., 0] + s[..., 1])[..., None].expand_as(out)                 # |cos|, |sin| <= 1
        rnd = 4 * U24 * (a.abs() + b.abs())[..., None].expand_as(out)         # fmul, fma and the q scale
        hm = lambda z: z.reshape(frames, N1, heads, 64).permute(0, 2, 1, 3).reshape(BH, N1, 64) * sc   # noqa: E731
        return hm(out), hm(s2), hm(rnd)
    refs = {"q": rotated(0, QSCALE), "k": rotated(D, 1.0)}
    vref = ref[:, 2 * D:].reshape(frames, N1, heads, 64).permute(0, 2, 3, 1).reshape(BH, 64, N1)
    vs = scale[:, 2 * D:].reshape(frames, N1, heads, 64).permute(0, 2, 3, 1).reshape(BH, 64, N1)
    for pair, (q, k, vT) in res.items():
        mode = "pair" if pair else "single"
        got = {"q": q[:BH * N1 * 64].view(BH, N1, 64), "k": k[:BH * N1 * 64].view(BH, N1, 64)}
        for name, (r, s, rnd) in refs.items():
            r16 = half_ulp16(torch.maximum(r.abs(), got[name].double().abs())) + rnd
            _check(f"rope qkv.{name} x{frames} {mode}", got[name], r, gamma(D) * s + r16, D, s, r16)
        vv = vT[:BH * 64 * N1p8].view(BH, 64, N1p8)
        r16 = half_ulp16(torch.maximum(vref.abs(), vv[:, :, :N1].double().abs()))
        _check(f"rope qkv.v x{frames} {mode}", vv[:, :, :N1], vref, gamma(D) * vs + r16, D, vs, r16)
        assert vv[:, :, N1:].isnan().all(), "v^T padding columns written"
        assert q[BH * N1 * 64:].isnan().all() and k[BH * N1 * 64:].isnan().all() and vT[BH * 64 * N1p8:].isnan().all()
    for a, b, name in zip(res[True], res[False], "qkv"):
        assert _bits_equal(a, b), f"rope qkv.{name}: CTA-pair and single-CTA results differ"


def _v3_state_dict(mlp, registers, seed, dim=128, depth=2, std=0.05):
    return ov3.random_state_dict(depth, dim, torch.Generator().manual_seed(seed), registers=registers,
                                 gated=mlp == "gated", hidden=344 if mlp == "gated" else 4 * dim, std=std)


def _extractor(attention, **kw):
    from dino_tracker_b200.vit import DinoV3Features
    return DinoV3Features(device=DEV, attention="fused" if attention.startswith("fused") else attention,
                          cta_pairs=attention == "fused", **kw)


ATTENTION = ["fused", "fused-single-cta", "materialized"]
FORWARD_CASES = ([("gelu", 4, "tokens", 0), ("gelu", 4, "tokens", 1), ("gated", 4, "tokens", 1), ("gelu", 0, "tokens", 1),
                  ("gated", 0, "tokens", 1)]
                 + [(mlp, 4, f, layer) for mlp in ("gelu", "gated") for f in ("queries", "keys", "values") for layer in (0, 1)])


@pytest.mark.parametrize("attention", ATTENTION)
@pytest.mark.parametrize("mlp,registers,facet,layer", FORWARD_CASES)
def test_forward_matches_oracle(mlp, registers, facet, layer, attention):
    """dim 128 (2 heads; gated: hidden 344), 2 blocks, three 98 x 126 frames at stride 8 (11 x 14 tokens)."""
    sd = _v3_state_dict(mlp, registers, seed=3)
    video = synth.random_video(3, 98, 126, seed=4)
    ref = ov3.dino_features_video(video.double(), {k: v.double() for k, v in sd.items()}, layer, stride=8, facet=facet)
    ex = _extractor(attention, state_dict=sd, layer=layer, stride=8, facet=facet)
    assert ex.n_registers == registers and ex.swiglu_hidden == (344 if mlp == "gated" else 0)
    _compare(f"dinov3 {mlp} R={registers} {facet}@{layer} [{attention}]", ex.features_chw(video).cpu(), ref.float())


@pytest.mark.parametrize("stride,attention,facet", [(8, "fused", "tokens"), (8, "fused-single-cta", "tokens"),
                                                    (8, "materialized", "tokens"), (8, "fused", "keys"),
                                                    (16, "fused", "tokens"), (16, "fused-single-cta", "tokens"),
                                                    (16, "materialized", "tokens"), (16, "fused", "queries")])
def test_vitl16_full_frame_against_gpu_oracle(stride, attention, facet):
    """ViT-L/16 widths (1024, 16 heads, 4 registers), 2 blocks, two 854 x 476 frames (58 x 105 tokens at stride 8,
    29 x 53 at 16), against the fp32 oracle on the GPU (TF32 off)."""
    import oracle
    oracle.use_exact_fp32()
    sd = _v3_state_dict("gelu", 4, seed=9, dim=1024, std=0.02)
    video = synth.random_video(2, FRAME_H, FRAME_W, seed=10)
    ex = _extractor(attention, state_dict=sd, layer=1, stride=stride, facet=facet)
    got = ex.features_chw(video).cpu()
    assert got.shape[-2:] == ((58, 105) if stride == 8 else (29, 53))
    del ex
    with torch.no_grad():
        ref = ov3.dino_features_video(video.to(DEV), {k: v.to(DEV) for k, v in sd.items()}, 1, stride=stride, facet=facet).cpu()
    _compare(f"vitl16 s{stride} {facet} [{attention}]", got, ref)


def test_matches_transformers_golden():
    """DinoV3Features at stride = patch = 16 against transformers' DINOv3ViTModel (vit_dinov3_small.npz)."""
    from oracle import make_golden_vit_dinov3 as mg
    g = dict(np.load(GOLDEN))
    for case in mg.CASES:
        ex = _extractor("fused", state_dict=mg.case_state_dict(case), layer=case["layer"], stride=16)
        _compare(f"golden {case['name']}", ex.features_chw(mg.case_video(case)).cpu(), torch.from_numpy(g[case["name"]]).float())


def test_get_dino_features_video_by_name():
    from dino_tracker_b200.vit import get_dino_features_video
    sd = _v3_state_dict("gelu", 4, seed=13, dim=384)
    video = synth.random_video(2, 98, 126, seed=14)
    got = get_dino_features_video(video, "dinov3_vits16", stride=8, layer=1, state_dict=sd, device=DEV)
    ref = ov3.dino_features_video(video.double(), {k: v.double() for k, v in sd.items()}, 1, stride=8)
    _compare("dinov3_vits16 by name", got, ref.float())


@pytest.mark.parametrize("attention", ATTENTION)
@pytest.mark.parametrize("facet", ["tokens", "keys"])
def test_dinov2_registers_matches_oracle(facet, attention):
    """DINOv2 with 4 registers (hub keys + register_tokens), 2 blocks, three 98 x 126 frames at stride 7: the position
    table is interpolated onto the grid, the registers carry none."""
    from dino_tracker_b200.vit import DinoV2Features
    g = torch.Generator().manual_seed(15)
    sd = ovf.random_state_dict(2, 128, g, n_pos=4, std=0.05)
    sd["register_tokens"] = torch.randn(1, 4, 128, generator=g) * 0.5
    video = synth.random_video(3, 98, 126, seed=16)
    ref = ov3.dino_features_video_reg(video, sd, 2, 1, facet=facet)
    ex = DinoV2Features(sd, heads=2, layer=1, device=DEV, attention="fused" if attention.startswith("fused") else attention,
                        cta_pairs=attention == "fused", facet=facet)
    assert ex.n_registers == 4
    _compare(f"dinov2 reg {facet} [{attention}]", ex.features_chw(video).cpu(), ref)


@pytest.mark.parametrize("mlp,facet", [("gelu", "tokens"), ("gated", "keys")])
def test_deterministic_and_batch_invariant(mlp, facet):
    sd = _v3_state_dict(mlp, 4, seed=5)
    video = synth.random_video(5, 98, 126, seed=6)
    ex = _extractor("fused", state_dict=sd, layer=1, facet=facet)
    a = ex(video).clone()
    b = ex(video).clone()
    assert torch.equal(a, b), f"non-deterministic: {(a - b).abs().max().item()}"
    c = ex(video[1:4]).clone()
    assert torch.equal(a[1:4], c), f"batch-dependent: {(a[1:4] - c).abs().max().item()}"
