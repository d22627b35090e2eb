"""GPU tests: wgmma ViT (fp16-operand GEMMs on CTA pairs or single CTAs + fused attention; TF32 GEMMs + materialised
attention as the validation path) against the fp32 oracle restatement (itself pinned to the live reference pipeline and to
transformers' DINOv2 block, see oracle/vit.py), and the attention kernel on its own against float64."""
import numpy as np
import pytest
import torch

from oracle import vit as ovit
from oracle import synth

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("attention", ["fused", "fused-single-cta", "materialized"])
@pytest.mark.parametrize("cfg", [dict(H=98, W=126, depth=2, dim=128, heads=2, layer=1, T=3),
                                 dict(H=112, W=140, depth=3, dim=192, heads=3, layer=1, T=2),
                                 dict(H=182, W=238, depth=1, dim=64, heads=1, layer=0, T=1)])
def test_vit_features_match_oracle(cfg, attention):
    from dino_tracker_b200.vit import DinoV2Features
    g = torch.Generator().manual_seed(3)
    sd = ovit.random_state_dict(cfg["depth"], cfg["dim"], g, n_pos=4, std=0.05)
    video = synth.random_video(cfg["T"], cfg["H"], cfg["W"], seed=4)
    ref = ovit.dino_features_video(video, sd, cfg["heads"], cfg["layer"])          # T x C x h x w
    ex = DinoV2Features(sd, heads=cfg["heads"], layer=cfg["layer"], device="cuda:0",
                        attention="fused" if attention.startswith("fused") else attention,
                        cta_pairs=attention == "fused")
    got = ex.features_chw(video).cpu()
    assert got.shape == ref.shape
    scale = ref.abs().max().item()
    err = (got - ref).abs().max().item()
    print(f"ViT[{attention}] max |diff| = {err:.3e} (max |ref| = {scale:.3f})")
    assert err <= 5e-3 * scale   # TF32 single-pass contractions (10-bit mantissa inputs), fp32 accumulation
    # cosine between corresponding tokens
    cos = torch.nn.functional.cosine_similarity(got.flatten(2), ref.flatten(2), dim=1)
    assert cos.min().item() > 0.9999


def test_pos_embed_interpolation_matches_oracle():
    from dino_tracker_b200.vit import interpolate_pos_embed
    pe = torch.randn(1, 1 + 37 * 37, 32)
    assert torch.equal(interpolate_pos_embed(pe, 67, 121), ovit.interpolate_pos_embed(pe, 67, 121))


def test_vit_is_deterministic_and_batch_invariant():
    """Frame features must not depend on which other frames share the call (frame sharding relies on it)."""
    from dino_tracker_b200.vit import DinoV2Features
    g = torch.Generator().manual_seed(5)
    sd = ovit.random_state_dict(2, 128, g, n_pos=4, std=0.05)
    video = synth.random_video(5, 98, 126, seed=6)
    ex = DinoV2Features(sd, heads=2, layer=1, device="cuda:0")
    a = ex(video).clone()
    b = ex(video).clone()
    assert torch.equal(a, b), f"non-deterministic: {(a - b).abs().max().item()}"
    c = ex(video[1:4]).clone()
    assert torch.equal(a[1:4], c), f"batch-dependent: {(a[1:4] - c).abs().max().item()}"


def _attention_reference(q, k, v, chunk=512):
    """softmax(q k^T / 8) v in float64 from the fp16-rounded operands the kernel sees.  q: [BH][N][64] (unscaled).
    Query rows go in chunks: at full frame length all scores at once would be BH x 8108^2 doubles."""
    q, k, v = q.double(), k.double(), v.double()
    out = torch.empty_like(q)
    for i in range(0, q.shape[1], chunk):
        p = torch.softmax(torch.einsum("hnd,hmd->hnm", q[:, i:i + chunk], k), dim=-1)
        out[:, i:i + chunk] = torch.einsum("hnm,hmd->hnd", p, v)
    return out


@pytest.mark.parametrize("case", ["random-small", "random-large", "ramp", "late-spike", "tail-1", "tail-63",
                                  "tail-63-f16", "full-random", "full-random-f16", "full-ramp", "full-ramp-f16",
                                  "full-late-spike", "full-late-spike-f16"])
def test_fused_attention_against_float64(case):
    """The attention kernel on its own (dinotrk_vit_attention): accumulator kept in registers across key tiles with an
    online running maximum -- 'ramp' and 'late-spike' make the row maxima jump by far more than 2^8 between key tiles, so
    the rescale of the accumulator (row sums included) matters on many tiles; the tail cases
    end the keys 1 / 63 columns into the last 64-key tile.  'full-*': one 854x476 frame's 8108 tokens (127 key tiles,
    the last one holding 44 keys), 16 heads (ViT-L), 2 frames.  '-f16': the fp16 store the forward's default path uses."""
    from dino_tracker_b200 import _lib
    lib = _lib.load()
    dev = "cuda:0"
    g = torch.Generator().manual_seed(11)
    full, out_f16 = case.startswith("full-"), case.endswith("-f16")
    pattern = case.removeprefix("full-").removesuffix("-f16")
    B, heads = 2, (16 if full else 3)
    N1 = 67 * 121 + 1 if full else {"tail-1": 64 * 5 + 1, "tail-63": 64 * 4 + 63}.get(pattern, 700)
    BH = B * heads
    q = torch.randn(BH, N1, 64, generator=g)
    k = torch.randn(BH, N1, 64, generator=g)
    v = torch.randn(BH, N1, 64, generator=g)
    if pattern == "random-large":
        q *= 6.0
    elif pattern == "ramp":       # score grows with the key index: ~16 log2 units per 64-key tile, every tile rescales
        q[:, :, 0] = 4.0
        k[:, :, 0] = torch.linspace(0, 240.0 * (N1 - 1) / 699, N1)[None]
    elif pattern == "late-spike":  # one late key dominates everything before it (row maxima jump by ~100 log2 units)
        u = torch.sign(torch.randn(64, generator=g))
        q = 0.2 * q + 3.0 * u
        k[:, N1 - 70] = 3.0 * u
    # the kernel's inputs: fp16, q pre-scaled by 64^-1/2 * log2(e)
    scale = 0.125 * 1.4426950408889634
    q16 = (q * scale).half()
    k16 = k.half()
    v16 = v.half()
    N1p = (N1 + 7) // 8 * 8
    vT = torch.zeros(BH, 64, N1p, dtype=torch.half)
    vT[:, :, :N1] = v16.transpose(1, 2)
    out = torch.full((B * N1, heads * 64), float("nan"), device=dev, dtype=torch.half if out_f16 else torch.float32)
    qd, kd, vd = q16.to(dev).contiguous(), k16.to(dev).contiguous(), vT.to(dev).contiguous()
    attention = lib.dinotrk_vit_attention_f16 if out_f16 else lib.dinotrk_vit_attention
    _lib.check(attention(_lib.ptr(qd), _lib.ptr(kd), _lib.ptr(vd), B, heads, N1, N1p, _lib.ptr(out), _lib.stream_ptr()),
               "vit_attention")
    torch.cuda.synchronize()
    # exp2(q16 . k) = exp((q16 / scale / 8) . k)
    ref = _attention_reference(qd.float() / scale / 8.0, kd.float(), v16.to(dev).float())
    got = out.view(B, N1, heads, 64).permute(0, 2, 1, 3).reshape(BH, N1, 64).double()
    assert torch.isfinite(got).all()
    err = (got - ref).abs()
    # fp16 P (2^-11 relative per probability) and fp16-exact operands: a few 1e-3 absolute on |v| ~ 1..4; the fp16 store
    # adds half an ulp of the output
    bound = torch.full_like(ref, 2e-3)
    if out_f16:
        _, e = torch.frexp(torch.maximum(ref.abs(), got.abs()))
        bound += torch.ldexp(torch.ones_like(ref), e.clamp_min(-13) - 12)
    print(f"attention[{case}] max |diff| = {err.max().item():.3e} (max |ref| = {ref.abs().max().item():.3f}), "
          f"worst error / bound = {(err / bound).max().item():.3f}")
    assert (err <= bound).all()


def test_vit_matches_reference_pipeline_golden():
    """CUDA ViT against the features the LIVE reference pipeline produced (tests/golden/vit_small.npz: the reference's
    get_dino_features_video / VitExtractor around a stand-in hub model with transformers' DINOv2 blocks; dim 384, 6 heads,
    2 blocks, tap 1, 98x126 frame)."""
    import os
    from oracle import make_golden as mg
    from dino_tracker_b200.vit import DinoV2Features
    cfg = mg.VIT_CASE
    g = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vit_small.npz")))
    sd = mg.vit_case_state_dict(cfg)
    video = synth.random_video(cfg["T"], cfg["H"], cfg["W"], seed=cfg["seed"] + 1)
    ex = DinoV2Features(sd, heads=cfg["heads"], layer=cfg["layer"], device="cuda:0")
    got = ex.features_chw(video).cpu().numpy()
    ref = g["features"]
    assert got.shape == ref.shape
    scale = np.abs(ref).max()
    err = np.abs(got - ref).max()
    print(f"ViT vs reference-pipeline golden: max |diff| = {err:.3e} (max |ref| = {scale:.3f})")
    assert err <= 5e-3 * scale
