"""CPU: the DINOv3 / DINOv2-with-registers oracle (oracle/vit_dinov3.py) against ``transformers``, the loader's key
conversion and RoPE pair permutation, and the golden file the GPU tests read.

``transformers``' DINOv3ViTModel and Dinov2WithRegistersModel run in float64 with seeded weights; at stride = patch the
oracle's block outputs with the prefix tokens dropped must match theirs.  DINOv3's RoPE angles are computed in float32
inside ``transformers`` (the oracle uses float64), so the bar is 1e-6 of the largest output, not float64 rounding."""
import os

import numpy as np
import pytest
import torch

from oracle import synth
from oracle import vit_dinov3 as ov3
from oracle import vit_swiglu_facets as ovf

transformers = pytest.importorskip("transformers")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vit_dinov3_small.npz")


def _close(got, ref, rel):
    scale = ref.abs().max().item()
    err = (got - ref).abs().max().item()
    assert err <= rel * scale, f"max |diff| {err:.3e} > {rel:g} x {scale:.3e}"


def _hf_dinov3(sd, depth, dim, registers, gated, hidden):
    cfg = transformers.DINOv3ViTConfig(hidden_size=dim, num_hidden_layers=depth, num_attention_heads=dim // 64,
                                       intermediate_size=hidden, num_register_tokens=registers, patch_size=16,
                                       use_gated_mlp=gated, hidden_act="silu" if gated else "gelu", layer_norm_eps=1e-5,
                                       rope_theta=100.0, key_bias=False, image_size=224)
    m = transformers.DINOv3ViTModel(cfg).double().eval()
    missing, unexpected = m.load_state_dict({k: v.double() for k, v in sd.items()}, strict=False)
    assert not unexpected and all("inv_freq" in k for k in missing), (missing, unexpected)
    return m


@pytest.mark.parametrize("registers,gated,size", [(4, False, (64, 96)), (0, False, (64, 96)), (4, True, (70, 100)),
                                                  (0, True, (64, 96)), (4, False, (70, 100))])
def test_oracle_matches_transformers_dinov3(registers, gated, size):
    """Every block's output, prefix dropped, at stride 16: R = 4 and 0, GELU and gated MLP, a frame that is a multiple of
    16 and one that is not (the hub crops the remainder; so does the stride-16 convolution)."""
    depth, dim, hidden = 2, 128, 344 if gated else 512
    sd = ov3.random_state_dict(depth, dim, torch.Generator().manual_seed(1), registers=registers, gated=gated,
                               hidden=hidden, std=0.05)
    m = _hf_dinov3(sd, depth, dim, registers, gated, hidden)
    video = synth.random_video(2, *size, seed=2).double()
    sd64 = {k: v.double() for k, v in sd.items()}
    with torch.no_grad():
        hs = m(pixel_values=ov3.normalize(video), output_hidden_states=True).hidden_states
        for layer in range(depth):
            ref = hs[layer + 1][:, 1 + registers:]
            got = ov3.vit_tokens(video, sd64, layer, stride=16)[:, 1 + registers:]
            _close(got, ref, 1e-6)


def test_oracle_matches_transformers_dinov2_registers():
    """DINOv2 with 4 registers, hub keys, on a 4 x 4 grid at stride 14 (the position table is not interpolated)."""
    depth, dim, heads, R = 2, 128, 2, 4
    g = torch.Generator().manual_seed(3)
    sd = ovf.random_state_dict(depth, dim, g, n_pos=4, std=0.05)
    sd["register_tokens"] = torch.randn(1, R, dim, generator=g) * 0.5
    cfg = transformers.Dinov2WithRegistersConfig(hidden_size=dim, num_hidden_layers=depth, num_attention_heads=heads,
                                                 mlp_ratio=4, num_register_tokens=R, patch_size=14, image_size=56,
                                                 layer_norm_eps=1e-6, layerscale_value=1.0)
    m = transformers.Dinov2WithRegistersModel(cfg).double().eval()
    hf = {"embeddings.cls_token": sd["cls_token"], "embeddings.mask_token": torch.zeros(1, dim),
          "embeddings.register_tokens": sd["register_tokens"], "embeddings.position_embeddings": sd["pos_embed"],
          "embeddings.patch_embeddings.projection.weight": sd["patch_embed.proj.weight"],
          "embeddings.patch_embeddings.projection.bias": sd["patch_embed.proj.bias"],
          "layernorm.weight": sd["norm.weight"], "layernorm.bias": sd["norm.bias"]}
    for i in range(depth):
        s, d = f"blocks.{i}.", f"encoder.layer.{i}."
        for n in ("norm1", "norm2", "mlp.fc1", "mlp.fc2"):
            hf[d + n + ".weight"], hf[d + n + ".bias"] = sd[s + n + ".weight"], sd[s + n + ".bias"]
        for j, n in enumerate(("query", "key", "value")):
            hf[d + f"attention.attention.{n}.weight"] = sd[s + "attn.qkv.weight"][j * dim:(j + 1) * dim]
            hf[d + f"attention.attention.{n}.bias"] = sd[s + "attn.qkv.bias"][j * dim:(j + 1) * dim]
        hf[d + "attention.output.dense.weight"], hf[d + "attention.output.dense.bias"] = sd[s + "attn.proj.weight"], sd[s + "attn.proj.bias"]
        hf[d + "layer_scale1.lambda1"], hf[d + "layer_scale2.lambda1"] = sd[s + "ls1.gamma"], sd[s + "ls2.gamma"]
    m.load_state_dict({k: v.double() for k, v in hf.items()}, strict=True)
    video = synth.random_video(2, 56, 56, seed=4).double()
    sd64 = {k: v.double() for k, v in sd.items()}
    with torch.no_grad():
        hs = m(pixel_values=ov3.normalize(video), output_hidden_states=True).hidden_states
        for layer in range(depth):
            _close(ov3.vit_tokens_reg(video, sd64, heads, layer, stride=14)[:, 1 + R:], hs[layer + 1][:, 1 + R:], 1e-12)


def test_rope_pair_permutation_keeps_scores():
    """The loader's q / k row order (dims (j, j + 32) -> columns (2j, 2j + 1)) with the pairwise rotation in that order
    gives float64-identical attention scores to rotate_half in the hub order, and the loader's table is the oracle's."""
    from dino_tracker_b200.vit import rope_perm, rope_table
    h, w, D = 5, 7, 128
    g = torch.Generator().manual_seed(5)
    q, k = torch.randn(h * w, D, generator=g, dtype=torch.float64), torch.randn(h * w, D, generator=g, dtype=torch.float64)
    cos, sin = ov3.rope_cos_sin(h, w)
    heads = lambda t: t.reshape(h * w, D // 64, 64).transpose(0, 1)   # noqa: E731
    ref = ov3.rotate(heads(q), cos, sin) @ ov3.rotate(heads(k), cos, sin).transpose(-2, -1)
    perm = rope_perm(D)
    assert sorted(perm.tolist()) == list(range(D)) and perm[:4].tolist() == [0, 32, 1, 33]
    tab = rope_table(h, w).double()                      # [P][32][2], float32-rounded
    assert (tab[..., 0] - cos[:, :32]).abs().max() < 1e-7 and (tab[..., 1] - sin[:, :32]).abs().max() < 1e-7
    c, s = cos[:, None, :32], sin[:, None, :32]

    def rot(t):   # the epilogue: (a, b) of pair j in columns (2j, 2j + 1)
        t = heads(t[:, perm]).transpose(0, 1).reshape(h * w, D // 64, 32, 2)
        a, b = t[..., 0], t[..., 1]
        return torch.stack((a * c - b * s, b * c + a * s), dim=-1).reshape(h * w, D // 64, 64).transpose(0, 1)
    got = rot(q) @ rot(k).transpose(-2, -1)
    assert (got - ref).abs().max().item() <= 1e-12 * ref.abs().max().item()


def test_loader_key_conversion():
    """dinov3_to_hub: qkv stacked with a zero k bias, the gated MLP as [gate; up] -> w12 and down -> w3."""
    from dino_tracker_b200.vit import dinov3_to_hub
    sd = ov3.random_state_dict(2, 128, torch.Generator().manual_seed(6), gated=True, hidden=344)
    hub = dinov3_to_hub(sd)
    a = "model.layer.1.attention."
    assert torch.equal(hub["blocks.1.attn.qkv.weight"],
                       torch.cat([sd[a + "q_proj.weight"], sd[a + "k_proj.weight"], sd[a + "v_proj.weight"]]))
    assert torch.equal(hub["blocks.1.attn.qkv.bias"][128:256], torch.zeros(128))
    assert torch.equal(hub["blocks.1.mlp.w12.weight"][:344], sd["model.layer.1.mlp.gate_proj.weight"])
    assert torch.equal(hub["blocks.1.mlp.w3.weight"], sd["model.layer.1.mlp.down_proj.weight"])
    assert hub["register_tokens"].shape == (1, 4, 128) and "pos_embed" not in hub


def test_patch_size_rule():
    from dino_tracker_b200.vit import patch_size
    assert [patch_size(n) for n in ("dinov2_vitl14", "dino_vits8", "dino_vitb8", "dinov2_vitl14_reg", "dinov3_vitl16",
                                    "dinov3_vits16plus")] == [14, 8, 8, 14, 16, 16]


def test_golden_matches_oracle():
    """tests/golden/vit_dinov3_small.npz (oracle/make_golden_vit_dinov3.py, a seeded transformers run) against the oracle
    at stride 16; the GPU tests read the same file without transformers."""
    from oracle import make_golden_vit_dinov3 as mg
    g = dict(np.load(GOLDEN))
    for case in mg.CASES:
        sd, video = mg.case_state_dict(case), mg.case_video(case)
        sd64 = {k: v.double() for k, v in sd.items()}
        got = ov3.dino_features_video(video.double(), sd64, case["layer"], stride=16)
        _close(got, torch.from_numpy(g[case["name"]]), 1e-6)


def test_extractor_rejects_width_and_stride():
    """Head dim 64 only (ViT-7B's 128 is refused), and 7 <= stride <= patch; both checked before any device work."""
    from dino_tracker_b200.vit import DinoV3Features
    sd = ov3.random_state_dict(1, 128, torch.Generator().manual_seed(7))
    for bad in (6, 17):
        with pytest.raises(ValueError, match="stride"):
            DinoV3Features(sd, stride=bad)
    sd["embeddings.cls_token"] = torch.zeros(1, 1, 160)
    with pytest.raises(ValueError, match="multiple of 64"):
        DinoV3Features(sd)
