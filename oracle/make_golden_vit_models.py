"""Generate ``tests/golden/vit_facets_small.npz`` and ``tests/golden/vit_g_small.npz`` by running the LIVE reference
(only where its sources are present), next to ``oracle/make_golden.py`` (whose ``vit_small`` case stays as it is):

    python -m oracle.make_golden_vit_models

Both cases run ``utils.get_dino_features_video`` + ``models/extractor.VitExtractor`` unmodified on the CPU; only
``torch.hub.load`` is replaced by a stand-in with the DinoVisionTransformer surface the extractor touches, whose blocks
are ``transformers``' Dinov2Layer (independent of ``oracle/``) carrying seeded weights.  For the facets the stand-in's
``attn.qkv`` is a real ``nn.Linear`` carrying the block's qkv weights, applied to the block's LayerNorm-1 output, so the
reference's qkv hook records what the hub model's would.

1. ``vit_facets_small``: the ``dinov2_vits14`` name and dims (384, 6 heads), 2 GELU blocks, queries / keys / values
   at layers 0 and 1, one 42 x 56 frame (5 x 7 tokens).
2. ``vit_g_small``: the ``dinov2_vitg14`` name (the reference derives C = 1536 from it), 24 heads, 2 SwiGLU blocks
   (Hd = 4096), ``layer=1`` passed explicitly (the name implies 40 blocks), one 98 x 126 frame, tokens and keys.  Its
   outputs are 1536 x 13 x 17 each, so the file keeps a seeded sample of 8192 entries of each plus float64 sums.
"""
import os

import numpy as np
import torch

from . import ref_harness, synth
from . import vit_swiglu_facets as ovf
from .make_golden import GOLDEN_DIR, hf_dinov2_layer

FACETS_CASE = dict(model_name="dinov2_vits14", dim=384, heads=6, depth=2, layers=(0, 1), H=42, W=56, T=1, seed=71,
                   std=0.05)
G_CASE = dict(model_name="dinov2_vitg14", dim=1536, heads=24, depth=2, layer=1, H=98, W=126, T=1, seed=81, std=0.03,
              n_sample=8192)


def hf_dinov2_swiglu_layer(dim, heads, sd, i):
    """Block i of a hub state dict with a SwiGLU MLP as ``transformers``' Dinov2Layer(use_swiglu_ffn=True): its
    weights_in / weights_out are the hub's w12 / w3 (x1 = first Hd rows of w12, as the hub's chunk(2) takes them)."""
    from transformers import Dinov2Config
    from transformers.models.dinov2.modeling_dinov2 import Dinov2Layer
    cfg = Dinov2Config(hidden_size=dim, num_attention_heads=heads, num_hidden_layers=1, mlp_ratio=4, layer_norm_eps=1e-6,
                       hidden_act="gelu", layerscale_value=1.0, use_swiglu_ffn=True, qkv_bias=True,
                       attention_probs_dropout_prob=0.0, hidden_dropout_prob=0.0, drop_path_rate=0.0)
    cfg._attn_implementation = "eager"
    layer = Dinov2Layer(cfg).eval()
    p = f"blocks.{i}."
    qkv_w, qkv_b = sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"]
    mapped = {
        "norm1.weight": sd[p + "norm1.weight"], "norm1.bias": sd[p + "norm1.bias"],
        "norm2.weight": sd[p + "norm2.weight"], "norm2.bias": sd[p + "norm2.bias"],
        "attention.attention.query.weight": qkv_w[:dim], "attention.attention.query.bias": qkv_b[:dim],
        "attention.attention.key.weight": qkv_w[dim:2 * dim], "attention.attention.key.bias": qkv_b[dim:2 * dim],
        "attention.attention.value.weight": qkv_w[2 * dim:], "attention.attention.value.bias": qkv_b[2 * dim:],
        "attention.output.dense.weight": sd[p + "attn.proj.weight"], "attention.output.dense.bias": sd[p + "attn.proj.bias"],
        "layer_scale1.lambda1": sd[p + "ls1.gamma"], "layer_scale2.lambda1": sd[p + "ls2.gamma"],
        "mlp.weights_in.weight": sd[p + "mlp.w12.weight"], "mlp.weights_in.bias": sd[p + "mlp.w12.bias"],
        "mlp.weights_out.weight": sd[p + "mlp.w3.weight"], "mlp.weights_out.bias": sd[p + "mlp.w3.bias"],
    }
    assert set(mapped) == set(layer.state_dict())
    layer.load_state_dict(mapped)
    return layer


def case_state_dict(cfg, swiglu):
    g = torch.Generator().manual_seed(cfg["seed"])
    sd = ovf.random_state_dict(cfg["depth"], cfg["dim"], g, n_pos=37, std=cfg["std"], swiglu=swiglu)
    for i in range(cfg["depth"]):   # LayerScale away from 1 so that its placement matters
        sd[f"blocks.{i}.ls1.gamma"] = 0.5 + torch.rand(cfg["dim"], generator=g)
        sd[f"blocks.{i}.ls2.gamma"] = 0.5 + torch.rand(cfg["dim"], generator=g)
    return sd


def case_video(cfg):
    return synth.random_video(cfg["T"], cfg["H"], cfg["W"], seed=cfg["seed"] + 1)


def sample_index(cfg, numel):
    """The seeded entries of a flattened output that vit_g_small.npz keeps."""
    return np.random.RandomState(cfg["seed"]).randint(0, numel, size=cfg["n_sample"]).astype(np.int64)


def _stand_in(sd, dim, heads, depth, swiglu):
    import torch.nn as nn
    make_layer = hf_dinov2_swiglu_layer if swiglu else hf_dinov2_layer

    class Block(nn.Module):
        def __init__(self, i):
            super().__init__()
            self.layer = make_layer(dim, heads, sd, i)
            self.attn = nn.Module()
            self.attn.qkv = nn.Linear(dim, 3 * dim)      # the qkv hook point, on the block's LayerNorm-1 output
            self.attn.qkv.weight.data.copy_(sd[f"blocks.{i}.attn.qkv.weight"])
            self.attn.qkv.bias.data.copy_(sd[f"blocks.{i}.attn.qkv.bias"])
            self.attn.attn_drop = nn.Identity()

        def forward(self, x):
            self.attn.qkv(self.layer.norm1(x))
            out = self.layer(x)
            return out[0] if isinstance(out, (tuple, list)) else out

    class StandIn(nn.Module):
        def __init__(self):
            super().__init__()
            self.patch_embed = nn.Module()
            self.patch_embed.proj = nn.Conv2d(3, dim, 14, stride=14)
            self.patch_embed.proj.weight.data.copy_(sd["patch_embed.proj.weight"])
            self.patch_embed.proj.bias.data.copy_(sd["patch_embed.proj.bias"])
            self.cls_token = nn.Parameter(sd["cls_token"].clone())
            self.pos_embed = nn.Parameter(sd["pos_embed"].clone())
            self.blocks = nn.ModuleList([Block(i) for i in range(depth)])

        def interpolate_pos_encoding(self, x, w, h):      # replaced by the reference (set_overlapping_patches)
            raise AssertionError("the reference must install its own position-embedding interpolation")

        def forward(self, x):                             # DinoVisionTransformer.prepare_tokens_with_masks + blocks
            B, nc, w, h = x.shape
            x = self.patch_embed.proj(x).flatten(2).transpose(1, 2)
            x = torch.cat((self.cls_token.expand(B, -1, -1), x), dim=1)
            x = x + self.interpolate_pos_encoding(x, w, h)
            for blk in self.blocks:
                x = blk(x)
            return x

    return StandIn().eval()


def _reference_features(video, cfg, sd, swiglu, facet, layer):
    ref_harness.install("cpu")
    import utils as ref_utils
    real_load = torch.hub.load
    torch.hub.load = lambda repo, model_name, *a, **kw: _stand_in(sd, cfg["dim"], cfg["heads"], cfg["depth"], swiglu)
    try:
        with torch.no_grad():
            return ref_utils.get_dino_features_video(video, model_name=cfg["model_name"], facet=facet, stride=7,
                                                     layer=layer, device="cpu")
    finally:
        torch.hub.load = real_load


def gen_facets_case(name, cfg=FACETS_CASE):
    sd, video = case_state_dict(cfg, swiglu=False), case_video(cfg)
    out = {}
    for layer in cfg["layers"]:
        for facet in ("queries", "keys", "values"):
            f = _reference_features(video, cfg, sd, False, facet, layer)
            out[f"{facet}_{layer}"] = f.numpy()
    np.savez_compressed(os.path.join(GOLDEN_DIR, name + ".npz"), **out)
    print(name, {k: (v.shape, float(np.abs(v).max())) for k, v in out.items()})


def gen_g_case(name, cfg=G_CASE):
    sd, video = case_state_dict(cfg, swiglu=True), case_video(cfg)
    out = {}
    for facet in ("tokens", "keys"):
        f = _reference_features(video, cfg, sd, True, facet, cfg["layer"]).numpy()
        idx = sample_index(cfg, f.size)
        out[f"{facet}_shape"] = np.array(f.shape)
        out[f"{facet}_idx"] = idx
        out[f"{facet}_vals"] = f.reshape(-1)[idx]
        out[f"{facet}_sums"] = np.array([f.astype(np.float64).sum(), np.abs(f.astype(np.float64)).sum()])
        out[f"{facet}_absmax"] = np.array(np.abs(f).max())
    np.savez_compressed(os.path.join(GOLDEN_DIR, name + ".npz"), **out)
    print(name, {k: v.tolist() for k, v in out.items() if k.endswith(("_shape", "_absmax"))})


def main():
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    torch.set_num_threads(8)
    gen_facets_case("vit_facets_small")
    gen_g_case("vit_g_small")


if __name__ == "__main__":
    main()
