"""Generate ``tests/golden/vit_dino_v1_small.npz`` by running the LIVE reference (only where its sources are present):

    python -m oracle.make_golden_vit_dino_v1

``utils.get_dino_features_video`` + ``models/extractor.VitExtractor`` run unmodified on the CPU with the names
``dino_vits8`` and ``dino_vitb8``, so the reference itself derives patch 8, the stride patch, the position-embedding
interpolation from a 28 x 28 grid, C and the grid.  Only ``torch.hub.load('facebookresearch/dino:main', name)`` is
replaced by a stand-in with the ``VisionTransformer`` surface the extractor touches; its blocks are ``transformers``'
``ViTLayer`` (pre-LN, no LayerScale; independent of ``oracle/``) carrying seeded weights, and its ``attn.qkv`` is a real
``nn.Linear`` with the block's qkv weights applied to the block's LayerNorm-1 output, so the reference's qkv hook fires.

Per name: 2 blocks with the real width and heads, ``layer=1`` passed explicitly (the names imply 12 blocks), one
36 x 50 frame (5 x 7 tokens at patch 8, stride 7), tokens and keys.
"""
import os

import numpy as np
import torch

from . import ref_harness, synth
from . import vit_dino_v1 as ov1
from .make_golden import GOLDEN_DIR

CASES = {"dino_vits8": dict(seed=91), "dino_vitb8": dict(seed=92)}
DEPTH, LAYER, H, W, T, STD = 2, 1, 36, 50, 1, 0.05
FACETS = ("tokens", "keys")


def hf_vit_layer(dim, heads, sd, i):
    """Block i of a DINO v1 hub state dict as ``transformers``' ViTLayer (LayerNorm eps 1e-6, qkv bias, exact GELU)."""
    from transformers import ViTConfig
    from transformers.models.vit.modeling_vit import ViTLayer
    cfg = ViTConfig(hidden_size=dim, num_attention_heads=heads, num_hidden_layers=1, intermediate_size=4 * dim,
                    hidden_act="gelu", layer_norm_eps=1e-6, qkv_bias=True, attention_probs_dropout_prob=0.0,
                    hidden_dropout_prob=0.0)
    cfg._attn_implementation = "eager"
    layer = ViTLayer(cfg).eval()
    p = f"blocks.{i}."
    qkv_w, qkv_b = sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"]
    mapped = {
        "layernorm_before.weight": sd[p + "norm1.weight"], "layernorm_before.bias": sd[p + "norm1.bias"],
        "layernorm_after.weight": sd[p + "norm2.weight"], "layernorm_after.bias": sd[p + "norm2.bias"],
        "attention.attention.query.weight": qkv_w[:dim], "attention.attention.query.bias": qkv_b[:dim],
        "attention.attention.key.weight": qkv_w[dim:2 * dim], "attention.attention.key.bias": qkv_b[dim:2 * dim],
        "attention.attention.value.weight": qkv_w[2 * dim:], "attention.attention.value.bias": qkv_b[2 * dim:],
        "attention.output.dense.weight": sd[p + "attn.proj.weight"], "attention.output.dense.bias": sd[p + "attn.proj.bias"],
        "intermediate.dense.weight": sd[p + "mlp.fc1.weight"], "intermediate.dense.bias": sd[p + "mlp.fc1.bias"],
        "output.dense.weight": sd[p + "mlp.fc2.weight"], "output.dense.bias": sd[p + "mlp.fc2.bias"],
    }
    assert set(mapped) == set(layer.state_dict())
    layer.load_state_dict(mapped)
    return layer


def case_state_dict(name):
    _, dim, _ = ov1.CONFIGS[name]
    return ov1.random_state_dict(DEPTH, dim, torch.Generator().manual_seed(CASES[name]["seed"]), std=STD)


def case_video(name):
    return synth.random_video(T, H, W, seed=CASES[name]["seed"] + 1)


def _stand_in(sd, dim, heads):
    import torch.nn as nn

    class Block(nn.Module):
        def __init__(self, i):
            super().__init__()
            self.layer = hf_vit_layer(dim, heads, sd, i)
            self.attn = nn.Module()
            self.attn.qkv = nn.Linear(dim, 3 * dim)      # the qkv hook point, on the block's LayerNorm-1 output
            self.attn.qkv.weight.data.copy_(sd[f"blocks.{i}.attn.qkv.weight"])
            self.attn.qkv.bias.data.copy_(sd[f"blocks.{i}.attn.qkv.bias"])
            self.attn.attn_drop = nn.Identity()

        def forward(self, x):
            self.attn.qkv(self.layer.layernorm_before(x))
            out = self.layer(x)
            return out[0] if isinstance(out, (tuple, list)) else out

    class StandIn(nn.Module):
        def __init__(self):
            super().__init__()
            self.patch_embed = nn.Module()
            self.patch_embed.proj = nn.Conv2d(3, dim, ov1.PATCH, stride=ov1.PATCH)
            self.patch_embed.proj.weight.data.copy_(sd["patch_embed.proj.weight"])
            self.patch_embed.proj.bias.data.copy_(sd["patch_embed.proj.bias"])
            self.cls_token = nn.Parameter(sd["cls_token"].clone())
            self.pos_embed = nn.Parameter(sd["pos_embed"].clone())
            self.blocks = nn.ModuleList([Block(i) for i in range(DEPTH)])

        def interpolate_pos_encoding(self, x, w, h):      # replaced by the reference (set_overlapping_patches)
            raise AssertionError("the reference must install its own position-embedding interpolation")

        def forward(self, x):                             # dino's VisionTransformer.prepare_tokens + blocks
            B, nc, w, h = x.shape
            x = self.patch_embed.proj(x).flatten(2).transpose(1, 2)
            x = torch.cat((self.cls_token.expand(B, -1, -1), x), dim=1)
            x = x + self.interpolate_pos_encoding(x, w, h)
            for blk in self.blocks:
                x = blk(x)
            return x

    return StandIn().eval()


def reference_features(name, facet):
    sd, video = case_state_dict(name), case_video(name)
    _, dim, heads = ov1.CONFIGS[name]
    ref_harness.install("cpu")
    import utils as ref_utils
    real_load = torch.hub.load
    hub_repos = []

    def load(repo, model_name, *a, **kw):
        hub_repos.append(repo)
        return _stand_in(sd, dim, heads)
    torch.hub.load = load
    try:
        with torch.no_grad():
            f = ref_utils.get_dino_features_video(video, model_name=name, facet=facet, stride=7, layer=LAYER, device="cpu")
    finally:
        torch.hub.load = real_load
    assert hub_repos == ["facebookresearch/dino:main"], hub_repos
    return f


def main(out_dir=GOLDEN_DIR):
    os.makedirs(out_dir, exist_ok=True)
    torch.set_num_threads(8)
    out = {}
    for name in CASES:
        for facet in FACETS:
            out[f"{name}_{facet}"] = reference_features(name, facet).numpy()
    np.savez_compressed(os.path.join(out_dir, "vit_dino_v1_small.npz"), **out)
    print("vit_dino_v1_small", {k: (v.shape, float(np.abs(v).max())) for k, v in out.items()})


if __name__ == "__main__":
    main()
