"""Oracle restatement of the DINO v1 backbones of the feature stage: ViT-S/8 and ViT-B/8 (SURVEY.md 8a row a1).

Test infrastructure (see ``oracle/__init__.py``).  The reference loads a name without ``v2`` from
``facebookresearch/dino:main`` (``models/extractor.py:25-28``) and gives it patch 8 when the name contains ``8``
(``:168-169``); the stride patch, the position-embedding interpolation (same ``(w = H_img, h = W_img)`` call as DINOv2),
the tap point and the facets are the reference's own code and are the same as for DINOv2 (``oracle/vit.py``,
``oracle/vit_swiglu_facets.py``, whose stem and qkv this module reuses).  What differs is the block, which belongs to
facebookresearch/dino's ``vision_transformer.Block`` (unpinned ``main``, absent from the reference tree): pre-LN with
LayerNorm eps 1e-6, MHA with qkv bias and scale head_dim**-0.5, exact-GELU MLP 4x, and **no LayerScale**:
``x += Attn(LN(x)); x += MLP(LN(x))``.  The hub state dict has DINOv2's key names without ``ls1.gamma`` /
``ls2.gamma``; its pos-embed grid is 28 x 28 (224-pixel training at patch 8) and its patch embedding 8 x 8.

Pinned by ``tests/golden/vit_dino_v1_small.npz`` from the live reference (``oracle/make_golden_vit_dino_v1.py``) and
cross-checked against ``transformers``' ``ViTLayer`` (tests/test_vit_dino_v1_oracle_cpu.py).
"""
import math

import torch
import torch.nn.functional as F

from . import vit as ovit
from . import vit_swiglu_facets as ovf

CONFIGS = {"dino_vits8": (12, 384, 6), "dino_vitb8": (12, 768, 12)}   # name: (depth, dim, heads)
PATCH, N_POS = 8, 28
FACETS = ovf.FACETS


def random_state_dict(depth, dim, gen, std=0.02):
    """Seeded DINO v1 weights with hub key names: ``oracle.vit.random_state_dict`` at patch 8 and a 28 x 28 pos-embed
    grid, LayerScale removed."""
    sd = ovit.random_state_dict(depth, dim, gen, n_pos=N_POS, patch=PATCH, std=std)
    return {k: v for k, v in sd.items() if not k.endswith(("ls1.gamma", "ls2.gamma"))}


def interpolate_pos_embed(pos_embed, n_h, n_w, H, W):
    """models/extractor.py:57-85 as the reference applies it to an H x W frame: the table unchanged only when the grid has
    N tokens and the frame is square in pixels (``npatch == N and w == h``), else bicubic to n_h x n_w with the +0.1
    trick.  (``oracle.vit.interpolate_pos_embed`` tests the grid's squareness instead; the two differ only for a
    non-square frame whose grid is square with N tokens, e.g. 197 x 198 pixels -> 28 x 28 at patch 8, stride 7.)"""
    N = pos_embed.shape[1] - 1
    if n_h * n_w == N and H == W:
        return pos_embed
    if n_h * n_w != N or n_h != n_w:
        return ovit.interpolate_pos_embed(pos_embed, n_h, n_w)
    dim, side = pos_embed.shape[-1], int(math.sqrt(N))
    patch_pos = pos_embed[:, 1:].reshape(1, side, side, dim).permute(0, 3, 1, 2)
    patch_pos = F.interpolate(patch_pos, scale_factor=((n_h + 0.1) / math.sqrt(N), (n_w + 0.1) / math.sqrt(N)),
                              mode="bicubic", align_corners=False, recompute_scale_factor=False)
    return torch.cat((pos_embed[:, 0][:, None], patch_pos.permute(0, 2, 3, 1).reshape(1, -1, dim)), dim=1)


def block_forward(x, sd, i, heads):
    """One DINO v1 block (no LayerScale)."""
    p = f"blocks.{i}."
    B, N, D = x.shape
    hd = D // heads
    t = ovf.qkv(x, sd, i).reshape(B, N, 3, heads, hd).permute(2, 0, 3, 1, 4)
    q, k, v = t[0] * hd ** -0.5, t[1], t[2]
    y = (torch.softmax(q @ k.transpose(-2, -1), dim=-1) @ v).transpose(1, 2).reshape(B, N, D)
    x = x + F.linear(y, sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
    y = F.layer_norm(x, (D,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], eps=1e-6)
    y = F.linear(F.gelu(F.linear(y, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"])), sd[p + "mlp.fc2.weight"],
                 sd[p + "mlp.fc2.bias"])
    return x + y


def vit_tokens(frames01, sd, heads, layer, stride=7, facet="tokens"):
    """frames01: B x 3 x H x W in [0, 1].  'tokens': block ``layer``'s output B x (1 + h w) x D; a facet: that block's
    query / key / value rows of its qkv Linear output."""
    if facet not in FACETS:
        raise ValueError(f"facet {facet} not supported")
    mean = torch.tensor(ovit.IMAGENET_MEAN, device=frames01.device)[None, :, None, None]
    std = torch.tensor(ovit.IMAGENET_STD, device=frames01.device)[None, :, None, None]
    x = F.conv2d((frames01 - mean) / std, sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=stride)
    B, D, n_h, n_w = x.shape
    x = torch.cat((sd["cls_token"].expand(B, -1, -1), x.flatten(2).transpose(1, 2)), dim=1)
    x = x + interpolate_pos_embed(sd["pos_embed"], n_h, n_w, *frames01.shape[-2:])
    for i in range(layer):
        x = block_forward(x, sd, i, heads)
    if facet == "tokens":
        return block_forward(x, sd, layer, heads)
    f = FACETS.index(facet) - 1
    return ovf.qkv(x, sd, layer)[..., f * D:(f + 1) * D]


def dino_features_video(video01, sd, heads, layer, stride=7, facet="tokens"):
    """utils.py:32-72 at patch 8: per-frame loop, cls dropped, -> T x C x h x w."""
    T, _, H, W = video01.shape
    ph, pw = 1 + (H - PATCH) // stride, 1 + (W - PATCH) // stride
    out = []
    for i in range(T):
        tok = vit_tokens(video01[i:i + 1], sd, heads, layer, stride, facet)
        out.append(tok[0, 1:].reshape(ph, pw, -1).permute(2, 0, 1))
    return torch.stack(out)
