"""Oracle restatement of the DINOv3 ViT feature stage and of DINOv2 with registers (float64-capable, any stride).

Test infrastructure (see ``oracle/__init__.py``).  No live reference runs DINOv3: the block arithmetic restates
``transformers``' ``DINOv3ViTModel`` (pre-LN block, LayerNorm eps 1e-5, MHA with scale 64^-1/2 and a rotary position
embedding on q and k of the patch tokens, LayerScale, MLP with exact GELU or the gated silu MLP), and is cross-checked
against it with seeded weights at stride = patch (tests/test_vit_dinov3_oracle_cpu.py).  State dicts use the
``transformers`` key names (``embeddings.*``, ``model.layer.{i}.*``), which is what a user of the released weights gets.

What the reference tracker adds, restated as for DINOv2 (``oracle/vit.py``): ImageNet normalisation, the patch embedding
at a stride below the patch, the tap = output of block ``layer`` before the final norm, the prefix tokens dropped and the
C x h x w layout.  The RoPE coordinates come from the token grid (h x w of ``make_geom``): ``(arange(n) + 0.5) / n`` per
axis mapped to [-1, 1], which is what ``transformers`` computes from the grid of non-overlapping patches at
stride = patch, and the analogue of the reference resampling DINOv2's position table onto the token grid.

DINOv2 with registers (hub ``dinov2_vit*14_reg``): the hub keys of ``oracle/vit.py`` plus ``register_tokens``
[1][R][D]; cls + patches get the (interpolated) position table, then the registers are inserted after cls without
position.  Cross-checked against ``transformers``' ``Dinov2WithRegistersModel`` on a grid whose table is not
interpolated.
"""
import math

import torch
import torch.nn.functional as F

from . import vit as ovit
from . import vit_swiglu_facets as ovf

FACETS = ovf.FACETS
HEAD_DIM = 64


def random_state_dict(depth, dim, gen, registers=4, gated=False, hidden=None, patch=16, std=0.02):
    """Seeded weights with ``transformers``' DINOv3ViTModel key names.  Every LayerNorm, LayerScale and bias is drawn
    away from its initial value so that each term of the block is exercised.  ``hidden``: MLP width (default 4 dim)."""
    hidden = hidden or 4 * dim

    def tn(*shape):
        return torch.randn(*shape, generator=gen) * std
    sd = {"embeddings.cls_token": tn(1, 1, dim) * 10, "embeddings.mask_token": torch.zeros(1, 1, dim),
          "embeddings.register_tokens": tn(1, registers, dim) * 10,
          "embeddings.patch_embeddings.weight": tn(dim, 3, patch, patch), "embeddings.patch_embeddings.bias": tn(dim),
          "norm.weight": torch.ones(dim), "norm.bias": torch.zeros(dim)}
    for i in range(depth):
        p = f"model.layer.{i}."
        sd[p + "norm1.weight"] = 1 + tn(dim); sd[p + "norm1.bias"] = tn(dim)
        for x in "qkv":
            sd[p + f"attention.{x}_proj.weight"] = tn(dim, dim) * 2
        sd[p + "attention.q_proj.bias"] = tn(dim); sd[p + "attention.v_proj.bias"] = tn(dim)
        sd[p + "attention.o_proj.weight"] = tn(dim, dim); sd[p + "attention.o_proj.bias"] = tn(dim)
        sd[p + "layer_scale1.lambda1"] = 1 + tn(dim)
        sd[p + "norm2.weight"] = 1 + tn(dim); sd[p + "norm2.bias"] = tn(dim)
        if gated:
            sd[p + "mlp.gate_proj.weight"] = tn(hidden, dim); sd[p + "mlp.gate_proj.bias"] = tn(hidden)
        sd[p + "mlp.up_proj.weight"] = tn(hidden, dim); sd[p + "mlp.up_proj.bias"] = tn(hidden)
        sd[p + "mlp.down_proj.weight"] = tn(dim, hidden); sd[p + "mlp.down_proj.bias"] = tn(dim)
        sd[p + "layer_scale2.lambda1"] = 1 + tn(dim)
    return sd


def n_registers(sd):
    t = sd.get("embeddings.register_tokens")
    return 0 if t is None else t.shape[1]


def rope_cos_sin(h, w, theta=100.0, dtype=torch.float64, device="cpu"):
    """cos, sin [h w][64] of the token grid (dims j and j + 32 share angle j; y angles first, then x)."""
    inv = theta ** (-torch.arange(16, dtype=torch.float64, device=device) / 16)
    cy = 2 * (torch.arange(h, dtype=torch.float64, device=device) + 0.5) / h - 1
    cx = 2 * (torch.arange(w, dtype=torch.float64, device=device) + 0.5) / w - 1
    yy, xx = torch.meshgrid(cy, cx, indexing="ij")
    coords = torch.stack((yy, xx), dim=-1).reshape(h * w, 2)
    ang = (2 * math.pi * coords[:, :, None] * inv).reshape(h * w, 32).tile(2)
    return ang.cos().to(dtype), ang.sin().to(dtype)


def rotate(t, cos, sin):
    """RoPE on the patch rows (the last cos.shape[0] tokens) of t [..., N, 64]; prefix rows unchanged."""
    n = cos.shape[0]
    pre, pat = t[..., :-n, :], t[..., -n:, :]
    half = torch.cat((-pat[..., 32:], pat[..., :32]), dim=-1)
    return torch.cat((pre, pat * cos + half * sin), dim=-2)


def qkv(x, sd, i, eps):
    """Block i's q / k / v Linear outputs on its LayerNorm-1 output, before RoPE (B x N x D each)."""
    p = f"model.layer.{i}."
    D = x.shape[-1]
    y = F.layer_norm(x, (D,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], eps=eps)
    a = p + "attention."
    return tuple(F.linear(y, sd[a + f"{c}_proj.weight"], sd.get(a + f"{c}_proj.bias")) for c in "qkv")


def block_forward(x, sd, i, cos, sin, eps):
    p = f"model.layer.{i}."
    B, N, D = x.shape
    heads = D // HEAD_DIM
    q, k, v = (t.reshape(B, N, heads, HEAD_DIM).transpose(1, 2) for t in qkv(x, sd, i, eps))
    q, k = rotate(q, cos, sin), rotate(k, cos, sin)
    y = (torch.softmax((q * HEAD_DIM ** -0.5) @ k.transpose(-2, -1), dim=-1) @ v).transpose(1, 2).reshape(B, N, D)
    x = x + F.linear(y, sd[p + "attention.o_proj.weight"], sd.get(p + "attention.o_proj.bias")) * sd[p + "layer_scale1.lambda1"]
    y = F.layer_norm(x, (D,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], eps=eps)
    m = p + "mlp."
    up = F.linear(y, sd[m + "up_proj.weight"], sd.get(m + "up_proj.bias"))
    if m + "gate_proj.weight" in sd:
        h = F.silu(F.linear(y, sd[m + "gate_proj.weight"], sd.get(m + "gate_proj.bias"))) * up
    else:
        h = F.gelu(up)
    return x + F.linear(h, sd[m + "down_proj.weight"], sd.get(m + "down_proj.bias")) * sd[p + "layer_scale2.lambda1"]


def normalize(frames01):
    mean = torch.tensor(ovit.IMAGENET_MEAN, device=frames01.device, dtype=frames01.dtype)[None, :, None, None]
    std = torch.tensor(ovit.IMAGENET_STD, device=frames01.device, dtype=frames01.dtype)[None, :, None, None]
    return (frames01 - mean) / std


def embed(pixels, sd, stride):
    """Patch embedding at `stride` of normalised pixels, then [cls, registers, patches]; also the token grid."""
    x = F.conv2d(pixels, sd["embeddings.patch_embeddings.weight"], sd["embeddings.patch_embeddings.bias"], stride=stride)
    B, D, h, w = x.shape
    pre = [sd["embeddings.cls_token"].reshape(1, 1, D).expand(B, -1, -1)]
    if n_registers(sd):
        pre.append(sd["embeddings.register_tokens"].expand(B, -1, -1))
    return torch.cat(pre + [x.flatten(2).transpose(1, 2)], dim=1), h, w


def vit_tokens(frames01, sd, layer, stride=16, facet="tokens", theta=100.0, eps=1e-5):
    """frames01: B x 3 x H x W in [0, 1].  'tokens': block ``layer``'s output B x (1 + R + h w) x D; a facet: that
    block's query / key / value Linear output (before RoPE), B x (1 + R + h w) x D."""
    if facet not in FACETS:
        raise ValueError(f"facet {facet} not supported")
    x, h, w = embed(normalize(frames01), sd, stride)
    cos, sin = rope_cos_sin(h, w, theta, x.dtype, x.device)
    for i in range(layer):
        x = block_forward(x, sd, i, cos, sin, eps)
    if facet == "tokens":
        return block_forward(x, sd, layer, cos, sin, eps)
    return qkv(x, sd, layer, eps)[FACETS.index(facet) - 1]


def dino_features_video(video01, sd, layer, stride=16, patch=16, facet="tokens", theta=100.0, eps=1e-5):
    """Per-frame loop, cls and registers dropped, -> T x C x h x w."""
    T, _, H, W = video01.shape
    ph, pw = 1 + (H - patch) // stride, 1 + (W - patch) // stride
    pre = 1 + n_registers(sd)
    out = []
    for i in range(T):
        tok = vit_tokens(video01[i:i + 1], sd, layer, stride, facet, theta, eps)
        out.append(tok[0, pre:].reshape(ph, pw, -1).permute(2, 0, 1))
    return torch.stack(out)


# ---- DINOv2 with registers (hub keys)
def vit_tokens_reg(frames01, sd, heads, layer, stride=7, facet="tokens"):
    """DINOv2 ``_reg``: as ``oracle.vit_swiglu_facets.vit_tokens`` with the registers inserted after cls (no
    position).  B x (1 + R + h w) x D."""
    x = F.conv2d(normalize(frames01), sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=stride)
    B, D, n_h, n_w = x.shape
    x = torch.cat((sd["cls_token"].expand(B, -1, -1), x.flatten(2).transpose(1, 2)), dim=1)
    x = x + ovit.interpolate_pos_embed(sd["pos_embed"], n_h, n_w)
    x = torch.cat((x[:, :1], sd["register_tokens"].expand(B, -1, -1), x[:, 1:]), dim=1)
    for i in range(layer):
        x = ovf.block_forward(x, sd, i, heads)
    if facet == "tokens":
        return ovf.block_forward(x, sd, layer, heads)
    f = FACETS.index(facet) - 1
    return ovf.qkv(x, sd, layer)[..., f * D:(f + 1) * D]


def dino_features_video_reg(video01, sd, heads, layer, stride=7, patch=14, facet="tokens"):
    T, _, H, W = video01.shape
    ph, pw = 1 + (H - patch) // stride, 1 + (W - patch) // stride
    pre = 1 + sd["register_tokens"].shape[1]
    out = []
    for i in range(T):
        tok = vit_tokens_reg(video01[i:i + 1], sd, heads, layer, stride, facet)
        out.append(tok[0, pre:].reshape(ph, pw, -1).permute(2, 0, 1))
    return torch.stack(out)
